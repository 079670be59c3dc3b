"""Cost of row weights (lfmq_set_row_weights) in the training step: weighted against unweighted, alternated, three runs
of each, at BASELINE configs[1] (bf16 cluster path), configs[2] (bf16 general path), a two-step fp32 UQ chain and the
linear model.  Prints the card, its power limit, the median ms per step of each run and the launches per step.

    python tools/bench_row_weights.py [--steps 50] [--warmup 10] [--out results.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from lfm_quant_b200.engine import DenseEngine, ForecastChainEngine, ForecasterEngine  # noqa: E402

F, O = 32, 16


def _card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def _cases():
    B, T = 4096, 48
    yield 'cfg1-bf16-cluster', B, T, lambda: ForecasterEngine(max_batch=B, seq_len=T, n_inputs=F, n_outputs=O,
                                                              num_hidden=256, num_layers=1, target_idx=3,
                                                              precision='bf16'), False
    yield 'cfg2-bf16-general', B, T, lambda: ForecasterEngine(max_batch=B, seq_len=T, n_inputs=F, n_outputs=O,
                                                              num_hidden=512, num_layers=2, target_idx=3,
                                                              precision='bf16', dropout=0.2, recurrent_dropout=0.2,
                                                              seed=5), False
    yield 'uq-chain-fp32', 256, 48, lambda: ForecastChainEngine(forecast_steps=2, weights=[1.0, 0.5], max_batch=256,
                                                                seq_len=48, n_inputs=F, n_outputs=O, num_hidden=256,
                                                                num_layers=1, target_idx=3, uq=True, dropout=0.1,
                                                                seed=3), True
    yield 'linear', B, 5, lambda: DenseEngine(max_batch=B, seq_len=5, n_inputs=F, n_outputs=O, target_idx=3), False


def _time(eng, chain, x, y, steps, warmup):
    step = (lambda i: eng.train_step(x, [y, y], i, 0.5)) if chain else (lambda i: eng.train_step(x, y, i, 0.5))
    for i in range(warmup):
        step(i)
    torch.cuda.synchronize()
    n0 = eng.launch_count
    ms = []
    for i in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        step(warmup + i)
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return float(np.median(ms)), (eng.launch_count - n0) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=10)
    ap.add_argument('--out', default='')
    a = ap.parse_args()
    torch.cuda.set_device(0)
    res = {'card': _card(), 'cases': {}}
    print('card: %s' % res['card'])
    for name, B, T, make, chain in _cases():
        rng = np.random.RandomState(0)
        x = torch.from_numpy(rng.normal(size=(B, T, F)).astype(np.float32)).cuda()
        y = torch.from_numpy(rng.normal(size=(B, O) if name == 'linear' else (B, T, O)).astype(np.float32)).cuda()
        w = torch.from_numpy(rng.uniform(0, 2, size=B).astype(np.float32)).cuda()
        eng = make()
        runs = {'unweighted': [], 'weighted': []}
        launches = {}
        for _ in range(3):
            for key in ('unweighted', 'weighted'):
                eng.set_row_weights(w if key == 'weighted' else None)
                t, n = _time(eng, chain, x, y, a.steps, a.warmup)
                runs[key].append(t)
                launches[key] = n
        eng.close()
        res['cases'][name] = {'ms': runs, 'launches_per_step': launches}
        print('%-20s unweighted %s ms  weighted %s ms  launches/step %s' % (
            name, ' '.join('%.3f' % v for v in runs['unweighted']), ' '.join('%.3f' % v for v in runs['weighted']),
            launches))
        time.sleep(0.5)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or '.', exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
