"""Train steps per second of a whole ensemble: N members trained one after another against the same N trained side by
side (one host thread and one CUDA stream each, every handle with a device share of 1/N), N = 1, 4, 8.

Shapes: the reference's default (lfm_quant.py flags: B=256, T=5, H=64, L=2; F=32, O=16) at fp32 and bf16, and
BASELINE configs[1] (B=4096, T=48, H=256, L=1) and configs[2] (B=4096, T=48, H=512, L=2, dropout 0.2) at bf16.

    python tools/bench_ensemble.py [--steps 50] [--warmup 5] [--members 1,4,8] [--cases ref_fp32,ref_bf16,cfg1,cfg2]

Prints one JSON line per (case, N) with the GPU's name and power limit; --out FILE also writes them there.
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'oracle'))

CASES = {
    'ref_fp32': dict(B=256, T=5, F=32, O=16, H=64, L=2, precision='fp32', dropout=0.0),
    'ref_bf16': dict(B=256, T=5, F=32, O=16, H=64, L=2, precision='bf16', dropout=0.0),
    'cfg1': dict(B=4096, T=48, F=32, O=16, H=256, L=1, precision='bf16', dropout=0.0),
    'cfg2': dict(B=4096, T=48, F=32, O=16, H=512, L=2, precision='bf16', dropout=0.2),
}


def gpu_info():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else 'unknown'


def make_members(c, n):
    import torch
    import lfm_oracle as orc
    from lfm_quant_b200.engine import ForecasterEngine
    members = []
    for i in range(n):
        rng = np.random.default_rng(i)
        eng = ForecasterEngine(max_batch=c['B'], seq_len=c['T'], n_inputs=c['F'], n_outputs=c['O'], num_hidden=c['H'],
                               num_layers=c['L'], target_idx=3, precision=c['precision'], dropout=c['dropout'],
                               seed=521 + i)
        eng.set_weights(orc.init_params(c['L'], c['F'], c['O'], c['H'], init_scale=1.0, seed=521 + i,
                                        dtype=np.float32))
        x = torch.from_numpy(rng.standard_normal((c['B'], c['T'], c['F']), dtype=np.float32)).cuda()
        y = torch.from_numpy(rng.standard_normal((c['B'], c['T'], c['O']), dtype=np.float32)).cuda()
        members.append((eng, x, y))
    torch.cuda.synchronize()
    return members


def run(members, steps, warmup, concurrent):
    """Seconds for `steps` train steps of every member after `warmup` untimed ones (host clock around work that ends in
    a device synchronise)."""
    import torch
    n = len(members)
    ready = threading.Barrier(n + 1)
    done = threading.Barrier(n + 1)
    step0 = [0] * n

    def member(i, count):
        eng, x, y = members[i]
        for k in range(count):
            eng.train_step(x, y, step0[i] + k, 0.6)
        step0[i] += count

    def thread(i):
        try:
            torch.cuda.set_device(0)
            s = torch.cuda.Stream()
            with torch.cuda.stream(s):
                member(i, warmup)
                s.synchronize()
                ready.wait()
                ready.wait()
                member(i, steps)
                s.synchronize()
            done.wait()
        except Exception:
            ready.abort()        # the main thread raises BrokenBarrierError instead of waiting for ever
            done.abort()
            raise

    if concurrent:
        for eng, _, _ in members:
            eng.set_device_share(1, n)
        threads = [threading.Thread(target=thread, args=(i,)) for i in range(n)]
        for t in threads:
            t.start()
        ready.wait()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ready.wait()
        done.wait()
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        for t in threads:
            t.join()
        for eng, _, _ in members:
            eng.set_device_share(1, 1)
        return dt
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        for i in range(n):
            member(i, warmup)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for i in range(n):
            member(i, steps)
        torch.cuda.synchronize()
        return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--members', default='1,4,8')
    ap.add_argument('--cases', default=','.join(CASES))
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('bench_ensemble needs a CUDA GPU')
    torch.cuda.set_device(0)
    gpu = gpu_info()
    lines = []
    for case in a.cases.split(','):
        c = CASES[case]
        for n in [int(v) for v in a.members.split(',')]:
            members = make_members(c, n)
            seq = run(members, a.steps, a.warmup, concurrent=False)
            con = run(members, a.steps, a.warmup, concurrent=True)
            res = {'case': case, 'members': n, 'steps_per_member': a.steps,
                   'shape': {k: c[k] for k in ('B', 'T', 'F', 'O', 'H', 'L', 'precision', 'dropout')},
                   'one_after_another_steps_per_s': n * a.steps / seq, 'side_by_side_steps_per_s': n * a.steps / con,
                   'speedup': seq / con, 'gpu': gpu}
            print(json.dumps(res), flush=True)
            lines.append(res)
            for eng, _, _ in members:
                eng.close()
            del members
            torch.cuda.empty_cache()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            for r in lines:
                f.write(json.dumps(r) + '\n')


if __name__ == '__main__':
    main()
