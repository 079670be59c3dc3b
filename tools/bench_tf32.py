"""fp32 against tf32 (LFMQ_PREC_TF32: the fp32 step with its GEMMs on tf32 tensor cores), train step and predict, at four
shapes, alternating the precisions inside one call; the step's split by lfmq_profile region (FWD / HEAD / BWD / WGRAD /
OPT) for both; and each region's GEMM FLOPs (computed here from the shapes) over its time.  A region also holds the
pointwise work around its GEMMs, so its rate is a lower bound on what the GEMMs reach; the H100 SXM data sheet's dense
figures are 67 TFLOP/s FP32 and 495 TFLOP/s TF32, at up to 700 W.  One JSON line per result, with the card and its
power limit read in the same run.

    python tools/bench_tf32.py [--iters 5] [--warmup 2] [--reps 3] [--cases uq_chain,gru,cfg2,ref]
    python tools/bench_tf32.py --dump out.npz      # an fp32 UQ chain's train-step outputs and gradients, for A/B builds
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'oracle'))

import lfm_oracle as orc  # noqa: E402
from lfm_quant_b200.engine import ForecastChainEngine, ForecasterEngine  # noqa: E402

DROP = dict(dropout=0.2, recurrent_dropout=0.1, seed=521)
# name: (B, T, F, O, H, L, cell, uq, forecast steps, dropouts, extra precisions)
CASES = {
    'uq_chain': (4096, 48, 32, 16, 256, 1, 'lstm', True, 2, DROP, ()),            # tools/bench_uq_chain.py
    'gru': (4096, 48, 32, 16, 256, 1, 'gru', False, 1, DROP, ()),
    'cfg2': (4096, 48, 32, 16, 512, 2, 'lstm', False, 1, dict(dropout=0.2, seed=521), ('bf16',)),   # BASELINE configs[2]
    'ref': (256, 5, 32, 16, 64, 2, 'lstm', False, 1, DROP, ()),                   # the reference's default shape
}


def _power_limit_w():
    try:
        r = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader,nounits', '-i',
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return float(r.stdout.strip().splitlines()[0])
    except Exception:
        return None


def _time(fn, warmup, iters):
    for i in range(warmup):
        fn(i)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(iters):
        fn(warmup + i)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def _engine(case, precision, train):
    B, T, F, O, H, L, cell, uq, S, drop, _ = CASES[case]
    kw = dict(max_batch=B, seq_len=T, n_inputs=F, n_outputs=O, num_hidden=H, num_layers=L, target_idx=3,
              precision=precision, train=train, forward_only=not train, rnn_cell=cell, uq=uq, **drop)
    w = orc.init_params(L, F, O, H, init_scale=1.0, seed=521, dtype=np.float32, rnn_cell=cell, uq=uq)
    if S == 1:
        eng = ForecasterEngine(**kw)
    else:
        eng = ForecastChainEngine(forecast_steps=S, weights=[1.0, 0.5][:S], **kw)
        for s in range(1, S):
            w += orc.init_params(1, F, O, H, init_scale=1.0, seed=521 + 7 * s, dtype=np.float32, rnn_cell=cell, uq=uq)
    eng.set_weights(w)
    return eng


def _data(case, rng):
    B, T, F, O, _, _, _, _, S, _, _ = CASES[case]
    x = torch.from_numpy(rng.standard_normal((B, T, F), dtype=np.float32)).cuda()
    ys = [torch.from_numpy(rng.standard_normal((B, T, O), dtype=np.float32)).cuda() for _ in range(S)]
    return x, (ys[0] if S == 1 else ys)


def _flops(case):
    """GEMM FLOPs of one train step per profiler region, summed over the stages (2 per multiply-add)."""
    B, T, F, O, H, L, cell, uq, S, _, _ = CASES[case]
    NG = 3 if cell == 'gru' else 4
    heads = 2 if uq else 1
    f = dict(fwd=0.0, head=0.0, bwd=0.0, wgrad=0.0)
    for s in range(S):
        for l in range(L if s == 0 else 1):
            I = F if l == 0 else H
            f['fwd'] += 2.0 * B * T * I * NG * H + 2.0 * B * (T - 1) * H * NG * H
            f['bwd'] += 2.0 * B * (T - 1) * NG * H * H
            f['wgrad'] += 2.0 * B * T * (I + H) * NG * H
            if l > 0 or s > 0:
                f['wgrad'] += 2.0 * B * T * NG * H * I          # dx
        f['head'] += heads * (2.0 * B * T * H * O * 3)          # forward, dW, dy
    return f


def _stages(eng):
    return getattr(eng, 'stages', [eng])


def _profile(case, eng, x, y, steps=2):
    for st in _stages(eng):
        st.profile(True)
    for i in range(steps):
        eng.train_step(x, y, i, 0.01)
    torch.cuda.synchronize()
    tot = {}
    for st in _stages(eng):
        for k, (ms, n) in st.profile_read().items():
            tot[k] = tot.get(k, 0.0) + ms / steps
        st.profile(False)
    return tot


def dump(path):
    """The fp32 UQ chain's forward outputs, train-step losses and gradients at a fixed seed: run it under two builds
    and compare the files bit for bit."""
    rng = np.random.default_rng(0)
    eng = _engine('uq_chain', 'fp32', train=True)
    x, ys = _data('uq_chain', rng)
    out = {}
    for i, t in enumerate(eng.forward(x, step=1)):
        out['forward_%d' % i] = t.cpu().numpy()
    out['backward'] = eng.backward(x, ys, step=1).cpu().numpy()
    for i, g in enumerate(eng.grads_list()):
        out['grad_%d' % i] = g
    for it in range(2):
        out['step_%d' % it] = eng.train_step(x, ys, it, 0.01).cpu().numpy()
    for i, w in enumerate(eng.get_weights(trainable_only=False)):
        out['weight_%d' % i] = w
    np.savez(path, **out)
    print(json.dumps(dict(case='dump', path=path, arrays=len(out))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--cases', default=','.join(CASES))
    ap.add_argument('--dump', default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_tf32 needs a CUDA device')
    if a.dump:
        return dump(a.dump)
    card, power = torch.cuda.get_device_name(), _power_limit_w()
    rng = np.random.default_rng(0)
    for case in a.cases.split(','):
        B, T, F, O, H, L, cell, uq, S, drop, extra = CASES[case]
        base = dict(case=case, B=B, T=T, F=F, O=O, H=H, L=L, cell=cell, uq=uq, forecast_steps=S, card=card,
                    power_limit_w=power, **drop)
        precs = ('fp32', 'tf32') + tuple(extra)
        x, y = _data(case, rng)
        engs = {p: _engine(case, p, train=True) for p in precs}
        times = {p: [] for p in precs}
        for _ in range(a.reps):           # alternate the precisions: drifts in clock or load hit both alike
            for p in precs:
                times[p].append(_time(lambda i: engs[p].train_step(x, y, i, 0.01), a.warmup, a.iters))
        flops = _flops(case)
        for p in precs:
            regions = _profile(case, engs[p], x, y) if p != 'bf16' else {}
            rates = {k: round(flops[k] / (regions[k] * 1e-3) / 1e12, 2) for k in flops if regions.get(k)}
            print(json.dumps(dict(base, what='train_step', precision=p, ms=round(float(np.median(times[p])), 3),
                                  ms_reps=[round(t, 3) for t in times[p]],
                                  regions_ms={k: round(v, 3) for k, v in regions.items()},
                                  region_gemm_tflops=rates, gemm_tflop_per_step=round(sum(flops.values()) / 1e12, 3))),
                  flush=True)
        for p in precs:
            engs[p].close()
        engs = {p: _engine(case, p, train=False) for p in precs}
        times = {p: [] for p in precs}
        for _ in range(a.reps):
            for p in precs:
                times[p].append(_time(lambda i: engs[p].forward(x, step=i), a.warmup, a.iters))
        for p in precs:
            print(json.dumps(dict(base, what='predict', precision=p, ms=round(float(np.median(times[p])), 3),
                                  ms_reps=[round(t, 3) for t in times[p]])), flush=True)
            engs[p].close()
        del engs, x, y
        torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
