"""Times the training-window attributions on one GPU: lfmq_influence_topk (engine.influence_topk), the fused 3xTF32 wgmma
GEMM with the streaming top-K epilogue, against the torch path a user would write today on the same GPU -- fp32 matmul
of the queries against column chunks of the pool, torch.topk of each chunk's scores both ways, and a merge with the
running lists -- once with TF32 off and once with it on.  Also times the pool's feature pass
(lfmq_influence_train_features) of a point and a UQ LSTM on its own.

Shapes: Nq = 16384 queries, Nt = 262144 training windows, K = 10; D = 256 with J = 1 (point) and J = 2 (UQ), and
D = 1536 (the linear model over T * F = 48 * 32), each with the appended one (D1 = D + 1).  Features are seeded random
draws with a lognormal spread of the pool's norms.  TFLOP/s counts the 2 Nq Nt D1 J useful operations.  Time over CUDA
events after a warm-up call; the torch path runs once after its warm-up.  The card's name and power limit are read in
the same run.  Prints one JSON line per case.

usage: python tools/bench_influence.py [--out FILE] [--reps K] [--cases point,uq,linear,features] [--nt NT]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from lfm_quant_b200.engine import ForecasterEngine, influence_topk  # noqa: E402

NQ, NT, K = 16384, 262144, 10
CASES = {'point': (256, 1), 'uq': (256, 2), 'linear': (1536, 1)}
CHUNK = 16384
T, F, O, H = 48, 32, 16, 256


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def features(nq, nt, d1, J, seed=0):
    g = torch.Generator(device='cuda').manual_seed(seed)
    a = torch.randn(nq, d1, device='cuda', generator=g)
    a[:, -1] = 1.0
    u = torch.randn(J, nt, d1, device='cuda', generator=g) * torch.exp(torch.randn(J, nt, 1, device='cuda', generator=g))
    s = torch.ones(J, nq, device='cuda')
    if J == 2:
        s[1] = torch.rand(nq, device='cuda', generator=g) * 0.9 + 0.1
    return a, u, s


def torch_topk(a, u, s, k):
    """chunked matmul + topk of each chunk both ways + merge with the running lists"""
    J, nt, _ = u.shape
    out = []
    for j in range(J):
        best_v = best_i = worst_v = worst_i = None
        for c0 in range(0, nt, CHUNK):
            sc = -(s[j][:, None] * (a @ u[j, c0:c0 + CHUNK].T))
            pv, pi = torch.topk(sc, k, dim=1)
            nv, ni = torch.topk(sc, k, dim=1, largest=False)
            pi, ni = pi + c0, ni + c0
            if best_v is not None:
                pv, sel = torch.topk(torch.cat([best_v, pv], 1), k, dim=1)
                pi = torch.gather(torch.cat([best_i, pi], 1), 1, sel)
                nv, sel = torch.topk(torch.cat([worst_v, nv], 1), k, dim=1, largest=False)
                ni = torch.gather(torch.cat([worst_i, ni], 1), 1, sel)
            best_v, best_i, worst_v, worst_i = pv, pi, nv, ni
        out.append((best_i, best_v, worst_i, worst_v))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out')
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--cases', default='point,uq,linear,features')
    ap.add_argument('--nt', type=int, default=NT)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    name = card()
    rows = []
    for case in args.cases.split(','):
        if case == 'features':
            for uq in (False, True):
                e = ForecasterEngine(max_batch=8192, seq_len=T, n_inputs=F, n_outputs=O, num_hidden=H, target_idx=3,
                                     precision='fp32', train=False, forward_only=True, uq=uq, dropout=0.2,
                                     recurrent_dropout=0.15)
                rng = np.random.RandomState(0)
                e.set_weights([rng.uniform(-0.1, 0.1, size=sp[1]) for sp in e.trainable_specs])
                x = torch.randn(args.nt, T, F, device='cuda')
                y = torch.randn(args.nt, T, O, device='cuda')
                ms = timed(lambda: e.influence_features(x, y), 1)
                rows.append(dict(case='features-' + ('uq' if uq else 'point'), Nt=args.nt, T=T, F=F, H=H,
                                 precision='fp32', ms=round(ms, 2), card=name))
                print(json.dumps(rows[-1]), flush=True)
                del x, y, e
                torch.cuda.empty_cache()
            continue
        D, J = CASES[case]
        a, u, s = features(NQ, args.nt, D + 1, J)
        flops = 2.0 * NQ * args.nt * (D + 1) * J
        ms = timed(lambda: influence_topk(a, u, s, K), args.reps)
        row = dict(case=case, Nq=NQ, Nt=args.nt, D1=D + 1, J=J, K=K, lfmq_ms=round(ms, 2),
                   lfmq_tflops=round(flops / ms / 1e9, 1), card=name)
        for tf32 in (False, True):
            torch.backends.cuda.matmul.allow_tf32 = tf32
            tms = timed(lambda: torch_topk(a, u, s, K), 1)
            key = 'torch_tf32' if tf32 else 'torch_fp32'
            row[key + '_ms'] = round(tms, 2)
            row[key + '_speedup'] = round(tms / ms, 2)
        torch.backends.cuda.matmul.allow_tf32 = False
        rows.append(row)
        print(json.dumps(row), flush=True)
        del a, u, s
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as fh:
            for r in rows:
                fh.write(json.dumps(r) + '\n')


if __name__ == '__main__':
    main()
