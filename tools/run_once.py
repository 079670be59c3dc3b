"""A few train steps (or forwards) of one bench workload, for profiler captures.

    python tools/run_once.py --workload cfg3 --steps 2 [--precision bf16] [--batch N]
"""
import argparse
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'oracle'))

import bench  # noqa: E402
from lfm_quant_b200.engine import ForecasterEngine  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--workload', default='cfg3')
    ap.add_argument('--precision', default='bf16')
    ap.add_argument('--steps', type=int, default=2)
    ap.add_argument('--batch', type=int, default=0)
    a = ap.parse_args()
    w = dict(bench.WORKLOADS[a.workload])
    if a.batch:
        w['B'] = a.batch
    predict = w['mode'] == 'predict'
    eng = ForecasterEngine(max_batch=w['B'], seq_len=w['T'], n_inputs=w['F'], n_outputs=w['O'], num_hidden=w['H'],
                           num_layers=w['L'], target_idx=3, train=not predict, precision=a.precision,
                           dropout=w['dropout'], forward_only=predict, seed=bench.SEED)
    eng.set_weights(bench.initial_weights(w))
    rng = np.random.default_rng(0)
    x, y = bench.synthetic(w['B'], rng, w)
    x, y = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()
    out = torch.empty(w['B'], w['T'], w['O'], device='cuda') if predict else None
    for i in range(a.steps):
        if predict:
            eng.forward(x, out=out)
        else:
            eng.train_step(x, y, i, 0.6)
    torch.cuda.synchronize()
    print('done', a.workload, a.precision, a.steps)


if __name__ == '__main__':
    main()
