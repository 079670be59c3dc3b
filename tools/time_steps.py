"""Per-region device timings of the train step / forward at the BASELINE shapes.

    python tools/time_steps.py [--precision bf16] [--batch 4096] [--steps 10]
"""
import argparse
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'oracle'))

import lfm_oracle as orc  # noqa: E402
from lfm_quant_b200.engine import ForecasterEngine  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--precision', default='bf16')
    ap.add_argument('--batch', type=int, default=4096)
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--predict-batch', type=int, default=65536)
    a = ap.parse_args()
    T, F, O, H = 48, 32, 16, 256
    rng = np.random.default_rng(0)
    w = orc.init_params(1, F, O, H, init_scale=1.0, seed=521, dtype=np.float32)
    B = a.batch
    eng = ForecasterEngine(max_batch=B, seq_len=T, n_inputs=F, n_outputs=O, num_hidden=H, target_idx=3,
                           precision=a.precision)
    eng.set_weights(w)
    x = torch.from_numpy(rng.standard_normal((B, T, F), dtype=np.float32)).cuda()
    y = torch.from_numpy(rng.standard_normal((B, T, O), dtype=np.float32)).cuda()
    for i in range(3):
        eng.train_step(x, y, i, 0.6)
    torch.cuda.synchronize()
    eng.profile(True)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(a.steps):
        eng.train_step(x, y, 3 + i, 0.6)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / a.steps
    reg = eng.profile_read()
    print('[train %s B=%d] %.3f ms/step  %.0f seq/s  regions(ms/step): %s' % (
        a.precision, B, ms, B / ms * 1e3, {k: round(v[0] / a.steps, 4) for k, v in reg.items()}))
    eng.profile(False)
    eng.close()
    del eng
    torch.cuda.empty_cache()
    PB = a.predict_batch
    eng = ForecasterEngine(max_batch=PB, seq_len=T, n_inputs=F, n_outputs=O, num_hidden=H, target_idx=3,
                           precision=a.precision, train=False, forward_only=True)
    eng.set_weights(w)
    xp = torch.from_numpy(rng.standard_normal((PB, T, F), dtype=np.float32)).cuda()
    out = torch.empty(PB, T, O, device='cuda')
    for i in range(2):
        eng.forward(xp, out=out)
    torch.cuda.synchronize()
    eng.profile(True)
    e0.record()
    for i in range(5):
        eng.forward(xp, out=out)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 5
    reg = eng.profile_read()
    print('[predict %s B=%d] %.3f ms/call  %.0f seq/s  regions(ms): %s' % (
        a.precision, PB, ms, PB / ms * 1e3, {k: round(v[0] / 5, 4) for k, v in reg.items() if v[1]}))


if __name__ == '__main__':
    main()
