"""What the bf16 cluster path computes at the benchmark's shape, written out so that two builds can be compared.

    python tools/dump_step_outputs.py --out DIR          # the build LFMQ_LIB_PATH selects (default: the in-tree one)
    python tools/dump_step_outputs.py --compare DIR_A DIR_B

With seeded inputs and weights, for B in {4096, 3940, 1000} at T=48 (30 tiles + 4 half tiles, 30 tiles + 2 half tiles
with a partial last one, 16 half tiles): the predictions of a forward-only handle, and for dropout 0 and 0.2 the
gradients of one backward (grads_list()) with the {loss, mse_0} tail of the gradient vector.

--compare requires predictions and the LSTM W, U, b gradients to be bit-identical, and the head gradients and the loss
to agree to 1e-5 relative (to the tensor's largest entry): those are sums over rows through the head's shared-memory
atomics, whose order varies from run to run.  Exit status 1 if anything differs beyond that.
"""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'oracle'))

BATCHES = (4096, 3940, 1000)
DROPOUTS = (0.0, 0.2)
T, F, O, H = 48, 32, 16, 256
HEAD_TOL = 1e-5
N_LSTM = 3                     # grads_list() starts with the LSTM kernel W, recurrent U and bias


def _problem(B, seed):
    import lfm_oracle as orc
    rng = np.random.RandomState(seed)
    params = orc.init_params(1, F, O, H, init_scale=0.3, seed=seed + 1, dtype=np.float32)
    x = rng.normal(size=(B, T, F)).astype(np.float32)
    y = rng.normal(size=(B, T, O)).astype(np.float32)
    y[0, :2, :] = 0.0          # zero-padded steps -> loss mask 0
    return params, x, y


def dump(out):
    import torch
    from lfm_quant_b200.engine import ForecasterEngine
    os.makedirs(out, exist_ok=True)
    kw = dict(seq_len=T, n_inputs=F, n_outputs=O, num_hidden=H, precision='bf16')
    for B in BATCHES:
        params, x, y = _problem(B, seed=B)
        xd, yd = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()
        eng = ForecasterEngine(max_batch=B, target_idx=3, train=False, forward_only=True, **kw)
        eng.set_weights(params)
        np.save(os.path.join(out, 'pred_B%d.npy' % B), eng.forward(xd).cpu().numpy())
        eng.close()
        for dropout in DROPOUTS:
            eng = ForecasterEngine(max_batch=B, target_idx=O - 1, dropout=dropout, **kw)
            eng.set_weights(params)
            eng.backward(xd, yd, step=3)
            arrays = {'g%d_%s' % (i, s[0]): g for i, (s, g) in enumerate(zip(eng.trainable_specs, eng.grads_list()))}
            arrays['tail'] = eng.grads[eng.n_trainable:eng.n_trainable + 2].cpu().numpy()
            np.savez(os.path.join(out, 'train_B%d_drop%g.npz' % (B, dropout)), **arrays)
            eng.close()
        print('B=%d written' % B, flush=True)


def _maxdiff(a, b):
    return float(np.max(np.abs(a.astype(np.float64) - b.astype(np.float64)))) if a.size else 0.0


def compare(da, db):
    bad = []
    for B in BATCHES:
        name = 'pred_B%d.npy' % B
        a, b = np.load(os.path.join(da, name)), np.load(os.path.join(db, name))
        ok = np.isfinite(a).all() and np.array_equal(a, b)
        print('%-26s %s  max|diff| %.3e' % (name, 'bit-identical' if ok else 'DIFFERS', _maxdiff(a, b)))
        bad += [] if ok else [name]
        for dropout in DROPOUTS:
            name = 'train_B%d_drop%g.npz' % (B, dropout)
            za, zb = np.load(os.path.join(da, name)), np.load(os.path.join(db, name))
            assert sorted(za.files) == sorted(zb.files), (za.files, zb.files)
            for key in sorted(za.files):
                a, b = za[key], zb[key]
                lstm = key.startswith('g') and int(key[1:].split('_')[0]) < N_LSTM
                if lstm:
                    ok = np.isfinite(a).all() and np.array_equal(a, b)
                    verdict = 'bit-identical' if ok else 'DIFFERS'
                else:
                    scale = max(float(np.max(np.abs(b))), 1e-30)
                    rel = _maxdiff(a, b) / scale
                    ok = np.isfinite(a).all() and rel <= HEAD_TOL
                    verdict = 'rel %.2e' % rel + ('' if ok else ' > %g' % HEAD_TOL)
                print('%-26s %-12s %s' % (name, key, verdict))
                bad += [] if ok else ['%s:%s' % (name, key)]
    print('OK' if not bad else 'MISMATCH: %s' % ', '.join(bad))
    return 0 if not bad else 1


def main():
    ap = argparse.ArgumentParser()
    g = ap.add_mutually_exclusive_group(required=True)
    g.add_argument('--out', metavar='DIR')
    g.add_argument('--compare', nargs=2, metavar=('DIR_A', 'DIR_B'))
    a = ap.parse_args()
    if a.out:
        dump(a.out)
        return 0
    return compare(*a.compare)


if __name__ == '__main__':
    sys.exit(main())
