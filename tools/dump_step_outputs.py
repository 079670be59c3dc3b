"""What each execution path computes for one step, written out so that two builds can be compared.

    python tools/dump_step_outputs.py --out DIR          # the build LFMQ_LIB_PATH selects (default: the in-tree one)
    python tools/dump_step_outputs.py --compare DIR_A DIR_B

With seeded inputs and weights:
  - the bf16 cluster path at the benchmark's shape, for B in {4096, 3940, 1000} at T=48 (30 tiles + 4 half tiles, 30
    tiles + 2 half tiles with a partial last one, 16 half tiles): the predictions of a forward-only handle, and for
    dropout 0 and 0.2 the gradients of one backward (grads_list()) with the {loss, mse_0} tail of the gradient vector;
  - the bf16 general path at BASELINE configs[2] (H=512, two layers, dropout 0.2, B=4096, T=48): the same;
  - the fp32 and tf32 steps of a point LSTM and of a two-step RNNUqRangeEstimate chain (B=256, T=48, H=64, dropout
    0.2): the predictions (and variances) of one forward, every stage's gradient vector with its loss tail, and the
    losses one backward returns.

--compare requires predictions and the recurrent layers' gradients to be bit-identical on every path.  On the fp32 and
tf32 paths, whose loss reductions run in a fixed order, it requires everything else to be bit-identical too.  On the
bf16 paths it requires the head and BatchNormalization gradients and the loss to agree to 1e-5 relative (to the
tensor's largest entry): those are sums over rows through the head's shared-memory atomics, whose order varies from run
to run.  Exit status 1 if anything differs beyond that.
"""
import argparse
import glob
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'oracle'))

BATCHES = (4096, 3940, 1000)
DROPOUTS = (0.0, 0.2)
T, F, O, H = 48, 32, 16, 256
GENERAL = dict(B=4096, H=512, L=2, dropout=0.2)      # BASELINE configs[2]
SMALL = dict(B=256, H=64)                            # the fp32 / tf32 steps
HEAD_TOL = 1e-5


def _problem(B, seed, L=1, hidden=H, uq=False, stages=1):
    import lfm_oracle as orc
    rng = np.random.RandomState(seed)
    params = orc.init_params(L, F, O, hidden, init_scale=0.3, seed=seed + 1, dtype=np.float32, uq=uq)
    for s in range(1, stages):         # one recurrent layer and the heads per extra stage
        params += orc.init_params(1, F, O, hidden, init_scale=0.3, seed=seed + 1 + 7 * s, dtype=np.float32, uq=uq)
    x = rng.normal(size=(B, T, F)).astype(np.float32)
    ys = []
    for _ in range(stages):
        y = rng.normal(size=(B, T, O)).astype(np.float32)
        if not uq:
            y[0, :2, :] = 0.0          # zero-padded steps -> loss mask 0 (the uq loss of a masked row is NaN)
        ys.append(y)
    return params, x, ys


def _grads(eng, prefix=''):
    arrays = {'g_%s%s' % (prefix, s[0]): g for s, g in zip(eng.trainable_specs, eng.grads_list())}
    arrays[prefix + 'tail'] = eng.grads[eng.n_trainable:].cpu().numpy()
    return arrays


def _dump_bf16(out, name, B, L, hidden, dropouts, seed):
    import torch
    from lfm_quant_b200.engine import ForecasterEngine
    kw = dict(seq_len=T, n_inputs=F, n_outputs=O, num_hidden=hidden, num_layers=L, precision='bf16')
    params, x, (y,) = _problem(B, seed, L=L, hidden=hidden)
    xd, yd = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()
    eng = ForecasterEngine(max_batch=B, target_idx=3, train=False, forward_only=True, **kw)
    eng.set_weights(params)
    np.savez(os.path.join(out, 'bf16_%s_pred.npz' % name), pred=eng.forward(xd).cpu().numpy())
    eng.close()
    for dropout in dropouts:
        eng = ForecasterEngine(max_batch=B, target_idx=O - 1, dropout=dropout, **kw)
        eng.set_weights(params)
        eng.backward(xd, yd, step=3)
        np.savez(os.path.join(out, 'bf16_%s_train_drop%g.npz' % (name, dropout)), **_grads(eng))
        eng.close()


def _dump_exact(out, precision, uq):
    import torch
    from lfm_quant_b200.engine import ForecastChainEngine, ForecasterEngine
    B, hidden = SMALL['B'], SMALL['H']
    stages = 2 if uq else 1
    params, x, ys = _problem(B, 17 + stages, hidden=hidden, uq=uq, stages=stages)
    kw = dict(max_batch=B, seq_len=T, n_inputs=F, n_outputs=O, num_hidden=hidden, target_idx=3, precision=precision,
              dropout=0.2, seed=521)
    xd, yds = torch.from_numpy(x).cuda(), [torch.from_numpy(y).cuda() for y in ys]
    if uq:
        eng = ForecastChainEngine(forecast_steps=stages, weights=[1.0, 0.5], uq=True, **kw)
        eng.set_weights(params)
        arrays = {'pred%d' % i: p.cpu().numpy() for i, p in enumerate(eng.forward(xd, step=3))}
        arrays['loss'] = eng.backward(xd, yds, step=3).cpu().numpy()
        for s, st in enumerate(eng.stages):
            arrays.update(_grads(st, 's%d_' % s))
    else:
        eng = ForecasterEngine(**kw)
        eng.set_weights(params)
        arrays = {'pred': eng.forward(xd, step=3).cpu().numpy()}
        eng.backward(xd, yds[0], step=3)
        arrays.update(_grads(eng))
    np.savez(os.path.join(out, 'exact_%s_%s.npz' % (precision, 'uq_chain2' if uq else 'point')), **arrays)
    eng.close()


def dump(out):
    os.makedirs(out, exist_ok=True)
    for B in BATCHES:
        _dump_bf16(out, 'cluster_B%d' % B, B, 1, H, DROPOUTS, seed=B)
        print('cluster B=%d written' % B, flush=True)
    g = GENERAL
    _dump_bf16(out, 'general', g['B'], g['L'], g['H'], (g['dropout'],), seed=7)
    print('general written', flush=True)
    for precision in ('fp32', 'tf32'):
        for uq in (False, True):
            _dump_exact(out, precision, uq)
    print('fp32 / tf32 written', flush=True)


def _maxdiff(a, b):
    return float(np.max(np.abs(a.astype(np.float64) - b.astype(np.float64)))) if a.size else 0.0


def compare(da, db):
    bad = []
    names = sorted(os.path.basename(p) for p in glob.glob(os.path.join(da, '*.npz')))
    assert names == sorted(os.path.basename(p) for p in glob.glob(os.path.join(db, '*.npz'))), 'different file sets'
    for name in names:
        za, zb = np.load(os.path.join(da, name)), np.load(os.path.join(db, name))
        assert sorted(za.files) == sorted(zb.files), (za.files, zb.files)
        for key in sorted(za.files):
            a, b = za[key], zb[key]
            exact = name.startswith('exact_') or key.startswith(('pred', 'g_lstm_', 'g_gru_'))
            if exact:
                ok = np.isfinite(a).all() and np.array_equal(a, b)
                verdict = 'bit-identical' if ok else 'DIFFERS max|diff| %.3e' % _maxdiff(a, b)
            else:
                scale = max(float(np.max(np.abs(b))), 1e-30)
                rel = _maxdiff(a, b) / scale
                ok = np.isfinite(a).all() and rel <= HEAD_TOL
                verdict = 'rel %.2e' % rel + ('' if ok else ' > %g' % HEAD_TOL)
            print('%-34s %-40s %s' % (name, key, verdict))
            bad += [] if ok else ['%s:%s' % (name, key)]
    print('OK (%d files)' % len(names) if not bad else 'MISMATCH: %s' % ', '.join(bad))
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
