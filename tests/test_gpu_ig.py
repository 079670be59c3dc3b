"""Integrated-gradients attributions of the point forecast (lfmq_integrated_gradients, ForecasterEngine.
integrated_gradients, NativeForecaster.attribute, --ig_steps): attr[b,t,f] = x[b,t,f] (1/M) sum_k df/dx[t,f] at
alpha_k x[b], alpha_k = (k + 1/2) / M, f = pred[b, T-1, target_idx], baseline 0.

Checked here: the fp64 oracle (tests/ig_oracle.py) at both precisions; the completeness gap against the oracle's; the
same bits across launch sizes, batch order, slices and repeated calls, with f_x and f_base equal to forward's target
column; the handle's state left untouched; the refused handles; and the CLI's attributions.npz."""
import ctypes
import os

import numpy as np
import pandas as pd
import pytest
import torch

import ig_oracle as igo
from util import make_problem, rel_err

pytestmark = pytest.mark.gpu
KW = dict(target_lambda=0.5, rnn_lambda=0.7, dropout=0.2, recurrent_dropout=0.15, seed=31)   # dropout off: train=0
# max abs error over max abs value against fp64 (tf32: the tf32 path's gradient bound).  Worst measured over CASES on
# an H100 80GB HBM3 at 700 W: fp32 8.7e-7, tf32 3.3e-3; the fp32 completeness gap against the oracle's 2.6e-6 of
# max |f_x - f_base| (DESIGN.md section 5d)
TOL = {'fp32': 1e-4, 'tf32': 1.1e-2}


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).cuda()


def _problem(B, T, F, O, H, L, cell, seed):
    P, x, y = make_problem(B, T, F, O, H, L, seed=seed, rnn_cell=cell)
    rng = np.random.RandomState(seed + 100)
    bn = dict(bn_mean=[rng.normal(size=H).astype(np.float32) * 0.3 for _ in range(L)],       # away from (0, 1)
              bn_var=[rng.uniform(0.4, 2.5, size=H).astype(np.float32) for _ in range(L)])
    return P, x, y, bn


def _engine(max_batch, T, F, O, H, L, cell, prec, P, bn, target_idx=1, **kw):
    from lfm_quant_b200.engine import ForecasterEngine
    args = dict(KW, train=False, forward_only=False)
    args.update(kw)
    eng = ForecasterEngine(max_batch=max_batch, seq_len=T, n_inputs=F, n_outputs=O, num_hidden=H, num_layers=L,
                           rnn_cell=cell, precision=prec, target_idx=target_idx, **args)
    eng.set_weights(P, bn_stats=list(zip(bn['bn_mean'], bn['bn_var'])))
    return eng


def _np(outs):
    return [t.cpu().numpy() for t in outs]


# (cell, L, M, B, T, F, O): every value of each axis appears; H = 64
CASES = [('lstm', 1, 8, 129, 5, 33, 17), ('gru', 2, 8, 129, 5, 33, 17), ('lstm', 2, 32, 1, 48, 1, 1),
         ('gru', 1, 1, 1, 48, 33, 17), ('lstm', 1, 32, 4096, 48, 33, 17), ('gru', 2, 1, 4096, 5, 1, 1),
         ('lstm', 2, 1, 129, 48, 1, 17), ('gru', 1, 32, 129, 48, 33, 1)]


@pytest.mark.parametrize('prec', ['fp32', 'tf32'])
@pytest.mark.parametrize('case', CASES, ids=['-'.join(map(str, c)) for c in CASES])
def test_attributions_match_the_fp64_oracle(prec, case):
    """Launches of 1000 rows (cut inside interpolants); the oracle runs three windows (a window's outputs depend on
    that window alone).  At fp32 the completeness gap also equals the oracle's at the same M."""
    cell, L, M, B, T, F, O = case
    H = 64
    P, x, _, bn = _problem(B, T, F, O, H, L, cell, seed=B + T + F)
    ti = O // 2
    eng = _engine(1000, T, F, O, H, L, cell, prec, P, bn, target_idx=ti)
    attr, f_x, f_base = _np(eng.integrated_gradients(_cuda(x), M))
    assert attr.shape == (B, T, F) and f_x.shape == (B,) and f_base.shape == (B,)
    sel = sorted({0, B // 2, B - 1})
    ref = igo.integrated_gradients(P, x[sel], M, num_layers=L, target_idx=ti, rnn_cell=cell, **bn)
    errs = [rel_err(g, r) for g, r in zip((attr[sel], f_x[sel], f_base[sel]), ref)]
    print('ig %s %s: rel err attr %.2e f_x %.2e f_base %.2e' % (prec, case, *errs))
    assert max(errs) < TOL[prec], errs
    if prec == 'fp32':
        gap = igo.completeness_gap(attr[sel].astype(np.float64), f_x[sel].astype(np.float64),
                                   f_base[sel].astype(np.float64))
        dgap = np.abs(gap - igo.completeness_gap(*ref)).max() / np.abs(ref[1] - ref[2]).max()
        print('ig %s %s: completeness gap vs oracle %.2e of |f_x - f_base|' % (prec, case, dgap))
        assert dgap < 1e-4, dgap
    eng.close()


@pytest.mark.parametrize('prec', ['fp32', 'tf32'])
@pytest.mark.parametrize('cell', ['lstm', 'gru'])
def test_same_bits_whatever_the_launches_order_or_batch(prec, cell):
    B, T, F, O, H, L, M = 37, 6, 8, 4, 64, 2, 5
    P, x, _, bn = _problem(B, T, F, O, H, L, cell, seed=3)
    xd = _cuda(x)
    res = []
    for mb in (50, B, 3 * B, M * B):
        eng = _engine(mb, T, F, O, H, L, cell, prec, P, bn)
        res.append(_np(eng.integrated_gradients(xd, M)))
        if mb == B:
            assert all(np.array_equal(a, b) for a, b in zip(res[-1], _np(eng.integrated_gradients(xd, M))))
            perm = np.random.RandomState(0).permutation(B)
            for a, b in zip(_np(eng.integrated_gradients(_cuda(x[perm]), M)), res[-1]):
                assert np.array_equal(a, b[perm])
            for a, b in zip(_np(eng.integrated_gradients(_cuda(x[5:20]), M)), res[-1]):
                assert np.array_equal(a, b[5:20])
            fwd = eng.forward(xd).cpu().numpy()[:, -1, 1]
            base = eng.forward(torch.zeros_like(xd)).cpu().numpy()[:, -1, 1]
            assert np.array_equal(res[-1][1], fwd) and np.array_equal(res[-1][2], base)
        eng.close()
    for r in res[1:]:
        for a, b in zip(r, res[0]):
            assert np.array_equal(a, b)


def _opt_slots(eng):
    p, n = ctypes.c_void_p(0), ctypes.c_int64(0)
    assert eng.lib.lfmq_opt_state_ptr(eng.handle, ctypes.byref(p), ctypes.byref(n)) == 0
    off = p.value - eng.workspace.data_ptr()
    return eng.workspace[off:off + 4 * n.value].view(torch.float32).cpu().numpy()


@pytest.mark.parametrize('prec', ['fp32', 'tf32'])
def test_attribution_leaves_the_handle_state_untouched(prec):
    """Parameters, the gradient buffer with its tail and the optimizer slots keep their bits, and the next train step is
    the same bits as on a handle that never attributed."""
    B, T, F, O, H, L = 64, 6, 8, 4, 64, 2
    P, x, y, bn = _problem(B, T, F, O, H, L, 'lstm', seed=7)
    xd, yd = _cuda(x), _cuda(y)
    a, b = (_engine(B, T, F, O, H, L, 'lstm', prec, P, bn, optimizer='Adam') for _ in range(2))
    for e in (a, b):
        e.train_step(xd, yd, 0, 0.01)
    before = (a.params.cpu().numpy(), a.grads.cpu().numpy(), _opt_slots(a))
    a.integrated_gradients(xd, 8)
    after = (a.params.cpu().numpy(), a.grads.cpu().numpy(), _opt_slots(a))
    for u, w in zip(before, after):
        assert np.array_equal(u, w)
    la, lb = a.train_step(xd, yd, 1, 0.01).cpu().numpy(), b.train_step(xd, yd, 1, 0.01).cpu().numpy()
    assert np.array_equal(la, lb)
    for u, w in zip((a.params, a.grads), (b.params, b.grads)):
        assert torch.equal(u, w)
    assert np.array_equal(_opt_slots(a), _opt_slots(b))
    a.close()
    b.close()


def test_refused_handles():
    from lfm_quant_b200 import _native as N
    from lfm_quant_b200.engine import DenseEngine
    T, F, O, H, L = 4, 6, 3, 64, 1
    P, x, _, bn = _problem(8, T, F, O, H, L, 'lstm', seed=1)
    xd = _cuda(x)
    for kw, code in ((dict(precision='bf16'), 3), (dict(precision='bf16x3', forward_only=True), 3),
                     (dict(forward_only=True), 1), (dict(train=True), 1)):
        prec = kw.pop('precision', 'fp32')
        eng = _engine(8, T, F, O, H, L, 'lstm', prec, P, bn, **kw)
        with pytest.raises(N.LfmqError, match='lfmq error %d' % code):
            eng.integrated_gradients(xd, 4)
        eng.close()
    from lfm_quant_b200.engine import ForecasterEngine
    uq = ForecasterEngine(max_batch=8, seq_len=T, n_inputs=F, n_outputs=O, num_hidden=H, uq=True, train=False)
    with pytest.raises(N.LfmqError, match='lfmq error 1'):
        uq.integrated_gradients(xd, 4)
    uq.close()
    dense = DenseEngine(max_batch=8, seq_len=T, n_inputs=F, n_outputs=O)
    n = ctypes.c_uint64(0)
    assert dense.lib.lfmq_integrated_gradients_work_bytes(dense.handle, 8, 4, ctypes.byref(n)) == 1
    dense.close()
    eng = _engine(8, T, F, O, H, L, 'lstm', 'fp32', P, bn)
    with pytest.raises(N.LfmqError, match='lfmq error 1'):
        eng.integrated_gradients(xd, 0)
    out = torch.empty(8 * T * F, device='cuda')
    rc = eng.lib.lfmq_integrated_gradients(eng.handle, xd.data_ptr(), 8, 4, out.data_ptr(), out.data_ptr(),
                                           out.data_ptr(), out.data_ptr(), 16, None)
    assert rc == 4 and b'work needs' in eng.lib.lfmq_last_error()
    eng.close()


def _model_cfg(argv):
    from lfm_quant_b200.scripts import base_config
    return base_config.get_configs(['--num_hidden', '64', '--num_layers', '1', '--batch_size', '16', '--dropout', '0.1']
                                   + argv)


def test_attribute_of_the_model_object():
    """The IG engine is fp32 for an fp32 or bf16 model and tf32 for a tf32 one, follows set_weights, and refuses uq and
    multi-step models."""
    from lfm_quant_b200.scripts.models.point_estimate.rnn_point_estimate import NativeForecaster
    T, F, O = 5, 12, 6
    x = np.random.RandomState(0).normal(size=(40, T, F)).astype(np.float32)
    for prec, ig_prec in (('fp32', 'fp32'), ('bf16', 'fp32'), ('tf32', 'tf32')):
        m = NativeForecaster(_model_cfg(['--train=False', '--precision', prec]), T, F, O, 2)
        attr, f_x, f_base = m.attribute(x, 4)
        assert m._ig_engine.precision == ig_prec and m._ig_engine.cfg.max_batch == 64
        assert attr.shape == (40, T, F) and f_x.shape == (40,)
        w = m.get_weights()
        w[0] = w[0] * 0.5
        m.set_weights(w)
        attr2 = m.attribute(x, 4)[0]
        assert not torch.equal(attr, attr2)
        ref = m._ig_engine.integrated_gradients(_cuda(x), 4)[0]
        assert torch.equal(attr2, ref)
        m.close()
    uq = NativeForecaster(_model_cfg(['--train=False', '--nn_type', 'RNNUqRangeEstimate', '--UQ=True']), T, F, O, 0,
                          uq=True)
    with pytest.raises(ValueError, match='attribute'):
        uq.attribute(x, 4)
    uq.close()


@pytest.fixture(scope='module')
def workdir(tmp_path_factory):
    from lfm_quant_b200.scripts.synthetic import write_open_dataset, write_system_test_conf
    d = tmp_path_factory.mktemp('ig')
    write_open_dataset(str(d / 'datasets' / 'open-dataset.dat'), n_keys=30, n_months=420, seed=9)
    write_system_test_conf(str(d / 'config' / 'system-test.conf'), str(d / 'datasets'), str(d / 'experiments'))
    os.environ.setdefault('LFM_QUANT_ROOT', str(d))
    return d


def test_cli_ig_steps(workdir):
    """Train at fp32, then predict with --ig_steps 16 at fp32 and tf32: preds.dat is byte for byte the file without the
    flag, and attributions.npz holds one row per preds.dat row, in its (date, gvkey) order, equal to
    NativeForecaster.attribute on the same batches of a model of that precision."""
    from lfm_quant_b200.scripts import configs
    from lfm_quant_b200.scripts import lfm_quant as cli
    from lfm_quant_b200.scripts.data_processing import Dataset
    from lfm_quant_b200.scripts.predict import Predict
    conf = str(workdir / 'config' / 'system-test.conf')
    extra = ['--model_dir', 'ig', '--dropout', '0.1']
    mdir = workdir / 'experiments' / 'ig'
    configs.reset()
    cli.main(['--config=' + conf, '--train=True'] + extra)
    configs.reset()
    cli.main(['--config=' + conf, '--train=False'] + extra)
    plain = (mdir / 'pred' / 'preds.dat').read_bytes()
    assert not (mdir / 'pred' / 'attributions.npz').exists()
    files = {}
    for prec in ('fp32', 'tf32'):
        flags = ['--ig_steps', '16', '--precision', prec]
        configs.reset()
        cli.main(['--config=' + conf, '--train=False'] + extra + flags)
        if prec == 'fp32':
            assert (mdir / 'pred' / 'preds.dat').read_bytes() == plain
        files[prec] = dict(np.load(mdir / 'pred' / 'attributions.npz'))
        df = pd.read_csv(mdir / 'pred' / 'preds.dat', sep=' ', dtype={'gvkey': str})
        z = files[prec]
        N = len(df)
        assert z['attr'].shape[0] == N and z['f_x'].shape == (N,) and z['f_base'].shape == (N,)
        assert np.array_equal(z['date'], df['date'].values) and list(z['gvkey']) == list(df['gvkey'])

        configs.reset()
        c = cli.get_configs(['--config=' + conf, '--train=False'] + extra + flags)
        p = Predict(c, Dataset(c))
        assert list(z['fields']) == p.dataset.fin_col_names + p.dataset.aux_col_names
        assert z['attr'].shape[1:] == (p.seq_len, p.n_inputs)
        p.model.load_weights(os.path.join(p.chkpts_dir, 'chkpt'))
        ref = [np.concatenate(v) for v in zip(*[_np(p.model.attribute(inp, 16)) for inp, _, _ in p._batches])]
        assert p.model._ig_engine.precision == prec
        for key, r in zip(('attr', 'f_x', 'f_base'), ref):
            assert np.array_equal(z[key], r), key
        gap = np.abs(z['attr'].reshape(N, -1).sum(1) - (z['f_x'] - z['f_base']))
        print('ig cli %s: %d rows, completeness gap max %.2e, max |f_x - f_base| %.2e'
              % (prec, N, gap.max(), np.abs(z['f_x'] - z['f_base']).max()))
        p.model.close()
    assert not np.array_equal(files['fp32']['attr'], files['tf32']['attr'])
    configs.reset()
