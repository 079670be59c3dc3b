"""GPU tests of tensor-core inference for the GRU cell and RNNUqRangeEstimate (csrc/rnn_tc.cu, forward-only handles):
LFMQ_PREC_BF16 and LFMQ_PREC_BF16X3 on the general path, MC dropout on uq handles, forward-only GRU chains and the CLI's
prediction run with --precision bf16x3 on models trained in fp32.

Checker = the fp64 oracle (orc.forward, orc.forward_uq, orc.forward_forecast).  Tolerances: bf16 3e-2, bf16x3 1e-4
(max-norm relative, as in test_gpu_generic.py).
"""
import os

import numpy as np
import pandas as pd
import pytest
import torch

import lfm_oracle as orc
from util import make_engine, make_problem, make_uq_problem, rel_err

pytestmark = pytest.mark.gpu

BF16_TOL = 3e-2
X3_TOL = 1e-4
TOLS = {'bf16': BF16_TOL, 'bf16x3': X3_TOL}


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).cuda()


# (B, T, F, O, H, L): every hidden size of the path, one to three layers, F not a multiple of 64, O < 16
GRU_SHAPES = [(200, 5, 20, 7, 64, 1), (130, 4, 33, 16, 128, 2), (300, 6, 32, 3, 256, 1), (129, 3, 9, 16, 512, 3),
              (140, 5, 70, 5, 192, 2)]


@pytest.mark.parametrize('precision', ['bf16', 'bf16x3'])
@pytest.mark.parametrize('shape', GRU_SHAPES)
def test_gru_forward_only_matches_oracle(shape, precision):
    B, T, F, O, H, L = shape
    params, x, _ = make_problem(B, T, F, O, H, L, seed=5, init_scale=0.5, rnn_cell='gru')
    eng = make_engine(B, T, F, O, H, L, train=False, forward_only=True, precision=precision, target_idx=O - 1,
                      rnn_cell='gru')
    eng.set_weights(params)
    preds = eng.forward(_cuda(x)).cpu().numpy()
    ref, _ = orc.forward(params, x.astype(np.float64), num_layers=L, rnn_cell='gru')
    err = rel_err(preds, ref)
    print('gru %s %s: max-norm rel err %.3e' % (precision, shape, err))
    assert np.isfinite(preds).all() and err < TOLS[precision]
    p2 = eng.forward(_cuda(x[:B - 37])).cpu().numpy()          # ragged call on the same handle
    assert rel_err(p2, ref[:B - 37]) < TOLS[precision]
    eng.close()


def test_gru_bf16x3_long_sequence_meets_the_fp32_tolerance():
    B, T, F, O, H, L = 64, 48, 32, 16, 256, 1
    params, x, _ = make_problem(B, T, F, O, H, L, seed=8, init_scale=0.5, rnn_cell='gru')
    eng = make_engine(B, T, F, O, H, L, train=False, forward_only=True, precision='bf16x3', target_idx=3, rnn_cell='gru')
    eng.set_weights(params)
    preds = eng.forward(_cuda(x)).cpu().numpy()
    ref, _ = orc.forward(params, x.astype(np.float64), num_layers=L, rnn_cell='gru')
    assert rel_err(preds, ref) < X3_TOL
    eng.close()


UQ_KW = dict(dropout=0.2, recurrent_dropout=0.1, seed=521)


@pytest.mark.parametrize('precision', ['bf16', 'bf16x3'])
@pytest.mark.parametrize('shape,cell', [((200, 6, 20, 7, 128, 2), 'lstm'), ((300, 5, 32, 16, 256, 1), 'lstm'),
                                        ((150, 6, 33, 5, 64, 1), 'gru'), ((130, 4, 32, 16, 256, 2), 'gru')])
def test_uq_forward_only_matches_oracle_with_mc_dropout(shape, cell, precision):
    B, T, F, O, H, L = shape
    params, x = make_uq_problem(B, T, F, O, H, L, seed=13, cell=cell)
    eng = make_engine(B, T, F, O, H, L, target_idx=O - 1, uq=True, rnn_cell=cell, train=False, forward_only=True,
                      precision=precision, **UQ_KW)
    eng.set_weights(params)
    xc = _cuda(x)
    pred, var = eng.forward(xc, step=4, row0=64)
    pred, var = pred.cpu().numpy(), var.cpu().numpy()
    rp, rv, _ = orc.forward_uq(params, x.astype(np.float64), num_layers=L, rnn_cell=cell, step=4, row0=64, **UQ_KW)
    tol = TOLS[precision]
    print('uq %s %s %s: pred %.3e var %.3e' % (cell, precision, shape, rel_err(pred, rp), rel_err(var, rv)))
    assert rel_err(pred, rp) < tol and rel_err(var, rv) < tol
    assert float(var.min()) >= 1e-6
    # the same (step, row0) draws the same masks: bit for bit; another step draws others
    p_again, v_again = eng.forward(xc, step=4, row0=64)
    np.testing.assert_array_equal(p_again.cpu().numpy(), pred)
    np.testing.assert_array_equal(v_again.cpu().numpy(), var)
    p_other, _ = eng.forward(xc, step=5, row0=64)
    assert rel_err(p_other.cpu().numpy(), pred) > 10 * tol
    eng.close()


@pytest.mark.parametrize('cell', ['lstm', 'gru'])
def test_uq_bf16x3_draws_the_masks_of_the_fp32_path(cell):
    """bf16x3 and fp32 handles agree to the fp32 tolerance at the same (step, row0): the Dropout and recurrent-dropout
    masks are the same sample on both paths."""
    B, T, F, O, H, L = 160, 8, 32, 16, 128, 2
    params, x = make_uq_problem(B, T, F, O, H, L, seed=17, cell=cell)
    outs = {}
    for precision in ('fp32', 'bf16x3'):
        eng = make_engine(B, T, F, O, H, L, target_idx=1, uq=True, rnn_cell=cell, train=False, forward_only=True,
                          precision=precision, **UQ_KW)
        eng.set_weights(params)
        p, v = eng.forward(_cuda(x), step=9, row0=1000)
        outs[precision] = (p.cpu().numpy(), v.cpu().numpy())
        eng.close()
    assert rel_err(outs['bf16x3'][0], outs['fp32'][0]) < X3_TOL
    assert rel_err(outs['bf16x3'][1], outs['fp32'][1]) < X3_TOL


def test_gru_chain_forward_only_bf16x3_matches_oracle():
    from lfm_quant_b200.engine import ForecastChainEngine
    B, T, F, O, H, L, S = 140, 6, 16, 8, 64, 1, 2
    rng = np.random.RandomState(3)
    P = orc.init_forecast_params(L, F, O, H, S, init_scale=0.5, seed=4, dtype=np.float64, rnn_cell='gru')
    P = [(p + rng.normal(size=p.shape) * 0.05).astype(np.float32).astype(np.float64) for p in P]
    x = rng.normal(size=(B, T, F)).astype(np.float32)
    eng = ForecastChainEngine(forecast_steps=S, weights=[1.0, 0.5], max_batch=B, seq_len=T, n_inputs=F, n_outputs=O,
                              num_hidden=H, num_layers=L, rnn_cell='gru', target_idx=1, train=False, forward_only=True,
                              precision='bf16x3')
    eng.set_weights(P)
    preds = eng.forward(_cuda(x))
    rp, _ = orc.forward_forecast(P, x.astype(np.float64), num_layers=L, forecast_steps=S, rnn_cell='gru')
    for s in range(S):
        assert rel_err(preds[s].cpu().numpy(), rp[s]) < X3_TOL, s
    eng.close()


@pytest.mark.parametrize('cell,kw', [
    ((128, 4, 32, 16, 256, 1), dict(rnn_cell='gru')),
    ((128, 4, 32, 16, 256, 1), dict(uq=True)),
])
def test_training_handles_are_still_refused(cell, kw):
    from lfm_quant_b200._native import LfmqError
    B, T, F, O, H, L = cell
    match = 'LSTM cell only' if 'rnn_cell' in kw else 'point-estimate head only'
    with pytest.raises(LfmqError, match=match):
        make_engine(B, T, F, O, H, L, precision='bf16', **kw)


# ---- the CLI: train in fp32, predict on tensor cores ------------------------------------------------------------------
@pytest.fixture(scope='module')
def cli_workdir(tmp_path_factory):
    from lfm_quant_b200.scripts.synthetic import write_open_dataset, write_system_test_conf
    d = tmp_path_factory.mktemp('infer_cells')
    write_open_dataset(str(d / 'datasets' / 'open-dataset.dat'), n_keys=30, n_months=420, seed=9)
    write_system_test_conf(str(d / 'config' / 'system-test.conf'), str(d / 'datasets'), str(d / 'experiments'))
    os.environ.setdefault('LFM_QUANT_ROOT', str(d))
    return d


@pytest.mark.parametrize('extra', [
    ['--rnn_cell', 'gru', '--model_dir', 'infer-gru'],
    ['--nn_type', 'RNNUqRangeEstimate', '--UQ=True', '--dropout', '0.1', '--recurrent_dropout', '0.1',
     '--model_dir', 'infer-uq'],
], ids=['gru', 'uq'])
def test_cli_predicts_an_fp32_trained_model_on_tensor_cores(cli_workdir, extra):
    from lfm_quant_b200.scripts import configs
    from lfm_quant_b200.scripts import lfm_quant as cli
    conf = str(cli_workdir / 'config' / 'system-test.conf')
    mdir = cli_workdir / 'experiments' / extra[extra.index('--model_dir') + 1]
    configs.reset()
    assert np.isfinite(cli.main(['--config=' + conf, '--train=True'] + extra))
    outs = {}
    for precision in ('fp32', 'bf16x3'):
        configs.reset()
        cli.main(['--config=' + conf, '--train=False', '--precision', precision] + extra)
        outs[precision] = pd.read_csv(mdir / 'pred' / 'preds.dat', sep=' ', dtype={'gvkey': str})
    configs.reset()
    a, b = outs['fp32'], outs['bf16x3']
    assert len(a) == len(b) > 100
    cols = ['norm_preds_1'] + (['norm_variance_1'] if '--UQ=True' in extra else [])
    for col in cols:
        va, vb = a[col].to_numpy(dtype=np.float64), b[col].to_numpy(dtype=np.float64)
        assert np.isfinite(vb).all(), col
        assert rel_err(vb, va) < X3_TOL, (col, rel_err(vb, va))
