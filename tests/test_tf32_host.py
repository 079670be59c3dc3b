"""LFMQ_PREC_TF32 without a GPU: the ABI constant, what the library accepts and refuses at create, the workspace, and
the rounding oracle (tests/tf32_oracle.py) against lfm_oracle."""
import ctypes as C

import numpy as np
import pytest

import lfm_oracle as orc
import tf32_oracle as t3
import uq_chain_oracle as uco
from lfm_quant_b200 import _native as N


def _cfg(**kw):
    c = N.LfmqConfig()
    c.struct_size = C.sizeof(N.LfmqConfig)
    c.max_batch, c.seq_len, c.n_inputs, c.n_outputs, c.num_hidden, c.num_layers = 32, 20, 33, 17, 64, 2
    c.target_idx = 3
    c.bn_epsilon = 1e-3
    c.train = 1
    for k, v in kw.items():
        setattr(c, k, v)
    return c


def _ws(**kw):
    n = C.c_uint64(0)
    N.check(N.load().lfmq_workspace_bytes(C.byref(_cfg(**kw)), C.byref(n)))
    return n.value


def test_tf32_constant_is_additive():
    lib = N.load()
    assert N.PREC_TF32 == 3
    assert lib.lfmq_abi_version() == 4
    n = C.c_uint64(0)
    for p in (7, 9):
        assert lib.lfmq_workspace_bytes(C.byref(_cfg(precision=p)), C.byref(n)) == 1      # LFMQ_ERR_ARG
    from lfm_quant_b200.engine import PRECISIONS
    assert PRECISIONS['tf32'] == N.PREC_TF32


@pytest.mark.parametrize('cell', [0, 1])
@pytest.mark.parametrize('uq', [0, 1])
@pytest.mark.parametrize('forward_only', [0, 1])
def test_tf32_workspace_is_the_fp32_paths(cell, uq, forward_only):
    """tf32 runs the fp32 path's buffers; its GEMMs stage every operand tile through registers, so there are no
    transposed weight copies or padding to carve: the workspace equals fp32's, and it holds the fp32 activations a
    forward-only bf16x3 handle leaves out."""
    kw = dict(rnn_cell=cell, uq=uq, forward_only=forward_only, max_batch=4096, seq_len=48, num_hidden=256)
    assert _ws(precision=N.PREC_TF32, **kw) == _ws(precision=N.PREC_FP32, **kw)
    assert _ws(precision=N.PREC_TF32, **kw) > _ws(precision=N.PREC_BF16X3, **dict(kw, forward_only=1))


def test_tf32_refuses_num_hidden_off_the_multiple_of_4():
    lib = N.load()
    n = C.c_uint64(0)
    for H in (6, 130, 1022):
        rc = lib.lfmq_workspace_bytes(C.byref(_cfg(precision=N.PREC_TF32, num_hidden=H)), C.byref(n))
        assert rc == 3, H                                                    # LFMQ_ERR_UNSUPPORTED
        assert b'multiple of 4' in lib.lfmq_last_error()
    for H in (4, 132, 1020):
        assert lib.lfmq_workspace_bytes(C.byref(_cfg(precision=N.PREC_TF32, num_hidden=H)), C.byref(n)) == 0


def test_dense_handle_refuses_tf32():
    lib = N.load()
    c = N.LfmqDenseConfig()
    c.struct_size = C.sizeof(N.LfmqDenseConfig)
    c.max_batch, c.seq_len, c.n_inputs, c.n_outputs, c.target_idx = 64, 5, 7, 3, 1
    c.precision = N.PREC_TF32
    n = C.c_uint64(0)
    assert lib.lfmq_dense_workspace_bytes(C.byref(c), C.byref(n)) == 3
    assert b'fp32 only' in lib.lfmq_last_error()


# ---- the rounding oracle -------------------------------------------------------------------------------------------
def test_round_tf32_is_nearest_ties_away():
    u = 2.0 ** -10                                   # one tf32 ulp at 1
    x = np.array([1 + u / 2, 1 + 1.5 * u, -(1 + u / 2), 1 + u / 2 - 2.0 ** -20, 1 + u / 2 + 2.0 ** -20, 3.0, 0.0])
    want = np.array([1 + u, 1 + 2 * u, -(1 + u), 1.0, 1 + u, 3.0, 0.0])
    np.testing.assert_array_equal(t3.round_tf32(x), want)
    r = t3.round_tf32(np.random.RandomState(0).normal(size=10000))
    assert not np.any(r.astype(np.float32).view(np.uint32) & 0x1FFF)


def _problem(cell, uq, S, L=2, B=5, T=6, F=7, O=3, H=8):
    rng = np.random.RandomState(S + L + (cell == 'gru'))
    if S > 1 and uq:
        P = uco.init_params(L, F, O, H, S, init_scale=0.5, seed=3, dtype=np.float64, rnn_cell=cell)
    elif S > 1:
        P = orc.init_forecast_params(L, F, O, H, S, init_scale=0.5, seed=3, dtype=np.float64, rnn_cell=cell)
    else:
        P = orc.init_params(L, F, O, H, init_scale=0.5, seed=3, dtype=np.float64, rnn_cell=cell, uq=uq)
    x = rng.normal(size=(B, T, F))
    ys = [rng.normal(size=(B, T, O)) for _ in range(S)]
    return P, x, ys


CASES = [('lstm', False, 1), ('gru', False, 1), ('lstm', True, 1), ('gru', True, 1), ('lstm', False, 2),
         ('gru', True, 2)]


def _run(cell, uq, S, P, x, ys):
    """A train step's outputs and gradients through the oracle for one model kind."""
    L = 2
    drop = dict(dropout=0.2, recurrent_dropout=0.1, seed=521, step=2, row0=9)
    lkw = dict(target_idx=2, target_lambda=0.5, rnn_lambda=0.7)
    if S == 1 and not uq:
        p, fc = orc.forward(P, x, num_layers=L, training=True, rnn_cell=cell, **drop)
        _, _, dp, _ = orc.loss_point_estimate(ys[0], p, **lkw)
        return [p], orc.backward(dp, fc, num_layers=L, rnn_cell=cell)
    if S == 1:
        p, v, fc = orc.forward_uq(P, x, num_layers=L, rnn_cell=cell, **drop)
        _, _, _, dp, dv = orc.loss_uq_estimate(ys[0], p, v, **lkw)
        return [p, v], orc.backward_uq(dp, dv, fc, num_layers=L, rnn_cell=cell)
    if not uq:
        ps, fc = orc.forward_forecast(P, x, num_layers=L, forecast_steps=S, training=True, rnn_cell=cell, **drop)
        _, _, dps = orc.loss_forecast(ys, ps, [1.0, 0.5], **lkw)
        return ps, orc.backward_forecast(dps, fc, rnn_cell=cell)
    ps, vs, fc = uco.forward(P, x, num_layers=L, forecast_steps=S, rnn_cell=cell, **drop)
    _, _, _, dps, dvs = uco.loss(ys, ps, vs, [1.0, 0.5], **lkw)
    return ps + vs, uco.backward(dps, dvs, fc, rnn_cell=cell)


@pytest.mark.parametrize('cell,uq,S', CASES)
def test_rounding_oracle_without_rounding_is_lfm_oracle(cell, uq, S):
    """rounding(False) runs the same Tf32Array machinery with nothing rounded: bit-equal to lfm_oracle.  With rounding,
    every output and gradient moves by about tf32's unit roundoff (2^-11) and no more than 1e-2 relative."""
    P, x, ys = _problem(cell, uq, S)
    ref_o, ref_g = _run(cell, uq, S, P, x, ys)
    with t3.rounding(False):
        o, g = t3.call(_run, cell, uq, S, P, x, ys)
    for a, b in zip(o + g, ref_o + ref_g):
        assert type(a) is np.ndarray
        np.testing.assert_array_equal(a, b)
    with t3.rounding():
        o, g = t3.call(_run, cell, uq, S, P, x, ys)
    worst = max(np.abs(a - b).max() / np.abs(b).max() for a, b in zip(o + g, ref_o + ref_g) if np.any(b))
    assert 1e-6 < worst < 1e-2, worst
    assert orc.np is np and uco.np is np
