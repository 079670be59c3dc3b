"""GPU tests of the bf16 tensor-core path (LFMQ_PREC_BF16): wgmma gate GEMMs with bf16 operands, fp32 accumulate.

bf16 operands carry 8 mantissa bits, so these tests use a bf16-level tolerance against the fp64 oracle (the fp32
parity mode is held to 1e-4 in test_gpu_parity.py) and additionally check the tensor-core path against the fp32
CUDA path at the BASELINE sizes.
"""
import numpy as np
import pytest
import torch

import lfm_oracle as orc
from util import make_engine, make_problem, rel_err

pytestmark = pytest.mark.gpu

BF16_TOL = 3e-2


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.mark.parametrize('B,T', [(300, 6), (128, 1), (700, 3)])
def test_bf16_forward_matches_oracle(B, T):
    F, O, H, L = 32, 16, 256, 1
    params, x, y = make_problem(B, T, F, O, H, L, seed=11, init_scale=0.3)
    eng = make_engine(B, T, F, O, H, L, train=False, forward_only=True, precision='bf16')
    eng.set_weights(params)
    preds = eng.forward(_cuda(x)).cpu().numpy()
    ref, _ = orc.forward(params, x.astype(np.float64), num_layers=L)
    assert np.isfinite(preds).all()
    assert rel_err(preds, ref) < BF16_TOL
    # ragged call on the same handle
    p2 = eng.forward(_cuda(x[:B - 37])).cpu().numpy()
    assert rel_err(p2, ref[:B - 37]) < BF16_TOL


def test_bf16_forward_small_inputs_and_outputs():
    B, T, F, O, H, L = 130, 4, 20, 7, 256, 1
    params, x, y = make_problem(B, T, F, O, H, L, seed=12, init_scale=0.3)
    eng = make_engine(B, T, F, O, H, L, train=False, forward_only=True, precision='bf16')
    eng.set_weights(params)
    preds = eng.forward(_cuda(x)).cpu().numpy()
    ref, _ = orc.forward(params, x.astype(np.float64), num_layers=L)
    assert rel_err(preds, ref) < BF16_TOL


def test_bf16_unsupported_shapes_fail_loudly():
    # H != 256 and L != 1 run the general tensor-core path since round 2 (tests/test_gpu_generic.py); what no tensor-core
    # path covers still fails at lfmq_create, never silently on another path
    from lfm_quant_b200._native import LfmqError
    with pytest.raises(LfmqError):
        make_engine(8, 4, 32, 16, 100, 1, precision='bf16')     # H not a multiple of 64
    with pytest.raises(LfmqError):
        make_engine(8, 4, 32, 16, 576, 1, precision='bf16')     # H > 512


def _oracle_grads(params, x, y, O, L=1, **kw):
    preds, fc = orc.forward(params, x.astype(np.float64), num_layers=L, **kw)
    loss, mse, dpred, _ = orc.loss_point_estimate(y.astype(np.float64), preds, target_idx=O - 1, target_lambda=0.5,
                                                  rnn_lambda=0.7)
    return loss, mse, orc.backward(dpred, fc, num_layers=L)


@pytest.mark.parametrize('B,T,F,O', [(300, 6, 32, 16), (128, 1, 32, 16), (200, 5, 20, 7)])
def test_bf16_gradients_match_oracle(B, T, F, O):
    H, L = 256, 1
    params, x, y = make_problem(B, T, F, O, H, L, seed=21, init_scale=0.3)
    eng = make_engine(B, T, F, O, H, L, target_idx=O - 1, precision='bf16')
    eng.set_weights(params)
    eng.backward(_cuda(x), _cuda(y))
    tail = eng.grads[eng.n_trainable:eng.n_trainable + 2].cpu().numpy()
    loss, mse, ref = _oracle_grads(params, x, y, O)
    assert tail[0] == pytest.approx(loss, rel=BF16_TOL)
    assert tail[1] == pytest.approx(mse, rel=BF16_TOL)
    for (name, _, _, _), g, r in zip(eng.trainable_specs, eng.grads_list(), ref):
        assert np.isfinite(g).all(), name
        if np.abs(r).max() == 0.0:            # e.g. dU at T=1 (h_prev = 0)
            assert np.abs(g).max() < 1e-6, name
            continue
        assert rel_err(g, r) < 2 * BF16_TOL, name
        cos = float(np.sum(g * r) / (np.linalg.norm(g) * np.linalg.norm(r) + 1e-30))
        assert cos > 0.999, (name, cos)


def test_bf16_dropout_matches_philox_oracle():
    B, T, F, O, H, L = 256, 4, 32, 16, 256, 1
    params, x, y = make_problem(B, T, F, O, H, L, seed=22, init_scale=0.3)
    eng = make_engine(B, T, F, O, H, L, target_idx=O - 1, precision='bf16', dropout=0.25, seed=99)
    eng.set_weights(params)
    eng.backward(_cuda(x), _cuda(y), step=5, row0=512)
    loss, mse, ref = _oracle_grads(params, x, y, O, dropout=0.25, training=True, seed=99, step=5, row0=512)
    tail = eng.grads[eng.n_trainable:eng.n_trainable + 2].cpu().numpy()
    assert tail[0] == pytest.approx(loss, rel=BF16_TOL)
    for (name, _, _, _), g, r in zip(eng.trainable_specs, eng.grads_list(), ref):
        assert rel_err(g, r) < 2 * BF16_TOL, name


def test_bf16_train_steps_track_oracle():
    B, T, F, O, H, L = 256, 6, 32, 16, 256, 1
    params, x, y = make_problem(B, T, F, O, H, L, seed=23, init_scale=0.3)
    cfg = dict(num_layers=L, target_idx=3, target_lambda=0.5, rnn_lambda=0.7, max_grad_norm=50.0, optimizer='SGD',
               max_norm=3.0, sgd_momentum=0.0, train=True)
    eng = make_engine(B, T, F, O, H, L, target_idx=3, optimizer='SGD', precision='bf16')
    eng.set_weights(params)
    p = [q.copy() for q in params]
    slots = orc.zero_slots('SGD', p)
    xc, yc = _cuda(x), _cuda(y)
    for it in range(3):
        out = eng.train_step(xc, yc, it, 0.05).cpu().numpy()
        p, mse, loss, raw, gn = orc.train_step(p, slots, x.astype(np.float64), y.astype(np.float64), it, cfg, lr=0.05)
        assert out[1] == pytest.approx(mse, rel=BF16_TOL), it
    for (name, _, _, _), w, r in zip(eng.trainable_specs, eng.get_weights(), p):
        assert rel_err(w, r) < BF16_TOL, name


def test_bf16_gradients_match_fp32_path_at_baseline_shape():
    """BASELINE cfg2 (B=4096, T=48): full-size BPTT on tensor cores vs the fp32 CUDA path."""
    B, T, F, O, H, L = 4096, 48, 32, 16, 256, 1
    params, x, y = make_problem(B, T, F, O, H, L, seed=24, init_scale=1.0, zero_rows=False)
    grads = {}
    for prec in ('fp32', 'bf16'):
        eng = make_engine(B, T, F, O, H, L, target_idx=3, precision=prec)
        eng.set_weights(params)
        eng.backward(_cuda(x), _cuda(y))
        grads[prec] = (eng.grads_list(), eng.grads[eng.n_trainable:eng.n_trainable + 2].cpu().numpy(),
                       [s[0] for s in eng.trainable_specs])
        eng.close()
        del eng
        torch.cuda.empty_cache()
    assert grads['bf16'][1][1] == pytest.approx(grads['fp32'][1][1], rel=BF16_TOL)
    for name, g, r in zip(grads['fp32'][2], grads['bf16'][0], grads['fp32'][0]):
        assert np.isfinite(g).all(), name
        cos = float(np.sum(g * r) / (np.linalg.norm(g) * np.linalg.norm(r) + 1e-30))
        assert cos > 0.995, (name, cos)
        assert rel_err(g, r) < 0.1, name


def test_bf16_matches_fp32_path_at_baseline_shape():
    """BASELINE cfg2 shape (B=4096, T=48, F=32, H=256): tensor-core forward vs the fp32 CUDA path."""
    B, T, F, O, H, L = 4096, 48, 32, 16, 256, 1
    params, x, y = make_problem(B, T, F, O, H, L, seed=13, init_scale=1.0, zero_rows=False)
    e32 = make_engine(B, T, F, O, H, L, train=False, forward_only=True, precision='fp32')
    e16 = make_engine(B, T, F, O, H, L, train=False, forward_only=True, precision='bf16')
    e32.set_weights(params)
    e16.set_weights(params)
    xc = _cuda(x)
    p32 = e32.forward(xc).cpu().numpy()
    p16 = e16.forward(xc).cpu().numpy()
    assert np.isfinite(p16).all()
    # error relative to the output scale, and its RMS
    scale = np.abs(p32).max()
    assert np.abs(p16 - p32).max() / scale < 6e-2
    assert np.sqrt(np.mean((p16 - p32) ** 2)) / np.sqrt(np.mean(p32 ** 2)) < 2e-2


def test_bf16_training_with_more_tiles_than_resident_clusters():
    """B = 4500 is 36 batch tiles (the last one ragged): the persistent recurrences run a second iteration per cluster,
    while clusters left without a tile in that round sit it out; this exercises the barrier phases carried across tiles
    (forward x_empty / h_written, backward exp_ready / recv_free / dpb_free) and the
    dz TMA-store coordinates of later tiles.  Gradients and loss vs the fp32 CUDA path."""
    B, T, F, O, H, L = 4500, 5, 32, 16, 256, 1
    params, x, y = make_problem(B, T, F, O, H, L, seed=31, init_scale=0.5)
    out = {}
    for prec in ('fp32', 'bf16'):
        eng = make_engine(B, T, F, O, H, L, target_idx=3, precision=prec)
        eng.set_weights(params)
        eng.backward(_cuda(x), _cuda(y))
        out[prec] = (eng.grads_list(), eng.grads[eng.n_trainable:eng.n_trainable + 2].cpu().numpy(),
                     [s[0] for s in eng.trainable_specs])
        eng.close()
    assert out['bf16'][1][0] == pytest.approx(out['fp32'][1][0], rel=BF16_TOL)
    assert out['bf16'][1][1] == pytest.approx(out['fp32'][1][1], rel=BF16_TOL)
    for name, g, r in zip(out['fp32'][2], out['bf16'][0], out['fp32'][0]):
        assert np.isfinite(g).all(), name
        cos = float(np.sum(g * r) / (np.linalg.norm(g) * np.linalg.norm(r) + 1e-30))
        assert cos > 0.999, (name, cos)
        assert rel_err(g, r) < 2 * BF16_TOL, name
