"""The two baselines on the GPU: the dense handle (MLPLinearPointEstimate's Dense(O) over the flattened window, its
MLP-branch loss and gradients, the optimizer) against the fp64 oracle in tests/dense_oracle.py, its determinism and
data-parallel decomposition, the naive forecast, and both models through the CLI on the synthetic dataset."""
import os
import shutil
import tempfile

import numpy as np
import pandas as pd
import pytest
import torch

import dense_oracle as do
import lfm_oracle as orc
from lfm_quant_b200 import _native as N
from lfm_quant_b200.engine import DenseEngine
from lfm_quant_b200.scripts import configs
from lfm_quant_b200.scripts import lfm_quant as cli
from lfm_quant_b200.scripts.synthetic import write_open_dataset, write_system_test_conf

pytestmark = pytest.mark.gpu

# (B, T, F, O): tiny, the CLI's (batch 32, T = 20, 16 financial + 16 aux fields), and B = 4096 at T = 48 whose
# weight gradient sums 32 row-block partials; O = 17 takes two column passes
SHAPES = [(5, 3, 4, 1), (32, 20, 32, 16), (4096, 48, 32, 16), (4096, 48, 300, 17), (4096, 48, 32, 7),
          (300, 6, 20, 17), (257, 4, 7, 1), (100, 80, 30, 3)]


def rel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-30))


def _problem(B, T, F, O, seed, scale=0.1):
    rng = np.random.RandomState(seed)
    x = rng.normal(size=(B, T * F)).astype(np.float32)
    W = rng.uniform(-scale, scale, size=(T * F, O)).astype(np.float32)
    b = rng.normal(scale=0.1, size=O).astype(np.float32)
    y = (x[:, -F:][:, :O] + rng.normal(size=(B, O))).astype(np.float32)
    y[::7] = 0.0                                        # rows whose targets are all zero
    return x, W, b, y


def _engine(B, T, F, O, **kw):
    e = DenseEngine(max_batch=B, seq_len=T, n_inputs=F, n_outputs=O, **kw)
    return e


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.mark.parametrize('shape', SHAPES)
@pytest.mark.parametrize('lam,huber', [(0.0, False), (0.5, False), (1.0, False), (0.5, True)])
def test_forward_loss_and_gradients_match_the_oracle(shape, lam, huber):
    B, T, F, O = shape
    tidx = O - 1 if O > 1 else 0
    x, W, b, y = _problem(B, T, F, O, seed=B + F + O)
    ref = do.dense_forward(x, W, b)
    r = np.abs(y - ref * (~np.all(y == 0, axis=1))[:, None])
    delta = float(np.median(r[r > 0]))                 # Huber residuals on both sides of delta
    e = _engine(B, T, F, O, target_idx=tidx, target_lambda=lam, huber_loss=huber, huber_delta=delta)
    e.set_weights([W, b])
    xd, yd = _cuda(x), _cuda(y)
    pred = e.forward(xd).cpu().numpy()
    assert rel(pred, ref) <= 1e-4
    kw = dict(target_idx=tidx, target_lambda=lam)
    out = e.loss(_cuda(ref.astype(np.float32)), yd).cpu().numpy()          # validation: MSE form
    assert rel(out, do.mlp_loss(y, ref.astype(np.float32), **kw)) <= 1e-4
    e.backward(xd, yd)
    tail = e.grads[e.n_trainable:e.n_trainable + 2].cpu().numpy()
    hk = dict(kw, huber=huber, huber_delta=delta)
    loss, mse0 = do.mlp_loss(y, ref, **hk)
    assert rel(tail[0], loss) <= 1e-4 and rel(tail[1], mse0) <= 1e-4
    dW, db = do.dense_grads(x, do.mlp_loss_grad(y, ref, **hk))
    gW, gb = e.grads_list()
    assert rel(gW, dW) <= 1e-4 and rel(gb, db) <= 1e-4


@pytest.mark.parametrize('opt,mom', [('Adadelta', 0.0), ('Adam', 0.0), ('SGD', 0.9)])
def test_three_train_steps_match_the_oracle(opt, mom):
    B, T, F, O, tidx, lr = 512, 12, 16, 6, 2, {'Adadelta': 0.6, 'Adam': 1e-3, 'SGD': 0.05}[opt]
    x, W, b, y = _problem(B, T, F, O, seed=5)
    clip = 0.05
    e = _engine(B, T, F, O, target_idx=tidx, target_lambda=0.5, optimizer=opt, sgd_momentum=mom, max_grad_norm=clip)
    e.set_weights([W, b])
    params = [W.astype(np.float64), b.astype(np.float64)]
    slots = orc.zero_slots(opt, params)
    for it in range(3):
        xs, ys = x[it * 160:it * 160 + 160], y[it * 160:it * 160 + 160]
        out = e.train_step(_cuda(xs), _cuda(ys), it, lr).cpu().numpy()
        gn = e.grads[e.n_trainable + 2].item()
        assert gn > clip                                # the clip bites
        params, loss, mse0 = do.train_step(params, slots, xs, ys, it, target_idx=tidx, target_lambda=0.5,
                                           optimizer=opt, lr=lr, max_grad_norm=clip, sgd_momentum=mom)
        assert rel(out[0], loss) <= 1e-4 and rel(out[1], mse0) <= 1e-4
        for w, r in zip(e.get_weights(), params):
            assert rel(w, r) <= 5e-4


def test_deterministic_and_row_independent():
    B, T, F, O = 4096, 48, 32, 16
    x, W, b, y = _problem(B, T, F, O, seed=9)
    e = _engine(B, T, F, O, target_idx=3)
    e.set_weights([W, b])
    xd, yd = _cuda(x), _cuda(y)
    e.backward(xd, yd)
    g1 = e.grads.clone()
    e.backward(xd, yd)
    assert torch.equal(g1, e.grads)                     # bit-identical
    p = e.forward(xd)
    perm = torch.from_numpy(np.random.RandomState(1).permutation(B)).cuda()
    assert torch.equal(e.forward(xd[perm].contiguous()), p[perm])
    for s0, n in ((0, 1), (17, 5), (1000, 999), (4095, 1)):
        assert torch.equal(e.forward(xd[s0:s0 + n].contiguous()), p[s0:s0 + n])


def test_row_slices_with_global_denominators_sum_to_the_full_batch():
    B, T, F, O = 1000, 10, 12, 5
    x, W, b, y = _problem(B, T, F, O, seed=4)
    e = _engine(B, T, F, O, target_idx=1, huber_loss=True, huber_delta=0.5)
    e.set_weights([W, b])
    xd, yd = _cuda(x), _cuda(y)
    e.backward(xd, yd)
    full = e.grads[:e.n_trainable + 2].double().clone()
    denom = e.mask_count(yd)
    assert denom.cpu().numpy().tolist() == [B, float((~np.all(y == 0, axis=1)).sum())]
    acc = torch.zeros_like(full)
    for a, z in ((0, 333), (333, 640), (640, 1000)):
        e.backward(xd[a:z].contiguous(), yd[a:z].contiguous(), row0=a, denom=denom)
        acc += e.grads[:e.n_trainable + 2].double()
    assert float((acc - full).abs().max() / full.abs().max()) <= 1e-6


def test_one_rank_gloo_train_step_dp_equals_train_step():
    import torch.distributed as dist
    B, T, F, O = 256, 8, 10, 4
    x, W, b, y = _problem(B, T, F, O, seed=2)
    a, c = (_engine(B, T, F, O, target_idx=2, max_grad_norm=0.1) for _ in range(2))
    a.set_weights([W, b])
    c.set_weights([W, b])
    init = tempfile.mktemp()
    dist.init_process_group('gloo', init_method='file://' + init, rank=0, world_size=1)
    try:
        xd, yd = _cuda(x), _cuda(y)
        for it in range(2):
            got = a.train_step_dp(xd, yd, it, 0.6, 0, a.loss_counts(yd))
            ref = c.train_step(xd, yd, it, 0.6)
            assert torch.equal(got, ref)
            assert torch.equal(a.params, c.params)
    finally:
        dist.destroy_process_group()
        os.path.exists(init) and os.remove(init)


def test_dense_handle_refuses_tensor_core_precisions():
    for prec in ('bf16', 'bf16x3'):
        with pytest.raises(N.LfmqError, match='fp32 only'):
            _engine(64, 4, 5, 3, precision=prec)


# ---- the CLI on the synthetic dataset --------------------------------------------------------------------------------
PRED_TAIL = ['targets_1', 'norm_preds_1', 'norm_variance_1', 'norm_targets_1', 'norm_squared_diff_1', 'preds_1',
             'variance_1', 'fcst_err_1', 'abs_err_1', 'unscaled_squared_err_1']


@pytest.fixture(scope='module')
def workdir(tmp_path_factory):
    d = tmp_path_factory.mktemp('baselines')
    write_open_dataset(str(d / 'datasets' / 'open-dataset.dat'), n_keys=30, n_months=420, seed=9)
    write_system_test_conf(str(d / 'config' / 'system-test.conf'), str(d / 'datasets'), str(d / 'experiments'))
    os.environ.setdefault('LFM_QUANT_ROOT', str(d))
    return d


def _main(workdir, *args):
    configs.reset()
    try:
        return cli.main(['--config=' + str(workdir / 'config' / 'system-test.conf')] + list(args))
    finally:
        configs.reset()


MLP = ['--nn_type', 'MLPLinearPointEstimate', '--init_scale', '0.02', '--max_epoch', '3']


def _preds(workdir, model_dir):
    return pd.read_csv(workdir / 'experiments' / model_dir / 'pred' / 'preds.dat', sep=' ', dtype={'gvkey': str})


def test_cli_mlp_linear_trains_predicts_and_restores_from_the_tf_container(workdir):
    valid = _main(workdir, *MLP, '--model_dir', 'mlp', '--train=True')
    mdir = workdir / 'experiments' / 'mlp'
    ep = pd.read_csv(mdir / 'train_log' / 'system-test-train-logs-epoch.csv')
    assert np.isfinite(valid) and np.isfinite(ep['valid_mse']).all()
    assert ep['valid_mse'].iloc[-1] < ep['valid_mse'].iloc[0]                   # it learns
    w = np.load(mdir / 'chkpts' / 'chkpt.lfmq.npz')
    assert sorted(w.files) == ['OUTPUT_1/bias', 'OUTPUT_1/kernel'] and w['OUTPUT_1/kernel'].shape == (20 * 32, 16)

    _main(workdir, *MLP, '--model_dir', 'mlp', '--train=False')
    out = _preds(workdir, 'mlp')
    cols = list(out.columns)
    assert cols[:3] == ['date', 'gvkey', 'seq_norm'] and cols[-10:] == PRED_TAIL
    assert cols[3:-10] == ['inp_t%d' % t for t in range(-19, 1)]
    assert len(out) > 100 and np.isfinite(out['norm_preds_1']).all()

    from lfm_quant_b200 import tf_checkpoint
    bundle = tf_checkpoint.read_bundle(str(mdir / 'chkpts' / 'chkpt'))
    assert {'layer_with_weights-0/kernel/.ATTRIBUTES/VARIABLE_VALUE',
            'layer_with_weights-0/bias/.ATTRIBUTES/VARIABLE_VALUE'} <= set(bundle)
    os.remove(mdir / 'chkpts' / 'chkpt.lfmq.npz')                               # the TF container alone
    _main(workdir, *MLP, '--model_dir', 'mlp', '--train=False')
    again = _preds(workdir, 'mlp')
    np.testing.assert_array_equal(again['norm_preds_1'].values, out['norm_preds_1'].values)


def test_cli_mlp_linear_ensemble_writes_ensemble_preds(workdir):
    ens = [*MLP, '--max_epoch', '1', '--model_dir', 'mlp-ens', '--num_procs', '2', '--NPE', '2']
    _main(workdir, *ens, '--train=True')
    _main(workdir, *ens, '--train=False')
    df = pd.read_csv(workdir / 'experiments' / 'mlp-ens' / 'ensemble_preds.dat', sep=' ', dtype={'gvkey': str})
    assert len(df) > 100 and np.isfinite(df['preds_1']).all()


def test_cli_naive_predicts_without_a_checkpoint_and_refuses_training(workdir):
    scales = workdir / 'experiments' / 'naive-scales.dat'
    if not scales.exists():                            # the scaling of a trained run (data_processing.py:151-165)
        _main(workdir, *MLP, '--max_epoch', '1', '--model_dir', 'naive-src', '--train=True')
        shutil.copy(workdir / 'experiments' / 'naive-src' / 'scales.dat', scales)
    naive = ['--nn_type', 'NaivePointEstimate', '--model_dir', 'naive', '--scalesfile', str(scales)]
    _main(workdir, *naive, '--train=False')
    assert not (workdir / 'experiments' / 'naive' / 'chkpts').exists()
    out = _preds(workdir, 'naive')
    assert list(out.columns)[-10:] == PRED_TAIL and len(out) > 100
    # the forecast is this year's value of the target field: the un-scaled last input step
    np.testing.assert_array_equal(out['preds_1'].values, out['inp_t0'].values)
    with pytest.raises(ValueError, match='no variables to train'):
        _main(workdir, *naive, '--train=True')


def test_cli_mlp_linear_refuses_multi_step(workdir):
    with pytest.raises(NotImplementedError, match='forecast_steps'):
        _main(workdir, *MLP, '--model_dir', 'mlp-s2', '--forecast_steps', '2', '--forecast_steps_weights', '0.5-0.5',
              '--train=True')


def test_naive_keeps_the_financial_fields_of_the_last_step(workdir):
    """naive_point_estimate.py:53-54 keeps the FIRST n_outputs input features; the batcher puts the financial fields
    first (inp_col_ids = fin_col_ids + aux_col_ids), so the forecast is last year's fundamentals."""
    from lfm_quant_b200.scripts import base_config
    from lfm_quant_b200.scripts.data_processing import Dataset
    from lfm_quant_b200.scripts.models.point_estimate.naive_point_estimate import NaivePointEstimate
    from lfm_quant_b200.scripts.synthetic import FIN_FIELDS
    configs.reset()
    c = base_config.get_configs(['--config=' + str(workdir / 'config' / 'system-test.conf'), '--nn_type',
                                 'NaivePointEstimate', '--train=True', '--model_dir', 'naive-ds'])
    ds = Dataset(c)
    ds.generate_dataset()
    configs.reset()
    O = ds.n_outputs
    assert list(ds.inp_col_ids[:O]) == list(ds.fin_col_ids)
    assert [ds.data.columns[i] for i in ds.inp_col_ids[:O]] == FIN_FIELDS
    x, y, _ = ds.get_batch(*next(iter(ds.train_set.batch(64))))
    assert x.shape == (64, ds.seq_len * ds.n_inputs) and y.shape == (64, O)
    c.train = False
    m = NaivePointEstimate(c, ds).model
    got = m.predict(x)
    np.testing.assert_array_equal(got, x.cpu().numpy().reshape(64, ds.seq_len, ds.n_inputs)[:, -1, :O])
