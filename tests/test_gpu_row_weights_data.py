"""Row weights from the data (--sample_weight_field, --recency_halflife; DESIGN.md section 6d) on the GPU:
- the device weight kernel (lfmq_row_weights) equals the host vector bit for bit on the synthetic dataset;
- a data-parallel weighted step (row shards with the all-reduced weighted counts) equals the one-rank step, for a point
  handle, a UQ handle and the linear model, and two gloo ranks of the CLI train the one-rank weighted model;
- the CLI trains with both flags and logs a finite, unweighted valid_mse; a 2-origin walk-forward with a half-life runs.
"""
import numpy as np
import pandas as pd
import pytest
import torch

from util import make_problem, rel_err

pytestmark = pytest.mark.gpu
F, O, TARGET = 12, 6, 2
WFLAGS = ['--sample_weight_field', 'mrkcap', '--recency_halflife', '5']


@pytest.fixture(scope='module')
def workdir(tmp_path_factory):
    from lfm_quant_b200.scripts.synthetic import write_open_dataset, write_system_test_conf
    d = tmp_path_factory.mktemp('rwd')
    write_open_dataset(str(d / 'datasets' / 'open-dataset.dat'), n_keys=30, n_months=420, seed=9)
    write_system_test_conf(str(d / 'config' / 'system-test.conf'), str(d / 'datasets'), str(d / 'experiments'))
    (d / 'experiments').mkdir()
    return d


@pytest.fixture()
def cli(workdir, monkeypatch):
    from lfm_quant_b200.scripts import configs
    from lfm_quant_b200.scripts import lfm_quant
    monkeypatch.setenv('LFM_QUANT_ROOT', str(workdir))
    monkeypatch.setenv('LFMQ_SEEDED_SHUFFLE', '1')
    conf = str(workdir / 'config' / 'system-test.conf')

    def main(*argv):
        configs.reset()
        try:
            return lfm_quant.main(['--config=' + conf] + list(argv))
        finally:
            configs.reset()
    return main


def test_device_weights_equal_the_host_vector(workdir):
    from lfm_quant_b200.scripts import base_config, configs
    from lfm_quant_b200.scripts.data_processing import Dataset
    configs.reset()
    c = base_config.get_configs(['--config=' + str(workdir / 'config' / 'system-test.conf'), '--model_dir', 'dev',
                                 '--experiments_dir', str(workdir / 'experiments')] + WFLAGS)
    configs.reset()
    ds = Dataset(c)
    ds.generate_dataset()
    inp = ds._dataset['train_X']
    host = ds.row_weights_host(inp)
    dev = ds.row_weights(inp, len(inp) + 7).cpu().numpy()
    assert np.array_equal(dev[:len(inp)], host) and not np.any(dev[len(inp):])
    assert host.min() >= 0 and host.max() > 0


# ---- data parallelism: shards with the all-reduced weighted counts sum to the one-rank step --------------------------
def _engine(kind, B):
    from lfm_quant_b200.engine import DenseEngine, ForecasterEngine
    if kind == 'dense':
        return DenseEngine(max_batch=B, seq_len=5, n_inputs=F, n_outputs=O, target_idx=TARGET)
    return ForecasterEngine(max_batch=B, seq_len=8, n_inputs=F, n_outputs=O, num_hidden=64, num_layers=1,
                            target_idx=TARGET, uq=(kind == 'uq'), dropout=0.1 if kind == 'uq' else 0.0, seed=4)


@pytest.mark.parametrize('kind', ['point', 'uq', 'dense'])
def test_two_rank_weighted_step_equals_the_one_rank_step(kind):
    B, cut = 300, 110
    rng = np.random.RandomState(51)
    if kind == 'dense':
        x = rng.normal(size=(B, 5, F)).astype(np.float32)
        y = rng.normal(size=(B, O)).astype(np.float32)
        y[::9] = 0.0
    else:
        _, x, y = make_problem(B, 8, F, O, 64, 1, seed=53, init_scale=0.3)
        if kind == 'uq':
            y = rng.normal(size=y.shape).astype(np.float32)     # a masked step makes the uq loss NaN
    w = rng.uniform(0, 2, size=B).astype(np.float32)
    w[::11] = 0.0
    cu = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731

    def padded(v):
        out = torch.zeros(B, dtype=torch.float32, device='cuda')
        out[:len(v)] = cu(v)
        return out
    one = _engine(kind, B)
    params = one.get_weights()
    wd = padded(w)
    one.set_row_weights(wd)
    one.backward(cu(x), cu(y), step=2, row0=0)
    n = one.n_trainable
    want = one.grads[:n + 2].cpu().numpy().copy()
    shards = [(0, cut), (cut, B)]
    engs = []
    counts = 0
    for a, b in shards:                      # rank r: its weights, its local counts; the sum is the all-reduce
        e = _engine(kind, B)
        e.set_weights(params)
        e.set_row_weights(padded(w[a:b]))
        counts = counts + e.loss_counts(cu(y[a:b]))
        engs.append(e)
    got = 0
    for (a, b), e in zip(shards, engs):
        e.backward(cu(x[a:b]), cu(y[a:b]), step=2, row0=a, denom=counts)
        got = got + e.grads[:n + 2].cpu().numpy()
    assert rel_err(got, want) <= 1e-5, rel_err(got, want)
    assert abs(counts[0].item() - float(w.astype(np.float64).sum())) <= 1e-4 * w.sum()
    for e in engs + [one]:
        e.close()


@pytest.mark.timeout(600)
def test_cli_two_ranks_train_the_one_rank_weighted_model(tmp_path):
    import socket
    import torch.multiprocessing as mp
    from lfm_quant_b200.scripts.synthetic import write_open_dataset, write_system_test_conf
    from test_gpu_dp_models import _cli_rank
    write_open_dataset(str(tmp_path / 'datasets' / 'open-dataset.dat'), n_keys=30, n_months=420, seed=9)
    write_system_test_conf(str(tmp_path / 'config' / 'system-test.conf'), str(tmp_path / 'datasets'),
                           str(tmp_path / 'experiments'))
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    mp.spawn(_cli_rank, args=(1, 0, str(tmp_path), WFLAGS, 'one'), nprocs=1, join=True)
    mp.spawn(_cli_rank, args=(2, port, str(tmp_path), WFLAGS, 'two'), nprocs=2, join=True)
    ex = tmp_path / 'experiments'
    for kind in ('batch', 'epoch'):
        one, two = (pd.read_csv(ex / m / 'train_log' / ('system-test-train-logs-%s.csv' % kind)) for m in ('one', 'two'))
        assert len(one) == len(two) > 1
        assert np.isfinite(two['mse']).all()
        assert rel_err(two['mse'].values, one['mse'].values) < 1e-4, kind


def test_cli_trains_weighted_and_validates_unweighted(workdir, cli):
    """Both flags train through the CLI: the logged training loss is the weighted one (it differs from the unweighted
    run's), and valid_mse, which goes through the unweighted lfmq_loss, is finite."""
    cli('--train=True', '--model_dir', 'w', '--max_epoch', '2', *WFLAGS)
    cli('--train=True', '--model_dir', 'u', '--max_epoch', '2')
    ex = workdir / 'experiments'
    w, u = (pd.read_csv(ex / m / 'train_log' / 'system-test-train-logs-epoch.csv') for m in ('w', 'u'))
    assert np.isfinite(w['valid_mse']).all() and np.isfinite(w['mse']).all()
    assert not np.array_equal(w['mse'].values, u['mse'].values)        # the training loss is weighted


def test_walk_forward_with_a_halflife_runs(workdir, cli):
    cli('--train=True', '--training_type', 'iterative', '--split_date', '199712', '--end_date', '199912',
        '--model_dir', 'wfw', '--recency_halflife', '3')
    ex = workdir / 'experiments' / 'wfw'
    assert (ex / 'walk_forward_preds.dat').stat().st_size > 0
    for origin in (199712, 199812):
        assert (ex / ('system-test-wf-%d' % origin) / 'chkpts').is_dir(), origin
