"""Training-window attributions on the GPU (lfmq_influence_*, _HandleEngine.influence_features, influence_topk).

Checked here: both feature passes against the fp64 oracle (tests/influence_oracle.py) for every model kind at fp32 and
tf32, with B not a multiple of the launch rows; the top-K lists and the pool total against fp64 over a grid of query
counts, pool sizes, widths, K and J; the tie rule on duplicated windows; the same bits on a repeated call, under another
batching of the queries and for a pool that shares a prefix; the refusals of the entry points; and the CLI on the
synthetic dataset (point, UQ and linear models, a bf16 model against fp32, and a walk-forward run)."""
import ctypes as C

import numpy as np
import pytest
import torch

import influence_oracle as io
import lfm_oracle as orc
from lfm_quant_b200 import _native as N
from lfm_quant_b200.engine import DenseEngine, ForecasterEngine, influence_topk

pytestmark = pytest.mark.gpu
KW = dict(target_idx=1, target_lambda=0.5, rnn_lambda=0.7)
ERR_ARG = 1


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).cuda()


def _problem(B, T, F, O, seed):
    rng = np.random.RandomState(seed)
    x = rng.normal(size=(B, T, F)).astype(np.float32)
    y = rng.normal(size=(B, T, O)).astype(np.float32)
    y[3, :2] = 0.0          # masked early steps
    y[5, -1] = 0.0          # masked last step
    y[7] = 0.0              # a window with every step masked
    return x, y


# (name, kind, cell, L)
KINDS = [('lstm-point-L2', 'point', 'lstm', 2), ('gru-point', 'point', 'gru', 1), ('lstm-uq', 'uq', 'lstm', 1),
         ('gru-uq-L2', 'uq', 'gru', 2)]


@pytest.mark.parametrize('precision,tol', [('fp32', 2e-5), ('tf32', 2e-2)])
@pytest.mark.parametrize('name,kind,cell,L', KINDS)
def test_recurrent_features_match_oracle(name, kind, cell, L, precision, tol):
    B, T, F, O, H = 100, 6, 5, 4, 64
    x, y = _problem(B, T, F, O, 3)
    P = orc.init_params(L, F, O, H, init_scale=0.5, seed=11, dtype=np.float64, rnn_cell=cell, uq=kind == 'uq')
    P = [p.astype(np.float32).astype(np.float64) for p in P]
    eng = ForecasterEngine(max_batch=48, seq_len=T, n_inputs=F, n_outputs=O, num_hidden=H, num_layers=L, rnn_cell=cell,
                           uq=kind == 'uq', precision=precision, train=False, forward_only=True, dropout=0.3,
                           recurrent_dropout=0.2, seed=5, **KW)
    eng.set_weights(P)
    u = eng.influence_features(_cuda(x), _cuda(y)).cpu().numpy()
    a, s = [t.cpu().numpy() for t in eng.influence_features(_cuda(x))]
    ru = io.train_features(kind, P, x, y, num_layers=L, rnn_cell=cell, **KW)
    ra, rs = io.query_features(kind, P, x, target_idx=KW['target_idx'], num_layers=L, rnn_cell=cell)
    assert np.all(np.isfinite(u))
    assert np.all(u[:, 7] == 0.0)
    for got, ref in ((u, ru), (a, ra), (s, rs)):
        assert got.shape == ref.shape
        err = np.max(np.abs(got - ref)) / max(np.max(np.abs(ref)), 1e-30)
        assert err < tol, (name, err)


@pytest.mark.parametrize('huber', [False, True])
def test_dense_features_match_oracle(huber):
    B, T, F, O = 100, 6, 5, 4
    x, y = _problem(B, T, F, O, 4)
    y = y[:, -1].copy()
    y[2] = 0.0
    rng = np.random.RandomState(9)
    P = [rng.normal(size=(T * F, O)) * 0.3, rng.normal(size=O) * 0.1]
    P = [p.astype(np.float32).astype(np.float64) for p in P]
    eng = DenseEngine(max_batch=48, seq_len=T, n_inputs=F, n_outputs=O, target_idx=KW['target_idx'],
                      target_lambda=KW['target_lambda'], huber_loss=huber, huber_delta=0.7, forward_only=True)
    eng.set_weights(P)
    u = eng.influence_features(_cuda(x), _cuda(y)).cpu().numpy()
    a, s = [t.cpu().numpy() for t in eng.influence_features(_cuda(x))]
    ru = io.train_features('dense', P, x, y, target_idx=KW['target_idx'], target_lambda=KW['target_lambda'],
                           huber=huber, huber_delta=0.7)
    ra, rs = io.query_features('dense', P, x, target_idx=KW['target_idx'])
    assert np.all(u[:, 2] == 0.0)
    for got, ref in ((u, ru), (a, ra), (s, rs)):
        assert got.shape == ref.shape
        assert np.max(np.abs(got - ref)) <= 2e-5 * max(np.max(np.abs(ref)), 1e-30)


def _random(Nq, Nt, D1, J, seed, zero_s=False):
    rng = np.random.RandomState(seed)
    a = rng.normal(size=(Nq, D1)).astype(np.float32)
    a[:, -1] = 1.0
    u = (rng.normal(size=(J, Nt, D1)) * rng.lognormal(0, 1, size=(J, Nt, 1))).astype(np.float32)
    s = np.ones((J, Nq), dtype=np.float32)
    if J == 2:
        s[1] = rng.uniform(0.05, 1.0, size=Nq)
        if zero_s:
            s[1, ::7] = 0.0
    return a, u, s


def _check_topk(a, u, s, K, got):
    pos_idx, pos_score, neg_idx, neg_score, total = [t.cpu().numpy() for t in got]
    a64, u64, s64 = (v.astype(np.float64) for v in (a, u, s))
    I = io.influence(a64, u64, s64)
    J, Nq, Nt = I.shape
    na = np.linalg.norm(a64, axis=1)
    nu = np.linalg.norm(u64, axis=2)
    ref = io.topk(I, K)
    for (idx, score, ridx, rscore, sign) in ((pos_idx, pos_score, ref[0], ref[1], 1.0),
                                             (neg_idx, neg_score, ref[2], ref[3], -1.0)):
        assert idx.shape == (Nq, J, K)
        # the same number of entries of each sign (no sign near the tolerance in these draws), padded alike
        for j in range(J):
            for q in range(Nq):
                n = int((ridx[q, j] >= 0).sum())
                tol = 2e-6 * s64[j, q] * na[q] * nu[j]
                sel = idx[q, j]
                assert np.all(sel[n:] == -1) and np.all(score[q, j, n:] == 0.0)
                assert np.all(sel[:n] >= 0), (j, q, sel[:n])
                f64 = I[j, q, sel[:n]]
                assert np.all(np.abs(score[q, j, :n] - f64) <= tol[sel[:n]] + 1e-30)
                if n:
                    kth = rscore[q, j, n - 1]
                    assert np.all(sign * f64 >= sign * kth - tol[sel[:n]] - 1e-30)
                assert len(set(sel[:n].tolist())) == n
    rtot = I.sum(axis=2).T
    bound = 1e-6 * (np.abs(I).sum(axis=2).T + 1e-30)
    assert np.all(np.abs(total - rtot) <= bound + 1e-5 * np.abs(rtot))


GRID = [(1, 1000, 65, 10, 1), (129, 1000, 257, 64, 2), (129, 70001, 65, 1, 1), (4096, 1000, 513, 10, 2),
        (129, 1000, 1537, 10, 1), (1, 70001, 257, 64, 2), (4096, 1, 65, 10, 1), (129, 1, 257, 64, 2)]


@pytest.mark.parametrize('Nq,Nt,D1,K,J', GRID)
def test_topk_matches_fp64(Nq, Nt, D1, K, J):
    a, u, s = _random(Nq, Nt, D1, J, seed=Nq + Nt + D1 + K, zero_s=True)
    qs = np.arange(Nq) if Nq <= 129 else np.random.RandomState(0).choice(Nq, 40, replace=False)
    got = influence_topk(_cuda(a), _cuda(u), _cuda(s), K)
    got = [t[torch.from_numpy(qs).cuda()] for t in got]
    _check_topk(a[qs], u, s[:, qs], K, got)


def test_duplicated_windows_list_lowest_index_first():
    a, u, s = _random(5, 600, 65, 1, seed=1)
    u[0, 300:] = u[0, :300]
    pos_idx, pos_score, neg_idx, neg_score, _ = [t.cpu().numpy() for t in influence_topk(_cuda(a), _cuda(u), _cuda(s),
                                                                                         10)]
    for idx, score in ((pos_idx, pos_score), (neg_idx, neg_score)):
        for q in range(5):
            i, sc = idx[q, 0], score[q, 0]
            assert np.all(sc[0::2] == sc[1::2])
            assert np.all(i[1::2] == i[0::2] + 300) and np.all(i[0::2] < 300)


def test_same_bits_across_calls_batching_and_pool_prefix():
    a, u, s = _random(300, 20000, 257, 2, seed=2)
    A, U, S = _cuda(a), _cuda(u), _cuda(s)
    r1 = [t.cpu().numpy() for t in influence_topk(A, U, S, 16)]
    r2 = [t.cpu().numpy() for t in influence_topk(A, U, S, 16)]
    for x1, x2 in zip(r1, r2):
        assert np.array_equal(x1, x2)
    sub = [t.cpu().numpy() for t in influence_topk(A[131:140], U, S[:, 131:140], 16)]
    for x1, x2 in zip(r1, sub):
        assert np.array_equal(x1[131:140], x2)
    # a pool holding the first 7000 windows: every window listed by both calls has the same score bits
    pre = [t.cpu().numpy() for t in influence_topk(A, U[:, :7000].contiguous(), S, 16)]
    for k in (0, 2):
        for q in range(300):
            for j in range(2):
                big = dict(zip(r1[k][q, j], r1[k + 1][q, j]))
                for i, sc in zip(pre[k][q, j], pre[k + 1][q, j]):
                    if i >= 0 and i in big:
                        assert big[i] == sc


def test_topk_refusals():
    lib = N.load()
    n = C.c_uint64(0)
    for args in ((0, 10, 65, 1, 5), (4, 0, 65, 1, 5), (4, 10, 65, 3, 5), (4, 10, 65, 1, 0), (4, 10, 65, 1, 65)):
        assert lib.lfmq_influence_topk_work_bytes(*args, C.byref(n)) == ERR_ARG
    nul = C.c_void_p(0)
    assert lib.lfmq_influence_topk(nul, nul, nul, 4, 10, 65, 1, 5, nul, nul, nul, nul, nul, nul, 0, nul) == ERR_ARG


@pytest.mark.parametrize('precision', ['bf16', 'bf16x3'])
def test_feature_refusals(precision):
    T, F, O, H = 4, 8, 4, 64
    eng = ForecasterEngine(max_batch=64, seq_len=T, n_inputs=F, n_outputs=O, num_hidden=H, precision=precision,
                           train=False, forward_only=True, **KW)
    n = C.c_uint64(0)
    assert eng.lib.lfmq_influence_features_work_bytes(eng.handle, C.byref(n)) == ERR_ARG
    x = torch.zeros(8, T, F, device='cuda')
    with pytest.raises(N.LfmqError):
        eng.influence_features(x)


# ---- the CLI on the synthetic dataset ----------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def workdir(tmp_path_factory):
    from lfm_quant_b200.scripts.synthetic import write_open_dataset, write_system_test_conf
    d = tmp_path_factory.mktemp('influence')
    write_open_dataset(str(d / 'datasets' / 'open-dataset.dat'), n_keys=30, n_months=420, seed=9)
    write_system_test_conf(str(d / 'config' / 'system-test.conf'), str(d / 'datasets'), str(d / 'experiments'))
    (d / 'experiments').mkdir()
    return d


@pytest.fixture()
def cli(workdir, monkeypatch):
    from lfm_quant_b200.scripts import configs
    from lfm_quant_b200.scripts import lfm_quant
    monkeypatch.setenv('LFM_QUANT_ROOT', str(workdir))
    conf = str(workdir / 'config' / 'system-test.conf')

    def main(*argv):
        configs.reset()
        try:
            return lfm_quant.main(['--config=' + conf] + list(argv))
        finally:
            configs.reset()
    main.conf = conf
    return main


def _split(cli, *argv):
    """the training and validation gvkeys a --train=True run with these flags draws"""
    from lfm_quant_b200.scripts import base_config, configs
    from lfm_quant_b200.scripts.data_processing import Dataset
    configs.reset()
    try:
        ds = Dataset(base_config.get_configs(['--config=' + cli.conf] + list(argv) + ['--train=True']))
    finally:
        configs.reset()
    return set(ds._train_gvkeys), set(ds._valid_gvkeys)


UQ = ['--nn_type', 'RNNUqRangeEstimate', '--UQ=True', '--dropout', '0.1', '--recurrent_dropout', '0.1']


@pytest.mark.parametrize('name,extra,J', [('point', ['--dropout', '0.1'], 1), ('uq', UQ, 2),
                                          ('linear', ['--nn_type', 'MLPLinearPointEstimate'], 1)])
def test_cli_writes_influence_npz_and_leaves_preds_dat_alone(workdir, cli, name, extra, J):
    m = workdir / 'experiments' / ('infl-' + name)
    args = ['--model_dir', 'infl-' + name] + extra
    cli(*args, '--train=True')
    train_keys, valid_keys = _split(cli, *args)
    got = {}
    for prec in ('fp32', 'bf16') if name != 'linear' else ('fp32',):
        cli(*args, '--train=False', '--precision', prec)
        plain = (m / 'pred' / 'preds.dat').read_bytes()
        cli(*args, '--train=False', '--precision', prec, '--influence_top_k', '5')
        assert (m / 'pred' / 'preds.dat').read_bytes() == plain, prec
        z = dict(np.load(m / 'pred' / 'influence.npz'))
        (m / 'pred' / 'influence.npz').unlink()
        N, Nt = z['date'].size, z['train_date'].size
        assert z['pos_idx'].shape == (N, J, 5) and z['neg_score'].shape == (N, J, 5) and z['total'].shape == (N, J)
        assert z['outputs'].tolist() == ['norm_preds_1', 'norm_variance_1'][:J]
        for k in ('pos_idx', 'neg_idx'):
            i = z[k][z[k] >= 0]
            assert i.size > 0 and i.max() < Nt
            keys = set(z['train_gvkey'][i].tolist())
            assert keys <= train_keys and not keys & valid_keys
        assert np.all(z['pos_score'][z['pos_idx'] >= 0] > 0) and np.all(z['neg_score'][z['neg_idx'] >= 0] < 0)
        got[prec] = z
    if 'bf16' in got:        # a bf16 model is explained through an fp32 handle of the same checkpoint
        for k in got['fp32']:
            assert np.array_equal(got['fp32'][k], got['bf16'][k]), k


def test_cli_walk_forward_lists_no_window_after_its_origin(workdir, cli):
    origins = [199612, 199712]
    args = ['--training_type', 'iterative', '--split_date', '199612', '--end_date', '199812', '--model_dir', 'infl-wf',
            '--NPE', '2']
    cli(*args, '--train=True')
    cli(*args, '--train=False', '--influence_top_k', '3')
    wf = workdir / 'experiments' / 'infl-wf'
    for o in origins:
        z = np.load(wf / ('system-test-wf-%d' % o) / 'pred' / 'influence.npz')
        assert z['train_date'].size > 0 and (z['train_date'] // 100).max() <= o
        listed = np.concatenate([z[k][z[k] >= 0] for k in ('pos_idx', 'neg_idx')])
        assert listed.size > 0 and (z['train_date'][listed] // 100).max() <= o
