"""Split-conformal intervals on the H100 (DESIGN.md section 5j): lfmq_conformal_* against conformal_oracle bit for bit,
lfmq_nearest_topk against fp64 with the influence test's criterion, and the CLI on the synthetic dataset for every model
kind, with preds.dat left byte-identical."""
import ctypes as C

import numpy as np
import pandas as pd
import pytest
import torch

import conformal_oracle as co
from lfm_quant_b200 import _native as N
from lfm_quant_b200.engine import conformal_apply, conformal_calibrate, conformal_scores, nearest_topk

pytestmark = pytest.mark.gpu
ERR_ARG = 1
LEVELS32 = list(np.round(np.linspace(0.02, 0.99, 32), 4))


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _problem(S, N, seed, scaled):
    rng = np.random.RandomState(seed)
    pred = rng.normal(size=(S, N)).astype(np.float32)
    y = (pred + rng.standard_t(4, size=(S, N))).astype(np.float32)
    y[rng.uniform(size=(S, N)) < 0.1] = np.nan
    y[:, ::97] = np.inf
    scale = rng.uniform(0.2, 3.0, size=(S, N)).astype(np.float32) if scaled else None
    return pred, y, scale


@pytest.mark.parametrize('S,Q,Nc,scaled', [(1, 1, 1, False), (2, 5, 9, True), (3, 32, 9, False), (1, 5, 4097, True),
                                           (3, 32, 4097, True), (2, 1, 4097, False), (3, 32, 10 ** 6, True)])
def test_calibrate_and_apply_match_oracle_bit_for_bit(S, Q, Nc, scaled):
    levels = [0.9] if Q == 1 else ([0.1, 0.5, 0.8, 0.9, 0.99] if Q == 5 else LEVELS32)
    pc, yc, sc = _problem(S, Nc, seed=S * 7 + Nc, scaled=scaled)
    pq, yq, sq = _problem(S, 3001, seed=S + Q, scaled=scaled)
    n_valid, srt, qhat = conformal_calibrate(_cuda(pc), _cuda(yc), levels, scale=None if sc is None else _cuda(sc))
    rn, rs, rq = co.calibrate(pc, yc, levels, sc)
    assert np.array_equal(n_valid.cpu().numpy(), rn)
    assert np.array_equal(qhat.cpu().numpy(), rq)
    got_s = srt.cpu().numpy()
    for s in range(S):
        assert np.array_equal(got_s[s, :rn[s]], rs[s, :rn[s]]) and np.isnan(got_s[s, rn[s]:]).all()
    if Nc < 20:      # small sets: some levels' rank exceeds n, so qhat is +inf
        assert np.isinf(rq).any()
    lo, hi, p = (t.cpu().numpy() for t in conformal_apply(_cuda(pq), (n_valid, srt, qhat), y=_cuda(yq),
                                                          scale=None if sq is None else _cuda(sq)))
    rlo, rhi, rp = co.apply(pq, rn, rs, rq, y=yq, scale=sq)
    assert np.array_equal(p, rp, equal_nan=True)
    for g, r in ((lo, rlo), (hi, rhi)):
        fin = np.isfinite(r)
        assert np.array_equal(np.isfinite(g), fin) and np.array_equal(g[~fin], r[~fin])
        assert np.all(np.abs(g[fin] - r[fin]) <= np.spacing(np.abs(r[fin])))
    r = conformal_scores(_cuda(pq), _cuda(yq), None if sq is None else _cuda(sq)).cpu().numpy()
    assert np.array_equal(r, co.scores(pq, yq, sq), equal_nan=True)
    # no target: NaN p-values, the same bounds
    lo2, _, p2 = conformal_apply(_cuda(pq), (n_valid, srt, qhat), scale=None if sq is None else _cuda(sq))
    assert np.isnan(p2.cpu().numpy()).all() and np.array_equal(lo2.cpu().numpy(), lo)


def test_conformal_refusals():
    lib = N.load()
    n = C.c_uint64(0)
    assert lib.lfmq_conformal_calibrate_work_bytes(0, 5, C.byref(n)) == ERR_ARG
    assert lib.lfmq_conformal_apply_work_bytes(1, 5, 5, 33, C.byref(n)) == ERR_ARG
    pred = torch.zeros(1, 5, device='cuda')
    for bad in ([0.5, 0.5], [0.0], [1.0], [0.1] * 33):
        with pytest.raises(N.LfmqError):
            conformal_calibrate(pred, pred, bad)
    nul = C.c_void_p(0)
    assert lib.lfmq_conformal_apply(nul, nul, nul, 1, 5, nul, nul, nul, 5, 1, nul, nul, nul, nul, 0, nul) == ERR_ARG


# ---- nearest pool rows -------------------------------------------------------------------------------------------
def _points(Nq, Nt, D1, seed):
    rng = np.random.RandomState(seed)
    b = (rng.normal(size=(Nt, D1)) * rng.lognormal(0, 0.5, size=(Nt, 1))).astype(np.float32)
    a = rng.normal(size=(Nq, D1)).astype(np.float32)
    a[: Nq // 2] = b[rng.randint(0, Nt, size=Nq // 2)] + 0.05 * a[: Nq // 2]      # queries near pool rows
    value = rng.uniform(0, 2, size=Nt).astype(np.float32)
    return a, b, value


def _check_nearest(a, b, value, K, got):
    idx, d2, mean = (t.cpu().numpy() for t in got)
    a64, b64 = a.astype(np.float64), b.astype(np.float64)
    ridx, rd2, _ = co.knn(a64, b64, K)
    na, nb = np.linalg.norm(a64, axis=1), np.linalg.norm(b64, axis=1)
    k = min(K, b.shape[0])
    assert np.all(idx[:, k:] == -1) and np.all(np.isinf(d2[:, k:]))
    for q in range(a.shape[0]):
        sel = idx[q, :k]
        assert np.all(sel >= 0) and len(set(sel.tolist())) == k
        f64 = ((a64[q] - b64[sel]) ** 2).sum(axis=1)
        # d2 is the fp64 distance of the difference, rounded to fp32 (the summation order may differ in the last bits)
        assert np.all(np.abs(d2[q, :k] - f64) <= 2 * np.spacing(np.float32(f64)).astype(np.float64)), q
        assert np.all(np.diff(d2[q, :k]) >= 0)
        # the shortlist ranks by the 3xTF32 score: a returned row is at most its tolerance beyond the fp64 K-th nearest
        tol = 2 * 2e-6 * na[q] * nb[sel] + 2e-6 * (na[q] ** 2 + nb[sel] ** 2)
        assert np.all(f64 <= rd2[q, k - 1] + tol), q
        assert np.isclose(mean[q], value[sel].astype(np.float64).mean(), rtol=1e-6)


GRID = [(1, 1000, 65, 10), (129, 1000, 257, 64), (129, 70001, 65, 1), (4096, 1000, 1537, 10), (1, 70001, 257, 64),
        (4096, 1, 65, 10), (129, 1, 257, 1), (129, 70001, 1537, 10)]


@pytest.mark.parametrize('Nq,Nt,D1,K', GRID)
def test_nearest_matches_fp64(Nq, Nt, D1, K):
    a, b, value = _points(Nq, Nt, D1, seed=Nq + Nt + D1 + K)
    qs = np.arange(Nq) if Nq <= 129 else np.random.RandomState(0).choice(Nq, 40, replace=False)
    got = nearest_topk(_cuda(a), _cuda(b), K, value=_cuda(value))
    sel = torch.from_numpy(qs).cuda()
    _check_nearest(a[qs], b, value, K, [got[0][sel], got[1][sel], got[2][sel]])


def test_near_duplicate_queries_get_exact_distances():
    # queries a hair from pool rows in a wide feature space: |a|^2 ~ 1e4 against d^2 ~ 1e-2, where the GEMM's score
    # alone cannot resolve the distance; the nearest row is the source row, with its fp64 distance
    rng = np.random.RandomState(5)
    b = (rng.normal(size=(3000, 1537)) * 3).astype(np.float32)
    src = rng.choice(3000, 64, replace=False)
    a = (b[src] + 3e-3 * rng.normal(size=(64, 1537))).astype(np.float32)
    idx, d2 = (t.cpu().numpy() for t in nearest_topk(_cuda(a), _cuda(b), 5)[:2])
    assert np.array_equal(idx[:, 0], src)
    f64 = ((a.astype(np.float64) - b[src].astype(np.float64)) ** 2).sum(axis=1)
    assert np.all(np.abs(d2[:, 0] - f64) <= 2 * np.spacing(np.float32(f64)).astype(np.float64))


def test_duplicated_rows_list_lowest_index_first():
    a, b, _ = _points(6, 600, 65, seed=3)
    b[300:] = b[:300]
    idx, d2 = (t.cpu().numpy() for t in nearest_topk(_cuda(a), _cuda(b), 10)[:2])
    for q in range(6):
        assert np.all(d2[q, 0::2] == d2[q, 1::2])
        assert np.all(idx[q, 1::2] == idx[q, 0::2] + 300) and np.all(idx[q, 0::2] < 300)


def test_same_bits_across_calls_batching_and_pool_prefix():
    a, b, value = _points(300, 20000, 257, seed=4)
    A, B, V = _cuda(a), _cuda(b), _cuda(value)
    r1 = [t.cpu().numpy() for t in nearest_topk(A, B, 16, value=V)]
    r2 = [t.cpu().numpy() for t in nearest_topk(A, B, 16, value=V)]
    for x1, x2 in zip(r1, r2):
        assert np.array_equal(x1, x2)
    sub = [t.cpu().numpy() for t in nearest_topk(A[131:140], B, 16, value=V)]
    for x1, x2 in zip(r1, sub):
        assert np.array_equal(x1[131:140], x2)
    pre = [t.cpu().numpy() for t in nearest_topk(A, B[:7000].contiguous(), 16)[:2]]
    for q in range(300):
        big = dict(zip(r1[0][q], r1[1][q]))
        for i, d in zip(pre[0][q], pre[1][q]):
            if i in big:
                assert big[i] == d


def test_nearest_refusals():
    lib = N.load()
    n = C.c_uint64(0)
    for args in ((0, 10, 65, 5), (4, 0, 65, 5), (4, 10, 0, 5), (4, 10, 65, 0), (4, 10, 65, 65)):
        assert lib.lfmq_nearest_topk_work_bytes(*args, C.byref(n)) == ERR_ARG
    nul = C.c_void_p(0)
    assert lib.lfmq_nearest_topk(nul, nul, nul, 4, 10, 65, 5, nul, nul, nul, nul, 0, nul) == ERR_ARG


# ---- the CLI on the synthetic dataset ----------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def workdir(tmp_path_factory):
    from lfm_quant_b200.scripts.synthetic import write_open_dataset, write_system_test_conf
    d = tmp_path_factory.mktemp('conformal')
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
    return main


UQ = ['--nn_type', 'RNNUqRangeEstimate', '--UQ=True', '--dropout', '0.1', '--recurrent_dropout', '0.1']
LEVELS = [0.5, 0.8, 0.9]
SPEC = '0.5-0.8-0.9'
# exact: the model predicts a window with the same bits in the calibration pass as in preds.dat (no dropout draw)
MODELS = [('lstm', [], [], [], 1, True), ('gru', ['--rnn_cell', 'gru'], [], [], 1, True),
          ('uq', UQ, [], [], 1, False), ('uq', UQ, ['--mc_samples', '8'], [], 1, False),
          ('chain', ['--forecast_steps', '2', '--forecast_steps_weights', '1.0-0.5'], [], [], 2, True),
          ('linear', ['--nn_type', 'MLPLinearPointEstimate'], [], [], 1, True),
          ('linear', ['--nn_type', 'MLPLinearPointEstimate'], [], ['--conformal_knn', '16'], 1, True),
          ('lstm', [], ['--precision', 'bf16'], [], 1, False)]


def _check_files(m, steps, exact):
    iv = pd.read_csv(m / 'pred' / 'intervals.dat', sep=' ', dtype={'gvkey': str})
    preds = pd.read_csv(m / 'pred' / 'preds.dat', sep=' ', dtype={'gvkey': str})
    assert len(iv) == len(preds) and iv['gvkey'].tolist() == preds['gvkey'].tolist()
    cov = pd.read_csv(m / 'pred' / 'coverage.dat', sep=' ')
    assert len(cov) == steps * len(LEVELS) * 4
    for s in range(1, steps + 1):
        for lv in ('50', '80', '90'):
            assert np.all(iv['norm_lo%s_%d' % (lv, s)] <= iv['norm_hi%s_%d' % (lv, s)])
            assert np.all(iv['lo%s_%d' % (lv, s)] <= iv['hi%s_%d' % (lv, s)])
        p = iv['pvalue_%d' % s]
        assert np.array_equal(np.isnan(p), np.isnan(preds['norm_targets_%d' % s]))
        assert np.all((p[p.notna()] > 0) & (p[p.notna()] <= 1))
    c = cov[cov.subset == 'calibration']
    assert (c['n'] > 0).all()
    if exact:       # the calibration windows' own scores: coverage >= l by construction
        assert np.all(c['coverage'].values >= c['level'].values - 1e-12), c
    return iv, cov


@pytest.mark.parametrize('name,extra,pred_extra,conf_extra,steps,exact', MODELS)
def test_cli_writes_intervals_and_leaves_preds_dat_alone(workdir, cli, name, extra, pred_extra, conf_extra, steps,
                                                         exact):
    model_dir = 'conf-%s-%d' % (name, steps)
    m = workdir / 'experiments' / model_dir
    args = ['--model_dir', model_dir] + extra
    if not (m / 'chkpts').exists():
        cli(*args, '--train=True')
    cli(*args, '--train=False', *pred_extra)
    plain = (m / 'pred' / 'preds.dat').read_bytes()
    cli(*args, '--train=False', *pred_extra, '--conformal_levels', SPEC, *conf_extra)
    assert (m / 'pred' / 'preds.dat').read_bytes() == plain
    _check_files(m, steps, exact)


def test_cli_naive_model(workdir, cli):
    import shutil
    scales = workdir / 'experiments' / 'naive-scales.dat'
    src = workdir / 'experiments' / 'conf-linear-1' / 'scales.dat'
    if not src.exists():
        cli('--model_dir', 'conf-linear-1', '--nn_type', 'MLPLinearPointEstimate', '--train=True')
    shutil.copy(src, scales)
    args = ['--nn_type', 'NaivePointEstimate', '--model_dir', 'conf-naive', '--scalesfile', str(scales),
            '--train=False']
    cli(*args)
    m = workdir / 'experiments' / 'conf-naive'
    plain = (m / 'pred' / 'preds.dat').read_bytes()
    cli(*args, '--conformal_levels', SPEC)
    assert (m / 'pred' / 'preds.dat').read_bytes() == plain
    _check_files(m, 1, True)


def test_cli_walk_forward_stitches_intervals(workdir, cli):
    origins = [199612, 199712]
    args = ['--training_type', 'iterative', '--split_date', '199612', '--end_date', '199812', '--model_dir', 'conf-wf',
            '--NPE', '2']
    cli(*args, '--train=True')
    cli(*args, '--train=False', '--conformal_levels', SPEC)
    wf = workdir / 'experiments' / 'conf-wf'
    iv = pd.read_csv(wf / 'walk_forward_intervals.dat', sep=' ', dtype={'gvkey': str})
    cov = pd.read_csv(wf / 'walk_forward_coverage.dat', sep=' ')
    preds = pd.read_csv(wf / 'walk_forward_preds.dat', sep=' ', dtype={'gvkey': str})
    assert len(iv) == len(preds) and sorted(set(iv['origin'])) == origins
    assert len(cov) == len(origins) * len(LEVELS) * 4 and sorted(set(cov['origin'])) == origins
