"""Predictive quantiles, ALE and Shapley attributions at the sizes and limits the predict driver runs them at: many
launches per call, cut inside a Monte-Carlo sample or a coalition copy, all 32 quantile levels out to 1e-4 and 0.9999,
up to 1024 ALE bins, and the cfg shape T = 48, F = 32.

At these sizes an fp64 model over every copy would take hours, so the reference is the fp64 analysis arithmetic
(tests/predictive_oracle.py, ale_oracle.py, shapley_oracle.py) fed by the library's own forward: each copy runs
through ForecastChainEngine.forward in the launches the analysis itself runs (max_batch rows, keyed row0 = a for ALE
and m * N + a for sample m of Shapley), so its outputs are the analysis's forwards bit for bit and what is checked is
the gather, pick, fold, binning and solver code.  The end-to-end fp64-model checks stay with the small sizes in
test_gpu_predictive.py, test_gpu_ale.py and test_gpu_shapley.py.  Every case prints its worst error."""
import numpy as np
import pytest
import torch
from scipy import special

import ale_oracle as alo
import importance_oracle as imo
import predictive_oracle as pdo
import shapley_oracle as sho
import test_gpu_predictive as tgp
from test_gpu_shapley import _params

pytestmark = pytest.mark.gpu
KW = tgp.KW
TIDX = KW['target_idx']
STEP, SEED = 5, 2024
EPS = 2.0 ** -24                       # the unit roundoff of fp32
# every level --pred_quantiles takes at once (LFMQ_DIST_MAX_LEVELS), from the 1e-4 tail to the 0.9999 one
LEVELS = [1e-4, 5e-4, 1e-3, 0.005, 0.01, 0.025, 0.05, 0.075, 0.1, 0.15, 0.2, 0.25, 0.3, 0.35, 0.4, 0.45, 0.5, 0.55, 0.6,
          0.65, 0.7, 0.75, 0.8, 0.85, 0.9, 0.95, 0.975, 0.99, 0.995, 0.999, 0.9995, 0.9999]
BANDS = [('tau <= 1e-3', lambda t: t <= 1e-3), ('1e-3 < tau < 0.01', lambda t: (t > 1e-3) & (t < 0.01)),
         ('0.01 <= tau <= 0.99', lambda t: (t >= 0.01) & (t <= 0.99)),
         ('0.99 < tau < 0.999', lambda t: (t > 0.99) & (t < 0.999)), ('tau >= 0.999', lambda t: t >= 0.999)]


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).cuda()


def _ulp(a):
    a = np.abs(np.asarray(a, dtype=np.float32))
    return (np.nextafter(a, np.float32(np.inf)) - a).astype(np.float64)


def _engine(S, T, F, O, H, L, *, max_batch, precision, cell='lstm', uq, drop=None):
    from lfm_quant_b200.engine import ForecastChainEngine
    args = dict(KW, train=False, forward_only=True)
    args.update(drop or {})
    return ForecastChainEngine(forecast_steps=S, weights=[1.0, 0.5][:S], max_batch=max_batch, seq_len=T, n_inputs=F,
                               n_outputs=O, num_hidden=H, num_layers=L, rnn_cell=cell, precision=precision, uq=uq,
                               **args)


def _forward_outputs(eng, row_key):
    """outputs(x_copy, m) -> [N, J] fp64: the explained outputs (pred_s, or tar_s and var_s, at [T-1, target_idx]) of
    ForecastChainEngine.forward over the copy in launches of max_batch rows, launch [a, a + n) keyed row0 =
    row_key(m, N) + a: the launches lfmq_chain_ale (row_key 0) and lfmq_chain_shapley (row_key m * N) run."""
    mb = eng.cfg.max_batch

    def f(x, m):
        xd = _cuda(x)
        N = xd.shape[0]
        base = row_key(m, N)
        outs = [eng.forward(xd[a:a + mb].contiguous(), step=STEP, row0=base + a) for a in range(0, N, mb)]
        return np.stack([torch.cat([o[j] for o in outs])[:, -1, TIDX].cpu().numpy() for j in range(len(outs[0]))],
                        axis=1).astype(np.float64)
    return f


# ---- predictive quantiles and scores --------------------------------------------------------------------------------
def _floor_variances(eng):
    """every stage's variance head at target_idx pushed far below the 1e-6 floor: var == 1e-6 in every sample"""
    P = eng.get_weights()
    names = [n for (_, n, _, _, tr) in eng.specs if tr]
    for i, n in enumerate(names):
        if 'OUTPUT_VARIANCE' in n and 'bias' in n:
            P[i] = P[i].copy()
            P[i][TIDX] = -40.0
        elif 'OUTPUT_VARIANCE' in n and 'kernel' in n:
            P[i] = P[i].copy()
            P[i][:, TIDX] *= 0.01
    eng.set_weights(P)


def _check_dist(name, eng, x, M, levels, floor=False):
    """forward_dist at `levels` against the fp64 mixture of the library's own samples (tgp._samples); prints the worst
    quantile error per level band in q-space (over the mixture's sd) and in F-space (|F(q) - tau| over
    min(tau, 1 - tau)), and returns them."""
    N, T, O = x.shape[0], eng.T, eng.O
    S = eng.S
    ys, y = tgp._targets(S, N, T, O, 17, nan_rows=(3,))
    y[5, -1, TIDX] += 40.0                                        # a target far in the tail
    ys = [_cuda(y)] * S
    _, q, sc = eng.forward_dist(_cuda(x), M, levels, ys=ys, step=STEP)
    q, sc = q.cpu().numpy().astype(np.float64), sc.cpu().numpy().astype(np.float64)
    # the library takes its levels in fp32: the reference solves for exactly those
    tau = np.asarray(levels, dtype=np.float32).astype(np.float64)
    worst_q, worst_F = np.zeros(len(tau)), np.zeros(len(tau))
    bad = []
    sc_worst = dict(crps=0.0, nll=0.0, pit=0.0)
    for s, (mu, v) in enumerate(tgp._samples(eng, x, M, STEP)):
        if floor:
            assert (v == np.float32(1e-6)).all()
        ref = pdo.quantiles_batch(mu, v, tau)
        sd = np.sqrt(v.mean(axis=1) + mu.var(axis=1))[:, None]
        err = np.abs(q[s] - ref)
        tol = np.maximum(1e-5 * sd, 2.0 * _ulp(ref))
        worst_q = np.maximum(worst_q, (err / sd).max(axis=0))
        z = (q[s][:, :, None] - mu[:, None, :]) / np.sqrt(v)[:, None, :]
        upper = tau > 0.5
        t = np.where(upper, 1.0 - tau, tau)
        Fs = special.ndtr(np.where(upper[None, :, None], -z, z)).mean(axis=2)
        worst_F = np.maximum(worst_F, (np.abs(Fs - t[None, :]) / t[None, :]).max(axis=0))
        for b, k in zip(*np.nonzero(err > tol)):
            bad.append((s, int(b), float(tau[k]), float(err[b, k] / sd[b, 0]), float(err[b, k] / _ulp(ref[b, k]))))
        assert (np.diff(q[s], axis=1) >= 0).all()
        for b in range(N):
            yb = float(y[b, -1, TIDX])
            if not np.isfinite(yb):
                assert np.isnan(sc[s, b]).all()
                continue
            r = [pdo.crps(mu[b], v[b], yb), pdo.nll(mu[b], v[b], yb), pdo.pit(mu[b], v[b], yb)]
            sc_worst['crps'] = max(sc_worst['crps'], abs(sc[s, b, 0] - r[0]) / abs(r[0]))
            sc_worst['nll'] = max(sc_worst['nll'], max(0.0, abs(sc[s, b, 1] - r[1]) - 2.0 ** -23 * abs(r[1])))
            sc_worst['pit'] = max(sc_worst['pit'], abs(sc[s, b, 2] - r[2]))
    for band, sel in BANDS:
        k = sel(tau)
        if k.any():
            print('dist %s %-20s worst |q - q_ref| / sd %.2e, worst |F(q) - tau| / min(tau, 1 - tau) %.2e'
                  % (name, band, worst_q[k].max(), worst_F[k].max()))
    print('dist %s per level |q - q_ref| / sd: %s' % (name, ' '.join('%g:%.1e' % (a, e) for a, e in
                                                                      zip(levels, worst_q))))
    print('dist %s scores: %s' % (name, {k: '%.2e' % w for k, w in sc_worst.items()}))
    assert not bad, '%d quantiles off, worst (stage, window, tau, err/sd, err/ulp): %s' % (
        len(bad), sorted(bad, key=lambda r: -r[3])[:8])
    assert sc_worst['crps'] <= 1e-5 and sc_worst['nll'] <= 1e-5 and sc_worst['pit'] <= 1e-6, sc_worst
    return worst_q, worst_F


# (name, precision, H): launches of 1024 rows over 8 samples of 1500 windows, cut inside the samples
@pytest.mark.parametrize('case', [('fp32', 'fp32', 64), ('bf16', 'bf16', 256)], ids=['fp32', 'bf16'])
def test_all_32_levels_across_launch_cuts(case):
    name, prec, H = case
    T, F, O, N, M = 8, 32, 16, 1500, 8
    eng, x = tgp._model(2, T, F, O, H, 1, N, seed=41, precision=prec, max_batch=1024)
    assert (M * N) % 1024 and N % 1024                            # launch cuts fall inside samples
    _check_dist('32-levels-' + name, eng, x, M, LEVELS)
    eng.close()


@pytest.mark.parametrize('M', [33, 1024])
def test_many_samples(M):
    """M = 33 puts one sample past a warp's lanes, M = 1024 gives the CRPS 523776 pairs per window"""
    T, F, O, N = 8, 32, 16, 48
    eng, x = tgp._model(1, T, F, O, 64, 1, N, seed=M, max_batch=1024)
    _check_dist('M%d' % M, eng, x, M, LEVELS)
    eng.close()


def test_multimodal_mixtures():
    T, F, O, N, M = 8, 32, 16, 200, 7        # the levels keep clear of the gaps k / 7 between the modes
    eng, x = tgp._model(2, T, F, O, 64, 1, N, seed=43, head_scale=300.0, max_batch=1024)
    mu, v = tgp._samples(eng, x, M, STEP)[0]
    assert np.median(np.ptp(mu, axis=1) / np.sqrt(v.max(axis=1))) > 20
    _check_dist('multimodal', eng, x, M, LEVELS)
    eng.close()


def test_variances_on_the_floor():
    """sd = 1e-3 in every component: the solver's bracket rule (1e-6 min_sd) is below the fp32 spacing of q, so the
    quantiles can only be as good as q's own rounding"""
    T, F, O, N, M = 8, 32, 16, 200, 7
    eng, x = tgp._model(1, T, F, O, 64, 1, N, seed=44, max_batch=1024)
    _floor_variances(eng)
    _check_dist('var-floor', eng, x, M, LEVELS, floor=True)
    eng.close()


# ---- ALE -------------------------------------------------------------------------------------------------------------
ALE_K = 1024
ALE_OUT = ('n_bins', 'edges', 'counts', 'ale', 'local_mean', 'local_sd')


def _ale_inputs(N, T, F, mb, seed):
    """(x, x_nf) [N,T,F] whose latest quarter forces every binning case.  x: field 0 with ~700 distinct values (N' > K >
    distinct, so quantiles repeat), field 1 with runs of ties across the launch cuts at mb and 2 mb, field 2 with -0 and
    +0 among its values, field 4 with two values.  x_nf adds +-inf and NaN to field 2 and leaves field 3 fewer finite
    values than bins; a window with a non-finite input forecasts NaN in every copy, so x_nf's bins are what it
    checks."""
    rng = np.random.RandomState(seed)
    x = rng.normal(size=(N, T, F)).astype(np.float32)
    last = x[:, -1, :]
    last[:, 0] = np.round(last[:, 0] * 100.0) / 100.0
    last[mb - 40:mb + 40, 1] = 0.3125
    last[2 * mb - 7:2 * mb + 50, 1] = -1.25
    last[1::17, 2] = -0.0
    last[2::17, 2] = 0.0
    last[:, 4] = np.where(rng.rand(N) < 0.3, -0.5, 0.75)
    x_nf = x.copy()
    last = x_nf[:, -1, :]
    last[::7, 2] = np.nan
    last[3::11, 2] = np.inf
    last[5::13, 2] = -np.inf
    last[np.arange(N) % 5 != 0, 3] = np.nan
    assert np.unique(x[:, -1, 0]).size < ALE_K < N and np.isfinite(last[:, 3]).sum() < ALE_K
    return x, x_nf


def _check_ale(name, eng, x, cols, K):
    """lfmq_chain_ale against ale_oracle.ale over the engine's own forward: bins, edges and counts exactly; local
    means, sds and the ALE within the rounding of the fp32 local effects (d = f(upper) - f(lower) is rounded once to
    fp32 per window; everything after is fp64)"""
    got = dict(zip(ALE_OUT, [t.cpu().numpy() for t in eng.ale(_cuda(x), np.asarray(cols), K, STEP)]))
    ref = alo.ale(x.astype(np.float64), cols, K, _forward_outputs(eng, lambda m, N: 0))
    for k in ('n_bins', 'counts'):
        assert np.array_equal(got[k], ref[k]), k
    assert np.array_equal(got['edges'], ref['edges'].astype(np.float32), equal_nan=True)
    worst = dict(local_mean=0.0, local_sd=0.0, ale=0.0)
    flat = x.reshape(x.shape[0], -1)
    for g, c in enumerate(cols):
        Kg = int(ref['n_bins'][g])
        for k in ('ale', 'local_mean', 'local_sd'):
            assert np.array_equal(np.isnan(got[k][g]), np.isnan(ref[k][g])), (k, g)
        if not Kg:
            continue
        d = ref['d'][g]
        _, b = alo.bins(flat[:, c], K)
        a = np.stack([np.abs(d[b == k]).mean(axis=0) for k in range(1, Kg + 1)])          # mean |d| per bin [Kg,J]
        mx = np.stack([np.abs(d[b == k]).max(axis=0) for k in range(1, Kg + 1)])
        if np.isnan(d).all():
            continue
        scale = np.nanmax(np.abs(d), axis=0)                                              # max |d| per output
        lm, ls = ref['local_mean'][g, :Kg], ref['local_sd'][g, :Kg]
        bounds = dict(local_mean=EPS * (a + np.abs(lm)), local_sd=EPS * (mx + ls),
                      ale=EPS * (np.abs(ref['ale'][g, :Kg + 1]) + 2.0 * a.sum(axis=0)))
        for k, bound in bounds.items():
            r = ref[k][g, :bound.shape[0]]
            e = np.abs(got[k][g, :bound.shape[0]] - r)
            ok = (e <= 2.0 * bound + 1e-12 * scale) | np.isnan(r)            # NaN in both: a window forecast NaN
            assert ok.all(), (name, k, g, float(np.nanmax(e / (bound + 1e-300))))
            if np.isfinite(r).any():
                worst[k] = max(worst[k], float(np.nanmax(e / scale)))
    print('ale %s: K=%d, n_bins %s; worst error / max|d|: %s' % (name, K, got['n_bins'][:6].tolist(),
                                                                 {k: '%.1e' % w for k, w in worst.items()}))
    return got


def test_ale_bf16_point_at_the_cfg_shape():
    T, F, O, H, L, mb = 48, 32, 16, 256, 1, 1024
    N = 3 * mb + 37
    P, _ = _params(T, F, O, H, L, 1, 'lstm', False, seed=51)
    x, x_nf = _ale_inputs(N, T, F, mb, seed=52)
    eng = _engine(1, T, F, O, H, L, max_batch=mb, precision='bf16', uq=False)
    eng.set_weights(P)
    cols = [(T - 1) * F + f for f in range(F)]
    got = _check_ale('bf16-point', eng, x, cols, ALE_K)
    assert got['n_bins'][0] < ALE_K and got['n_bins'][4] == 1 and got['n_bins'][5] == ALE_K
    assert all(np.isfinite(got['ale'][g, :got['n_bins'][g] + 1]).all() for g in range(F))
    # non-finite values sort last and have no bin; field 3 has fewer finite values than bins
    got = _check_ale('bf16-point-non-finite', eng, x_nf, cols[:6], ALE_K)
    for f in (2, 3):
        assert got['counts'][f].sum() == np.isfinite(x_nf[:, -1, f]).sum()
    assert got['n_bins'][3] == np.unique(x_nf[:, -1, 3][np.isfinite(x_nf[:, -1, 3])]).size - 1
    # K > N: every window of a 600-window subset has a bin of its own after the first
    sub = x[:600]
    got = _check_ale('bf16-point-K>N', eng, sub, cols[:3] + cols[5:8], ALE_K)
    assert got['n_bins'][3] == np.unique(sub[:, -1, 5]).size - 1
    eng.close()


def test_ale_gru_uq_chain():
    T, F, O, H, L, S, mb = 48, 32, 16, 64, 1, 2, 1024
    N = 3 * mb + 37
    P, _ = _params(T, F, O, H, L, S, 'gru', True, seed=53)
    x, _ = _ale_inputs(N, T, F, mb, seed=54)
    eng = _engine(S, T, F, O, H, L, max_batch=mb, precision='tf32', cell='gru', uq=True, drop=tgp.DROP)
    eng.set_weights(P)
    cols = [(T - 1) * F + f for f in range(12)]
    _check_ale('tf32-gru-uq-S2', eng, x, cols, ALE_K)
    eng.close()


# ---- Shapley ---------------------------------------------------------------------------------------------------------
def _check_shapley(name, eng, x, cg, G, M):
    """lfmq_chain_shapley against shapley_oracle.shapley over the engine's own forward.  The library sums in fp64 and
    rounds each output once, so phi (|phi| <= 2 max|f|), f_x and f_bg are within 2 u max|f| per output, well inside
    the M G u max|f| that fp32 sums would need; additivity per window within the roundings of its G + 2 outputs."""
    phi, f_x, f_bg = [t.cpu().numpy().astype(np.float64) for t in eng.shapley(_cuda(x), cg, M, SEED, STEP)]
    f = _forward_outputs(eng, lambda m, N: m * N)
    ref = sho.shapley(x, cg, G, M, SEED, f)           # the copies only move x's fp32 values; the sums are fp64
    fmax = np.maximum(np.abs(ref[1]).max(axis=0), np.abs(ref[2]).max(axis=0))                # [K]
    tol = 2.0 * EPS * fmax
    errs = [np.abs(phi - ref[0]).max(axis=(0, 2)), np.abs(f_x - ref[1]).max(axis=0), np.abs(f_bg - ref[2]).max(axis=0)]
    gap = np.abs(phi.sum(axis=2) - (f_x - f_bg))                                             # [N,K]
    gap_tol = 2.0 * EPS * (np.abs(ref[0]).sum(axis=2) + np.abs(ref[1]) + np.abs(ref[2]))
    print('shapley %s N=%d G=%d M=%d: error / (u max|f|): phi %s, f_x %s, f_bg %s; additivity / its bound %.2f'
          % (name, x.shape[0], G, M, *[np.array2string(e / (tol / 2.0), precision=3) for e in errs],
             (gap / gap_tol).max()))
    for what, e in zip(('phi', 'f_x', 'f_bg'), errs):
        assert (e <= tol).all(), (what, e / tol)
    assert (gap <= gap_tol).all(), (gap / gap_tol).max()
    assert (np.abs(ref[0]).max(axis=(0, 2)) > 0).all()
    return f_x, f


def test_shapley_bf16_point_at_the_cfg_shape():
    """N = 9000 in launches of 4096 (two full launches and a tail), G = 32 field groups, M = 3: the last sample has no
    antithetic partner"""
    T, F, O, H, L, mb, N, M = 48, 32, 16, 256, 1, 4096, 9000, 3
    P, _ = _params(T, F, O, H, L, 1, 'lstm', False, seed=61)
    x = np.random.RandomState(62).normal(size=(N, T, F)).astype(np.float32)
    eng = _engine(1, T, F, O, H, L, max_batch=mb, precision='bf16', uq=False)
    eng.set_weights(P)
    cg, G = imo.field_groups(T, F)
    f_x, f = _check_shapley('bf16-point', eng, x, cg, G, M)
    fwd = f(x, 0)
    assert np.array_equal(f_x, fwd), int((f_x != fwd).sum())        # a point model's f_x is its forward, bit for bit
    eng.close()


def test_shapley_bf16_uq_chain_on_the_general_path():
    T, F, O, H, L, S, mb, N, M = 48, 32, 16, 128, 1, 2, 1024, 3109, 4
    P, _ = _params(T, F, O, H, L, S, 'lstm', True, seed=63)
    x = np.random.RandomState(64).normal(size=(N, T, F)).astype(np.float32)
    eng = _engine(S, T, F, O, H, L, max_batch=mb, precision='bf16', uq=True, drop=tgp.DROP)
    eng.set_weights(P)
    cg, G = imo.quarter_groups(T, F)
    _check_shapley('bf16-uq-S2-general', eng, x, cg, G, M)
    eng.close()


# ---- the engine's scratch cache --------------------------------------------------------------------------------------
def _analyses(T, F):
    cg, _ = imo.quarter_groups(T, F)
    cols = [(T - 1) * F + f for f in range(4)]
    ys = {}

    def dist(eng, x):
        N = x.shape[0]
        if N not in ys:
            ys[N] = tgp._targets(eng.S, N, T, eng.O, 71, nan_rows=(1,))[0]
        return eng.forward_dist(_cuda(x), 5, LEVELS, ys=ys[N], step=STEP)[1:]
    return dict(dist=dist,
                shapley=lambda eng, x: eng.shapley(_cuda(x), cg, 3, SEED, STEP),
                ale=lambda eng, x: eng.ale(_cuda(x), np.asarray(cols), 64, STEP))


@pytest.mark.parametrize('which', ['dist', 'shapley', 'ale'])
def test_a_reused_engine_gives_a_fresh_engines_bits(which):
    """small, large, then small again on one engine (its scratch grown and reused) against a fresh engine per call"""
    T, F, O, H, L, S = 8, 16, 8, 64, 1, 2
    P, _ = _params(T, F, O, H, L, S, 'lstm', True, seed=72)
    x = np.random.RandomState(73).normal(size=(2600, T, F)).astype(np.float32)
    run = _analyses(T, F)[which]

    def engine():
        eng = _engine(S, T, F, O, H, L, max_batch=1024, precision='fp32', uq=True, drop=tgp.DROP)
        eng.set_weights(P)
        return eng
    sizes = (100, 2600, 100)
    one = engine()
    reused = [[t.cpu().numpy() for t in run(one, x[:n])] for n in sizes]
    one.close()
    for n, got in zip(sizes, reused):
        fresh = engine()
        want = [t.cpu().numpy() for t in run(fresh, x[:n])]
        fresh.close()
        for a, b in zip(got, want):
            assert np.array_equal(a, b, equal_nan=True), (which, n)
