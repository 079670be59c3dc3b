"""CPU tests of point-estimate ensembles (runtime/model_execution.py:154-199 of the reference): the members' configs and
model-k.conf files, the GPU each member runs on and its device share, ensemble_preds.dat against an independent checker of the reference's
aggregation, the refusal of misaligned members, and the CTA budget a device share leaves a persistent launch."""
import ctypes as C
import os
import random

import numpy as np
import pandas as pd
import pytest

from ensemble_checker import expected_ensemble_frame
from lfm_quant_b200 import _native as N
from lfm_quant_b200.scripts import base_config, configs
from lfm_quant_b200.scripts.runtime import model_execution as me


@pytest.fixture()
def fresh_flags():
    configs.reset()
    yield
    configs.reset()


def _config(tmp_path, *extra):
    (tmp_path / 'exp').mkdir(exist_ok=True)
    return base_config.get_configs(['--experiments_dir', str(tmp_path / 'exp'), '--model_dir', 'ens', '--name', 'm',
                                    '--seed', '77', '--num_procs', '3'] + list(extra))


@pytest.mark.parametrize('num_gpu', [1, 2])
def test_member_seeds_directories_confs_and_gpus(fresh_flags, tmp_path, num_gpu):
    c = _config(tmp_path, '--num_gpu', str(num_gpu), '--NPE', '3')
    experiment_dir, members = me.member_configs(c)
    assert experiment_dir == os.path.join(str(tmp_path / 'exp'), 'ens')
    draw = random.Random(77)
    seeds = [77, draw.randint(0, 1000), draw.randint(0, 1000)]
    assert [m.seed for m in members] == seeds
    assert [m.member_id for m in members] == [0, 1, 2]
    assert [m.model_dir for m in members] == [os.path.join(experiment_dir, 'm-%d' % k) for k in range(3)]
    assert [m.default_gpu for m in members] == ['/gpu:%d' % (k % num_gpu) for k in range(3)]
    assert all(m.num_procs == 1 and m.NPE == 1 for m in members)
    assert c.seed == 77 and c.num_procs == 3 and c.model_dir == 'ens'          # the ensemble's config is left alone
    for m in members:
        path = me.write_member_conf(m)
        assert path == os.path.join(m.model_dir, 'model-%d.conf' % m.member_id)
        lines = open(path).read().splitlines()
        assert lines == sorted(lines) and '--seed       %d ' % m.seed in lines
        assert '--forecast_steps_weights       1.0' in lines and '--piecewise_lr_values       0.5-0.1-0.05-0.1' in lines
        assert not any(l.startswith('--dont_scale_fields') for l in lines)      # unset flags are left out
        configs.reset()
        back = base_config.get_configs(['--config', path])                    # the member runs alone from its file
        for k in ('seed', 'member_id', 'model_dir', 'default_gpu', 'num_procs', 'NPE', 'name', 'train',
                  'forecast_steps_weights', 'piecewise_lr_boundaries', 'learning_rate'):
            assert getattr(back, k) == getattr(m, k), k


@pytest.mark.parametrize('num_gpu,npe,shares', [(1, 3, [3, 3, 3]), (2, 3, [2, 1, 2]), (2, 2, [2, 1, 2]),
                                                (1, 2, [2, 2, 2])])
def test_members_run_with_their_device_share_and_the_ensemble_file_is_written(fresh_flags, tmp_path, monkeypatch,
                                                                              num_gpu, npe, shares):
    """ModelExecution runs each member once (stubbed here), with 1/min(NPE, members on its GPU) of that GPU, then
    aggregates what the members wrote."""
    calls = []
    frames = _member_frames(3, 1, seed=4)

    def fake_member(cfg, share_den):
        calls.append((cfg.member_id, cfg.default_gpu, share_den, cfg.train))
        if cfg.train:
            os.makedirs(os.path.join(cfg.model_dir, 'train_log'), exist_ok=True)
            pd.DataFrame({'epoch': [0, 1], 'valid_mse': [0.5 + cfg.member_id, 0.25 + cfg.member_id]}).to_csv(
                os.path.join(cfg.model_dir, 'train_log', cfg.name + '-train-logs-epoch.csv'), index=False)
        else:
            os.makedirs(os.path.join(cfg.model_dir, 'pred'), exist_ok=True)
            frames[cfg.member_id].to_csv(os.path.join(cfg.model_dir, 'pred', cfg.preds_fname), sep=' ', index=False)

    monkeypatch.setattr(me.ModelExecution, 'member_execution', staticmethod(fake_member))
    c = _config(tmp_path, '--num_gpu', str(num_gpu), '--NPE', str(npe))
    assert me.ModelExecution(c)() == [0.25, 1.25, 2.25]
    assert sorted(calls) == [(k, '/gpu:%d' % (k % num_gpu), shares[k], True) for k in range(3)]
    calls.clear()
    c.train = False
    df = me.ModelExecution(c)()
    assert sorted(calls) == [(k, '/gpu:%d' % (k % num_gpu), shares[k], False) for k in range(3)]
    written = pd.read_csv(os.path.join(str(tmp_path / 'exp'), 'ens', 'ensemble_preds.dat'), sep=' ',
                          dtype={'gvkey': str})
    back = [pd.read_csv(os.path.join(str(tmp_path / 'exp'), 'ens', 'm-%d' % k, 'pred', 'preds.dat'), sep=' ',
                        dtype={'gvkey': str}) for k in range(3)]
    pd.testing.assert_frame_equal(written, expected_ensemble_frame(back, 1), check_exact=False, rtol=1e-12)
    pd.testing.assert_frame_equal(df, expected_ensemble_frame(back, 1), check_exact=False, rtol=1e-12)


def test_a_failing_member_stops_the_members_that_have_not_started(fresh_flags, tmp_path, monkeypatch):
    """With NPE = 1 the members run one at a time: once member 0 fails, at most the member its worker thread already
    took up runs, the others are cancelled, and member 0's error is raised."""
    import time
    ran = []

    def fake_member(cfg, share_den):
        ran.append(cfg.member_id)
        if cfg.member_id == 0:
            raise RuntimeError('member 0 failed')
        time.sleep(0.2)

    monkeypatch.setattr(me.ModelExecution, 'member_execution', staticmethod(fake_member))
    c = _config(tmp_path, '--num_procs', '6', '--NPE', '1')
    with pytest.raises(RuntimeError, match='member 0 failed'):
        me.ModelExecution(c)()
    assert ran[0] == 0 and set(ran) <= {0, 1}


def test_ensembles_refuse_torchrun(fresh_flags, tmp_path, monkeypatch):
    monkeypatch.setenv('WORLD_SIZE', '2')
    monkeypatch.setattr(me.ModelExecution, 'member_execution', staticmethod(lambda cfg, share: pytest.fail('ran')))
    with pytest.raises(NotImplementedError, match='torchrun'):
        me.ModelExecution(_config(tmp_path))()


def _member_frames(n, steps, seed, rows=40):
    """preds.dat frames of n members (predict.py's columns) over the same rows, different predictions."""
    rng = np.random.RandomState(seed)
    base = {'date': np.repeat([20031231, 20041231], rows // 2), 'gvkey': ['%06d' % (1000 + i % 7) for i in range(rows)],
            'seq_norm': rng.uniform(10, 500, rows)}
    tar = {s: rng.normal(size=rows) for s in range(1, steps + 1)}
    for s in tar:
        tar[s][3] = np.nan                                   # a window whose target does not exist yet
    out = []
    for _ in range(n):
        d = dict(base)
        for s in range(1, steps + 1):
            ns = str(s)
            d['targets_' + ns] = tar[s] * 100
            d['norm_preds_' + ns] = rng.normal(size=rows)
            d['norm_variance_' + ns] = np.zeros(rows)
            d['norm_targets_' + ns] = tar[s]
            d['norm_squared_diff_' + ns] = np.square(d['norm_targets_' + ns] - d['norm_preds_' + ns])
            d['preds_' + ns] = d['norm_preds_' + ns] * 100 + rng.normal(size=rows)
            d['variance_' + ns] = np.zeros(rows)
            d['fcst_err_' + ns] = np.abs((d['targets_' + ns] - d['preds_' + ns]) / d['targets_' + ns])
            d['abs_err_' + ns] = np.abs(d['targets_' + ns] - d['preds_' + ns])
            d['unscaled_squared_err_' + ns] = np.square(d['abs_err_' + ns] / d['seq_norm'])
        out.append(pd.DataFrame(d))
    return out


@pytest.mark.parametrize('n,steps', [(2, 1), (3, 1), (5, 2)])
def test_ensemble_preds_equal_the_reference_aggregation(n, steps):
    frames = _member_frames(n, steps, seed=n)
    got = me.ensemble_point_estimate(frames, steps)
    want = expected_ensemble_frame([f.copy() for f in frames], steps)
    pd.testing.assert_frame_equal(got, want, check_exact=False, rtol=1e-12)
    assert list(got.columns) == list(frames[0].columns)
    np.testing.assert_allclose(got['norm_preds_1'], np.mean([f['norm_preds_1'] for f in frames], axis=0))
    pd.testing.assert_frame_equal(frames[0], _member_frames(n, steps, seed=n)[0])      # the members are not modified


def test_misaligned_members_are_refused():
    frames = _member_frames(3, 1, seed=2)
    shuffled = frames[1].iloc[::-1].reset_index(drop=True)
    other_key = frames[2].copy()
    other_key.loc[5, 'gvkey'] = '999999'
    for bad, k in ((shuffled, 1), (other_key, 2), (frames[1].iloc[:-1], 1)):
        members = list(frames)
        members[k] = bad
        with pytest.raises(ValueError, match='member %d' % k):
            me.ensemble_point_estimate(members, 1)


def _budget(sm, per_sm, num, den):
    out = C.c_int64(-1)
    N.check(N.load().lfmq_persistent_cta_budget(sm, per_sm, num, den, C.byref(out)))
    return out.value


def test_persistent_cta_budget_of_a_device_share():
    assert _budget(132, 2, 1, 1) == 264 and _budget(132, 1, 5, 5) == 132          # the whole device, as before
    assert _budget(132, 2, 1, 2) == 66 and _budget(132, 1, 1, 3) == 44 and _budget(132, 2, 2, 3) == 88
    assert _budget(132, 1, 1, 8) == 16 and _budget(132, 4, 1, 200) == 0
    for n in range(2, 17):               # shares summing to 1 never count on more CTAs than the machine has SMs
        assert n * _budget(132, 2, 1, n) <= 132
        assert _budget(132, 2, 1, n) + _budget(132, 2, n - 1, n) <= 132
    lib = N.load()
    out = C.c_int64(0)
    for bad in ((0, 1, 1, 1), (132, 0, 1, 1), (132, 1, 0, 1), (132, 1, 3, 2)):
        assert lib.lfmq_persistent_cta_budget(*bad, C.byref(out)) != 0, bad
    assert lib.lfmq_persistent_cta_budget(132, 1, 1, 1, None) != 0
    assert lib.lfmq_set_device_share(None, 1, 2) != 0 and b'num <= den' in lib.lfmq_last_error()
