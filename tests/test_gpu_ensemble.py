"""Ensembles on the GPU: handles trained at the same time on their own streams and host threads compute what they
compute one after another, on every path (fp32 SIMT, bf16 cluster kernels, bf16 general path with device shares, with
persistent launches kept and with persistent launches given up), and the CLI trains and predicts a 3-member ensemble end
to end (runtime/model_execution.py:154-199 of the reference)."""
import os
import pickle
import threading

import numpy as np
import pandas as pd
import pytest

from ensemble_checker import expected_ensemble_frame
from util import make_engine, make_problem

pytestmark = pytest.mark.gpu

N_MEMBERS, STEPS = 3, 3
# name -> shape, engine options.  bf16_general: the general path at a shape whose backward steps run as ONE persistent
# launch alone on the GPU (64 CTAs per half-batch chain), which a share of 1/3 (44 CTAs) turns into one launch per time
# step.  bf16_general_persistent: the reference's default shape, whose 2-CTA persistent launches fit any share of 1/3,
# so three of them run at the same time, each with its own step-barrier counters.
CASES = {
    'fp32': dict(B=256, T=5, F=32, O=16, H=64, L=2, kw=dict(precision='fp32', dropout=0.1)),
    'bf16_cluster': dict(B=1024, T=8, F=32, O=16, H=256, L=1, kw=dict(precision='bf16')),
    'bf16_general': dict(B=4096, T=8, F=32, O=16, H=512, L=2, kw=dict(precision='bf16', dropout=0.2,
                                                                      recurrent_dropout=0.1)),
    'bf16_general_persistent': dict(B=256, T=5, F=32, O=16, H=64, L=2, kw=dict(precision='bf16', dropout=0.1,
                                                                               recurrent_dropout=0.1)),
}


def _members(case):
    import torch
    c = CASES[case]
    B, T, F, O, H, L = (c[k] for k in 'BTFOHL')
    engines, data = [], []
    for i in range(N_MEMBERS):
        params, x, y = make_problem(B, T, F, O, H, L, seed=20 + i)
        eng = make_engine(B, T, F, O, H, L, target_idx=3, train=True, seed=100 + i, **c['kw'])
        eng.set_weights(params)
        engines.append(eng)
        data.append((torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()))
    torch.cuda.synchronize()
    return engines, data


def _train(engines, data, concurrent):
    """STEPS train steps of every member on a stream of its own; concurrent: all members at once, one host thread each.
    Returns each member's losses, weights, and the kernels launched."""
    import torch
    losses = [None] * len(engines)
    errors = []
    start = threading.Barrier(len(engines)) if concurrent else None

    def member(i):
        try:
            torch.cuda.set_device(0)
            s = torch.cuda.Stream()
            with torch.cuda.stream(s):
                if start is not None:
                    start.wait()
                out = [engines[i].train_step(data[i][0], data[i][1], k, 0.6) for k in range(STEPS)]
                losses[i] = torch.stack(out)
            s.synchronize()
        except Exception as e:          # surfaced by the caller
            errors.append(e)
            if start is not None:
                start.abort()

    n0 = engines[0].launch_count
    if concurrent:
        threads = [threading.Thread(target=member, args=(i,)) for i in range(len(engines))]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
    else:
        for i in range(len(engines)):
            member(i)
    if errors:
        raise errors[0]
    launches = engines[0].launch_count - n0
    return [l.cpu().numpy() for l in losses], [e.get_weights(trainable_only=False) for e in engines], launches


@pytest.mark.parametrize('case', list(CASES))
def test_concurrent_handles_compute_what_they_compute_one_after_another(case):
    one, one_data = _members(case)
    seq_losses, seq_weights, seq_launches = _train(one, one_data, concurrent=False)
    for e in one:
        e.close()
    many, many_data = _members(case)
    for e in many:
        e.set_device_share(1, N_MEMBERS)
    con_losses, con_weights, con_launches = _train(many, many_data, concurrent=True)
    for e in many:
        e.close()
    for i in range(N_MEMBERS):
        assert np.isfinite(seq_losses[i]).all() and seq_losses[i][-1, 1] != seq_losses[(i + 1) % N_MEMBERS][-1, 1]
        if case == 'fp32':
            np.testing.assert_array_equal(con_losses[i], seq_losses[i])
            for a, b in zip(con_weights[i], seq_weights[i]):
                np.testing.assert_array_equal(a, b)
        else:   # the bound of test_gpu_generic.py::test_persistent_steps_equal_one_launch_per_step
            np.testing.assert_allclose(con_losses[i], seq_losses[i], rtol=1e-6, atol=1e-9)
            for a, b in zip(con_weights[i], seq_weights[i]):
                np.testing.assert_allclose(a, b, rtol=1e-6, atol=1e-9)
    if case == 'bf16_general':      # the shares turned persistent launches into one launch per time step
        assert con_launches > seq_launches
    else:
        assert con_launches == seq_launches
    if case == 'bf16_general_persistent':
        # the same handles with a budget of one CTA take one launch per time step: so the runs above, alone and side by
        # side, both ran the persistent launches
        stepped, stepped_data = _members(case)
        for e in stepped:
            e.set_device_share(1, 132)
        _, _, stepped_launches = _train(stepped, stepped_data, concurrent=False)
        for e in stepped:
            e.close()
        assert stepped_launches > seq_launches


@pytest.fixture(scope='module')
def workdir(tmp_path_factory):
    from lfm_quant_b200.scripts.synthetic import write_open_dataset, write_system_test_conf
    d = tmp_path_factory.mktemp('ens')
    write_open_dataset(str(d / 'datasets' / 'open-dataset.dat'), n_keys=30, n_months=420, seed=9)
    write_system_test_conf(str(d / 'config' / 'system-test.conf'), str(d / 'datasets'), str(d / 'experiments'))
    (d / 'experiments').mkdir()          # an ensemble needs an existing experiments_dir (model_execution.py:169-170)
    return d


def test_cli_trains_and_predicts_a_three_member_ensemble(workdir, monkeypatch):
    from lfm_quant_b200.scripts import configs
    from lfm_quant_b200.scripts import lfm_quant as cli
    monkeypatch.setenv('LFM_QUANT_ROOT', str(workdir))
    monkeypatch.setenv('LFMQ_SEEDED_SHUFFLE', '1')        # the batch order follows the seed: training is repeatable
    conf = str(workdir / 'config' / 'system-test.conf')
    ens = ['--config=' + conf, '--num_procs', '3', '--NPE', '3', '--model_dir', 'ens']
    configs.reset()
    valid = cli.main(ens + ['--train=True'])
    assert len(valid) == 3 and np.isfinite(valid).all()
    edir = workdir / 'experiments' / 'ens'
    mdirs = [edir / ('system-test-%d' % k) for k in range(3)]
    for k, m in enumerate(mdirs):
        for f in ('model-%d.conf' % k, 'scales.dat', 'chkpts/chkpt.lfmq.npz', 'chkpts/chkpt.index',
                  'train_log/system-test-train-logs-epoch.csv', 'train_log/system-test-train-logs-batch.csv'):
            assert (m / f).is_file(), (k, f)
        log = pd.read_csv(m / 'train_log' / 'system-test-train-logs-epoch.csv')
        assert log['valid_mse'].min() == pytest.approx(valid[k])
    w = [np.load(m / 'chkpts' / 'chkpt.lfmq.npz') for m in mdirs]
    assert not np.array_equal(w[0]['lstm_1/kernel'], w[1]['lstm_1/kernel'])       # seeds differ

    # each member trains alone (num_procs 1) from its model-k.conf, in a directory of its own, what it trained beside
    # the others: the same split, scaler, logged losses and weights
    for k, m in enumerate(mdirs):
        alone = workdir / 'experiments' / ('alone-%d' % k)
        configs.reset()
        cli.main(['--config=' + str(m / ('model-%d.conf' % k)), '--train=True', '--model_dir', str(alone)])
        a, b = (pickle.load(open(str(d / 'scales.dat'), 'rb')) for d in (alone, m))
        for key in ('center', 'scale'):
            np.testing.assert_array_equal(a[key], b[key])
        la, lb = (pd.read_csv(d / 'train_log' / 'system-test-train-logs-epoch.csv') for d in (alone, m))
        pd.testing.assert_frame_equal(la[['epoch', 'mse', 'valid_mse']], lb[['epoch', 'mse', 'valid_mse']])
        wa = np.load(alone / 'chkpts' / 'chkpt.lfmq.npz')
        assert set(wa.files) == set(w[k].files)
        for name in wa.files:
            np.testing.assert_array_equal(wa[name], w[k][name], err_msg=name)

    configs.reset()
    df = cli.main(ens + ['--train=False'])
    members = [pd.read_csv(m / 'pred' / 'preds.dat', sep=' ', dtype={'gvkey': str}) for m in mdirs]
    assert len(members[0]) > 100
    written = pd.read_csv(edir / 'ensemble_preds.dat', sep=' ', dtype={'gvkey': str})
    want = expected_ensemble_frame(members, 1)
    pd.testing.assert_frame_equal(df, want, check_exact=False, rtol=1e-12)
    pd.testing.assert_frame_equal(written, want, check_exact=False, rtol=1e-12)
    assert not np.array_equal(members[0]['norm_preds_1'].values, members[1]['norm_preds_1'].values)

    # each member predicts alone (num_procs 1) from its model-k.conf -- its seed, its directory -- what it predicted
    # beside the others
    for k, m in enumerate(mdirs):
        configs.reset()
        cli.main(['--config=' + str(m / ('model-%d.conf' % k)), '--train=False', '--preds_fname', 'alone.dat'])
        alone = pd.read_csv(m / 'pred' / 'alone.dat', sep=' ', dtype={'gvkey': str})
        pd.testing.assert_frame_equal(alone, members[k])
    configs.reset()
