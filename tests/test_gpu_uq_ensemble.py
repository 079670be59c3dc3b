"""Monte-Carlo prediction of a UQ model at the GPU's width, and the ensemble file it leads to: NativeForecaster.predict_mc
runs on a forward-only engine of min(samples * batch_size, MC_ROWS) rows per launch, and `--mc_samples S` writes
ensemble_preds.dat (ModelExecution.write_uq_ensemble) next to preds.dat.

Checked here: the wide engine gives the moments of the model's batch_size handle bit for bit, in one library call per
batch; it follows load_weights / set_weights and close releases it; and the CLI writes the same preds.dat as the
batch_size handle does, and ensemble_preds.dat = the host aggregation of that file."""
import io
import os

import numpy as np
import pandas as pd
import pytest
import torch

pytestmark = pytest.mark.gpu
T, F, O = 5, 12, 6


def _cfg(argv):
    from lfm_quant_b200.scripts import base_config, configs
    configs.reset()
    return base_config.get_configs(['--num_hidden', '64', '--num_layers', '1', '--batch_size', '256', '--dropout',
                                    '0.2', '--recurrent_dropout', '0.15', '--train=False', '--nn_type',
                                    'RNNUqRangeEstimate', '--UQ=True'] + argv)


def _model(prec, stages):
    from lfm_quant_b200.scripts.models.point_estimate.rnn_point_estimate import NativeForecaster
    argv = ['--precision', prec, '--forecast_steps', str(stages), '--forecast_steps_weights',
            '-'.join(['1.0', '0.5'][:stages])]
    return NativeForecaster(_cfg(argv), T, F, O, 1, uq=True)


def _perturbed(m, seed):
    rng = np.random.RandomState(seed)
    return [w + rng.normal(size=w.shape).astype(np.float32) * 0.05 if w.ndim == 2 else w for w in m.get_weights()]


class _Calls(object):
    """Counts the calls of the library's Monte-Carlo entry points (and passes them through)."""

    def __init__(self, monkeypatch, lib):
        self.n = 0
        for name in ('lfmq_forward_uq_mc', 'lfmq_chain_forward_uq_mc'):
            fn = getattr(lib, name)
            monkeypatch.setattr(lib, name, self._wrap(fn))

    def _wrap(self, fn):
        def call(*args):
            self.n += 1
            return fn(*args)
        return call


@pytest.mark.parametrize('prec', ['fp32', 'bf16', 'bf16x3'])
@pytest.mark.parametrize('stages', [1, 2])
@pytest.mark.parametrize('samples', [2, 32, 64])
def test_wide_engine_gives_the_batch_size_handles_moments(monkeypatch, prec, stages, samples):
    """A full batch of 256 windows and a short last batch of 100.  samples = 64 needs 16384 rows, more than MC_ROWS:
    the wide engine cuts its launches.  Each predict_mc is one lfmq_*forward_uq_mc call."""
    from lfm_quant_b200.scripts.models.point_estimate import rnn_point_estimate as rpe
    m = _model(prec, stages)
    m.set_weights(_perturbed(m, 3))
    x = torch.from_numpy(np.random.RandomState(1).normal(size=(256, T, F)).astype(np.float32)).cuda()
    calls = _Calls(monkeypatch, m.engine.lib)
    for xb in (x, x[:100].contiguous()):
        before = calls.n
        got = m.predict_mc(xb, samples)
        assert calls.n == before + 1
        wide = m._mc_engine
        assert wide is not None and wide is not m.engine
        assert wide.cfg.max_batch == min(samples * 256, rpe.MC_ROWS) and m.engine.cfg.max_batch == 256
        ref = m.engine.forward_mc(xb, samples, step=m._calls, row0=0)
        assert len(got) == stages
        for g, r in zip(got, ref):
            for a, b in zip(g, r):
                assert torch.equal(a, b)
    m.close()


def test_one_sample_keeps_the_batch_size_handle():
    m = _model('bf16', 1)
    x = torch.from_numpy(np.random.RandomState(2).normal(size=(256, T, F)).astype(np.float32)).cuda()
    got = m.predict_mc(x, 1)
    assert m._mc_engine is None
    for a, b in zip(got[0], m.engine.forward_mc(x, 1, step=m._calls)[0]):
        assert torch.equal(a, b)
    m.close()


@pytest.mark.parametrize('prec', ['fp32', 'bf16'])
def test_weights_set_after_the_first_prediction_reach_the_wide_engine(tmp_path, prec):
    """load_weights and set_weights after the first predict_mc: its output is the new weights' output; close releases
    both engines."""
    m, other = _model(prec, 2), _model(prec, 2)
    other.set_weights(_perturbed(other, 7))
    other.save_weights(str(tmp_path / 'chkpt'))
    x = torch.from_numpy(np.random.RandomState(3).normal(size=(256, T, F)).astype(np.float32)).cuda()
    first = m.predict_mc(x, 16)
    m.load_weights(str(tmp_path / 'chkpt'))
    got = m.predict_mc(x, 16)
    ref = other.engine.forward_mc(x, 16, step=m._calls)
    assert not torch.equal(got[0][0], first[0][0])
    for g, r in zip(got, ref):
        for a, b in zip(g, r):
            assert torch.equal(a, b)
    w = _perturbed(m, 9)
    m.set_weights(w)
    other.set_weights(w)
    got = m.predict_mc(x, 16)
    for g, r in zip(got, other.engine.forward_mc(x, 16, step=m._calls)):
        for a, b in zip(g, r):
            assert torch.equal(a, b)
    wide = m._mc_engine
    m.close()
    assert m._mc_engine is None
    assert all(not e.handle.value for e in wide.stages + m.engine.stages)
    other.close()


@pytest.fixture(scope='module')
def workdir(tmp_path_factory):
    from lfm_quant_b200.scripts.synthetic import write_open_dataset, write_system_test_conf
    d = tmp_path_factory.mktemp('uqens')
    write_open_dataset(str(d / 'datasets' / 'open-dataset.dat'), n_keys=30, n_months=420, seed=9)
    write_system_test_conf(str(d / 'config' / 'system-test.conf'), str(d / 'datasets'), str(d / 'experiments'))
    os.environ.setdefault('LFM_QUANT_ROOT', str(d))
    return d


@pytest.mark.parametrize('steps', [1, 2])
def test_cli_writes_ensemble_preds(workdir, monkeypatch, steps):
    """Train at fp32, then predict with --mc_samples 16 at fp32 and bf16.  preds.dat is byte for byte what the
    batch_size handle writes (MC_ROWS = 1 keeps predict_mc on it); ensemble_preds.dat is the host aggregation of that
    preds.dat, with pred_var_k = preds_k / sqrt(variance_k).  A prediction without the flag writes no ensemble file."""
    from lfm_quant_b200.scripts import configs
    from lfm_quant_b200.scripts import lfm_quant as cli
    from lfm_quant_b200.scripts.models.point_estimate import rnn_point_estimate as rpe
    from lfm_quant_b200.scripts.runtime.model_execution import ensemble_uq_estimate
    conf = str(workdir / 'config' / 'system-test.conf')
    extra = ['--nn_type', 'RNNUqRangeEstimate', '--UQ=True', '--dropout', '0.1', '--recurrent_dropout', '0.1',
             '--model_dir', 'ens-%d' % steps, '--forecast_steps', str(steps), '--forecast_steps_weights',
             '-'.join(['1.0', '0.5'][:steps])]
    mdir = workdir / 'experiments' / ('ens-%d' % steps)
    configs.reset()
    cli.main(['--config=' + conf, '--train=True'] + extra)
    ens = mdir / 'ensemble_preds.dat'

    def predict(argv):
        if ens.exists():
            ens.unlink()
        configs.reset()
        cli.main(['--config=' + conf, '--train=False'] + extra + argv)
        return (mdir / 'pred' / 'preds.dat').read_bytes(), ens.read_bytes() if ens.exists() else None

    for prec in ('fp32', 'bf16'):
        flags = ['--mc_samples', '16', '--precision', prec]
        wide = predict(flags)
        with monkeypatch.context() as mp:
            mp.setattr(rpe, 'MC_ROWS', 1)
            narrow = predict(flags)
        assert wide[0] == narrow[0] and wide[1] == narrow[1], prec
        preds = pd.read_csv(io.BytesIO(wide[0]), sep=' ', dtype={'gvkey': str})
        buf = io.StringIO()
        ensemble_uq_estimate(preds, steps).to_csv(buf, sep=' ', index=False)
        assert buf.getvalue().encode() == wide[1], prec
        # preds as the aggregation read them; the file's values exactly as written
        got = pd.read_csv(io.BytesIO(wide[1]), sep=' ', dtype={'gvkey': str}, float_precision='round_trip')
        for s in range(1, steps + 1):
            np.testing.assert_array_equal(got['pred_var_%d' % s],
                                          preds['preds_%d' % s] / np.sqrt(preds['variance_%d' % s]))
        assert [c for c in got.columns if c.endswith('_50')] == (['norm_preds_%d_50' % s for s in range(1, steps + 1)]
                                                                 + ['preds_%d_50' % s for s in range(1, steps + 1)])
        assert not any(c.startswith('norm_preds_var_') for c in got.columns)
    assert predict([])[1] is None
    configs.reset()
