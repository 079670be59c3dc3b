"""--mc_samples on the host: the flag, and which runs take more than one Monte-Carlo dropout sample (UQ prediction
only).  The samples themselves are checked on the GPU (tests/test_gpu_mc_samples.py)."""
import pytest

from lfm_quant_b200.scripts import base_config, configs


@pytest.fixture()
def fresh_flags():
    configs.reset()
    yield
    configs.reset()


def test_mc_samples_flag_defaults_to_one_sample(fresh_flags):
    assert base_config.get_configs([]).mc_samples == 1
    assert base_config.get_configs(['--mc_samples', '16']).mc_samples == 16


@pytest.mark.parametrize('argv', [
    ['--mc_samples', '4', '--train=False'],                                                       # a point estimate
    ['--mc_samples', '4', '--train=True', '--nn_type', 'RNNUqRangeEstimate', '--UQ=True'],        # training
    ['--mc_samples', '0', '--train=False', '--nn_type', 'RNNUqRangeEstimate', '--UQ=True'],
])
def test_mc_samples_outside_uq_prediction_is_refused(fresh_flags, monkeypatch, argv):
    from lfm_quant_b200.scripts.runtime.model_execution import ModelExecution
    monkeypatch.setattr(ModelExecution, 'single_execution', staticmethod(lambda cfg: 'ran'))
    with pytest.raises(ValueError, match='--mc_samples'):
        ModelExecution(base_config.get_configs(argv))()


def test_mc_samples_runs_uq_prediction_in_one_process(fresh_flags, monkeypatch):
    """--mc_samples > 1 is a single execution; num_procs > 1 UQ prediction stays refused."""
    from lfm_quant_b200.scripts.runtime.model_execution import ModelExecution
    seen = []
    monkeypatch.setattr(ModelExecution, 'single_execution', staticmethod(lambda cfg: seen.append(cfg.mc_samples) or 'ran'))
    c = base_config.get_configs(['--mc_samples', '16', '--train=False', '--nn_type', 'RNNUqRangeEstimate', '--UQ=True'])
    assert ModelExecution(c)() == 'ran' and seen == [16]
    c.num_procs = 4
    with pytest.raises(NotImplementedError):
        ModelExecution(c)()
