"""ensemble_preds.dat of a UQ prediction with Monte-Carlo samples, on the host: ensemble_uq_estimate and calibrated_z
against the reference's post-processing (tests/golden/reference_uq_ensemble.npz, made by make_reference_uq_ensemble.py
from the unmodified utils/post_processing.py), and which runs write the file."""
import io
import os

import numpy as np
import pandas as pd
import pytest

from lfm_quant_b200.scripts import base_config, configs
from lfm_quant_b200.scripts.runtime import model_execution as me

GOLDEN = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'reference_uq_ensemble.npz'))
CASES = sorted({k.split('/')[0] for k in GOLDEN.files if not k.startswith('iso/')})
ISO = sorted({k.split('/')[1] for k in GOLDEN.files if k.startswith('iso/')})
STEPS = {'one_step': 1, 'two_steps': 2, 'all_nan': 1, 'few_rows': 1, 'out_of_range': 2}
REL = 1e-12


def _frame(text):
    return pd.read_csv(io.StringIO(str(text)), sep=' ', dtype={'gvkey': str})


def _assert_frames_match(got, ref):
    assert list(got.columns) == list(ref.columns)
    for c in ref.columns:
        if c == 'gvkey':
            assert list(got[c]) == list(ref[c])
            continue
        a, b = got[c].to_numpy(dtype=np.float64), ref[c].to_numpy(dtype=np.float64)
        assert np.array_equal(np.isnan(a), np.isnan(b)), c
        ok = ~np.isnan(b)
        assert np.all(np.abs(a[ok] - b[ok]) <= REL * np.abs(b[ok])), (c, np.max(np.abs(a[ok] - b[ok])))


def test_fixture_covers_the_cases():
    assert CASES == sorted(STEPS)
    out = _frame(GOLDEN['out_of_range/out_csv'])
    assert out['preds_1_50'].notna().all() and out['preds_2_50'].isna().all()       # level outside the fitted range
    assert _frame(GOLDEN['all_nan/out_csv'])['preds_1_50'].isna().all()
    assert len(np.unique(GOLDEN['few_rows/freq'][:, 0])) < 100                       # tied frequencies


@pytest.mark.parametrize('case', CASES)
def test_aggregation_matches_the_reference(case, capsys):
    """Columns, their order, NaN positions and values to 1e-12 relative; the same 'Scaled MSE' lines."""
    frame = _frame(GOLDEN[case + '/in_csv'])
    got = me.ensemble_uq_estimate(frame, STEPS[case])
    assert capsys.readouterr().out == str(GOLDEN[case + '/stdout'])
    # as the file is written and read back: the reference's frame went through the same to_csv
    buf = io.StringIO()
    got.to_csv(buf, sep=' ', index=False)
    _assert_frames_match(_frame(buf.getvalue()), _frame(GOLDEN[case + '/out_csv']))
    _assert_frames_match(got, _frame(GOLDEN[case + '/out_csv']))
    assert 'norm_preds_var_1' in frame.columns and 'norm_preds_var_1' not in got.columns


@pytest.mark.parametrize('case', [c for c in CASES if c != 'all_nan'])
def test_coverage_and_calibrated_z_match_the_reference(case):
    frame = _frame(GOLDEN[case + '/in_csv'])
    preds = sorted(c for c in frame.columns if 'preds' in c and 'preds_var' not in c)
    freq = np.stack([me.coverage(frame[p].values, frame[p.replace('preds', 'variance')].values,
                                 frame[p.replace('preds', 'targets')].values, me.CALIBRATION_Z) for p in preds], 1)
    assert np.array_equal(freq, GOLDEN[case + '/freq'])
    z = np.array([me.calibrated_z(freq[:, i], me.CALIBRATION_Z, me.CERTAINTY_LEVEL) for i in range(freq.shape[1])])
    ref = GOLDEN[case + '/z']
    assert np.array_equal(np.isnan(z), np.isnan(ref))
    ok = ~np.isnan(ref)
    assert np.all(np.abs(z[ok] - ref[ok]) <= REL * np.abs(ref[ok])), (z, ref)


@pytest.mark.parametrize('name', ISO)
def test_isotonic_helper_matches_scikit_learn(name):
    """A single distinct frequency (a constant fit), levels below and above the range (NaN), a level on a fitted point,
    and a decreasing run that the fit pools."""
    g = lambda k: GOLDEN['iso/%s/%s' % (name, k)]
    got = me.calibrated_z(g('freq'), me.CALIBRATION_Z, float(g('level')))
    ref = float(g('out')[0])
    if np.isnan(ref):
        assert np.isnan(got)
    else:
        assert abs(got - ref) <= REL * abs(ref), (got, ref)


def test_point_ensemble_output_is_unchanged(capsys):
    """ensemble_point_estimate shares the error recomputation: the same columns and prints as the reference's
    aggregate_point_estimate of one frame (its preds columns, means of one member, pass through)."""
    frame = _frame(GOLDEN['two_steps/in_csv'])
    got = me.ensemble_point_estimate([frame, frame.copy()], 2)
    lines = capsys.readouterr().out.splitlines()
    assert lines == ['Scaled MSE for step %d: %1.4f' % (s, frame['norm_squared_diff_%d' % s].mean()) for s in (1, 2)]
    assert list(got.columns) == list(frame.columns)
    for c in ('abs_err_2', 'fcst_err_1', 'unscaled_squared_err_2', 'norm_squared_diff_1'):
        np.testing.assert_allclose(got[c], frame[c], rtol=1e-12)


@pytest.fixture()
def fresh_flags():
    configs.reset()
    yield
    configs.reset()


@pytest.mark.parametrize('flags, writes', [
    (['--mc_samples', '16'], True),
    (['--mc_samples', '1'], False),
    ([], False),
])
def test_ensemble_preds_is_written_for_mc_prediction_only(fresh_flags, monkeypatch, tmp_path, flags, writes):
    """A stubbed single execution writes pred/preds.dat (the two-step fixture frame); ModelExecution then writes
    <experiments_dir>/<model_dir>/ensemble_preds.dat = ensemble_uq_estimate of it, only with --mc_samples > 1."""
    text = str(GOLDEN['two_steps/in_csv'])

    def single_execution(cfg):
        os.makedirs(os.path.join(cfg.experiments_dir, cfg.model_dir, 'pred'))
        with open(os.path.join(cfg.experiments_dir, cfg.model_dir, 'pred', cfg.preds_fname), 'w') as fh:
            fh.write(text)
        return 'ran'

    monkeypatch.setattr(me.ModelExecution, 'single_execution', staticmethod(single_execution))
    c = base_config.get_configs(['--train=False', '--nn_type', 'RNNUqRangeEstimate', '--UQ=True', '--forecast_steps',
                                 '2', '--forecast_steps_weights', '1.0-0.5', '--experiments_dir', str(tmp_path),
                                 '--model_dir', 'm'] + flags)
    assert me.ModelExecution(c)() == 'ran'
    path = tmp_path / 'm' / 'ensemble_preds.dat'
    assert path.exists() == writes
    assert (tmp_path / 'm' / 'pred' / 'preds.dat').read_text() == text
    if writes:
        got = pd.read_csv(path, sep=' ', dtype={'gvkey': str})
        _assert_frames_match(got, _frame(GOLDEN['two_steps/out_csv']))


def test_training_writes_no_ensemble_preds(fresh_flags, monkeypatch, tmp_path):
    monkeypatch.setattr(me.ModelExecution, 'single_execution', staticmethod(lambda cfg: 'trained'))
    c = base_config.get_configs(['--train=True', '--nn_type', 'RNNUqRangeEstimate', '--UQ=True',
                                 '--experiments_dir', str(tmp_path), '--model_dir', 'm'])
    assert me.ModelExecution(c)() == 'trained'
    assert not (tmp_path / 'm').exists()
