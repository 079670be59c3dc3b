"""Independent checker of ensemble_preds.dat: what the reference's point-estimate aggregation (utils/post_processing.py,
aggregate_point_estimate) produces, computed here with DataFrame arithmetic.  Member 0's frame, its columns in their
order, with every column whose name contains 'preds' replaced by the members' element-wise mean, and per forecast step s
    norm_squared_diff_s    = (norm_targets_s - norm_preds_s)^2
    abs_err_s              = |targets_s - preds_s|
    fcst_err_s             = abs_err_s / |targets_s|
    unscaled_squared_err_s = (abs_err_s / seq_norm)^2
recomputed from the averaged predictions; every other column is member 0's."""
import numpy as np


def expected_ensemble_frame(frames, forecast_steps):
    averaged = [c for c in frames[0].columns if 'preds' in c]
    expected = frames[0].copy()
    expected[averaged] = sum(f[averaged] for f in frames) / len(frames)
    for s in range(1, forecast_steps + 1):
        tar, pred = expected['targets_%d' % s].to_numpy(), expected['preds_%d' % s].to_numpy()
        gap = np.abs(tar - pred)
        expected['norm_squared_diff_%d' % s] = (expected['norm_targets_%d' % s].to_numpy() -
                                                expected['norm_preds_%d' % s].to_numpy()) ** 2
        expected['abs_err_%d' % s] = gap
        expected['fcst_err_%d' % s] = gap / np.abs(tar)
        expected['unscaled_squared_err_%d' % s] = (gap / expected['seq_norm'].to_numpy()) ** 2
    return expected
