"""ModelExecution (reference: scripts/runtime/model_execution.py:19-241): ``fixed_dates`` training / prediction of
one config in-process.  A point-estimate ensemble (num_procs > 1, :154-199) runs its members in this process too: NPE of
them at a time, each on its own host thread and CUDA stream, side by side on the GPU(s) (DESIGN.md
section 6a).  The reference starts one ``lfm_quant.py`` process per member instead (:142).  The candidates of a
hyper-parameter search generation run the same way (run_candidates, DESIGN.md section 6b), and so do the origins of a
walk-forward backtest (training_type ``iterative``, which the reference leaves unbuilt; DESIGN.md section 6c).  The
ensembles' post-processing (utils/post_processing.py) is here too: ensemble_point_estimate, and ensemble_uq_estimate of
a UQ prediction with Monte-Carlo samples (DESIGN.md section 5c)."""
from __future__ import absolute_import, division, print_function

import copy
import os
import pathlib
import random
import traceback
from collections import Counter
from concurrent.futures import FIRST_EXCEPTION, ThreadPoolExecutor, wait
from itertools import cycle

import numpy as np
import pandas as pd
import scipy.optimize
import scipy.stats

from .. import base_config
from ..predict import FACTOR_MAX_SCORES, factor_names, factor_tables


def member_configs(config):
    """The N = num_procs members of a point-estimate ensemble (model_execution.py:162-190): member k has member_id k,
    model_dir <experiments_dir>/<model_dir>/<name>-k (absolute, so that the member's files land there whatever the
    working directory), default_gpu /gpu:(k mod num_gpu), and num_procs = NPE = 1.  Member 0 keeps config.seed; the
    others draw theirs from random.Random(config.seed) where the reference draws from the unseeded global generator
    (:187-188), so an ensemble can be reproduced.  Returns (<experiments_dir>/<model_dir>, [configs])."""
    assert os.path.isdir(config.experiments_dir), "Experiments dir  %s does not exist" % config.experiments_dir
    experiment_dir = os.path.join(os.path.abspath(config.experiments_dir), config.model_dir)
    gpus = cycle(range(config.num_gpu))
    seeds = random.Random(config.seed)
    members = []
    for k in range(config.num_procs):
        c = copy.deepcopy(config)
        c.member_id = k
        c.model_dir = os.path.join(experiment_dir, '%s-%d' % (config.name, k))
        c.default_gpu = '/gpu:%d' % next(gpus)
        if k > 0:
            c.seed = seeds.randint(0, 1000)
        c.num_procs = 1
        c.NPE = 1
        members.append(c)
    return experiment_dir, members


def add_months(yyyymm, months):
    """The YYYYMM date `months` months after `yyyymm` (before it when negative)."""
    m = (yyyymm // 100) * 12 + yyyymm % 100 - 1 + months
    return (m // 12) * 100 + m % 12 + 1


def walk_forward_origins(split_date, end_date, stride):
    """The origins of a walk-forward backtest (DESIGN.md section 6c): d_0 = split_date, d_k = d_0 + k·stride months,
    every d_k < end_date.  All dates YYYYMM."""
    if stride < 1:
        raise ValueError('--stride %d: walk-forward origins are stride >= 1 months apart' % stride)
    origins = []
    while add_months(split_date, len(origins) * stride) < end_date:
        origins.append(add_months(split_date, len(origins) * stride))
    return origins


def check_walk_forward(config):
    """Raises ValueError, naming the flag, for a walk-forward config (training_type iterative) that cannot run."""
    c = config
    if c.split_date is None or not (1 <= c.split_date % 100 <= 12 and c.start_date < c.split_date < c.end_date):
        raise ValueError('--split_date %s: training_type iterative needs the first origin, a YYYYMM date strictly '
                         'between --start_date %s and --end_date %s' % (c.split_date, c.start_date, c.end_date))
    walk_forward_origins(c.split_date, c.end_date, c.stride)
    if c.forecast_n > c.stride:
        # training at origin d keeps windows dated <= d - stride; their targets lie forecast_n months later
        raise ValueError('--forecast_n %d > --stride %d: the targets of an origin\'s last training windows would lie '
                         'after the origin' % (c.forecast_n, c.stride))
    if c.num_procs > 1:
        raise ValueError('--num_procs %d: training_type iterative trains one model per origin, not an ensemble'
                         % c.num_procs)
    if c.cdrs_inference:
        raise ValueError('--cdrs_inference: training_type iterative backtests on the datafile, not on CDRS data')
    if c.scalesfile and 'Naive' not in c.nn_type:
        raise ValueError('--scalesfile %s: with training_type iterative every origin fits scales.dat on its own data '
                         'and predicts with it' % c.scalesfile)
    if int(os.environ.get('WORLD_SIZE', '1')) > 1:
        raise ValueError('torchrun (WORLD_SIZE %s): training_type iterative runs its origins side by side in one '
                         'process and cannot be combined with data parallelism; run it without torchrun'
                         % os.environ['WORLD_SIZE'])


def origin_configs(config):
    """The origins of a walk-forward backtest: origin k at d_k runs in <experiments_dir>/<model_dir>/<name>-wf-<d_k>
    (absolute) as fixed_dates runs with member_id k, default_gpu /gpu:(k mod num_gpu), num_procs = NPE = 1 and the
    backtest's seed.  Its training keeps start_date and ends at d_k; its prediction covers d_k + 1 month through
    min(d_k + stride months, end_date).  Returns (<experiments_dir>/<model_dir>, [(d_k, training config, prediction
    config)])."""
    assert os.path.isdir(config.experiments_dir), "Experiments dir  %s does not exist" % config.experiments_dir
    experiment_dir = os.path.join(os.path.abspath(config.experiments_dir), config.model_dir)
    gpus = cycle(range(config.num_gpu))
    out = []
    for k, origin in enumerate(walk_forward_origins(config.split_date, config.end_date, config.stride)):
        c = copy.deepcopy(config)
        c.training_type = 'fixed_dates'
        c.member_id = k
        c.model_dir = os.path.join(experiment_dir, '%s-wf-%d' % (config.name, origin))
        c.default_gpu = '/gpu:%d' % next(gpus)
        c.num_procs = 1
        c.NPE = 1
        train, pred = copy.deepcopy(c), c
        train.train = True
        train.end_date = origin
        pred.train = False
        pred.start_date = add_months(origin, 1)
        pred.end_date = min(add_months(origin, config.stride), config.end_date)
        if getattr(config, 'influence_top_k', 0) > 0 or getattr(config, 'conformal_levels', None) is not None:
            # the origin's own training draw: the attribution pool, the conformal calibration set
            pred.pool_dates = (train.start_date, train.end_date)
        # an origin predicts only its stride's months: the factor backtest runs once, over the stitched frame
        pred.factor_quantiles = 0
        pred.factor_return_field, pred.factor_horizon = None, 1
        out.append((origin, train, pred))
    return experiment_dir, out


def stitch_walk_forward(frames, origins):
    """walk_forward_preds.dat: the origins' preds.dat frames in origin order, each row with its origin (YYYYMM)."""
    return pd.concat([f.assign(origin=o) for f, o in zip(frames, origins)], ignore_index=True)


def write_conf(flags, path):
    """Writes the flags {name: value} to `path` in the file format the reference writes for an ensemble member or a
    search candidate (model_execution.py:130-140, genetic_algorithm.py:171-182): one line per flag that has a value, in
    order of the flag names.  A scalar (also a NumPy scalar, as values read from a CSV file are) is written as
    ``--name<7 spaces>value`` with a trailing space; a list or tuple as its items joined by '-'."""
    lines = []
    for name in sorted(flags):
        value = flags[name]
        if isinstance(value, (list, tuple)):
            lines.append('--%s       %s\n' % (name, '-'.join(str(item) for item in value)))
        elif isinstance(value, (bool, int, float, str, np.bool_, np.integer, np.floating)):
            lines.append('--%s       %s \n' % (name, value))
    with open(path, 'w') as fh:
        fh.writelines(lines)
    return path


def write_member_conf(config):
    """<member dir>/model-<member_id>.conf (write_conf).  ``lfm_quant.py --config`` on the file runs the member
    alone."""
    pathlib.Path(config.model_dir).mkdir(parents=True, exist_ok=True)
    return write_conf(config.as_dict(), os.path.join(config.model_dir, 'model-%d.conf' % config.member_id))


def ensemble_point_estimate(frames, forecast_steps):
    """ensemble_preds.dat of a point-estimate ensemble (the reference's aggregate_point_estimate,
    utils/post_processing.py:39-81) from the members' preds.dat frames: member 0's frame, every column whose name holds
    'preds' averaged over the members, and each forecast step's squared scaled error, absolute error, relative error
    and seq_norm-scaled squared error recomputed from those averages.  The members must hold the same (date, gvkey) rows
    in the same order, which the reference assumes without checking; here a mismatch raises ValueError."""
    keys = frames[0][['date', 'gvkey']].reset_index(drop=True)
    for k, f in enumerate(frames[1:], 1):
        if len(f) != len(keys) or not f[['date', 'gvkey']].reset_index(drop=True).equals(keys):
            raise ValueError('ensemble member %d predicted other (date, gvkey) rows than member 0, or in another order; '
                             'the members cannot be averaged row by row' % k)
    out = frames[0].copy()
    averaged = [c for c in out.columns if 'preds' in c]
    out[averaged] = np.stack([f[averaged].to_numpy(dtype=np.float64) for f in frames]).mean(axis=0)
    _recompute_errors(out, forecast_steps)
    _print_scaled_mse(out, forecast_steps)
    return out


def _recompute_errors(out, forecast_steps):
    """Each forecast step's squared scaled error, absolute error, relative error and seq_norm-scaled squared error,
    recomputed in place from the frame's predictions (utils/post_processing.py:62-73)."""
    for s in range(1, forecast_steps + 1):
        target, pred = out['targets_%d' % s], out['preds_%d' % s]
        err = (target - pred).abs()
        out['norm_squared_diff_%d' % s] = (out['norm_targets_%d' % s] - out['norm_preds_%d' % s]) ** 2
        out['abs_err_%d' % s] = err
        out['fcst_err_%d' % s] = err / target.abs()
        out['unscaled_squared_err_%d' % s] = (err / out['seq_norm']) ** 2


def _weighted_scaled_mse(df, config):
    """The mean squared scaled error of a predictions frame, weighted over the forecast steps
    (model_execution.py:70-72)."""
    valid_loss = 0
    for i in range(config.forecast_steps):
        valid_loss += df['norm_squared_diff_' + str(i + 1)].mean() * config.forecast_steps_weights[i]
    return valid_loss


def _print_scaled_mse(out, forecast_steps):
    for s in range(1, forecast_steps + 1):
        print("Scaled MSE for step %i: %1.4f" % (s, out['norm_squared_diff_%d' % s].mean()))


# The reference calibrates its lower bounds at this one level (post_processing.py:91-92): the interval that holds 50 % of
# the true values, over the z-scores of 100 p-values (:109-110).
CERTAINTY_LEVEL = 0.5
CALIBRATION_Z = scipy.stats.norm.ppf(np.linspace(0.0001, 0.999999, 100))


def coverage(pred, var, target, z):
    """The fraction of the true values inside pred ± z·sqrt(var), for each z (post_processing.py:126-144).  A NaN target
    counts as outside, and the denominator is the number of non-NaN targets."""
    sd = np.sqrt(var)
    zc = np.asarray(z, dtype=np.float64)[:, None]
    inside = np.less_equal(pred - zc * sd, target) & np.less_equal(target, pred + zc * sd)
    return inside.sum(axis=1) / (len(target) - np.isnan(target).sum())


def calibrated_z(freq, z, level):
    """sklearn.isotonic.IsotonicRegression().fit(freq, z).predict([level])[0] without scikit-learn: the increasing
    least-squares fit of z on freq, tied frequencies merged into the mean of their z, linear between the fitted points,
    NaN outside [min freq, max freq].  A single distinct frequency gives a constant fit, at every level."""
    freq, z = np.asarray(freq, dtype=np.float64), np.asarray(z, dtype=np.float64)
    order = np.lexsort((z, freq))
    freq, z = freq[order], z[order]
    xs, first, counts = np.unique(freq, return_index=True, return_counts=True)
    ys = scipy.optimize.isotonic_regression(np.add.reduceat(z, first) / counts, weights=counts.astype(np.float64),
                                            increasing=True).x
    if len(ys) == 1:
        return float(ys[0])
    if not xs[0] <= level <= xs[-1]:
        return np.nan
    # the interior points of a flat run are dropped, as scikit-learn does, so that a level on a fitted point takes the
    # same segment and rounds the same way
    keep = np.ones(len(ys), dtype=bool)
    keep[1:-1] = (ys[1:-1] != ys[:-2]) | (ys[1:-1] != ys[2:])
    xs, ys = xs[keep], ys[keep]
    hi = int(np.clip(np.searchsorted(xs, level), 1, len(xs) - 1))      # scipy.interpolate.interp1d, kind='linear'
    lo = hi - 1
    return float((ys[hi] - ys[lo]) / (xs[hi] - xs[lo]) * (level - xs[lo]) + ys[lo])


def ensemble_uq_estimate(frame, forecast_steps):
    """ensemble_preds.dat of a UQ prediction with Monte-Carlo dropout samples: what the reference's
    aggregate_uq_estimate (utils/post_processing.py:83-124) returns for the one frame `frame` (preds.dat as read_results
    reads it) at certainty level 0.5.  The frame already holds the ensemble's moments, so the mean over one member and
    its zero variance leave them as they are.

    The norm_preds_var_<k> columns are dropped first.  Added: pred_var_<k> = preds_<k> / sqrt(variance_<k>), the error
    columns recomputed, and the calibrated lower bounds <pred field>_50 = pred - z_50 · sqrt(variance) of every
    prediction column, where z_50 is the z-score whose interval covers 50 % of the true values (calibrated_z over
    coverage).  When every target is NaN (a prediction for dates without targets) the lower bounds are NaN."""
    out = frame.drop(columns=[c for c in frame.columns if c.startswith('norm_preds_var_')])
    pred_fields = sorted(c for c in out.columns if 'preds' in c)
    var_fields = sorted(c for c in out.columns if 'variance' in c)
    tar_fields = sorted(c for c in out.columns if 'targets' in c)
    if not (len(pred_fields) == len(var_fields) == len(tar_fields)
            and all(p.split('_')[-1] == v.split('_')[-1] for p, v in zip(pred_fields, var_fields))):
        raise ValueError('a UQ prediction holds one variance and one target column per prediction column; got %s, %s '
                         'and %s' % (pred_fields, var_fields, tar_fields))
    for p, v in zip(pred_fields, var_fields):
        if 'norm' not in p:
            out['pred_var_' + p.split('_')[-1]] = out[p] / np.sqrt(out[v])
    _recompute_errors(out, forecast_steps)
    suffix = '_%d' % int(CERTAINTY_LEVEL * 100)
    if out[tar_fields[0]].isnull().all():
        for p in pred_fields:
            out[p + suffix] = np.nan
        return out
    for p, v, t in zip(pred_fields, var_fields, tar_fields):
        pred, var = out[p].values, out[v].values
        z = calibrated_z(coverage(pred, var, out[t].values, CALIBRATION_Z), CALIBRATION_Z, CERTAINTY_LEVEL)
        out[p + suffix] = pred - z * np.sqrt(var)
    _print_scaled_mse(out, forecast_steps)
    return out


def candidate_config(conf_path):
    """The config that ``lfm_quant.py --config <conf_path>`` runs: the file parsed with the forecaster's flag schema."""
    from .. import configs, lfm_quant
    configs.reset()
    return lfm_quant.get_configs(['--config', conf_path])


def run_candidates(conf_paths, npe):
    """Trains (or, with train False, predicts) the hyper-parameter search candidates whose model.conf files are
    `conf_paths`, in this process, `npe` at a time: each on its own host thread and CUDA stream, on its GPU (the last
    character of default_gpu), with a device share of 1/min(npe, candidates on that GPU) (DESIGN.md section 6b).  Each
    runs what ``lfm_quant.py --config <its model.conf>`` runs alone, and writes the same files.

    A candidate that fails -- its file does not parse, the library refuses its config, or it raises while it runs --
    does not stop the others: its error is printed and returned.  Returns one entry per candidate, None or the error.
    A default_gpu that is not a CUDA device of this process is an error of the search and raises."""
    import torch
    errors = [None] * len(conf_paths)
    candidates = {}
    for i, path in enumerate(conf_paths):
        try:
            c = candidate_config(path)
            if c.training_type == 'iterative' or c.cdrs_inference or c.num_procs > 1:
                raise NotImplementedError('a search candidate runs as one fixed_dates model (training_type '
                                          'fixed_dates, no cdrs_inference, num_procs 1); %s asks for more' % path)
            candidates[i] = c
        except (Exception, SystemExit) as e:        # argparse exits on a value it cannot convert
            print('candidate %s refused: %r' % (path, e))
            errors[i] = e
    visible = torch.cuda.device_count() if torch.cuda.is_available() else 0
    for c in candidates.values():
        gpu = str(c.default_gpu)[-1]
        if not (gpu.isdigit() and int(gpu) < visible):
            raise RuntimeError('search candidate %s: default_gpu %s is not a CUDA device of this process (%d visible); '
                               'set num_gpu to at most the number of GPUs' % (c.member_id, c.default_gpu, visible))
    if not candidates:
        return errors
    npe = max(1, min(int(npe), len(candidates)))
    on_gpu = Counter(c.default_gpu for c in candidates.values())

    def run(i):
        c = candidates[i]
        try:
            ModelExecution.member_execution(c, min(npe, on_gpu[c.default_gpu]))
            return None
        except Exception as e:
            print('candidate %s failed:\n%s' % (conf_paths[i], traceback.format_exc()))
            return e

    with ThreadPoolExecutor(max_workers=npe) as pool:
        for i, err in zip(list(candidates), pool.map(run, list(candidates))):
            errors[i] = err
    return errors


def check_conformal(c):
    """Refuses --conformal_levels / --conformal_knn where they cannot run, before any work."""
    levels, knn = getattr(c, 'conformal_levels', None), getattr(c, 'conformal_knn', 0)
    if knn != 0:
        bad = ['conformal_knn must be in [1, 64] (0 = off)' if not 0 < knn <= 64 else None,
               'it scales conformal intervals: set --conformal_levels' if levels is None else None,
               'a UQ model is scaled by its own sigma' if c.UQ else None,
               'NaivePointEstimate has no features to find neighbours in' if 'Naive' in c.nn_type else None,
               'it needs forecast_steps = 1' if c.forecast_steps != 1 else None]
        bad = [b for b in bad if b]
        if bad:
            raise ValueError('--conformal_knn %d: the normalised conformal score divides each error by the mean error '
                             'of the K nearest training windows; %s' % (knn, '; '.join(bad)))
    if levels is None:
        return
    bad = ['they are calibrated at prediction (--train=False)' if c.train else None,
           'they calibrate one model, not an ensemble (num_procs = 1)' if getattr(c, 'num_procs', 1) > 1 else None,
           'the calibration set is the validation split: validation_size must be > 0'
           if not c.validation_size > 0 else None]
    bad = [b for b in bad if b]
    if bad:
        raise ValueError('--conformal_levels %s: split-conformal intervals; %s' % (levels, '; '.join(bad)))
    base_config.conformal_levels(levels)


def check_factor(c):
    """Refuses --factor_quantiles / --factor_return_field / --factor_horizon where they cannot run, before any work;
    the return field is checked against the datafile's header and values."""
    q, field, horizon = (getattr(c, 'factor_quantiles', 0), getattr(c, 'factor_return_field', None),
                         getattr(c, 'factor_horizon', 1))
    if q == 0:
        if field or horizon != 1:
            raise ValueError('--factor_return_field / --factor_horizon: they add the ret measure to a factor '
                             'backtest; set --factor_quantiles')
        return
    G = len(factor_names(c.forecast_steps, c.UQ))
    bad = ['factor_quantiles must be in [2, 100] (0 = off)' if not 2 <= q <= 100 else None,
           'it ranks forecasts at prediction (--train=False)' if c.train else None,
           'it ranks the forecasts of one model, not an ensemble (num_procs = 1)'
           if getattr(c, 'num_procs', 1) > 1 else None,
           'forecast_steps %d gives %d factors, more than %d' % (c.forecast_steps, G, FACTOR_MAX_SCORES)
           if G > FACTOR_MAX_SCORES else None,
           'a walk-forward backtest reads the current yield from walk_forward_preds.dat: '
           'set --write_inp_to_out_file=True'
           if c.training_type == 'iterative' and not c.write_inp_to_out_file else None]
    bad = [b for b in bad if b]
    if bad:
        raise ValueError('--factor_quantiles %d: a lookahead factor backtest; %s' % (q, '; '.join(bad)))
    if horizon < 1:
        raise ValueError('--factor_horizon %d: ret compounds the returns of the H >= 1 months after each date' % horizon)
    if field:
        path = os.path.join(c.data_dir, c.datafile)
        header = pd.read_csv(path, sep=' ', nrows=0).columns
        numeric = field in header and field not in ('date', 'gvkey')
        if numeric:
            try:
                pd.to_numeric(pd.read_csv(path, sep=' ', usecols=[field])[field], errors='raise')
            except (ValueError, TypeError):
                numeric = False
        if not numeric:
            raise ValueError('--factor_return_field %s: not a numeric column of %s' % (field, c.datafile))


def check_row_weights(c):
    """The refusals of --sample_weight_field / --recency_halflife that need no data (DESIGN.md section 6d); the field's
    values are checked when the dataset loads."""
    if getattr(c, 'recency_halflife', 0.0) < 0:
        raise ValueError('--recency_halflife %g: the half-life is in years, > 0 (0 = off)' % c.recency_halflife)
    weighted = bool(getattr(c, 'sample_weight_field', '')) or getattr(c, 'recency_halflife', 0.0) > 0
    if weighted and c.train and 'Naive' in c.nn_type:
        raise ValueError('--sample_weight_field / --recency_halflife: %s has nothing to train' % c.nn_type)


class ModelExecution(object):

    def __init__(self, config):
        self.config = config

    def __call__(self):
        if self.config.mc_samples != 1 and (self.config.mc_samples < 1 or not self.config.UQ or self.config.train):
            raise ValueError('--mc_samples %d: Monte-Carlo dropout samples are drawn at UQ prediction only (--UQ=True '
                             '--train=False); a point estimate predicts with dropout off, and training and validation '
                             'take one sample' % self.config.mc_samples)
        c = self.config
        if c.ig_steps != 0 and (c.ig_steps < 0 or c.train or c.UQ or c.nn_type != 'RNNPointEstimate'
                                or c.forecast_steps != 1):
            raise ValueError('--ig_steps %d: integrated-gradients attributions explain the forecast of a trained '
                             'RNNPointEstimate with forecast_steps = 1 at prediction (--train=False, --UQ=False), with '
                             'ig_steps >= 1 interpolants (0 = off)' % c.ig_steps)
        if c.perm_importance != 0 and (c.perm_importance < 0 or c.train or 'Naive' in c.nn_type):
            raise ValueError('--perm_importance %d: permutation importance measures how a trained model uses its inputs, '
                             'at prediction (--train=False), with perm_importance >= 1 repeats (0 = off); '
                             'NaivePointEstimate has no model to measure' % c.perm_importance)
        if c.shapley_samples != 0 and (c.shapley_samples < 0 or c.train or 'Naive' in c.nn_type):
            raise ValueError('--shapley_samples %d: Shapley attributions explain the forecasts of a trained model, at '
                             'prediction (--train=False), with shapley_samples >= 1 permutation samples (0 = off); '
                             'NaivePointEstimate has no model to explain' % c.shapley_samples)
        if c.ale_bins != 0 and (c.ale_bins < 0 or c.train or 'Naive' in c.nn_type):
            raise ValueError('--ale_bins %d: accumulated local effects explain the forecasts of a trained model, at '
                             'prediction (--train=False), with ale_bins >= 1 quantile bins per field (0 = off); '
                             'NaivePointEstimate has no model to explain' % c.ale_bins)
        if getattr(c, 'influence_top_k', 0) != 0:
            bad = ['influence_top_k must be in [1, 64]' if not 0 < c.influence_top_k <= 64 else None,
                   'it explains a trained model at prediction (--train=False)' if c.train else None,
                   'NaivePointEstimate has no model to explain' if 'Naive' in c.nn_type else None,
                   'it needs forecast_steps = 1' if c.forecast_steps != 1 else None,
                   'it explains one model, not an ensemble (num_procs = 1)' if getattr(c, 'num_procs', 1) > 1 else None]
            bad = [b for b in bad if b]
            if bad:
                raise ValueError('--influence_top_k %d: training-window attributions list, for every forecast, the '
                                 'training windows that push it up and down the most; %s' % (c.influence_top_k,
                                                                                              '; '.join(bad)))
        if getattr(c, 'pred_quantiles', None) is not None:
            if not c.UQ or c.train:
                raise ValueError('--pred_quantiles %s: predictive quantiles are those of a UQ model\'s Monte-Carlo '
                                 'dropout mixture, at prediction (--UQ=True --train=False)' % c.pred_quantiles)
            base_config.pred_quantile_levels(c.pred_quantiles)
        check_conformal(c)
        check_factor(c)
        check_row_weights(c)
        if c.training_type == 'iterative':
            check_walk_forward(c)
            return self.walk_forward_execution()
        return self.fixed_dates_execution()

    @staticmethod
    def read_results(config):
        """Validation metrics after training, predictions after inference (model_execution.py:31-78).  A walk-forward
        config (training_type iterative) reads its stitched predictions, walk_forward_preds.dat, after either."""
        try:
            if config.training_type == 'iterative':
                df = pd.read_csv(os.path.join(config.experiments_dir, config.model_dir, 'walk_forward_preds.dat'),
                                 sep=' ', dtype={'gvkey': str})
                return _weighted_scaled_mse(df, config), None, df
            if config.train:
                df = pd.read_csv(os.path.join(config.experiments_dir, config.model_dir, 'train_log',
                                              config.name + '-train-logs-epoch.csv'), sep=',')
                df = df.sort_values(by='valid_mse').reset_index()
                return df.iloc[0]['valid_mse'], None, None
            df = pd.read_csv(os.path.join(config.experiments_dir, config.model_dir, 'pred', config.preds_fname),
                             sep=' ', dtype={'gvkey': str})
            return _weighted_scaled_mse(df, config), None, df
        except FileNotFoundError:
            print("Output file not found")
            return np.inf, np.inf, None

    @staticmethod
    def single_execution(config):
        """model_execution.py:81-111; the GPU is the last character of ``default_gpu`` (:88)."""
        import torch
        gpu = str(config.default_gpu)[-1]
        if gpu.isdigit() and torch.cuda.is_available() and int(gpu) < torch.cuda.device_count():
            torch.cuda.set_device(int(gpu))
        from ..data_processing import CDRSInferenceData, Dataset
        from ..predict import Predict
        from ..train import Train
        dataset = CDRSInferenceData(config) if config.cdrs_inference else Dataset(config)
        if config.train:
            print("Training")
            return Train(config, dataset).train()
        print("Prediction")
        return Predict(config, dataset).predict()

    @staticmethod
    def member_execution(config, share_den):
        """One member of an ensemble on the calling thread: its GPU (the last character of default_gpu), a stream of
        its own for every call, and 1/share_den of the GPU for the co-residency of its persistent launches.  Then
        Train or Predict as a single execution."""
        import torch
        from ..data_processing import Dataset
        from ..predict import Predict
        from ..train import Train
        gpu = str(config.default_gpu)[-1]
        if not (gpu.isdigit() and torch.cuda.is_available() and int(gpu) < torch.cuda.device_count()):
            raise RuntimeError('ensemble member %d: default_gpu %s is not a CUDA device of this process (%d visible)'
                               % (config.member_id, config.default_gpu,
                                  torch.cuda.device_count() if torch.cuda.is_available() else 0))
        torch.cuda.set_device(int(gpu))
        stream = torch.cuda.Stream()
        with torch.cuda.stream(stream):
            runner = (Train if config.train else Predict)(config, Dataset(config))
            if runner.model.engine is not None:           # NaivePointEstimate runs no kernels of its own
                runner.model.engine.set_device_share(1, share_den)
            out = runner.train() if config.train else runner.predict()
        stream.synchronize()
        return out

    @classmethod
    def run_members(cls, members, npe):
        """member_execution of every config in `members`, NPE at a time on host threads of their own.  A member that
        raises stops the run: members that have not started never start, the running ones finish, then its exception
        is raised."""
        npe = max(1, min(int(npe), len(members)))
        # at most min(NPE, members on that GPU) members run on one GPU at a time: their shares sum to at most 1
        on_gpu = Counter(m.default_gpu for m in members)
        with ThreadPoolExecutor(max_workers=npe) as pool:
            futures = [pool.submit(cls.member_execution, m, min(npe, on_gpu[m.default_gpu])) for m in members]
            wait(futures, return_when=FIRST_EXCEPTION)
            failed = [f for f in futures if f.done() and not f.cancelled() and f.exception() is not None]
            if failed:
                pool.shutdown(cancel_futures=True)
                raise failed[0].exception()

    def walk_forward_execution(self):
        """A walk-forward backtest (training_type iterative, DESIGN.md section 6c): with train True every origin
        trains (origin_configs), NPE at a time side by side like ensemble members; then, with train True or False,
        every origin predicts its months the same way.  Writes <experiments_dir>/<model_dir>/walk_forward_preds.dat
        (stitch_walk_forward) and returns that frame."""
        cfg = self.config
        experiment_dir, origins = origin_configs(cfg)
        if cfg.train:
            for _, train, _ in origins:
                write_member_conf(train)
            self.run_members([train for _, train, _ in origins], cfg.NPE)
        elif 'Naive' not in cfg.nn_type:          # the naive forecast has no checkpoint to load
            for origin, _, pred in origins:
                if not os.path.isdir(pred.model_dir):
                    raise FileNotFoundError('walk-forward origin %d has no directory %s: train the origins first '
                                            '(--train=True)' % (origin, pred.model_dir))
        preds = [pred for _, _, pred in origins]
        for p in preds:
            pathlib.Path(p.model_dir).mkdir(parents=True, exist_ok=True)
            write_conf(p.as_dict(), os.path.join(p.model_dir, 'predict-%d.conf' % p.member_id))
        self.run_members(preds, cfg.NPE)
        frames = []
        for origin, _, pred in origins:
            path = os.path.join(pred.model_dir, 'pred', cfg.preds_fname)
            if not os.path.isfile(path):
                raise RuntimeError('walk-forward origin %d wrote no %s' % (origin, path))
            if pred.UQ and pred.mc_samples > 1:
                self.write_uq_ensemble(pred)
            # read back exactly, so that the stitched rows are the origins' rows as they wrote them
            frames.append(pd.read_csv(path, sep=' ', dtype={'gvkey': str}, float_precision='round_trip'))
        df = stitch_walk_forward(frames, [origin for origin, _, _ in origins])
        df.to_csv(os.path.join(experiment_dir, 'walk_forward_preds.dat'), sep=' ', index=False)
        if cfg.perm_importance > 0:         # how the importance drifts across the origins
            stitch_walk_forward([pd.read_csv(os.path.join(pred.model_dir, 'pred', 'importance.dat'), sep=' ',
                                             dtype={'group': str}, float_precision='round_trip')
                                 for _, _, pred in origins], [origin for origin, _, _ in origins]).to_csv(
                os.path.join(experiment_dir, 'walk_forward_importance.dat'), sep=' ', index=False)
        if cfg.ale_bins > 0:
            stitch_walk_forward([pd.read_csv(os.path.join(pred.model_dir, 'pred', 'ale.dat'), sep=' ',
                                             dtype={'field': str}, float_precision='round_trip')
                                 for _, _, pred in origins], [origin for origin, _, _ in origins]).to_csv(
                os.path.join(experiment_dir, 'walk_forward_ale.dat'), sep=' ', index=False)
        if getattr(cfg, 'pred_quantiles', None) is not None:
            stitch_walk_forward([pd.read_csv(os.path.join(pred.model_dir, 'pred', 'quantiles.dat'), sep=' ',
                                             dtype={'gvkey': str}, float_precision='round_trip')
                                 for _, _, pred in origins], [origin for origin, _, _ in origins]).to_csv(
                os.path.join(experiment_dir, 'walk_forward_quantiles.dat'), sep=' ', index=False)
        if getattr(cfg, 'conformal_levels', None) is not None:      # each origin calibrated on its own draw
            for name, key in (('intervals', 'gvkey'), ('coverage', 'subset')):
                stitch_walk_forward([pd.read_csv(os.path.join(pred.model_dir, 'pred', name + '.dat'), sep=' ',
                                                 dtype={key: str}, float_precision='round_trip')
                                     for _, _, pred in origins], [origin for origin, _, _ in origins]).to_csv(
                    os.path.join(experiment_dir, 'walk_forward_%s.dat' % name), sep=' ', index=False)
        if getattr(cfg, 'factor_quantiles', 0) > 0:       # the out-of-sample backtest over every origin's months
            per_date, summary = factor_tables(df, cfg)
            per_date.to_csv(os.path.join(experiment_dir, 'walk_forward_factor_dates.dat'), sep=' ', index=False)
            summary.to_csv(os.path.join(experiment_dir, 'walk_forward_factor.dat'), sep=' ', index=False)
        _print_scaled_mse(df, cfg.forecast_steps)
        return df

    def point_estimate_ensemble(self):
        """model_execution.py:154-199 in one process.  Training returns every member's best validation MSE, as
        read_results reads it; prediction writes every member's pred/<preds_fname>, then
        <experiments_dir>/<model_dir>/ensemble_preds.dat (ensemble_point_estimate), and returns that frame."""
        cfg = self.config
        assert cfg.num_procs > 1
        if int(os.environ.get('WORLD_SIZE', '1')) > 1:
            raise NotImplementedError('an ensemble (num_procs > 1) runs its members side by side in one process and '
                                      'cannot be combined with torchrun data parallelism; run it without torchrun')
        experiment_dir, members = member_configs(cfg)
        for m in members:
            write_member_conf(m)
        self.run_members(members, cfg.NPE)
        results = [self.read_results(m) for m in members]
        if cfg.train:
            return [r[0] for r in results]
        frames = [r[2] for r in results]
        missing = [m.member_id for m, f in zip(members, frames) if f is None]
        if missing:
            raise RuntimeError('ensemble members %s wrote no %s' % (missing, cfg.preds_fname))
        df = ensemble_point_estimate(frames, cfg.forecast_steps)
        df.to_csv(os.path.join(experiment_dir, 'ensemble_preds.dat'), sep=' ', index=False)
        return df

    @classmethod
    def write_uq_ensemble(cls, config):
        """<experiments_dir>/<model_dir>/ensemble_preds.dat of a prediction with mc_samples > 1 Monte-Carlo samples
        (ensemble_uq_estimate of pred/<preds_fname> as read_results reads it), the file the reference's UQ ensemble
        writes (model_execution.py:237-241).  Returns that frame, or None when there are no predictions to read."""
        frame = cls.read_results(config)[2]
        if frame is None:
            return None
        df = ensemble_uq_estimate(frame, config.forecast_steps)
        df.to_csv(os.path.join(config.experiments_dir, config.model_dir, 'ensemble_preds.dat'), sep=' ', index=False)
        return df

    def uq_estimate_execution(self):
        """runtime/model_execution.py:201-241: training, or prediction with one process, is a single execution.  A
        prediction with mc_samples > 1 holds the samples' moments and is followed by the ensemble's post-processing
        (write_uq_ensemble).  The multi-process MC-dropout ensemble (num_procs > 1 at predict time) is not built."""
        if self.config.train or self.config.num_procs == 1:
            out = self.single_execution(self.config)
            if not self.config.train and self.config.mc_samples > 1:
                self.write_uq_ensemble(self.config)
            return out
        raise NotImplementedError('UQ ensemble prediction (num_procs > 1) fans out whole predictions through files; run '
                                  'one lfm_quant.py per member')

    def fixed_dates_execution(self):
        if self.config.UQ:
            return self.uq_estimate_execution()
        if self.config.num_procs == 1:
            return self.single_execution(self.config)
        return self.point_estimate_ensemble()
