"""Flag schema of the forecaster -- every flag of scripts/lfm_quant.py:23-106 and scripts/base_config.py:12-96,
same names, types and defaults -- plus the native-path extensions at the bottom.

``get_configs(argv=None, list_sep='-')`` reproduces the post-processing of scripts/lfm_quant.py:108-129
(unrollings from years, '-'-separated lists); scripts/base_config.py:115 splits forecast_steps_weights on ','
instead, available as ``list_sep=','``.
"""
from __future__ import absolute_import, division, print_function

import numpy as np

from . import configs

_STRING = 's'
_INT = 'i'
_FLOAT = 'f'
_BOOL = 'b'

# (name, kind, default, doc)
SCHEMA = [
    ('name', _STRING, 'test', 'A name for the config.'),
    ('datafile', _STRING, None, 'a datafile name.'),
    ('scalesfile', _STRING, None, 'Optional file for storing scaling params'),
    ('default_gpu', _STRING, '/gpu:0', 'The default GPU to use e.g., /gpu:0'),
    ('nn_type', _STRING, 'RNNPointEstimate', 'Model type'),
    ('active_field', _STRING, 'active', 'Key column name header for active indicator'),
    ('date_field', _STRING, 'date', 'Name of data column.'),
    ('key_field', _STRING, 'gvkey', 'Key column name header in datafile'),
    ('target_field', _STRING, 'oiadpq_ttm', 'Target column name header in datafile'),
    ('scale_field', _STRING, 'mrkcap', 'Feature to scale inputs by'),
    ('financial_fields', _STRING, 'saleq_ttm-ltq_mrq', 'Shared input and target field names'),
    ('aux_fields', _STRING, 'rel_mom1m-rel_mom9m', 'non-target, input only fields'),
    ('dont_scale_fields', _STRING, None, 'Names of fields to not scale'),
    ('data_dir', _STRING, 'datasets', 'The data directory'),
    ('model_dir', _STRING, 'test-model', 'Model directory'),
    ('experiments_dir', _STRING, './', 'Experiments directory'),
    ('rnn_cell', _STRING, 'lstm', 'lstm or gru'),
    ('activation_fn', _STRING, 'relu', 'MLP activation function in tf.nn.*'),
    ('num_inputs', _INT, -1, ''),
    ('num_outputs', _INT, -1, ''),
    ('target_idx', _INT, None, ''),
    ('min_unrollings', _INT, 5, 'Min number of unrolling steps'),
    ('max_unrollings', _INT, 5, 'Max number of unrolling steps'),
    ('min_years', _INT, None, 'Alt to min_unrollings'),
    ('max_years', _INT, None, 'Alt to max_unrollings'),
    ('pls_years', _INT, None, 'Alt to max_years. max_years = min_year+pls_years'),
    ('stride', _INT, 12, 'How many steps to skip per unrolling'),
    ('batch_size', _INT, 256, 'Size of each batch'),
    ('num_layers', _INT, 2, 'Numer of RNN layers'),
    ('forecast_n', _INT, 12, 'How many steps to forecast into the future'),
    ('num_hidden', _INT, 64, 'Number of hidden layer units'),
    ('init_scale', _FLOAT, 1.0, 'Initial scale for weights'),
    ('max_grad_norm', _FLOAT, 50.0, 'Gradient clipping'),
    ('start_date', _INT, 197501, 'First date to train on as YYYYMM'),
    ('end_date', _INT, 199912, 'Last date to train on as YYYYMM'),
    ('split_date', _INT, None, 'Date to split train/test on as YYYYMM: the first origin of training_type iterative'),
    ('train', _BOOL, True, 'Train model otherwise inference only'),
    ('dropout', _FLOAT, 0.0, 'Dropout rate for hidden layers'),
    ('recurrent_dropout', _FLOAT, 0.0, 'Dropout rate for recurrent connections'),
    ('log_squasher', _BOOL, True, 'Squash large normalized inputs with natural log function'),
    ('data_scaler', _STRING, 'RobustScaler', 'sklearn scaling algorithm or None if no scaling'),
    ('optimizer', _STRING, 'Adadelta', 'Any tensorflow optimizer in tf.train'),
    ('learning_rate', _FLOAT, 0.6, 'The initial starting learning rate'),
    ('lr_decay', _FLOAT, 1.0, 'Learning rate decay for exponential decay'),
    ('validation_size', _FLOAT, 0.3, 'Size of validation set as %, ie. 0.3 = 30% of data'),
    ('target_lambda', _FLOAT, 0.5, 'How much to weight last step vs. all steps in loss'),
    ('rnn_lambda', _FLOAT, 0.7, 'How much to weight last step vs. all steps in loss'),
    ('max_epoch', _INT, 1, 'Stop after max_epochs'),
    ('early_stop', _INT, 1, 'Early stop parameter'),
    ('seed', _INT, 521, 'Seed for deterministic training'),
    ('UQ', _BOOL, False, 'Uncertainty Quantification Mode'),
    ('l2_alpha', _FLOAT, 0.0, 'L2 regularization for weight parameters.'),
    ('recurrent_l2_alpha', _FLOAT, 0.0, 'L2 regularization for recurrent weight parameters.'),
    ('huber_loss', _BOOL, False, 'Use huber loss instead of mse'),
    ('huber_delta', _FLOAT, 1.0, 'delta for huber loss'),
    ('forecast_steps', _INT, 1, 'How many future predictions need to me made'),
    ('forecast_steps_weights', _STRING, '1.0', 'weights for the forecast steps'),
    ('logging_interval', _INT, 100, 'Number of batches for logging interval during training'),
    ('write_inp_to_out_file', _BOOL, True, 'Write input sequence to the output files'),
    ('training_type', _STRING, 'fixed_dates', 'Choose between "fixed_dates" and "iterative" training; "iterative" is a '
                                              'walk-forward backtest: one model trained through each origin split_date '
                                              '+ k*stride months, each predicting the stride months after it'),
    ('NPE', _INT, 1, 'Number of Parallel Executions'),
    ('num_procs', _INT, 1, 'Total number of training/prediction processes'),
    ('num_gpu', _INT, 1, 'NUmber of GPUs'),
    ('load_saved_weights', _BOOL, False, 'Load weights saved in the checkpoint directory'),
    ('epoch_logging_interval', _INT, 1, 'Number of batches for logging interval during training'),
    ('decay_steps', _INT, 1500, 'Number of training steps between decay steps'),
    ('initializer', _STRING, 'GlorotUniform', 'variable initializers available in Keras'),
    ('use_custom_init', _BOOL, True, 'Use RandomUniform initializer with init_scale values'),
    ('aux_masking', _BOOL, False, 'Mask aux features of all time steps except the last one with 0'),
    ('max_norm', _INT, 3, 'Max Norm for kernel constraint'),
    ('sgd_momentum', _FLOAT, 0.0, 'momentum for SGD optimizer'),
    ('end_learning_rate', _FLOAT, 0.01, 'end lr for polynomial decay'),
    ('decay_power', _FLOAT, 0.5, 'power to decay the learning rate with for polynomial decay'),
    ('piecewise_lr_boundaries', _STRING, '4000-5500-5500', 'boundaries for piecewise constant lr'),
    ('piecewise_lr_values', _STRING, '0.5-0.1-0.05-0.1', 'values for piecewise constant lr'),
    ('lr_schedule', _STRING, 'ExponentialDecay', 'Learning rate scheduler'),
    ('preds_fname', _STRING, 'preds.dat', 'Name of the prediction file'),
    ('member_id', _INT, 1, 'Id of member in a population'),
    ('cdrs_inference', _BOOL, False, 'If the execution is for inference on CDRS data'),
    ('use_external_cdrs_data', _BOOL, False, 'True if CDRS data is provided externally (base_config.py:91)'),
    ('cdrs_src_fname', _STRING, 'cdrs-src.dat', 'Filename of the CDRS source file'),
    ('cdrs_ml_fname', _STRING, 'cdrs-ml-data.dat', 'Filename of the CDRS ML data file'),
    ('model_ranking_fname', _STRING, './model-ranking.dat', 'Model Ranking File Name'),
    ('model_ranking_factor', _STRING, 'pred_var_entval', 'Model ranking factor'),
    ('cdrs_inference_date', _STRING, None, "CDRS Inference date. Format: '%Y-%m-%d' "),
    # ---- native-path extensions (not in the reference) -------------------------------------------------
    ('precision', _STRING, 'fp32', "'fp32' (parity mode), 'tf32' (the fp32 step with tf32 tensor-core GEMMs: any "
                                   "cell, head and forecast_steps), 'bf16' (tensor-core gate GEMMs) or 'bf16x3'"),
    ('mc_samples', _INT, 1, 'Monte-Carlo dropout samples per window at UQ prediction; more than 1 also writes the '
                            "UQ ensemble's ensemble_preds.dat with the calibrated lower bounds"),
    ('ig_steps', _INT, 0, 'Integrated-gradients interpolants per window at point-estimate prediction; more than 0 also '
                          'writes pred/attributions.npz: which input fields and quarters drive each forecast'),
    ('perm_importance', _INT, 0, 'Permutation-importance repeats at prediction; more than 0 also writes '
                                 'pred/importance.dat: how much the loss on the predicted windows rises when one input '
                                 'field, or one quarter, is shuffled across them'),
    ('shapley_samples', _INT, 0, 'Shapley permutation samples (antithetic pairs) per window at prediction; more than 0 '
                                 'also writes pred/shapley.npz: how much each input field and each quarter moves every '
                                 'window\'s forecast (and a UQ model\'s variance) away from a donor window\'s'),
    ('ale_bins', _INT, 0, 'Quantile bins per input field for accumulated local effects at prediction; more than 0 '
                          'also writes pred/ale.dat: in which direction and with what shape the forecast (and a UQ '
                          'model\'s variance) responds to each input field\'s latest value'),
    ('influence_top_k', _INT, 0, 'Training windows listed per forecast at prediction (1 to 64); more than 0 also '
                                 'writes pred/influence.npz: for every predicted window the K windows of the training '
                                 'split whose gradient step pushes its forecast (and a UQ model\'s variance) up the most '
                                 'and the K that push it down the most, with the summed influence of the whole split'),
    ('pred_quantiles', _STRING, None, "'-'-separated levels in (0, 1), e.g. 0.05-0.25-0.5-0.75-0.95, at UQ prediction; "
                                      'writes pred/quantiles.dat (the quantiles of each window\'s Monte-Carlo dropout '
                                      'mixture, with its CRPS, log score and PIT) and pred/calibration.dat; unset = off'),
    ('conformal_levels', _STRING, None, "'-'-separated coverage levels in (0, 1), e.g. 0.5-0.8-0.9, at prediction; "
                                        'writes pred/intervals.dat (every forecast\'s split-conformal interval, '
                                        'calibrated on the held-out validation companies, with its conformal p-value) '
                                        'and pred/coverage.dat; unset = off'),
    ('conformal_knn', _INT, 0, 'Training windows whose mean absolute error scales each conformal interval (1 to 64) '
                               'of a point or linear model with forecast_steps = 1: the normalised score; 0 = off'),
    ('factor_quantiles', _INT, 0, 'Quantile buckets (2 to 100) of a lookahead factor backtest at prediction: each '
                                  'date\'s companies ranked by forecast yield (preds / seq_norm) and by current yield '
                                  '(inp_t0 / seq_norm), scored against the realised yield; writes pred/factor_dates.dat '
                                  'and pred/factor.dat (walk_forward_factor*.dat in a walk-forward run); 0 = off'),
    ('factor_return_field', _STRING, None, 'Datafile column of each row\'s simple return over the month that ends at '
                                           'its date: adds the measure ret, the compounded return over the '
                                           'factor_horizon months after each forecast date; unset = off'),
    ('factor_horizon', _INT, 1, 'Months compounded into the factor backtest\'s ret measure (>= 1)'),
    ('sample_weight_field', _STRING, None, 'Datafile column that weighs each training window in the training loss, read '
                                         'raw at the window\'s last input row (NaN counts as 0; negative or infinite '
                                         'values are refused); unset = off.  Ignored with --train=False'),
    ('recency_halflife', _FLOAT, 0.0, 'Half-life in years of a recency weight 2^(-months / (12 Y)) on each training '
                                      'window, months counted back from the latest last-input date of the training '
                                      'set (per walk-forward origin); 0 = off.  Ignored with --train=False'),
]

_DEFINERS = {_STRING: configs.DEFINE_string, _INT: configs.DEFINE_integer, _FLOAT: configs.DEFINE_float,
             _BOOL: configs.DEFINE_boolean}


def define_flags():
    for name, kind, default, doc in SCHEMA:
        _DEFINERS[kind](name, default, doc)


def get_configs(argv=None, list_sep='-'):
    """Registers the schema and returns the parsed ConfigValues (scripts/lfm_quant.py:19-129)."""
    define_flags()
    c = configs.ConfigValues(argv)
    # scripts/lfm_quant.py:110-123
    if c.min_unrollings is None:
        c.min_unrollings = c.num_unrollings
    if c.max_unrollings is None:
        c.max_unrollings = c.num_unrollings
    if c.min_years is not None:
        c.min_unrollings = c.min_years * (12 // c.stride)
        if c.max_years is not None:
            c.max_unrollings = c.max_years * (12 // c.stride)
        elif c.pls_years is None:
            c.max_unrollings = c.min_unrollings
        else:
            c.max_unrollings = (c.min_years + c.pls_years) * (12 // c.stride)
    # scripts/lfm_quant.py:125-127
    c.forecast_steps_weights = [float(v) for v in str(c.forecast_steps_weights).split(list_sep)]
    if list_sep == '-':     # scripts/lfm_quant.py:126-127; scripts/base_config.py:115 leaves these two as strings
        c.piecewise_lr_boundaries = [float(v) for v in str(c.piecewise_lr_boundaries).split('-')]
        c.piecewise_lr_values = [float(v) for v in str(c.piecewise_lr_values).split('-')]
    return c


MAX_PRED_QUANTILES = 32      # lfmq_chain_forward_uq_dist's cap on the levels


MAX_CONFORMAL_LEVELS = 32    # lfmq_conformal_calibrate's cap on the levels


def pred_quantile_levels(spec):
    """The levels of --pred_quantiles: None when unset, else the '-'-separated floats, which must be strictly
    increasing inside (0, 1), at most MAX_PRED_QUANTILES of them.  A malformed value raises ValueError."""
    return _levels(spec, 'pred_quantiles', MAX_PRED_QUANTILES)


def conformal_levels(spec):
    """The coverage levels of --conformal_levels, parsed and checked as pred_quantile_levels parses its levels, at most
    MAX_CONFORMAL_LEVELS of them."""
    return _levels(spec, 'conformal_levels', MAX_CONFORMAL_LEVELS)


def _levels(spec, flag, cap):
    if spec is None or str(spec).strip() == '':
        return None
    try:
        levels = [float(v) for v in str(spec).split('-')]
    except ValueError:
        raise ValueError("--%s %s: expected '-'-separated levels such as 0.05-0.5-0.95" % (flag, spec))
    if not 1 <= len(levels) <= cap:
        raise ValueError('--%s %s: between 1 and %d levels' % (flag, spec, cap))
    if any(not 0.0 < v < 1.0 for v in levels) or any(b <= a for a, b in zip(levels, levels[1:])):
        raise ValueError('--%s %s: the levels must be strictly increasing inside (0, 1)' % (flag, spec))
    if any(not 0.0 < v < 1.0 for v in np.float32(levels)) or any(np.diff(np.float32(levels)) <= 0):
        raise ValueError('--%s %s: the levels must stay distinct inside (0, 1) in single precision' % (flag, spec))
    return levels
