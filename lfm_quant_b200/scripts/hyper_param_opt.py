#!/usr/bin/env python3
"""Hyper-parameter search CLI (reference: scripts/hyper_param_opt.py):

    hyper_param_opt.py [--config=FILE] --search_algorithm genetic|grid_search|doe [flags]

The flag schema is the reference's, in its order.  The flags of the model that a search may tune are list flags:
``--num_hidden 32 64 128`` makes num_hidden tunable over three values, a single value keeps it constant.  Every
candidate is written as <experiments_dir>/<name>/opt_run/<name>-<id>/model.conf, which ``lfm_quant.py --config``
runs alone, and its best validation MSE goes to opt_hist.csv.  The candidates of a generation train in this process,
NPE at a time, side by side on the GPU (DESIGN.md section 6b).

LFM_QUANT_ROOT must be set, and data_dir is taken relative to it; the reference names the variable DEEP_QUANT_ROOT.
"""
from __future__ import absolute_import, division, print_function

import os
import sys

if __package__ in (None, ''):       # executed as a script: make the package importable
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
    from lfm_quant_b200.scripts import configs
    from lfm_quant_b200.scripts.param_search.optimization import HPOptimization
else:
    from . import configs
    from .param_search.optimization import HPOptimization

# (name, definer, default, doc), in the reference's order: the order of the tunable flags is that of the grid
SCHEMA = [
    ('name', configs.DEFINE_string, 'hpo-test', 'A name for the search'),
    ('datafile', configs.DEFINE_string, 'source-ml-data-v8-100M.dat', 'Data file name'),
    ('predict_datafile', configs.DEFINE_string, None, 'Data file for predictions, if not datafile'),
    ('mse_outfile', configs.DEFINE_string, None, 'File for the MSE values of the predict phase'),
    ('scalesfile', configs.DEFINE_string, None, 'Optional file for the scaling parameters'),
    ('default_gpu', configs.DEFINE_string, '/gpu:0', 'Default GPU, e.g. /gpu:0'),
    ('nn_type', configs.DEFINE_string, 'RNNPointEstimate', 'Model type'),
    ('active_field', configs.DEFINE_string, 'active', 'Column of the active indicator'),
    ('date_field', configs.DEFINE_string, 'date', 'Column of the date'),
    ('key_field', configs.DEFINE_string, 'gvkey', 'Column of the key'),
    ('target_field', configs.DEFINE_string, 'oiadpq_ttm', 'Column of the target'),
    ('scale_field', configs.DEFINE_string, 'mrkcap', 'Feature the inputs are scaled by'),
    ('financial_fields', configs.DEFINE_string, 'saleq_ttm-ltq_mrq', 'Input and target fields'),
    ('aux_fields', configs.DEFINE_string, 'rel_mom1m-rel_mom9m', 'Input-only fields'),
    ('dont_scale', configs.DEFINE_string, None, 'Fields not to scale'),
    ('data_dir', configs.DEFINE_string, 'datasets', 'Data directory, relative to LFM_QUANT_ROOT'),
    ('model_dir', configs.DEFINE_string, 'test-model', 'Model directory'),
    ('experiments_dir', configs.DEFINE_string, './', 'Experiments directory'),
    ('rnn_cell', configs.DEFINE_list_string, 'lstm', 'lstm or gru'),
    ('activation_fn', configs.DEFINE_list_string, 'relu', 'MLP activation function'),
    ('num_inputs', configs.DEFINE_integer, -1, ''),
    ('num_outputs', configs.DEFINE_integer, -1, ''),
    ('target_idx', configs.DEFINE_integer, None, ''),
    ('min_unrollings', configs.DEFINE_list_integer, 5, 'Min number of unrolling steps'),
    ('max_unrollings', configs.DEFINE_list_integer, 5, 'Max number of unrolling steps'),
    ('min_years', configs.DEFINE_list_integer, None, 'Alternative to min_unrollings'),
    ('max_years', configs.DEFINE_list_integer, None, 'Alternative to max_unrollings'),
    ('pls_years', configs.DEFINE_integer, None, 'Alternative to max_years: max_years = min_years + pls_years'),
    ('stride', configs.DEFINE_list_integer, 12, 'Steps skipped per unrolling'),
    ('batch_size', configs.DEFINE_list_integer, 256, 'Batch size'),
    ('num_layers', configs.DEFINE_list_integer, 2, 'Number of RNN layers'),
    ('forecast_n', configs.DEFINE_integer, 12, 'Steps forecast into the future'),
    ('num_hidden', configs.DEFINE_list_integer, 64, 'Hidden units'),
    ('init_scale', configs.DEFINE_list_float, 1.0, 'Initial scale of the weights'),
    ('max_grad_norm', configs.DEFINE_list_float, 50.0, 'Gradient clipping'),
    ('start_date', configs.DEFINE_integer, 197501, 'First training date, YYYYMM'),
    ('end_date', configs.DEFINE_integer, 199812, 'Last training date, YYYYMM'),
    ('split_date', configs.DEFINE_integer, None, 'Date of the train/test split'),
    ('train', configs.DEFINE_boolean, True, 'Train, otherwise predict'),
    ('dropout', configs.DEFINE_list_float, 0.0, 'Dropout rate of the hidden layers'),
    ('recurrent_dropout', configs.DEFINE_list_float, 0.3, 'Dropout rate of the recurrent connections'),
    ('log_squasher', configs.DEFINE_boolean, True, 'Squash large normalized inputs with the natural log'),
    ('data_scaler', configs.DEFINE_list_string, 'RobustScaler', 'sklearn scaler, or None'),
    ('optimizer', configs.DEFINE_list_string, 'Adadelta', 'Optimizer'),
    ('learning_rate', configs.DEFINE_list_float, 0.6, 'Initial learning rate'),
    ('lr_decay', configs.DEFINE_list_float, 0.96, 'Learning rate decay'),
    ('validation_size', configs.DEFINE_float, 0.3, 'Share of the data held out for validation'),
    ('target_lambda', configs.DEFINE_list_float, 0.5, 'Weight of the last step against all steps in the loss'),
    ('rnn_lambda', configs.DEFINE_list_float, 0.7, 'Weight of the last step against all steps in the loss'),
    ('max_epoch', configs.DEFINE_integer, 35, 'Stop after max_epoch epochs'),
    ('early_stop', configs.DEFINE_integer, 15, 'Early stop parameter'),
    ('seed', configs.DEFINE_integer, 521, 'Seed of the training and of the search'),
    ('UQ', configs.DEFINE_boolean, False, 'Uncertainty quantification mode'),
    ('l2_alpha', configs.DEFINE_list_float, 0.0, 'L2 regularization of the weights'),
    ('recurrent_l2_alpha', configs.DEFINE_float, 0.0, 'L2 regularization of the recurrent weights'),
    ('huber_loss', configs.DEFINE_list_boolean, False, 'Huber loss instead of MSE'),
    ('huber_delta', configs.DEFINE_list_float, 1.0, 'Delta of the Huber loss'),
    ('forecast_steps', configs.DEFINE_integer, 1, 'Number of future predictions'),
    ('forecast_steps_weights', configs.DEFINE_string, '1.0', 'Weights of the forecast steps, comma separated'),
    ('logging_interval', configs.DEFINE_integer, 100, 'Batches between training log lines'),
    ('write_inp_to_out_file', configs.DEFINE_boolean, True, 'Write the input sequence to the output files'),
    ('training_type', configs.DEFINE_string, 'fixed_dates', 'fixed_dates or iterative'),
    ('member_id', configs.DEFINE_integer, 1, 'Id of a member of the population'),
    ('load_saved_weights', configs.DEFINE_boolean, False, 'Load the weights saved in the checkpoint directory'),
    ('epoch_logging_interval', configs.DEFINE_integer, 1, 'Epochs between log lines'),
    ('preds_fname', configs.DEFINE_string, 'preds.dat', 'Name of the prediction file'),
    ('num_procs', configs.DEFINE_integer, 1, 'Number of training/prediction processes'),
    # the search's own flags
    ('NPE', configs.DEFINE_integer, 1, 'Candidates trained at the same time'),
    ('search_algorithm', configs.DEFINE_string, 'genetic', 'genetic, grid_search or doe'),
    ('generations', configs.DEFINE_integer, 5, 'Generations of the genetic algorithm'),
    ('pop_size', configs.DEFINE_integer, 16, 'Population size of the genetic algorithm'),
    ('num_gpu', configs.DEFINE_integer, 1, 'GPUs the candidates are spread over, round robin'),
    ('mutate_rate', configs.DEFINE_float, 0.2, 'Mutation rate of the genetic algorithm'),
    ('objective', configs.DEFINE_string, 'mse', 'mse or uq_loss'),
    ('init_pop', configs.DEFINE_string, None, 'Pickled initial population (save_latest_pop writes one)'),
    ('save_latest_pop', configs.DEFINE_boolean, False, 'Pickle each generation before it trains'),
    ('doe_file', configs.DEFINE_string, None, 'Design of experiments CSV file'),
    ('decay_steps', configs.DEFINE_integer, 100000, 'Training steps between learning rate decays'),
    ('initializer', configs.DEFINE_string, 'GlorotUniform', 'Weight initializer'),
    ('use_custom_init', configs.DEFINE_boolean, True, 'RandomUniform initializer with init_scale'),
    ('aux_masking', configs.DEFINE_boolean, False, 'Mask the aux features of all steps but the last with 0'),
    ('max_norm', configs.DEFINE_integer, None, 'Max norm of the kernel constraint'),
    ('sgd_momentum', configs.DEFINE_float, 0.0, 'Momentum of the SGD optimizer'),
    ('end_learning_rate', configs.DEFINE_float, 0.01, 'End learning rate of the polynomial decay'),
    ('decay_power', configs.DEFINE_float, 0.5, 'Power of the polynomial decay'),
    ('piecewise_lr_boundaries', configs.DEFINE_string, None, 'Boundaries of the piecewise constant learning rate'),
    ('piecewise_lr_values', configs.DEFINE_string, None, 'Values of the piecewise constant learning rate'),
    ('lr_schedule', configs.DEFINE_string, 'ExponentialDecay', 'Learning rate schedule'),
    # native-path extension (not in the reference), tunable like the model flags
    ('precision', configs.DEFINE_list_string, 'fp32', "'fp32', 'tf32', 'bf16' or 'bf16x3'"),
]


def get_configs(argv=None):
    """The search config (reference: hyper_param_opt.py:16-119).  Registers the schema on a fresh flag parser, parses
    `argv` (default sys.argv), and leaves the parser empty again, so that the candidates' model.conf files parse with
    the forecaster's own schema.  data_dir is joined to LFM_QUANT_ROOT and forecast_steps_weights split on ','.
    ``config`` is cleared: the candidates do not carry the search's config file."""
    root = os.environ.get('LFM_QUANT_ROOT')
    assert root is not None, "Environment Variable LFM_QUANT_ROOT not set"
    configs.reset()
    for name, define, default, doc in SCHEMA:
        define(name, default, doc)
    c = configs.ConfigValues(argv)
    c.data_dir = os.path.join(root, c.data_dir)
    c.forecast_steps_weights = [float(x) for x in c.forecast_steps_weights.split(',')]
    c.config = None
    configs.reset()
    return c


def main(argv=None):
    return HPOptimization(get_configs(argv))()


if __name__ == "__main__":
    main()
