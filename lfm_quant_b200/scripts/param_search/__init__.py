"""Hyper-parameter search: genetic algorithm, grid search and design of experiments (reference: scripts/param_search/).
Entry point: scripts/hyper_param_opt.py."""
