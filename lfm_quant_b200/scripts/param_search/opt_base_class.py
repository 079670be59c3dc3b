"""OptimizerBaseClass (reference: scripts/param_search/opt_base_class.py): what the three searches share.

A search config (scripts/hyper_param_opt.py) holds list flags; a list with more than one value is a tunable
variable, a list with one value a constant.  Each search builds generations of candidate configs (single values
everywhere), writes each candidate's model.conf, has the generation trained (``execute``; by default
runtime.model_execution.run_candidates, NPE candidates at a time in this process) and records every candidate in
opt_hist.csv.

Candidate draws use one private ``random.Random`` per search, fed with the reference's call sequence on the global
generator, so that a search can be reproduced and draws what the reference draws.
"""
from __future__ import absolute_import, division, print_function

import copy
import os
import random
from itertools import cycle

import numpy as np
import pandas as pd

from ..runtime.model_execution import run_candidates, write_conf

_SCALARS = (bool, int, float, str, np.bool_, np.integer, np.floating)
# flags of this project that the reference's search schema does not have (scripts/hyper_param_opt.py)
EXTENSION_FLAGS = ('precision',)


class OptimizerBaseClass(object):
    """Base class of the search algorithms.  `execute(conf_paths, npe)` trains the candidates of a generation and
    returns one entry per candidate, None or the error it failed with (run_candidates)."""

    # opt_hist.csv: these columns, then the sorted tunable variables, then the sorted constant ones.  The fifth column
    # holds the second value _read_results returns (DOE: valid_uq_loss).
    hist_columns = ['id', 'gen', 'objective', 'valid_mse', 'valid_mse_fcst']

    def __init__(self, search_config, execute=None):
        self.search_config = search_config
        self.objective = search_config.objective
        self.search_config_dict = search_config.as_dict()
        self.all_vars, self.constant_vars, self.tunable_vars = [], [], []
        for k, v in self.search_config_dict.items():        # flag-definition order: the grid's product order
            self.all_vars.append(k)
            if isinstance(v, (list, tuple)) and len(v) > 1:
                self.tunable_vars.append(k)
            elif isinstance(v, (list, tuple)):
                self.constant_vars.append(k)

        self.NPE = search_config.NPE
        self.num_gpu = search_config.num_gpu
        self.num_gens = search_config.generations
        self.pop_size = search_config.pop_size
        self.init_pop = search_config.init_pop
        self.mutate_rate = search_config.mutate_rate
        self.vars_keep_type = ['forecast_steps_weights']     # a list in every candidate
        self.execute = execute or run_candidates

        self.rng = random.Random(search_config.seed)
        self.gpu_id_iterable = cycle(list(range(self.num_gpu)))
        self._id = 0
        self._cur_pop = None
        self.opt_hist = pd.DataFrame(columns=self.hist_columns + sorted(self.tunable_vars) +
                                     sorted(self.constant_vars))
        self.exp_dirname = os.path.join(search_config.experiments_dir, search_config.name)
        self.opt_run_dir = os.path.join(self.exp_dirname, 'opt_run')

    def _refuse_uq(self):
        """Genetic and grid search score the validation MSE only and refuse UQ models, as the reference does; here
        before the first generation trains rather than after."""
        if self.search_config.UQ:
            raise NotImplementedError('%s scores the validation MSE of point-estimate models; UQ=True is searched '
                                      'with search_algorithm doe' % type(self).__name__)

    def _new_member(self):
        return self._number(copy.deepcopy(self.search_config))

    def _number(self, config):
        """Gives `config` the next member id, its model_dir <name>/opt_run/<name>-<id> (relative to experiments_dir)
        and the next GPU, round robin over num_gpu."""
        self._id += 1
        config.member_id = self._id
        config.model_dir = os.path.join(self.search_config.name, 'opt_run',
                                        self.search_config.name + '-' + str(self._id))
        config.default_gpu = '/gpu:' + str(next(self.gpu_id_iterable))
        return config

    def _set_constants(self, config):
        for var in self.constant_vars:
            if var not in self.vars_keep_type:
                config.__dict__['__configs'][var] = self.search_config_dict[var][0]

    def _check_scalars(self, config):
        for k, v in config.as_dict().items():
            if k not in self.vars_keep_type:
                assert v is None or isinstance(v, _SCALARS), \
                    "All configuration parameters should have singular value. Received %r for param %s" % (v, k)

    def _prepare(self, config):
        """Flags set on a candidate just before it trains (genetic and grid search: a training run of one process)."""
        config.train = True
        config.num_procs = 1
        config.NPE = 1

    def _write_conf(self, config):
        """<experiments_dir>/<model_dir>/model.conf; ``lfm_quant.py --config`` on it runs the candidate alone."""
        model_dir = os.path.join(self.search_config.experiments_dir, config.model_dir)
        os.makedirs(model_dir, exist_ok=True)
        return write_conf(config.as_dict(), os.path.join(model_dir, 'model.conf'))

    @staticmethod
    def _train_log(config):
        """The candidate's epoch log, as train.py writes it."""
        return pd.read_csv(os.path.join(config.experiments_dir, config.model_dir, 'train_log',
                                        config.name + '-train-logs-epoch.csv'), sep=',')

    def _train_population(self, gen):
        """Records the current population in opt_hist, trains it, and records each candidate's result (inf for a
        candidate that failed).  Returns [(objective value, second value, config)] in population order."""
        for m in self._cur_pop:
            self.opt_hist.loc[m.member_id, 'id'] = m.member_id
            self.opt_hist.loc[m.member_id, 'gen'] = gen
            for var in self.tunable_vars + self.constant_vars:
                self.opt_hist.loc[m.member_id, var] = m.__dict__['__configs'][var]

        for m in self._cur_pop:
            self._prepare(m)
        errors = self.execute([self._write_conf(m) for m in self._cur_pop], self.NPE)
        results = [(np.inf, np.inf, m) if err is not None else self._read_results(m) + (m,)
                   for m, err in zip(self._cur_pop, errors)]

        for res in results:
            member_id = res[-1].member_id
            self.opt_hist.loc[member_id, 'objective'] = res[0]
            self.opt_hist.loc[member_id, 'valid_mse'] = res[0]
            self.opt_hist.loc[member_id, self.hist_columns[4]] = res[1]
        return results

    def _write_hist(self, directory):
        self.opt_hist.to_csv(os.path.join(directory, 'opt_hist.csv'), sep=',', index=False)
