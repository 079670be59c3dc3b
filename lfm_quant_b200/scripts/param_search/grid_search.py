"""GridSearch (reference: scripts/param_search/grid_search.py): every combination of the tunable values
(``itertools.product`` in flag-definition order), NPE combinations per generation.

Kept from the reference:
- ``num_gens = len(combinations) // NPE``: a remainder of fewer than NPE combinations is not trained;
- ``_read_results`` returns (forecast-space MSE, validation MSE), the other way round from the genetic algorithm, so
  opt_hist's ``objective`` and ``valid_mse`` columns hold the forecast-space MSE and ``valid_mse_fcst`` the validation
  MSE.
Divergences: UQ=True is refused before anything trains; directories are created with their parents.
"""
from __future__ import absolute_import, division, print_function

import os
from itertools import product

import numpy as np

from .opt_base_class import OptimizerBaseClass


class GridSearch(OptimizerBaseClass):

    def __init__(self, search_config, execute=None):
        super(GridSearch, self).__init__(search_config, execute)
        self._refuse_uq()
        os.makedirs(self.opt_run_dir, exist_ok=True)
        self.doe = list(product(*[self.search_config_dict[k] for k in self.tunable_vars]))
        print("Tunable Params")
        print(self.tunable_vars)
        self.num_gens = len(self.doe) // self.NPE
        self.pop_size = self.NPE

    def _get_gen(self, gen_num):
        return [self._build_config(m) for m in self.doe[gen_num * self.NPE:(gen_num + 1) * self.NPE]]

    def _build_config(self, member):
        """The candidate of one combination: member[i] is the value of tunable_vars[i]."""
        assert len(member) == len(self.tunable_vars)
        config = self._new_member()
        self._set_constants(config)
        for var, value in zip(self.tunable_vars, member):
            if var not in self.vars_keep_type:
                config.__dict__['__configs'][var] = value
        self._check_scalars(config)
        return config

    @staticmethod
    def _read_results(config):
        if config.UQ:
            raise NotImplementedError('grid search scores point-estimate models only')
        try:
            df = GridSearch._train_log(config).sort_values(by='valid_mse').reset_index()
            valid_loss, valid_loss_fcst = df.iloc[0]['valid_mse'], df.iloc[0]['valid_mse_fcst']
        except FileNotFoundError:
            valid_loss, valid_loss_fcst = np.inf, np.inf
        return valid_loss_fcst, valid_loss

    def run(self):
        print("Starting GRID search ...")
        for i in range(self.num_gens):
            print("Gen %i" % (i + 1))
            self._cur_pop = self._get_gen(i)
            self._train_population(i + 1)
            self._write_hist(self.opt_run_dir)
