"""DOE (reference: scripts/param_search/doe.py): the rows of a design-of-experiments CSV file (doe_file), NPE rows per
generation; every column of a row is set on its candidate.

Kept from the reference:
- a row may carry ``member_id`` (then the candidate keeps the search's model_dir unless the row sets ``model_dir``
  too) and ``train`` (False: the candidate predicts, and is scored by the weighted mean of preds.dat's
  ``norm_squared_diff_<step>`` columns);
- UQ models are scored by the best epoch's validation UQ loss; opt_hist's fifth column is ``valid_uq_loss`` (None
  for point estimates) and its ``objective`` column holds the validation MSE;
- columns that are not flags are set too (the reference's ``drop`` of them does not drop);
- a ``name`` column names the experiment directory, and opt_hist.csv is written there, not under opt_run;
- the candidates keep the search's NPE, num_procs and train values (none is reset before training).
Divergence: directories are created with their parents (the reference needs <name>/opt_run to exist for candidates
without member_id).
"""
from __future__ import absolute_import, division, print_function

import copy
import os

import numpy as np
import pandas as pd

from .opt_base_class import OptimizerBaseClass


class DOE(OptimizerBaseClass):

    hist_columns = ['id', 'gen', 'objective', 'valid_mse', 'valid_uq_loss']

    def __init__(self, search_config, execute=None):
        super(DOE, self).__init__(search_config, execute)
        assert search_config.doe_file is not None, 'search_algorithm doe needs a doe_file'
        self.doe = pd.read_csv(search_config.doe_file, sep=',')
        if 'name' in self.doe.columns:
            self.exp_dirname = os.path.join(search_config.experiments_dir, self.doe['name'].iloc[0])
        os.makedirs(self.exp_dirname, exist_ok=True)
        self.num_gens = int(np.ceil(self.doe.shape[0] / self.NPE))
        self.pop_size = self.NPE

    def _get_gen(self, gen_num):
        pop = self.doe.iloc[gen_num * self.NPE:(gen_num + 1) * self.NPE]
        return [self._build_config(pop.iloc[i]) for i in range(pop.shape[0])]

    def _build_config(self, member):
        """The candidate of one row (a pandas Series)."""
        if 'member_id' in member.index:
            config = copy.deepcopy(self.search_config)
            config.default_gpu = '/gpu:' + str(next(self.gpu_id_iterable))
        else:
            config = self._new_member()
        self._set_constants(config)
        for var in member.index:
            config.__dict__['__configs'][var] = member[var]
        self._check_scalars(config)
        return config

    def _prepare(self, config):
        pass

    @staticmethod
    def _read_results(config):
        """(validation MSE, validation UQ loss or None) of the best epoch -- by UQ loss for UQ models, by MSE
        otherwise -- or, for a candidate that predicted, (weighted preds.dat MSE, None); inf, inf when the file is
        missing."""
        try:
            if config.train:
                df = DOE._train_log(config)
                if not config.UQ:
                    df = df.sort_values(by='valid_mse').reset_index()
                    return df.iloc[0]['valid_mse'], None
                df = df.sort_values(by='valid_uq_loss').reset_index()
                return df.iloc[0]['valid_mse'], df.iloc[0]['valid_uq_loss']
            df = pd.read_csv(os.path.join(config.experiments_dir, config.model_dir, 'pred', config.preds_fname),
                             sep=' ', dtype={'gvkey': str})
            valid_loss = 0
            for i in range(config.forecast_steps):
                valid_loss += df['norm_squared_diff_' + str(i + 1)].mean() * config.forecast_steps_weights[i]
            return valid_loss, None
        except FileNotFoundError:
            return np.inf, np.inf

    def run(self):
        print("Starting DOE ...")
        for i in range(self.num_gens):
            print("Gen %i" % (i + 1))
            self._cur_pop = self._get_gen(i)
            self._train_population(i + 1)
            self._write_hist(self.exp_dirname)
