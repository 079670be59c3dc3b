"""GeneticAlgorithm (reference: scripts/param_search/genetic_algorithm.py).

Generation 1 is pop_size random candidates (or the rows of doe_file, or the population pickled at init_pop).  Each
next generation: the candidates sorted by validation MSE, the better half kept as parents, and every child a
crossover of two parents (each flag from the second parent with probability 1/2), mutated with probability
mutate_rate (one tunable flag redrawn).  Member ids keep increasing across generations.

Kept from the reference:
- the draws, in order: ``seed(seed)`` before the initial population and again at the start of ``run``; one
  ``choice`` per tunable flag per initial member; per child one ``shuffle(parents)``, one ``random()`` per flag of
  the config, one ``random()`` against mutate_rate and, if it mutates, ``choice`` of the flag and of its value;
- the sort key is the validation MSE (``results[i][0]``), and opt_hist's ``objective`` column holds it;
- with doe_file the file is read as strings, and NPE = pop_size = its number of rows;
- the population is pickled before each generation trains, so the file holds the generation about to train.
Divergences: the draws come from a private ``random.Random``; the crossover draws for the project's ``precision``
flag only where it is tunable (a constant one is the same in every member), so a search the reference can express
makes the reference's draws; UQ=True is refused before anything trains (the reference raises after the first
generation has trained); directories are created with their parents.
"""
from __future__ import absolute_import, division, print_function

import copy
import os
import pickle

import numpy as np
import pandas as pd

from .opt_base_class import EXTENSION_FLAGS, OptimizerBaseClass


class GeneticAlgorithm(OptimizerBaseClass):

    def __init__(self, search_config, execute=None):
        super(GeneticAlgorithm, self).__init__(search_config, execute)
        self._refuse_uq()
        if search_config.doe_file:
            self.doe = pd.read_csv(search_config.doe_file, sep=',', dtype=object)
            self.NPE = self.doe.shape[0]
            self.pop_size = self.NPE
        os.makedirs(self.opt_run_dir, exist_ok=True)
        self._cur_pop = self._init_population()

    def _init_population(self):
        self.rng.seed(self.search_config.seed)
        pop = []
        for i in range(self.pop_size):
            config = self._new_member()
            self._set_constants(config)
            if self.search_config.doe_file:
                member = self.doe.iloc[i]
                for var in member.index:
                    config.__dict__['__configs'][var] = member[var]
            else:
                for var in self.tunable_vars:
                    if var not in self.vars_keep_type:
                        config.__dict__['__configs'][var] = self.rng.choice(self.search_config_dict[var])
            self._check_scalars(config)
            pop.append(config)
        return pop

    @staticmethod
    def _read_results(config):
        """(validation MSE, its forecast-space counterpart) of the best epoch by validation MSE; inf, inf when the
        candidate wrote no log."""
        if config.UQ:
            raise NotImplementedError('the genetic algorithm scores point-estimate models only')
        try:
            df = GeneticAlgorithm._train_log(config).sort_values(by='valid_mse').reset_index()
            return df.iloc[0]['valid_mse'], df.iloc[0]['valid_mse_fcst']
        except FileNotFoundError:
            return np.inf, np.inf

    def _get_next_gen(self, results):
        assert isinstance(results, (list, tuple))
        results = sorted(results, key=lambda x: x[0])
        parents = [x[-1] for x in results[:len(results) // 2]]
        self._cur_pop = []
        for _ in range(self.pop_size):
            self.rng.shuffle(parents)
            child = self._cross_over(parents[0], parents[1])
            if self.rng.random() <= self.mutate_rate:
                child = self._mutate(child)
            self._cur_pop.append(child)
        return self._cur_pop

    def _cross_over(self, p1, p2):
        child = copy.deepcopy(p1)
        flags = child.__dict__['__configs']
        for flag in list(flags):
            if flag in EXTENSION_FLAGS and flag not in self.tunable_vars:
                continue        # constant in every member: no draw, so the draws stay the reference's
            if self.rng.random() >= 0.5:
                flags[flag] = p2.__dict__['__configs'][flag]
        self._number(child)         # its own id, directory and GPU, whichever parent the draws took them from
        return child

    def _mutate(self, mem):
        flag = self.rng.choice(self.tunable_vars)
        mem.__dict__['__configs'][flag] = self.rng.choice(self.search_config_dict[flag])
        return mem

    def run(self):
        self.rng.seed(self.search_config.seed)
        print("Starting GA search ...")
        if self.init_pop:
            with open(self.init_pop, 'rb') as fh:
                self._cur_pop = pickle.load(fh)
        assert isinstance(self._cur_pop, (list, tuple))
        for i in range(self.num_gens):
            gen = i + 1
            print("Gen %i" % gen)
            if self.search_config.save_latest_pop:
                latest = os.path.join(self.exp_dirname, '_latest_pop')
                os.makedirs(latest, exist_ok=True)
                with open(os.path.join(latest, 'latest_pop.pkl'), 'wb') as fh:
                    pickle.dump(self._cur_pop, fh)
            results = self._train_population(gen)
            self._cur_pop = self._get_next_gen(results)
            self._write_hist(self.opt_run_dir)
