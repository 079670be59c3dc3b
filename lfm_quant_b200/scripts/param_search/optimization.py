"""HPOptimization (reference: scripts/param_search/optimization.py): runs the search that search_algorithm names."""
from __future__ import absolute_import, division, print_function

import os

from .doe import DOE
from .genetic_algorithm import GeneticAlgorithm
from .grid_search import GridSearch

ALGORITHMS = {'genetic': GeneticAlgorithm, 'grid_search': GridSearch, 'doe': DOE}


class HPOptimization(object):

    def __init__(self, search_config, execute=None):
        self.search_config = search_config
        self.execute = execute

    def __call__(self):
        algorithm = self.search_config.search_algorithm
        if algorithm not in ALGORITHMS:
            raise NotImplementedError('search_algorithm %r: choose one of %s' % (algorithm, ', '.join(ALGORITHMS)))
        if int(os.environ.get('WORLD_SIZE', '1')) > 1:
            raise NotImplementedError('a hyper-parameter search trains its candidates side by side in one process and '
                                      'cannot be combined with torchrun data parallelism; run it without torchrun')
        search = ALGORITHMS[algorithm](self.search_config, self.execute)
        search.run()
        return search
