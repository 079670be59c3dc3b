"""MLPLinearPointEstimate (reference: scripts/models/point_estimate/mlp_linear_point_estimate.py:17-77): the linear
regression baseline, one Dense(n_outputs) layer OUTPUT_1 with a bias over the flattened input window [B, T*F]
(data_processing.py:363-365), kernel drawn by Initializer.get_initializer(), no MaxNorm and no regulariser.  It runs on
a dense handle of the native library (DenseEngine); the model object has the same Keras subset as the recurrent
forecaster's, and ``model(inp)`` / ``model.predict(inp)`` return [B, n_outputs]."""
from __future__ import absolute_import, division, print_function

import numpy as np

from ..model_base_class import BaseModelClass
from ...model_utils.initializers import Initializer
from ...model_utils.optimizers import Optimizers
from .rnn_point_estimate import NativeForecaster


class NativeDenseForecaster(NativeForecaster):
    """NativeForecaster over one DenseEngine stage: the same model object, whose TF-format container holds OUTPUT_1 as
    ``layer_with_weights-0``."""

    title = 'MLPLinearPointEstimate'
    _flat_outputs = True          # model.predict returns [B, n_outputs]

    def _build_engine(self, config, seq_len, n_inputs, n_outputs, target_idx):
        from ....engine import DenseEngine, ForecastChainEngine
        if config.forecast_steps != 1:
            raise NotImplementedError('MLPLinearPointEstimate has one output (mlp_linear_point_estimate.py:66-77); '
                                      'forecast_steps = %d needs one per step, which the reference cannot train '
                                      'either' % config.forecast_steps)
        self._engine_kw = dict(
            max_batch=config.batch_size, seq_len=seq_len, n_inputs=n_inputs, n_outputs=n_outputs,
            target_idx=target_idx, precision=getattr(config, 'precision', 'fp32'), optimizer=config.optimizer,
            target_lambda=config.target_lambda, max_grad_norm=config.max_grad_norm, sgd_momentum=config.sgd_momentum,
            huber_loss=bool(config.huber_loss), huber_delta=config.huber_delta, forward_only=not config.train)
        engine = DenseEngine(**self._engine_kw)
        specs = [(n, s) for (n, s, _, tr) in engine.specs if tr]
        rng = np.random.RandomState(config.seed)
        kernel = Initializer(config).get_initializer()(specs[0][1], rng)      # :69-73
        engine.set_weights([np.asarray(kernel, dtype=np.float32), np.zeros(specs[1][1], dtype=np.float32)])
        return ForecastChainEngine(stages=[engine])

    def _new_wide_engine(self, rows):
        from ....engine import DenseEngine, ForecastChainEngine
        return ForecastChainEngine(stages=[DenseEngine(**dict(self._engine_kw, max_batch=rows, forward_only=True))])


class MLPLinearPointEstimate(BaseModelClass):
    """Builds the linear baseline with the shapes of the dataset."""

    def __init__(self, config, dataset):
        self.config = config
        self.dataset = dataset
        self.seq_len = self.dataset.seq_len
        self.n_inputs = self.dataset.n_inputs
        self.n_outputs = self.dataset.n_outputs
        self.forecast_steps = self.config.forecast_steps
        self.opt = Optimizers(self.config)
        self.initializer = Initializer(self.config)
        super(MLPLinearPointEstimate, self).__init__(self.seq_len, self.n_inputs, self.n_outputs)
        self.model = NativeDenseForecaster(self.config, self.seq_len, self.n_inputs, self.n_outputs,
                                           self.dataset.target_index)
