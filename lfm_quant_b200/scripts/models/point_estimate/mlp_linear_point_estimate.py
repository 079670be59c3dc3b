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
from .rnn_point_estimate import NativeForecaster, _Variable


class NativeDenseForecaster(NativeForecaster):
    """The Keras-subset model object of NativeForecaster over a DenseEngine: __call__, predict, predict_device,
    train_step, trainable_variables, save_weights / load_weights (``.lfmq.npz`` and the TF-format container, where
    OUTPUT_1 is ``layer_with_weights-0``), summary."""

    def __init__(self, config, seq_len, n_inputs, n_outputs, target_idx):
        from ....engine import DenseEngine
        self.config = config
        self.uq = False
        if config.forecast_steps != 1:
            raise NotImplementedError('MLPLinearPointEstimate has one output (mlp_linear_point_estimate.py:66-77); '
                                      'forecast_steps = %d needs one per step, which the reference cannot train '
                                      'either' % config.forecast_steps)
        self.engine = DenseEngine(
            max_batch=config.batch_size, seq_len=seq_len, n_inputs=n_inputs, n_outputs=n_outputs,
            target_idx=target_idx, precision=getattr(config, 'precision', 'fp32'), optimizer=config.optimizer,
            target_lambda=config.target_lambda, max_grad_norm=config.max_grad_norm, sgd_momentum=config.sgd_momentum,
            huber_loss=bool(config.huber_loss), huber_delta=config.huber_delta, forward_only=not config.train)
        specs = [(n, s) for (n, s, _, tr) in self.engine.specs if tr]
        rng = np.random.RandomState(config.seed)
        kernel = Initializer(config).get_initializer()(specs[0][1], rng)      # :69-73
        self.engine.set_weights([np.asarray(kernel, dtype=np.float32), np.zeros(specs[1][1], dtype=np.float32)])
        self.trainable_variables = [_Variable(self, i, n, s) for i, (n, s) in enumerate(specs)]
        self._calls = 0

    def summary(self):
        lines = ['Model: "MLPLinearPointEstimate" (native sm_90a, precision=%s)' % self.engine.precision,
                 '%-44s %-16s %10s' % ('Variable', 'Shape', 'Param #'), '=' * 72]
        for name, shape, _, _ in self.engine.specs:
            lines.append('%-44s %-16s %10d' % (name, str(tuple(shape)), int(np.prod(shape))))
        lines += ['=' * 72, 'Total params: %d' % self.engine.n_total, 'Trainable params: %d' % self.engine.n_trainable]
        return '\n'.join(lines)


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
