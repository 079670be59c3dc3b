"""RNNUqRangeEstimate -- the reference's recurrent uncertainty-quantification model
(scripts/models/uq_range_estimate/rnn_uq_range_estimate.py:24-159) on the native engine: the same LSTM|GRU -> BN ->
Dropout trunk as RNNPointEstimate with dropout ALWAYS active (``training=True`` is a literal there, :86,88), a target
head OUTPUT_TARGET_1 and a variance head OUTPUT_VARIANCE_1 followed by max(softplus, 1e-6)
(model_utils/custom_layers.py:12-13).  ``model(inp)`` / ``model.predict(inp)`` return [target_preds, variance_preds];
with forecast_steps > 1 (:114-157) the list [tar_1, var_1, .., tar_S, var_S] of the forecast chain."""
from __future__ import absolute_import, division, print_function

from ...model_utils.initializers import Initializer
from ...model_utils.optimizers import Optimizers
from ..model_base_class import BaseModelClass
from ..point_estimate.rnn_point_estimate import NativeForecaster


class RNNUqRangeEstimate(BaseModelClass):

    def __init__(self, config, dataset):
        self.config = config
        self.dataset = dataset
        self.seq_len = self.dataset.seq_len
        self.n_inputs = self.dataset.n_inputs
        self.n_outputs = self.dataset.n_outputs
        self.forecast_steps = self.config.forecast_steps
        self.n_layers = self.config.num_layers
        self.n_hidden_units = self.config.num_hidden
        self.opt = Optimizers(self.config)
        self.initializer = Initializer(self.config)
        super(RNNUqRangeEstimate, self).__init__(self.seq_len, self.n_inputs, self.n_outputs)
        self.model = self._build_model()

    def _build_model(self):
        return NativeForecaster(self.config, self.seq_len, self.n_inputs, self.n_outputs, self.dataset.target_index,
                                uq=True)
