"""NaivePointEstimate (reference: scripts/models/point_estimate/naive_point_estimate.py:17-58): next year's fundamentals
equal this year's.  The prediction is the last time step of the input window cropped to its first n_outputs features,
the financial fields (data_processing.py:82-83: the input columns are the financial fields, then the aux fields).
Cropping1D(cropping=(0, F - O)) there removes the LAST F - O features, whatever its comment says.

The model has no variables: there is nothing to train (the reference's apply_gradients gets an empty list), so
``--train=True`` is refused, and prediction loads no checkpoint (predict.py:90-93).  The forecast is a selection of
inputs, not arithmetic: ``model.predict(inp)`` returns the [B, O] slice of the batch already on the GPU."""
from __future__ import absolute_import, division, print_function

import numpy as np

from ..model_base_class import BaseModelClass


class NaiveForecaster(object):
    """The model object: __call__ / predict / predict_device -> x[:, T-1, :O] of the [B, T, F] (or [B, T*F]) batch."""

    engine = None
    trainable_variables = []

    def __init__(self, seq_len, n_inputs, n_outputs, target_idx=0):
        self.T, self.F, self.O = seq_len, n_inputs, n_outputs
        self.target_idx = target_idx

    def predict_device(self, inp):
        import torch
        x = inp if isinstance(inp, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(inp, dtype=np.float32))
        return x.reshape(x.shape[0], self.T, self.F)[:, self.T - 1, :self.O]

    def __call__(self, inp, training=None):
        return self.predict_device(inp)

    def predict(self, inp, batch_size=None):
        return self.predict_device(inp).cpu().numpy()

    def conformal_forecast(self, inp):
        """(pred [1,B], None): the forecast of the target field, whose score is |y - pred| (DESIGN.md section 5j)."""
        return self.predict_device(inp)[:, self.target_idx].unsqueeze(0).contiguous(), None

    def conformal(self, cal_batches, query_windows, levels, knn=0, query_forecast=None, query_targets=None,
                  pool_batches=None):
        """Split-conformal intervals of the naive forecast, as NativeForecaster.conformal (no kNN score: the naive
        forecast has no features)."""
        from .rnn_point_estimate import conformal_intervals
        if int(knn) > 0:
            raise ValueError('conformal: NaivePointEstimate has no head-input features for the kNN score')
        if query_forecast is None:
            query_forecast = self.conformal_forecast(query_windows)
        return conformal_intervals(self.conformal_forecast, cal_batches, query_windows, query_forecast, query_targets,
                                   levels)

    def load_weights(self, prefix):
        return None

    def reset_states(self):
        return None

    def count_params(self):
        return 0

    def get_weights(self):
        return []

    def summary(self):
        return ('Model: "NaivePointEstimate" (last input step, first %d of %d features; no variables)\n'
                'Total params: 0' % (self.O, self.F))


class NaivePointEstimate(BaseModelClass):

    def __init__(self, config, dataset):
        self.config = config
        self.dataset = dataset
        self.seq_len = self.dataset.seq_len
        self.n_inputs = self.dataset.n_inputs
        self.n_outputs = self.dataset.n_outputs
        if config.train:
            raise ValueError('NaivePointEstimate has no variables to train: it predicts the last input step. Run it '
                             'with --train=False (no checkpoint is needed)')
        if config.forecast_steps != 1:
            raise NotImplementedError('NaivePointEstimate has one output (naive_point_estimate.py:45-58); '
                                      'forecast_steps = %d' % config.forecast_steps)
        super(NaivePointEstimate, self).__init__(self.seq_len, self.n_inputs, self.n_outputs)
        # the target field's index, which the conformal intervals read
        self.model = NaiveForecaster(self.seq_len, self.n_inputs, self.n_outputs, getattr(dataset, 'target_index', 0))
