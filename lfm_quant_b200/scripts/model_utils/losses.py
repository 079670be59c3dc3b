"""Losses(config, target_idx).weight_adjusted_mse (reference: scripts/model_utils/losses.py:19-135) and
Losses.weight_adjusted_uq_loss (:137-284), evaluated by the model's engine (ForecastChainEngine.loss / loss_uq: the
one stage's lfmq_loss / lfmq_loss_uq, or lfmq_chain_loss / lfmq_chain_loss_uq over the forecast steps).  The MLP
branch of weight_adjusted_mse (:100-115, MLPLinearPointEstimate) is lfmq_loss on a dense handle in its MSE form, the
form validation evaluates; its Huber form is the training loss, evaluated inside the training step (lfmq_backward)."""
from __future__ import absolute_import, division, print_function

import numpy as np


class _Scalar(object):
    """Device scalar with the ``.numpy()`` the drivers call (train.py:199,336)."""

    def __init__(self, t):
        self._t = t

    def numpy(self):
        return float(self._t.item()) if hasattr(self._t, 'item') else float(self._t)

    def __float__(self):
        return self.numpy()


class Losses(object):

    def __init__(self, config, target_idx, engine=None):
        self.config = config
        self.target_idx = target_idx
        self.engine = engine

    def bind(self, engine):
        self.engine = engine

    def weight_adjusted_mse(self, y_true, y_pred, is_validation=False):
        """losses.py:19-53: per-step loss / mse, linearly weighted -- one native call over the S pairs."""
        assert self.config.forecast_steps > 0, 'forecasts_steps should be a positive integer. %i was provided' % \
            self.config.forecast_steps
        assert isinstance(y_true, (list, tuple)), \
            'arguments to loss function need to be a list [y_true], [y_true1, y_true2, ..]'
        assert isinstance(y_pred, (list, tuple)), \
            'arguments to loss function need to be a list [y_pred], [y_pred1, y_pred2, ..]'
        if 'RNN' not in self.config.nn_type and 'MLP' not in self.config.nn_type:
            raise NotImplementedError('%s NN type not implemented' % self.config.nn_type)      # losses.py:117-119
        if 'MLP' in self.config.nn_type and self.config.huber_loss and not is_validation:
            raise NotImplementedError('the Huber training loss of the MLP branch (losses.py:102-105) is evaluated by '
                                      'the training step; Losses evaluates the MSE form (is_validation=True)')
        S = self.config.forecast_steps
        assert len(y_true) == S and len(y_pred) == S
        self._step_weights()
        out = self.engine.loss([self._to(p) for p in y_pred], [self._to(y) for y in y_true])
        return _Scalar(out[0]), _Scalar(out[1])

    def weight_adjusted_uq_loss(self, y_true, y_pred, y_var):
        """losses.py:137-178: (uq_loss, uq_loss_last_tar, mse), each with ``.numpy()``, each summed over the forecast
        steps with config.forecast_steps_weights."""
        assert self.config.UQ, "weight_adjusted_mse is only available for uq range estimate models. UQ should be True"
        assert self.config.forecast_steps > 0, 'forecasts_steps should be a positive integer. %i was provided' % \
            self.config.forecast_steps
        for name, v in (('y_true', y_true), ('y_pred', y_pred), ('y_var', y_var)):
            assert isinstance(v, (list, tuple)), \
                'arguments to loss function need to be a list [%s], [%s1, %s2, ..]' % (name, name, name)
        if 'RNN' not in self.config.nn_type:
            raise NotImplementedError('only RNN uq range estimates are built on this path')
        S = self.config.forecast_steps
        for name, v in (('y_true', y_true), ('y_pred', y_pred), ('y_var', y_var)):
            assert len(v) >= S, '%s holds %d forecast steps, forecast_steps is %d' % (name, len(v), S)
        self._step_weights()
        out = self.engine.loss_uq([self._to(p) for p in y_pred[:S]], [self._to(v) for v in y_var[:S]],
                                  [self._to(y) for y in y_true[:S]])
        return _Scalar(out[0]), _Scalar(out[1]), _Scalar(out[2])

    def _step_weights(self):
        """losses.py:41-45,165-170: one weight per forecast step; the weights of a single step become [1.0].  The
        engine weighs the steps with the weights it was built with."""
        S, w = self.config.forecast_steps, self.config.forecast_steps_weights
        assert S == 1 or len(w) == S
        if len(w) == S == 1:
            self.config.forecast_steps_weights = [1.0]
        assert self.engine is not None, 'Losses is not bound to a native engine'

    def _to(self, a):
        """An ndarray or tensor as a contiguous fp32 tensor on the engine's device."""
        import torch
        t = a if isinstance(a, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32))
        return t.to(self.engine.device, torch.float32).contiguous()
