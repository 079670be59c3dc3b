"""Losses(config, target_idx).weight_adjusted_mse (reference: scripts/model_utils/losses.py:19-135), evaluated by
the native loss kernel (lfmq_loss; lfmq_chain_loss for forecast_steps > 1), and Losses.weight_adjusted_uq_loss
(:137-284) by lfmq_loss_uq (lfmq_chain_loss_uq for forecast_steps > 1).  The MLP branch of weight_adjusted_mse
(:100-115, MLPLinearPointEstimate) is lfmq_loss on a dense handle in its MSE form, the form validation evaluates; its
Huber form is the training loss, evaluated inside the training step (lfmq_backward)."""
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
        if S == 1:
            if len(self.config.forecast_steps_weights) == 1:
                self.config.forecast_steps_weights = [1.0]       # losses.py:44-45
            return self._get_loss_point_estimate(y_true[0], y_pred[0], is_validation)
        # losses.py:36-51: per-step loss / mse, linearly weighted -- one native call over the S pairs
        assert len(y_true) == S and len(y_pred) == S
        assert len(self.config.forecast_steps_weights) == S
        import torch
        assert self.engine is not None, 'Losses is not bound to a native engine'
        dev = self.engine.device
        to = lambda a: (a if isinstance(a, torch.Tensor) else
                        torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32))).to(dev, torch.float32).contiguous()
        out = self.engine.loss([to(p) for p in y_pred], [to(y) for y in y_true])
        return _Scalar(out[0]), _Scalar(out[1])

    def _get_loss_point_estimate(self, y_true, y_pred, is_validation=False):
        import torch
        assert self.engine is not None, 'Losses is not bound to a native engine'
        dev = self.engine.device
        to = lambda a: a if isinstance(a, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32))
        yt = to(y_true).to(dev, torch.float32).contiguous()
        yp = to(y_pred).to(dev, torch.float32).contiguous()
        out = self.engine.loss(yp, yt)
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
        if S == 1:
            if len(self.config.forecast_steps_weights) == 1:
                self.config.forecast_steps_weights = [1.0]
        else:
            assert len(self.config.forecast_steps_weights) == S     # losses.py:164-166
        import torch
        assert self.engine is not None, 'Losses is not bound to a native engine'
        dev = self.engine.device
        to = lambda a: (a if isinstance(a, torch.Tensor) else
                        torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32))).to(dev, torch.float32).contiguous()
        if S == 1:
            out = self.engine.loss_uq(to(y_pred[0]), to(y_var[0]), to(y_true[0]))
        else:                       # losses.py:159-177: per-step losses with their own masks, linearly weighted
            out = self.engine.loss_uq([to(p) for p in y_pred[:S]], [to(v) for v in y_var[:S]],
                                      [to(y) for y in y_true[:S]])
        return _Scalar(out[0]), _Scalar(out[1]), _Scalar(out[2])
