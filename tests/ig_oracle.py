"""fp64 integrated gradients of the point forecast f(x) = pred[b, T-1, target_idx] (lfmq_integrated_gradients), built
from lfm_oracle's forward caches and lstm_backward / gru_backward with need_dx=True, seeded by the one-hot at
[T-1, target_idx].  Dropout off, BatchNormalization in its inference affine form, baseline x' = 0, midpoint rule
alpha_k = (k + 1/2) / M."""
import numpy as np

import lfm_oracle as orc


def forecast(params, x, *, num_layers, target_idx, rnn_cell='lstm', bn_mean=None, bn_var=None):
    """f(x) [B] and the forward cache."""
    preds, fcache = orc.forward(params, np.asarray(x, dtype=np.float64), num_layers=num_layers, training=False,
                                bn_mean=bn_mean, bn_var=bn_var, rnn_cell=rnn_cell)
    return preds[:, -1, target_idx], fcache


def input_gradient(params, x, *, num_layers, target_idx, rnn_cell='lstm', bn_mean=None, bn_var=None):
    """df/dx [B,T,F] and f(x) [B]."""
    f, (caches, _, Wo) = forecast(params, x, num_layers=num_layers, target_idx=target_idx, rnn_cell=rnn_cell,
                                  bn_mean=bn_mean, bn_var=bn_var)
    B, T = x.shape[:2]
    dpred = np.zeros((B, T, Wo.shape[1]))
    dpred[:, -1, target_idx] = 1.0
    dy = dpred @ Wo.T
    for l in range(num_layers - 1, -1, -1):
        lc, _, _, inv, gamma, _ = caches[l]
        dy = (orc.lstm_backward if rnn_cell == 'lstm' else orc.gru_backward)(dy * gamma * inv, lc, need_dx=True)[3]
    return dy, f


def integrated_gradients(params, x, steps, **kw):
    """(attr [B,T,F], f(x) [B], f(0) [B]) with `steps` midpoint-rule interpolants."""
    x = np.asarray(x, dtype=np.float64)
    total = np.zeros_like(x)
    for k in range(steps):
        total += input_gradient(params, (k + 0.5) / steps * x, **kw)[0]
    f_x = forecast(params, x, **kw)[0]
    f_base = forecast(params, np.zeros_like(x), **kw)[0]
    return x * total / steps, f_x, f_base


def completeness_gap(attr, f_x, f_base):
    """sum_{t,f} attr[b] - (f_x[b] - f_base[b]) [B]: the quadrature error of the midpoint rule."""
    return attr.reshape(attr.shape[0], -1).sum(axis=1) - (f_x - f_base)
