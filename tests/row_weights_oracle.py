"""fp64 oracle of the row-weighted training loss (DESIGN.md section 6d): every mean of the point-estimate loss
(losses.py:55-98), of the UQ loss (losses.py:180-284) and of the linear model's MLP branch (losses.py:69-75,100-115)
becomes a weighted mean over the windows of the batch.  ``w=None`` is the unweighted arithmetic of oracle/lfm_oracle.py.
A weighted count of 0 divides as 1."""
import numpy as np

import lfm_oracle as orc


def _nz(d):
    return d if d != 0 else d.dtype.type(1.0)


def loss_point(y_true, y_pred, w=None, *, target_idx, target_lambda, rnn_lambda):
    """(loss, mse_0, dLoss/dpred) of the RNN point branch with window weights w [B] (None: unweighted)."""
    if w is None:
        loss, mse, dpred, _ = orc.loss_point_estimate(y_true, y_pred, target_idx=target_idx,
                                                      target_lambda=target_lambda, rnn_lambda=rnn_lambda)
        return loss, mse, dpred
    B, T, K = y_true.shape
    dt = y_pred.dtype
    w = np.asarray(w, dtype=dt)
    mask = (~np.all(y_true == 0.0, axis=-1)).astype(dt)
    d_all = y_pred * mask[..., None] - y_true
    Bg = _nz(w.sum())
    Mg = _nz((w[:, None] * mask).sum())
    wd2 = w[:, None, None] * d_all ** 2
    mse_0 = wd2[:, -1, target_idx].sum() / Bg
    mse_1 = wd2[:, -1, :].sum() / (Bg * K)
    mse_2 = wd2.sum() / (Mg * K)
    p1, p2 = dt.type(target_lambda), dt.type(rnn_lambda)
    loss = p1 * mse_0 + (1 - p1) * (p2 * mse_1 + (1 - p2) * mse_2)
    coef = np.full((B, T, K), (1 - p1) * (1 - p2) / (K * Mg), dtype=dt)
    coef[:, -1, :] += (1 - p1) * p2 / (Bg * K)
    coef[:, -1, target_idx] += p1 / Bg
    dpred = 2.0 * d_all * coef * mask[..., None] * w[:, None, None]
    return loss, mse_0, dpred


def point_grads(params, x, y, w, cfg):
    """(loss, mse_0, gradients in Keras order) of one weighted training batch of a point model, no dropout."""
    L = cfg['num_layers']
    cell = cfg.get('rnn_cell', 'lstm')
    preds, fc = orc.forward(params, x.astype(np.float64), num_layers=L, training=True, rnn_cell=cell)
    loss, mse, dpred = loss_point(y.astype(np.float64), preds, w, target_idx=cfg['target_idx'],
                                  target_lambda=cfg['target_lambda'], rnn_lambda=cfg['rnn_lambda'])
    return loss, mse, orc.backward(dpred, fc, num_layers=L, rnn_cell=cell)


def loss_dense(y_true, y_pred, w=None, *, target_idx, target_lambda):
    """(loss, mse_0, dLoss/dpred) of the linear model's MSE branch over [B, O] with window weights w."""
    B, O = y_true.shape
    w = np.ones(B) if w is None else np.asarray(w, dtype=np.float64)
    mask = (~np.all(y_true == 0.0, axis=-1)).astype(np.float64)
    r = y_true - y_pred * mask[:, None]
    Bg = _nz(w.sum())
    mse_0 = (w * r[:, target_idx] ** 2).sum() / Bg
    mall = (w[:, None] * r ** 2).sum() / (Bg * O)
    loss = target_lambda * mse_0 + (1 - target_lambda) * mall
    g = np.full((B, O), (1 - target_lambda) / (Bg * O))
    g[:, target_idx] += target_lambda / Bg
    return loss, mse_0, -2.0 * r * g * mask[:, None] * w[:, None]
