"""fp64 restatement of the reference's two baselines, the oracle of the dense handle (lfmq_dense_create).  Paths are
relative to the reference's scripts/.

- MLPLinearPointEstimate (models/point_estimate/mlp_linear_point_estimate.py:66-77): one Dense(O) over x [B, T*F].
- NaivePointEstimate (models/point_estimate/naive_point_estimate.py:45-58): the last step's first O features.
- The MLP branch of Losses._get_loss_point_estimate (model_utils/losses.py:69-75,100-115), MSE and Keras Huber forms,
  and its gradient.
- One training step (train.py:178-199): the clip and optimizers of oracle/lfm_oracle.py, no MaxNorm.
"""
import numpy as np

import lfm_oracle as orc


def dense_forward(x, W, b):
    """mlp_linear_point_estimate.py:69-73: Dense(O)(x) with x [B, T*F] (or [B, T, F], flattened as
    data_processing.py:363-364 does)."""
    x = np.asarray(x, dtype=np.float64)
    return x.reshape(x.shape[0], -1) @ np.asarray(W, dtype=np.float64) + np.asarray(b, dtype=np.float64)


def naive_forecast(x, seq_len, n_inputs, n_outputs):
    """naive_point_estimate.py:47-56: Reshape to [T, F], Cropping1D((T-1, 0)) keeps the last step,
    Cropping1D((0, F-O)) on the features keeps the FIRST O of them."""
    return np.asarray(x).reshape(-1, seq_len, n_inputs)[:, seq_len - 1, :n_outputs]


def _huber(r, delta):
    """keras.losses.Huber per element: 0.5 r^2 if |r| <= delta else delta (|r| - delta / 2)."""
    a = np.abs(r)
    return np.where(a <= delta, 0.5 * r * r, delta * (a - 0.5 * delta))


def _huber_grad(r, delta):
    return np.where(np.abs(r) <= delta, r, delta * np.sign(r))


def mlp_loss(y_true, y_pred, *, target_idx, target_lambda, huber=False, huber_delta=1.0, batch_global=None):
    """losses.py:69-75,100-115: returns (loss, mse_0).  Rows whose targets are all zero have their predictions zeroed
    (:69-75) and still count in both means.  huber: the Huber form (:102-105, training only).  batch_global: the
    denominator B of the whole data-parallel batch (then the values are this shard's contributions)."""
    y = np.asarray(y_true, dtype=np.float64)
    p = np.asarray(y_pred, dtype=np.float64)
    B, O = y.shape
    Bg = B if batch_global is None else batch_global
    mask = (~np.all(y == 0.0, axis=-1)).astype(np.float64)
    r = y - p * mask[:, None]
    f = _huber(r, huber_delta) if huber else r * r
    mse_0 = f[:, target_idx].sum() / Bg
    mse_all = f.sum() / (Bg * O)
    return target_lambda * mse_0 + (1.0 - target_lambda) * mse_all, mse_0


def mlp_loss_grad(y_true, y_pred, *, target_idx, target_lambda, huber=False, huber_delta=1.0, batch_global=None):
    """dLoss/dy_pred of mlp_loss, [B, O]."""
    y = np.asarray(y_true, dtype=np.float64)
    p = np.asarray(y_pred, dtype=np.float64)
    B, O = y.shape
    Bg = B if batch_global is None else batch_global
    mask = (~np.all(y == 0.0, axis=-1)).astype(np.float64)
    r = y - p * mask[:, None]
    df = _huber_grad(r, huber_delta) if huber else 2.0 * r
    w = np.full(O, (1.0 - target_lambda) / (Bg * O))
    w[target_idx] += target_lambda / Bg
    return -mask[:, None] * df * w[None, :]


def dense_grads(x, dpred):
    """(dW, db) of Dense(O) for dLoss/dpred [B, O]."""
    x = np.asarray(x, dtype=np.float64)
    x = x.reshape(x.shape[0], -1)
    return x.T @ dpred, dpred.sum(axis=0)


def train_step(params, slots, x, y, it, *, target_idx, target_lambda, optimizer, lr, max_grad_norm,
               sgd_momentum=0.0, huber=False, huber_delta=1.0):
    """Train._train_step_point (train.py:178-199) of MLPLinearPointEstimate: forward, loss, gradients,
    tf.clip_by_global_norm, apply_gradients.  params = [W, b] (fp64), slots as lfm_oracle.zero_slots.
    Returns (new_params, loss, mse_0)."""
    W, b = params
    pred = dense_forward(x, W, b)
    kw = dict(target_idx=target_idx, target_lambda=target_lambda, huber=huber, huber_delta=huber_delta)
    loss, mse_0 = mlp_loss(y, pred, **kw)
    grads = list(dense_grads(x, mlp_loss_grad(y, pred, **kw)))
    if max_grad_norm > 0:
        grads, _ = orc.clip_by_global_norm(grads, max_grad_norm)
    new = orc.optimizer_update(optimizer, [W, b], grads, slots, lr, it, sgd_momentum=sgd_momentum)
    return new, loss, mse_0
