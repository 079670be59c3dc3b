"""CPU oracle of RNNUqRangeEstimate with forecast_steps >= 1 (reference
models/uq_range_estimate/rnn_uq_range_estimate.py:62-157, model_utils/losses.py:137-178, train.py:201-225).  TEST
INFRASTRUCTURE ONLY.  Composes the building blocks of oracle/lfm_oracle.py (the recurrent trunk, the uq heads and loss,
the single-step uq backward, the step tail) into the multi-step uq graph; forecast_steps = 1 is exactly
lfm_oracle.forward_uq / loss_uq_estimate / backward_uq."""
import numpy as np

import lfm_oracle as orc


def param_names(num_layers, forecast_steps, rnn_cell='lstm'):
    """trainable_variables order: the single-step uq model's (lfm_oracle.param_names(..., uq=True)), then per extra step
    s one recurrent layer numbered on from the trunk (:129-147), its BatchNormalization, OUTPUT_TARGET_{s+1} and
    OUTPUT_VARIANCE_{s+1} (:152-155)."""
    names = orc.param_names(num_layers, rnn_cell, uq=True)
    for s in range(1, forecast_steps):
        l = num_layers + s
        names += ['%s_%d/kernel' % (rnn_cell, l), '%s_%d/recurrent_kernel' % (rnn_cell, l), '%s_%d/bias' % (rnn_cell, l),
                  'batch_normalization_%d/gamma' % (l - 1), 'batch_normalization_%d/beta' % (l - 1)]
        for head in ('OUTPUT_TARGET_%d' % (s + 1), 'OUTPUT_VARIANCE_%d' % (s + 1)):
            names += [head + '/kernel', head + '/bias']
    return names


def init_params(num_layers, n_inputs, n_outputs, num_hidden, forecast_steps, init_scale=1.0, seed=521,
                dtype=np.float32, rnn_cell='lstm'):
    out = orc.init_params(num_layers, n_inputs, n_outputs, num_hidden, init_scale, seed, dtype, rnn_cell, uq=True)
    for s in range(1, forecast_steps):       # one recurrent layer on the raw feature width + its two heads
        out += orc.init_params(1, n_inputs, n_outputs, num_hidden, init_scale, seed + 7 * s, dtype, rnn_cell, uq=True)
    return out


def forward(params, x, *, num_layers, forecast_steps, dropout=0.0, recurrent_dropout=0.0, seed=0, step=0, row0=0,
            rnn_cell='lstm'):
    """model(inp) -> ([tar_1 .. tar_S], [var_1 .. var_S]) and the cache for ``backward``.  Stage 0 is
    lfm_oracle.forward_uq; stage s >= 1 runs one more recurrent layer + BatchNormalization + Dropout (both dropouts
    always on, ``training=True`` at :137,147) and OUTPUT_TARGET_{s+1} / OUTPUT_VARIANCE_{s+1} (:152-155) over the window
    shifted by one, the appended step built from the previous TARGET output (``outputs[-2]``, :118) and the aux features
    of the last original step (:71,121).  Dropout streams continue the trunk's layer numbering (layer num_layers + s - 1),
    as in lfm_oracle.forward_forecast."""
    O = params[5 * num_layers].shape[1]
    n0 = 5 * num_layers + 4
    p0, v0, fc0 = orc.forward_uq(params[:n0], x, num_layers=num_layers, dropout=dropout,
                                 recurrent_dropout=recurrent_dropout, seed=seed, step=step, row0=row0,
                                 rnn_cell=rnn_cell)
    preds, vars_, caches = [p0], [v0], [fc0]
    aux = x[:, -1:, O:]
    prev_input = x
    for s in range(1, forecast_steps):
        new_step = np.concatenate([preds[-1][:, -1:, :], aux], axis=2)
        cur_input = np.concatenate([prev_input, new_step], axis=1)[:, 1:, :]
        prev_input = cur_input
        ps = params[n0 + 9 * (s - 1):n0 + 9 * s]
        cur, lc = orc._trunk(ps[:5], cur_input, num_layers=1, dropout=dropout, recurrent_dropout=recurrent_dropout,
                             training=True, seed=seed, step=step, row0=row0, bn_mean=None, bn_var=None,
                             rnn_cell=rnn_cell, layer0=num_layers + s - 1)
        Wt, bt, Wv, bv = ps[5:9]
        a = cur @ Wv + bv
        preds.append(cur @ Wt + bt)
        vars_.append(np.maximum(orc.softplus(a), x.dtype.type(orc.VAR_FLOOR)))
        caches.append((lc, cur, Wt, Wv, a))
    return preds, vars_, (caches, num_layers, forecast_steps, O)


def loss(y_trues, preds, vars_, weights, **kw):
    """Losses.weight_adjusted_uq_loss over the forecast steps (losses.py:159-177): every step's (uq_loss,
    uq_loss_last_tar, mse) with its own mask counts, each summed with ``weights``.  Returns the three sums and the
    weighted dLoss/dpred_s, dLoss/dvar_s of sum_s w_s uq_loss_s."""
    tot = tot_last = tot_mse = 0.0
    dpreds, dvars = [], []
    for y, p, v, w in zip(y_trues, preds, vars_, weights):
        l, u, m, dp, dv = orc.loss_uq_estimate(y.astype(p.dtype), p, v, **kw)
        tot += w * l
        tot_last += w * u
        tot_mse += w * m
        dpreds.append(w * dp)
        dvars.append(w * dv)
    return tot, tot_last, tot_mse, dpreds, dvars


def backward(dpreds, dvars, fcache, *, rnn_cell='lstm'):
    """tape.gradient(uq_loss, trainable_variables) (train.py:218) in ``param_names`` order.  Each stage's variance head
    passes its gradient as lfm_oracle.backward_uq does; the input gradient of stage s flows into the last time step of
    the earlier TARGET predictions only (variances never feed forward)."""
    caches, num_layers, S, O = fcache
    dpreds = [d.copy() for d in dpreds]
    B, T, _ = dpreds[0].shape
    extra = []
    for s in range(S - 1, 0, -1):
        lc, y_last, Wt, Wv, a = caches[s]
        dp = dpreds[s]
        da = dvars[s] * np.where(orc.softplus(a) > orc.VAR_FLOOR, orc.sigmoid(a), 0.0)
        H = Wt.shape[0]
        y2 = y_last.reshape(B * T, H)
        g = [None] * 9
        g[5] = y2.T @ dp.reshape(B * T, O)
        g[6] = dp.reshape(B * T, O).sum(axis=0)
        g[7] = y2.T @ da.reshape(B * T, O)
        g[8] = da.reshape(B * T, O).sum(axis=0)
        dy = dp @ Wt.T + da @ Wv.T
        (lcache, hs, mean, inv, gamma, dmask) = lc[0]
        if dmask is not None:
            dy = dy * dmask
        g[3] = np.sum(dy * (hs - mean) * inv, axis=(0, 1))
        g[4] = np.sum(dy, axis=(0, 1))
        cell_bwd = orc.lstm_backward if rnn_cell == 'lstm' else orc.gru_backward
        dW, dU, db, dx = cell_bwd(dy * gamma * inv, lcache, need_dx=True)
        g[0], g[1], g[2] = dW, dU, db
        for j in range(s):                       # appended steps inside this window
            dpreds[s - 1 - j][:, -1, :] += dx[:, T - 1 - j, :O]
        extra = g + extra
    g0 = orc.backward_uq(dpreds[0], dvars[0], caches[0], num_layers=num_layers, rnn_cell=rnn_cell)
    return g0 + extra


def train_step(params, slots, x, ys, it, cfg, *, row0=0, lr):
    """Train._train_step_uq_range (train.py:201-225) of the multi-step graph: forward, the weighted uq loss, its
    gradients, clip_by_global_norm over every stage's variables, the optimizer, MaxNorm on every recurrent kernel.
    Returns (new_params, mse, uq_loss, grads_before_clip, grad_norm, uq_loss_last_tar), the sums weighted with
    cfg['forecast_steps_weights'] -- the reference's step returns (uq_loss_last_tar, mse)."""
    L, S = cfg['num_layers'], cfg['forecast_steps']
    cell = cfg.get('rnn_cell', 'lstm')
    preds, vars_, fc = forward(params, x, num_layers=L, forecast_steps=S, dropout=cfg.get('dropout', 0.0),
                               recurrent_dropout=cfg.get('recurrent_dropout', 0.0), seed=cfg.get('seed', 0), step=it,
                               row0=row0, rnn_cell=cell)
    uq, uq_last, mse, dpreds, dvars = loss(ys, preds, vars_, cfg['forecast_steps_weights'], target_idx=cfg['target_idx'],
                                           target_lambda=cfg['target_lambda'], rnn_lambda=cfg['rnn_lambda'])
    grads = backward(dpreds, dvars, fc, rnn_cell=cell)
    raw = [g.copy() for g in grads]
    gn = None
    if cfg.get('max_grad_norm', 0.0) > 0:
        grads, gn = orc.clip_by_global_norm(grads, cfg['max_grad_norm'])
    new = orc.optimizer_update(cfg.get('optimizer', 'Adadelta'), params, grads, slots, lr, it,
                               sgd_momentum=cfg.get('sgd_momentum', 0.0))
    for k in [5 * l for l in range(L)] + [5 * L + 4 + 9 * (s - 1) for s in range(1, S)]:
        new[k] = orc.max_norm_constraint(new[k], cfg.get('max_norm', 3))
    return new, mse, uq, raw, gn, uq_last
