"""fp64 oracle of permutation importance (lfmq_chain_permutation_importance, DESIGN.md section 5e).  TEST
INFRASTRUCTURE ONLY.  The bijection pi_{seed,g,r} in NumPy, the permuted copies, and the loss rows of every model kind
from the existing oracles' forwards and losses (oracle/lfm_oracle.py, tests/uq_chain_oracle.py, tests/dense_oracle.py),
with the dropout masks of window i keyed by its index (row0 = 0 over the whole held-out set)."""
import numpy as np

import dense_oracle as dno
import lfm_oracle as orc
import uq_chain_oracle as uco


def permutation(N, seed, group, repeat):
    """[pi(0), .., pi(N-1)]: a 4-round Feistel network on [0, 2^m) (m the smallest even integer >= 2 with 2^m >= N,
    halves of h = m / 2 bits), round j keyed by philox4x32_10(R, j, group, repeat; seed_lo, seed_hi)[0], cycle-walked
    from v = i until v < N."""
    m = 2
    while (1 << m) < N:
        m += 2
    h = np.uint32(m // 2)
    mask = np.uint32((1 << (m // 2)) - 1)
    k0, k1 = seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF
    out = np.empty(N, dtype=np.int64)
    todo = np.arange(N)
    v = np.arange(N, dtype=np.uint32)
    while todo.size:
        L, R = v >> h, v & mask
        for j in range(4):
            f = orc.philox4x32_10(R, np.uint32(j), np.uint32(group), np.uint32(repeat), k0, k1)[0]
            L, R = R, L ^ (f & mask)
        v = (L << h) | R
        done = v < N
        out[todo[done]] = v[done]
        todo, v = todo[~done], v[~done]
    return out


def permuted_copy(x, col_group, g, pi):
    """Copy (g, r) of x [N,T,F] or [N,T*F]: the columns c = t * F + f with col_group[c] == g from window pi(i)."""
    N = x.shape[0]
    flat = x.reshape(N, -1)
    out = flat.copy()
    cols = np.asarray(col_group) == g
    out[:, cols] = flat[pi][:, cols]
    return out.reshape(x.shape)


def importance(x, col_group, G, repeats, seed, loss_row):
    """out [1 + G * repeats, 3]: row 0 loss_row(x), row 1 + g * repeats + r loss_row(copy (g, r))."""
    N = x.shape[0]
    rows = [loss_row(x)]
    for g in range(G):
        for r in range(repeats):
            rows.append(loss_row(permuted_copy(x, col_group, g, permutation(N, seed, g, r))))
    return np.array(rows, dtype=np.float64)


def field_groups(T, F):
    return np.tile(np.arange(F, dtype=np.int32), T), F


def quarter_groups(T, F):
    return np.repeat(np.arange(T, dtype=np.int32), F), T


def point_loss(P, ys, weights, *, num_layers, rnn_cell, target_idx, target_lambda, rnn_lambda, bn_mean=None,
               bn_var=None):
    """{loss, mse_0, 0} of a point chain with dropout off (lfmq_loss, lfmq_chain_loss)."""
    ys = [np.asarray(y, dtype=np.float64) for y in ys]
    S = len(ys)

    def row(x):
        x = np.asarray(x, dtype=np.float64)
        if S == 1:
            preds = [orc.forward(P, x, num_layers=num_layers, rnn_cell=rnn_cell, bn_mean=bn_mean, bn_var=bn_var)[0]]
        else:
            preds = orc.forward_forecast(P, x, num_layers=num_layers, forecast_steps=S, rnn_cell=rnn_cell)[0]
        loss, mse = orc.loss_forecast(ys, preds, weights, target_idx=target_idx, target_lambda=target_lambda,
                                      rnn_lambda=rnn_lambda)[:2]
        return [loss, mse, 0.0]
    return row


def uq_loss(P, ys, weights, *, num_layers, rnn_cell, dropout, recurrent_dropout, seed, step, target_idx,
            target_lambda, rnn_lambda):
    """{uq_loss, uq_loss_last_tar, mse} of a uq chain with its dropout on, window i's masks keyed by row i at `step`."""
    ys = [np.asarray(y, dtype=np.float64) for y in ys]

    def row(x):
        preds, vars_, _ = uco.forward(P, np.asarray(x, dtype=np.float64), num_layers=num_layers, forecast_steps=len(ys),
                                      dropout=dropout, recurrent_dropout=recurrent_dropout, seed=seed, step=step,
                                      row0=0, rnn_cell=rnn_cell)
        return list(uco.loss(ys, preds, vars_, weights, target_idx=target_idx, target_lambda=target_lambda,
                             rnn_lambda=rnn_lambda)[:3])
    return row


def dense_loss(W, b, y, *, target_idx, target_lambda):
    """{loss, mse_0, 0} of the linear model, the MLP branch's MSE form (lfmq_loss on a dense handle)."""
    y = np.asarray(y, dtype=np.float64)

    def row(x):
        pred = dno.dense_forward(np.asarray(x, dtype=np.float64), W, b)
        return list(dno.mlp_loss(y, pred, target_idx=target_idx, target_lambda=target_lambda)) + [0.0]
    return row

