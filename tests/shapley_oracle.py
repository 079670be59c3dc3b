"""fp64 oracle of the Shapley attributions (lfmq_chain_shapley, DESIGN.md section 5f).  TEST INFRASTRUCTURE ONLY.  The
draws (donor windows and group orderings, from the bijection of tests/importance_oracle.py), the coalition copies and
the estimator, over the explained outputs of every model kind from the existing oracles' forwards
(oracle/lfm_oracle.py, tests/uq_chain_oracle.py, tests/dense_oracle.py), with the dropout masks of window i in sample m
keyed by row m * N + i."""
import numpy as np

import dense_oracle as dno
import importance_oracle as imo
import lfm_oracle as orc
import uq_chain_oracle as uco

DONOR_KEY, ORDER_KEY = 0x40000000, 0x40000001


def draws(N, G, samples, seed):
    """(donors, orders): donors[p] [N] the donor window of every window in pair p, orders[m] [G] the group ordering of
    sample m (an odd sample reverses its partner's)."""
    donors = [imo.permutation(N, seed, DONOR_KEY, p) for p in range((samples + 1) // 2)]
    orders = []
    for m in range(samples):
        orders.append(imo.permutation(G, seed, ORDER_KEY, m // 2) if m % 2 == 0 else orders[m - 1][::-1].copy())
    return donors, orders


def coalition_copy(x, col_group, rank, k, donor):
    """Copy (m, k) of x [N,T,F] or [N,T*F]: the columns whose group ranks >= k (rank [G]) from window donor[i]."""
    N = x.shape[0]
    flat = x.reshape(N, -1)
    take = np.asarray(rank)[np.asarray(col_group)] >= k
    return np.where(take[None, :], flat[donor], flat).reshape(x.shape)


def shapley(x, col_group, G, samples, seed, outputs):
    """(phi [N,K,G], f_x [N,K], f_bg [N,K]) in fp64.  outputs(x_copy, m) -> [N,K]: the explained outputs of sample m."""
    N = x.shape[0]
    donors, orders = draws(N, G, samples, seed)
    phi = f_x = f_bg = None
    for m in range(samples):
        o = orders[m]
        rank = np.empty(G, dtype=np.int64)
        rank[o] = np.arange(G)
        prev = None
        for k in range(G + 1):
            v = np.asarray(outputs(coalition_copy(x, col_group, rank, k, donors[m // 2]), m), dtype=np.float64)
            if phi is None:
                K = v.shape[1]
                phi, f_x, f_bg = np.zeros((N, K, G)), np.zeros((N, K)), np.zeros((N, K))
            if k == 0:
                f_bg += v
            else:
                phi[:, :, o[k - 1]] += v - prev
            if k == G:
                f_x += v
            prev = v
    return phi / samples, f_x / samples, f_bg / samples


def point_outputs(P, *, num_layers, rnn_cell, forecast_steps, target_idx):
    """pred_s[:, T-1, target_idx] of every stage of a point chain, dropout off."""
    def f(x, m):
        x = np.asarray(x, dtype=np.float64)
        if forecast_steps == 1:
            preds = [orc.forward(P, x, num_layers=num_layers, rnn_cell=rnn_cell)[0]]
        else:
            preds = orc.forward_forecast(P, x, num_layers=num_layers, forecast_steps=forecast_steps,
                                         rnn_cell=rnn_cell)[0]
        return np.stack([p[:, -1, target_idx] for p in preds], axis=1)
    return f


def uq_outputs(P, *, num_layers, rnn_cell, forecast_steps, dropout, recurrent_dropout, seed, step, target_idx):
    """tar_1, var_1, .., tar_S, var_S at [:, T-1, target_idx] of a uq chain, window i of sample m keyed by row
    m * N + i at `step`."""
    def f(x, m):
        x = np.asarray(x, dtype=np.float64)
        preds, vars_, _ = uco.forward(P, x, num_layers=num_layers, forecast_steps=forecast_steps, dropout=dropout,
                                      recurrent_dropout=recurrent_dropout, seed=seed, step=step, row0=m * x.shape[0],
                                      rnn_cell=rnn_cell)
        return np.stack([a[:, -1, target_idx] for pv in zip(preds, vars_) for a in pv], axis=1)
    return f


def dense_outputs(W, b, *, target_idx):
    """pred[:, target_idx] of the linear model over the flattened window."""
    def f(x, m):
        return dno.dense_forward(np.asarray(x, dtype=np.float64), W, b)[:, target_idx:target_idx + 1]
    return f
