"""fp64 oracle of the training-window attributions (lfmq_influence_*, DESIGN.md section 5i).  TEST INFRASTRUCTURE ONLY.

TracIn at the checkpoint, restricted to the output head, with every dropout off: I_j(t, q) = -grad_theta l_t .
grad_theta f^j_q = -s_jq (~a_q . u_jt), where l_t is the training loss of a batch holding window t alone (B = 1, its own
mask counts, masked elements 0), ~a = (a; 1) is the head input with a one appended, u_jt = sum_tau G_j[t, tau] ~a_{t,tau}
with G = dl_t / d(head output j at [tau, target_idx]) (the variance head's pre-softplus activation), s_0 = 1 and s_1 =
sigmoid(pre_q), 0 where the 1e-6 variance floor binds."""
import numpy as np

import lfm_oracle as orc


def head_inputs(kind, P, x, *, num_layers=1, rnn_cell='lstm'):
    """(a [B,Ta,D], pred [B,Ta,O], var, pre) in fp64: kind 'point', 'uq' (var, pre [B,T,O]) or 'dense' (Ta = 1, a is the
    flattened window)."""
    x = np.asarray(x, dtype=np.float64)
    if kind == 'dense':
        a = x.reshape(x.shape[0], 1, -1)
        return a, a @ P[0] + P[1], None, None
    if kind == 'point':
        pred, (_, cur, _) = orc.forward(P, x, num_layers=num_layers, rnn_cell=rnn_cell)
        return cur, pred, None, None
    pred, var, (_, cur, _, _, pre) = orc.forward_uq(P, x, num_layers=num_layers, rnn_cell=rnn_cell)
    return cur, pred, var, pre


def _floor_gate(pre):
    return np.where(orc.softplus(pre) > orc.VAR_FLOOR, orc.sigmoid(pre), 0.0)


def window_grads(kind, pred, var, pre, y, *, target_idx, target_lambda, rnn_lambda=0.0, huber=False, huber_delta=1.0):
    """G [J,B,Ta]: each window's one-window loss gradient at column target_idx of the head outputs, 0 where masked."""
    y = np.asarray(y, dtype=np.float64)
    B = y.shape[0]
    if kind == 'dense':
        m = (~np.all(y == 0.0, axis=-1)).astype(np.float64)
        O = y.shape[-1]
        g = (1 - target_lambda) / O + target_lambda
        r = y[:, target_idx] - pred[:, 0, target_idx] * m
        df = (np.where(np.abs(r) > huber_delta, np.sign(r) * huber_delta, r) if huber else 2.0 * r)
        return (-m * g * df)[None, :, None]
    J = 2 if kind == 'uq' else 1
    G = np.zeros((J, B) + y.shape[1:2])
    for b in range(B):
        yb, pb = y[b:b + 1], pred[b:b + 1]
        m = ~np.all(yb == 0.0, axis=-1)[0]
        with np.errstate(divide='ignore', invalid='ignore'):
            if kind == 'point':
                _, _, dpred, _ = orc.loss_point_estimate(yb, pb, target_idx=target_idx, target_lambda=target_lambda,
                                                         rnn_lambda=rnn_lambda)
                G[0, b] = np.where(m, dpred[0, :, target_idx], 0.0)
            else:
                _, _, _, dpred, dvar = orc.loss_uq_estimate(yb, pb, var[b:b + 1], target_idx=target_idx,
                                                            target_lambda=target_lambda, rnn_lambda=rnn_lambda)
                G[0, b] = np.where(m, dpred[0, :, target_idx], 0.0)
                G[1, b] = np.where(m, dvar[0, :, target_idx] * _floor_gate(pre[b, :, target_idx]), 0.0)
    return G


def train_features(kind, P, x, y, **kw):
    """u [J,B,D+1]."""
    nl = dict(num_layers=kw.pop('num_layers', 1), rnn_cell=kw.pop('rnn_cell', 'lstm'))
    a, pred, var, pre = head_inputs(kind, P, x, **nl)
    G = window_grads(kind, pred, var, pre, y, **kw)
    at = np.concatenate([a, np.ones(a.shape[:2] + (1,))], axis=-1)
    return np.einsum('jbt,btd->jbd', G, at)


def query_features(kind, P, x, *, target_idx, **nl):
    """(a [B,D+1], s [J,B])."""
    a, pred, var, pre = head_inputs(kind, P, x, **nl)
    at = np.concatenate([a[:, -1], np.ones((a.shape[0], 1))], axis=-1)
    s = [np.ones(a.shape[0])]
    if kind == 'uq':
        s.append(_floor_gate(pre[:, -1, target_idx]))
    return at, np.stack(s)


def influence(a, u, s):
    """I [J,Nq,Nt] = -s_jq (a_q . u_jt) in fp64."""
    a, u, s = (np.asarray(v, dtype=np.float64) for v in (a, u, s))
    return -s[:, :, None] * np.einsum('qd,jtd->jqt', a, u)


def topk(I, K):
    """(pos_idx, pos_score, neg_idx, neg_score) [Nq,J,K] of I [J,Nq,Nt]: the K largest positive and the K most negative
    influences, ties to the lower index, padded with -1 / 0."""
    J, Nq, Nt = I.shape
    out = [np.full((Nq, J, K), -1, dtype=np.int64), np.zeros((Nq, J, K)),
           np.full((Nq, J, K), -1, dtype=np.int64), np.zeros((Nq, J, K))]
    idx = np.arange(Nt)
    for j in range(J):
        for q in range(Nq):
            row = I[j, q]
            for k, sign in ((0, 1.0), (2, -1.0)):
                sel = idx[sign * row > 0]
                order = np.lexsort((sel, -sign * row[sel]))[:K]
                out[k][q, j, :order.size] = sel[order]
                out[k + 1][q, j, :order.size] = row[sel[order]]
    return out
