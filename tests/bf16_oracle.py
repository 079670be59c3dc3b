"""fp64 restatement of the bf16 tensor-core paths that rounds to bf16 exactly where the kernels round.  TEST-SIDE ONLY.

The fp64 oracle (oracle/lfm_oracle.py) is the model; this file is the model *as the LFMQ_PREC_BF16 kernels evaluate it*:
the same graph (L layers of LSTM or GRU, BatchNormalization with moving statistics, Dropout, recurrent dropout with the
oracle's Philox masks, the head, the weighted-MSE loss, BPTT), in fp64, with ``rb`` (fp32 -> bf16, round to nearest
even) applied to every tensor a kernel stores or feeds to a tensor core as bf16.  What is left between it and a kernel
is (1) fp32 accumulation order and (2) the approximate nonlinearities: ``tanh.approx.f32`` in the forward cell updates
(the sigmoid is written as 0.5 tanh(z/2) + 0.5, the identity the kernels use, but its tanh is the exact one here) and
``tanh.approx.bf16x2`` for tanh(c) in the backward gate algebra (modelled as rb(tanh(c))).  Neither is modelled.

Rounding plans, one per path (file:line in lfm_quant_b200/csrc):

``cluster`` -- lstm_tc.cu, H = 256, L = 1, LSTM, no recurrent dropout
  * x_t                               xh_fill_x_kernel, lstm_tc.cu:91-111 (xh cols 256..)
  * h_t, the next step's A operand    lstm_tc.cu:378-380 (xh row t+1); the head and the dW/dU GEMM read the same bf16 h
  * W, U as packed (x 0.5 on i|f|o)   pack_weights_body, lstm_tc.cu:117-143; the 0.5 is exact, the bias stays fp32
  * saved gates i|f|g|o, cell states  lstm_tc.cu:290-310 (save_chunk), :377 (held chunks)
  * head without Dropout: bf16(Wo gamma inv) for pred and for dLoss/dh (WoTp / WoSp, pack_head_body lstm_tc.cu:621-635);
    bias bo + sum_j (beta - gamma mean inv)_j Wo_j in fp32 (:637-653); dLoss/dpred tile bf16 (head_tc_kernel
    lstm_tc.cu:824-830), dbo from the fp32 dLoss/dpred (:817); dWo, dgamma, dbeta folded from h^T bf16(dpred) and the
    fp32 column sums (head_fold_kernel lstm_tc.cu:984-1007)
  * head with Dropout (head_rows_kernel lstm_tc.cu:441-608): everything fp32 on the bf16 h, dLoss/dh stored as bf16
    (dhout, :575); dWo from the fp32 Dropout(BN(h)) and fp32 dLoss/dpred (head_wgrad_kernel :883-951)
  * backward: U as packed (Ubk, pack_ubk_body :657-665); dLoss/dh_{t-1} = dz_t U^T reduce-scattered over the 4 CTAs of
    a cluster: the own 64-unit slice stays fp32, the three foreign partial slices arrive as bf16 (lstm_tc.cu:1243-1250,
    1328-1330); the FUSED head term dpred (Wo gamma inv)^T joins the own slice in fp32 (:1053-1055, :1311)
  * gate algebra in packed bf16x2 (lstm_tc.cu:1259-1273): dh = bf16(dhout + bf16(rec)) (FUSED: bf16(rec)),
    tc = bf16(tanh c), every bf16x2 mul / fma rounds once; the carried dLoss/dc stays fp32; dz stored bf16
  * dW, dU, db = bf16 xh^T bf16 dz over all rows, fp32 accumulation (wgrad GEMM, lstm_tc.cu:1345-1366)

``general`` -- rnn_tc.cu, any H multiple of 64 up to 512, any L, both dropouts; also GRU and UQ forward-only handles
  * x_t cast to bf16 (in[0])          gcast_x_kernel rnn_tc.cu:635-662
  * h_t (hseq) and the masked h_t * mask (hmseq, recurrent dropout): the A operand is the masked copy rounded once
                                      epi_fwd rnn_tc.cu:218-233, epi_gru_fwd :296-310 (GRU carries h in fp32, :295)
  * W, U as packed (x 0.5 on the sigmoid gates, exact); the backward's Ub = bf16(U), Wb = bf16(W)
                                      gpack_kernel rnn_tc.cu:683-732
  * layer inputs in[l] = bf16(Dropout(BN(bf16 h))) for l > 0 and the head input in[L]   gbn_drop_fwd_kernel :763-803
  * saved gates i|f|g|o and cell states                                               epi_fwd :234-241
  * head: pred = bf16(y) bf16(Wo) + bo (fp32 bias), gpack_head_kernel :737-748, epi_head :429; dLoss/dpred stored
    bf16 (hdpb, :439-444), dbo from fp32 dpred (:445); dy = bf16(bf16(dpred) bf16(Wo)^T) (EPI_STORE :394-402);
    dWo = bf16(y)^T bf16(dpred)
  * UQ heads: [pred | var] = bf16(y) [bf16(Wo) | bf16(Wv)] + fp32 biases, softplus floor  epi_head_uq :453-468
  * BN/Dropout backward: fp32 on bf16 dy and bf16 h, dhout = bf16(d gamma inv)           gbn_drop_bwd_kernel :808-868
  * backward step: rec = dz_{t+1} bf16(U)^T times the recurrent mask, rounded once; then the same bf16x2 gate algebra as
    the cluster path (epi_bwd :352-388), dz stored bf16
  * dW = bf16(in)^T dz, dU = bf16(masked h_{t-1})^T dz, db = colsum(bf16 dz) (gen_wgrad :1368-1382, gcolsum :885-909);
    dLoss/d(input) of layers above the first = bf16(dz bf16(W)^T) (EPI_STORE, :1603-1620)

With ``rb`` replaced by the identity each plan is the fp64 oracle's own arithmetic (tests/test_bf16_oracle_host.py
holds it to orc.forward / orc.backward / orc.forward_uq to 1e-12).
"""
from __future__ import annotations

import numpy as np

import lfm_oracle as orc


def rb(a):
    """fp32 -> bf16, round to nearest even, on the uint32 view of the fp32 value; returned as float64.  fp64 input is
    first rounded to fp32 (the kernels compute in fp32).  Overflow -> +-inf; NaN -> 0x7FFF, the canonical NaN of
    cvt.rn.bf16.f32 (NaN payloads are not portable: torch's CPU conversion gives 0xFFFF)."""
    shape = np.shape(a)
    f = np.ascontiguousarray(np.asarray(a, dtype=np.float32)).reshape(-1)
    u = f.view(np.uint32).astype(np.uint64)
    r = (u + np.uint64(0x7FFF) + ((u >> np.uint64(16)) & np.uint64(1))) & np.uint64(0xFFFF0000)
    r = np.where(np.isnan(f), np.uint64(0x7FFF0000), r).astype(np.uint32)
    return r.view(np.float32).astype(np.float64).reshape(shape)


def identity(a):
    return np.asarray(a, dtype=np.float64)


PATHS = ('cluster', 'general')


class Plan:
    """The rounding plan of one tensor-core path.  ``r`` is rb, or the identity for the fp64 oracle's arithmetic."""

    def __init__(self, path, r=rb):
        assert path in PATHS, path
        self.path = path
        self.r = r


def _sig(z):
    return 0.5 * np.tanh(0.5 * z) + 0.5        # the kernels' sigmoid (fwd_gates lstm_tc.cu:177-186, epi_fwd :207-211)


def _lstm_fwd(p, inp, W, U, b, rmask):
    r = p.r
    B, T, _ = inp.shape
    H = U.shape[0]
    Wr, Ur = r(W), r(U)
    c = np.zeros((B, H))
    hA = np.zeros((B, H))
    hs, hAs, cs = np.empty((B, T, H)), np.empty((B, T, H)), np.empty((B, T, H))
    gates = np.empty((B, T, 4 * H))
    for t in range(T):
        hAs[:, t] = hA
        z = inp[:, t] @ Wr + hA @ Ur + b
        i, f = _sig(z[:, :H]), _sig(z[:, H:2 * H])
        g, o = np.tanh(z[:, 2 * H:3 * H]), _sig(z[:, 3 * H:])
        c = f * c + i * g
        h = o * np.tanh(c)
        hs[:, t] = r(h)
        hA = hs[:, t] if rmask is None else r(h * rmask)
        gates[:, t] = r(np.concatenate([i, f, g, o], axis=1))
        cs[:, t] = r(c)
    return dict(hs=hs, hA=hAs, gates=gates, cs=cs)


def _gru_fwd(p, inp, W, U, b2, rmask):
    r = p.r
    B, T, _ = inp.shape
    H = U.shape[0]
    Wr, Ur = r(W), r(U)
    h = np.zeros((B, H))
    hA = np.zeros((B, H))
    hs = np.empty((B, T, H))
    for t in range(T):
        xz = inp[:, t] @ Wr
        hz = hA @ Ur
        z = _sig(xz[:, :H] + hz[:, :H] + (b2[0, :H] + b2[1, :H]))
        rr = _sig(xz[:, H:2 * H] + hz[:, H:2 * H] + (b2[0, H:2 * H] + b2[1, H:2 * H]))
        n = np.tanh(xz[:, 2 * H:] + b2[0, 2 * H:] + rr * (hz[:, 2 * H:] + b2[1, 2 * H:]))
        h = z * h + (1.0 - z) * n              # carried in fp32, unrounded (epi_gru_fwd rnn_tc.cu:293-295)
        hs[:, t] = r(h)
        hA = hs[:, t] if rmask is None else r(h * rmask)
    return dict(hs=hs)


def forward(p, params, x, *, num_layers, dropout=0.0, recurrent_dropout=0.0, training=False, seed=0, step=0, row0=0,
            bn_mean=None, bn_var=None, rnn_cell='lstm', uq=False):
    """orc.forward (orc.forward_uq with ``uq``) as path ``p.path`` evaluates it.  Returns (preds, cache) or
    (pred, var, cache).  ``training``: Dropout / recurrent dropout active (uq: always, as orc.forward_uq)."""
    L = num_layers
    training = training or uq
    if p.path == 'cluster':
        assert L == 1 and rnn_cell == 'lstm' and not uq and not (training and recurrent_dropout > 0)
    r = p.r
    B, T, _ = x.shape
    cur = r(x)
    layers = []
    for l in range(L):
        W, U, b, gamma, beta = params[5 * l:5 * l + 5]
        H = U.shape[0]
        mean = np.zeros(H) if bn_mean is None else np.asarray(bn_mean[l], dtype=np.float64)
        var = np.ones(H) if bn_var is None else np.asarray(bn_var[l], dtype=np.float64)
        rmask = None
        if training and recurrent_dropout > 0.0:
            rmask = orc.dropout_mask(seed, step, 2 * l + 1, row0, B, H, recurrent_dropout)
        st = (_lstm_fwd if rnn_cell == 'lstm' else _gru_fwd)(p, cur, W, U, b, rmask)
        inv = 1.0 / np.sqrt(var + orc.BN_EPS)
        y = gamma * (st['hs'] - mean) * inv + beta
        dmask = None
        if training and dropout > 0.0:
            dmask = orc.dropout_mask(seed, step, 2 * l, row0, B, T * H, dropout).reshape(B, T, H)
            y = y * dmask
        layers.append(dict(st, inp=cur, W=W, U=U, gamma=gamma, beta=beta, mean=mean, inv=inv, dmask=dmask,
                           rmask=rmask))
        cur = r(y) if p.path == 'general' else y
    top = layers[-1]
    head = 'general'
    if p.path == 'cluster':
        head = 'rows' if top['dmask'] is not None else 'fold'
    cache = dict(layers=layers, y=cur, params=params, L=L, head=head)
    if uq:
        Wt, bt, Wv, bv = params[5 * L:5 * L + 4]
        pred = cur @ r(Wt) + bt
        var = np.maximum(orc.softplus(cur @ r(Wv) + bv), orc.VAR_FLOOR)
        return pred, var, cache
    Wo, bo = params[5 * L], params[5 * L + 1]
    if head == 'fold':
        a = top['gamma'] * top['inv']
        c = top['beta'] - top['gamma'] * top['mean'] * top['inv']
        preds = top['hs'] @ r(a[:, None] * Wo) + (bo + c @ Wo)
    elif head == 'rows':
        preds = cur @ Wo + bo
    else:
        preds = cur @ r(Wo) + bo
    return preds, cache


def _exchange(p, dz, Ur, head):
    """The cluster backward's dLoss/dh_{t-1}: per 64-unit slice q, the own partial (rank q) in fp32 plus the three
    foreign partials as bf16, plus (FUSED) the head term in fp32."""
    B = dz.shape[0]
    H = Ur.shape[0]
    dz4 = dz.reshape(B, 4, 4, 64)          # gate, rank, unit of the rank's slice
    U4 = Ur.reshape(H, 4, 4, 64)
    slot = np.arange(H) // 64
    rec = np.zeros((B, H)) if head is None else head.copy()
    for rank in range(4):
        P = dz4[:, :, rank].reshape(B, 256) @ U4[:, :, rank].reshape(H, 256).T
        rec += np.where(slot == rank, P, p.r(P))
    return rec


def _lstm_bwd(p, ly, dhout, head_dh, need_dx):
    r = p.r
    gates, cs = ly['gates'], ly['cs']
    B, T, H = cs.shape
    Ur = r(ly['U'])
    rmask = ly['rmask']
    dc = np.zeros((B, H))
    dz_all = np.empty((B, T, 4 * H))
    dz_next = None
    for t in range(T - 1, -1, -1):
        i, f = gates[:, t, :H], gates[:, t, H:2 * H]
        g, o = gates[:, t, 2 * H:3 * H], gates[:, t, 3 * H:]
        ct = cs[:, t]
        cp = cs[:, t - 1] if t > 0 else np.zeros((B, H))
        if p.path == 'cluster':
            hd = None if head_dh is None else head_dh[:, t]
            rec = _exchange(p, dz_next, Ur, hd) if dz_next is not None else (np.zeros((B, H)) if hd is None else hd)
        else:
            rec = np.zeros((B, H)) if dz_next is None else dz_next @ Ur.T
            if rmask is not None:
                rec = rec * rmask
        dh = r(rec) if dhout is None else r(dhout[:, t] + r(rec))
        tc = r(np.tanh(ct))
        omtc = r(1.0 - tc * tc)
        t1 = r(r(dh * o) * omtc)
        dcn = dc + t1
        dc = dcn * f
        dcn2 = r(dcn)
        zi = r(dcn2 * r(g * r(i - i * i)))
        zf = r(dcn2 * r(cp * r(f - f * f)))
        zg = r(dcn2 * r(i * r(1.0 - g * g)))
        zo = r(r(dh * tc) * r(o - o * o))
        dz_next = np.concatenate([zi, zf, zg, zo], axis=1)
        dz_all[:, t] = dz_next
    inp = ly['inp']
    dz2 = dz_all.reshape(B * T, 4 * H)
    dW = inp.reshape(B * T, -1).T @ dz2
    dU = ly['hA'].reshape(B * T, H).T @ dz2
    db = dz2.sum(axis=0)
    dx = r(dz_all @ r(ly['W']).T) if need_dx else None
    return dW, dU, db, dx


def backward(p, dpred, cache):
    """Gradients in Keras order (orc.backward), as path ``p.path`` computes them."""
    r = p.r
    layers, y, params, L, head = cache['layers'], cache['y'], cache['params'], cache['L'], cache['head']
    Wo = params[5 * L]
    B, T, O = dpred.shape
    H = Wo.shape[0]
    grads = [None] * (5 * L + 2)
    grads[5 * L + 1] = dpred.sum(axis=(0, 1))
    head_dh = None
    dy = None
    top = layers[-1]
    if head == 'general':
        dpb = r(dpred)
        grads[5 * L] = y.reshape(-1, H).T @ dpb.reshape(-1, O)
        dy = r(dpb @ r(Wo).T)
    elif head == 'rows':
        grads[5 * L] = y.reshape(-1, H).T @ dpred.reshape(-1, O)
        dy = dpred @ Wo.T
    else:
        dpb = r(dpred)
        a = top['gamma'] * top['inv']
        c = top['beta'] - top['gamma'] * top['mean'] * top['inv']
        G = top['hs'].reshape(-1, H).T @ dpb.reshape(-1, O)
        csum = dpred.sum(axis=(0, 1))
        grads[5 * L] = a[:, None] * G + c[:, None] * csum[None, :]
        dbeta = Wo @ csum
        grads[5 * L - 1] = dbeta
        grads[5 * L - 2] = top['inv'] * ((Wo * G).sum(axis=1) - top['mean'] * dbeta)
        head_dh = dpb @ r(a[:, None] * Wo).T
    for l in range(L - 1, -1, -1):
        ly = layers[l]
        dhout = None
        if dy is not None:
            d = dy if ly['dmask'] is None else dy * ly['dmask']
            grads[5 * l + 3] = np.sum(d * (ly['hs'] - ly['mean']) * ly['inv'], axis=(0, 1))
            grads[5 * l + 4] = np.sum(d, axis=(0, 1))
            dhout = r(d * (ly['gamma'] * ly['inv']))
        dW, dU, db, dx = _lstm_bwd(p, ly, dhout, head_dh, need_dx=l > 0)
        grads[5 * l], grads[5 * l + 1], grads[5 * l + 2] = dW, dU, db
        dy = dx
    return grads


def train_step(p, params, slots, x, y, it, cfg, lr, bn_mean=None, bn_var=None, row0=0):
    """orc.train_step (point estimate) with the forward and backward of path ``p.path``; the optimizer, clip and MaxNorm
    run in fp64 as in the oracle.  Returns (new_params, mse_0, loss, grads_before_clip)."""
    L = cfg['num_layers']
    preds, fc = forward(p, params, x, num_layers=L, dropout=cfg.get('dropout', 0.0),
                        recurrent_dropout=cfg.get('recurrent_dropout', 0.0), training=cfg.get('train', True),
                        seed=cfg.get('seed', 0), step=it, row0=row0, bn_mean=bn_mean, bn_var=bn_var)
    loss, mse, dpred, _ = orc.loss_point_estimate(np.asarray(y, dtype=np.float64), preds, target_idx=cfg['target_idx'],
                                                  target_lambda=cfg['target_lambda'], rnn_lambda=cfg['rnn_lambda'])
    grads = backward(p, dpred, fc)
    raw = [g.copy() for g in grads]
    if cfg.get('max_grad_norm', 0.0) > 0:
        grads, _ = orc.clip_by_global_norm(grads, cfg['max_grad_norm'])
    new = orc.optimizer_update(cfg.get('optimizer', 'Adadelta'), params, grads, slots, lr, it,
                               sgd_momentum=cfg.get('sgd_momentum', 0.0))
    for l in range(L):
        new[5 * l] = orc.max_norm_constraint(new[5 * l], cfg.get('max_norm', 3))
    return new, mse, loss, raw
