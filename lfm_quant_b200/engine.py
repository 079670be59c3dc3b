"""Thin Python owners of the native handles: one handle engine per handle (ForecasterEngine, DenseEngine), and
ForecastChainEngine, the engine of every model object, over one handle or a forecast chain of them.

PyTorch is used for device allocation, streams and torch.distributed only; every piece of arithmetic
happens in lfm_quant_b200/_lfmq.so through the C-ABI of include/lfmq.h.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _native as N

# config.precision -> LFMQ_PREC_*.  'tf32' runs the fp32 step with its GEMMs on tensor cores (tf32 operands, fp32
# accumulation); dense handles refuse everything but 'fp32' in the library.
PRECISIONS = {'fp32': N.PREC_FP32, 'bf16': N.PREC_BF16, 'bf16x3': N.PREC_BF16X3, 'tf32': N.PREC_TF32}


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _scratch(owner, key, work_bytes, *args):
    """The caller scratch of one analysis: a device uint8 buffer of at least the bytes its lfmq_*_work_bytes query
    reports for args, kept on `owner` under `key` and grown as needed."""
    n = C.c_uint64(0)
    N.check(work_bytes(*args, C.byref(n)))
    bufs = owner.__dict__.setdefault('_scratch_bufs', {})
    if key not in bufs or bufs[key].numel() < n.value:
        bufs[key] = torch.empty(max(n.value, 1), dtype=torch.uint8, device=owner.device)
    return bufs[key]


class _TopkScratch(object):
    """Keeps the scratch of influence_topk, nearest_topk and conformal_calibrate between calls without an engine."""

    def __init__(self, device):
        self.device = device


def influence_topk(a, u, s, k, owner=None):
    """lfmq_influence_topk: for the query features a [Nq,D1], s [J,Nq] and the pool's training features u [J,Nt,D1] (all
    device fp32), the device tensors (pos_idx, pos_score, neg_idx, neg_score) [Nq,J,K] -- the K training windows with the
    largest positive and the most negative influences, index -1 and score 0 where fewer have that sign -- and total
    [Nq,J], the summed influence of the whole pool.  `owner` (an engine) keeps the scratch between calls."""
    a, u, s = a.contiguous(), u.contiguous(), s.contiguous()
    J, Nt, D1 = u.shape
    Nq, K = a.shape[0], int(k)
    assert a.shape == (Nq, D1) and s.shape == (J, Nq), (tuple(a.shape), tuple(u.shape), tuple(s.shape))
    lib = N.load()
    work = _scratch(owner if owner is not None else _TopkScratch(a.device), 'influence_topk',
                    lib.lfmq_influence_topk_work_bytes, Nq, Nt, D1, J, K)
    pos_idx = torch.empty(Nq, J, K, dtype=torch.int32, device=a.device)
    neg_idx = torch.empty_like(pos_idx)
    pos_score = torch.empty(Nq, J, K, dtype=torch.float32, device=a.device)
    neg_score = torch.empty_like(pos_score)
    total = torch.empty(Nq, J, dtype=torch.float32, device=a.device)
    N.check(lib.lfmq_influence_topk(_ptr(a), _ptr(u), _ptr(s), Nq, Nt, D1, J, K, _ptr(pos_idx), _ptr(pos_score),
                                    _ptr(neg_idx), _ptr(neg_score), _ptr(total), _ptr(work), work.numel(), _stream()))
    return pos_idx, pos_score, neg_idx, neg_score, total


def nearest_topk(a, b, k, value=None, owner=None):
    """lfmq_nearest_topk: for the queries a [Nq,D1] and the pool b [Nt,D1] (device fp32), the device tensors idx
    [Nq,K] (int32, nearest first, ties to the lower row, -1 past Nt) and d2 [Nq,K] (squared distances, +inf past Nt),
    and with value [Nt] also mean [Nq], the mean value of the listed rows (else None).  `owner` keeps the scratch."""
    a, b = a.contiguous(), b.contiguous()
    Nq, D1 = a.shape
    Nt, K = b.shape[0], int(k)
    assert b.shape == (Nt, D1), (tuple(a.shape), tuple(b.shape))
    if value is not None:
        value = value.contiguous()
        assert value.shape == (Nt,) and value.dtype == torch.float32, tuple(value.shape)
    lib = N.load()
    work = _scratch(owner if owner is not None else _TopkScratch(a.device), 'nearest_topk',
                    lib.lfmq_nearest_topk_work_bytes, Nq, Nt, D1, K)
    idx = torch.empty(Nq, K, dtype=torch.int32, device=a.device)
    d2 = torch.empty(Nq, K, dtype=torch.float32, device=a.device)
    mean = torch.empty(Nq, dtype=torch.float32, device=a.device) if value is not None else None
    N.check(lib.lfmq_nearest_topk(_ptr(a), _ptr(b), _ptr(value), Nq, Nt, D1, K, _ptr(idx), _ptr(d2), _ptr(mean),
                                  _ptr(work), work.numel(), _stream()))
    return idx, d2, mean


def _conformal_args(pred, y, scale):
    """pred, y and scale as contiguous device fp32 [S,N] (y, scale may be None)."""
    pred = pred.contiguous()
    assert pred.dim() == 2 and pred.is_cuda and pred.dtype == torch.float32, (tuple(pred.shape), pred.dtype)
    out = [pred]
    for t in (y, scale):
        if t is not None:
            t = t.contiguous()
            assert t.shape == pred.shape and t.dtype == torch.float32, (tuple(t.shape), t.dtype)
        out.append(t)
    return out


def conformal_scores(pred, y, scale=None):
    """lfmq_conformal_scores: the nonconformity scores r = |y - pred| (/ scale) [S,N] of device fp32 [S,N] arrays, NaN
    where y is not finite."""
    pred, y, scale = _conformal_args(pred, y, scale)
    S, n = pred.shape
    lib = N.load()
    r = torch.empty_like(pred)
    N.check(lib.lfmq_conformal_scores(_ptr(pred), _ptr(y), _ptr(scale), S, n, _ptr(r), None, 0, _stream()))
    return r


def conformal_calibrate(pred, y, levels, scale=None, owner=None):
    """lfmq_conformal_calibrate: of the calibration windows' pred, y (and scale) [S,Nc] and the host `levels`, the device
    tensors n_valid [S] (int32), sorted [S,Nc] (each step's scores ascending, NaN last) and qhat [S,Q] (+inf where the
    rank exceeds n_valid).  `owner` keeps the scratch."""
    pred, y, scale = _conformal_args(pred, y, scale)
    S, nc = pred.shape
    lv = np.ascontiguousarray(levels, dtype=np.float64)
    Q = int(lv.size)
    lib = N.load()
    work = _scratch(owner if owner is not None else _TopkScratch(pred.device), 'conformal',
                    lib.lfmq_conformal_calibrate_work_bytes, S, nc)
    n_valid = torch.empty(S, dtype=torch.int32, device=pred.device)
    sorted_ = torch.empty_like(pred)
    qhat = torch.empty(S, max(Q, 1), dtype=torch.float32, device=pred.device)
    N.check(lib.lfmq_conformal_calibrate(_ptr(pred), _ptr(y), _ptr(scale), S, nc,
                                         lv.ctypes.data_as(C.c_void_p), Q, _ptr(n_valid), _ptr(sorted_), _ptr(qhat),
                                         _ptr(work), work.numel(), _stream()))
    return n_valid, sorted_, qhat


def conformal_apply(pred, calibration, y=None, scale=None):
    """lfmq_conformal_apply: the intervals of the query windows pred (y, scale) [S,N] from conformal_calibrate's
    (n_valid, sorted, qhat): the device tensors lower, upper [S,N,Q] and pvalue [S,N] (NaN where y is None or not
    finite)."""
    pred, y, scale = _conformal_args(pred, y, scale)
    n_valid, sorted_, qhat = calibration
    S, n = pred.shape
    nc, Q = sorted_.shape[1], qhat.shape[1]
    assert sorted_.shape[0] == S and qhat.shape[0] == S and n_valid.shape == (S,)
    lib = N.load()
    lower = torch.empty(S, n, Q, dtype=torch.float32, device=pred.device)
    upper = torch.empty_like(lower)
    pvalue = torch.empty_like(pred)
    N.check(lib.lfmq_conformal_apply(_ptr(pred), _ptr(y), _ptr(scale), S, n, _ptr(sorted_.contiguous()),
                                     _ptr(n_valid.contiguous()), _ptr(qhat.contiguous()), nc, Q, _ptr(lower),
                                     _ptr(upper), _ptr(pvalue), None, 0, _stream()))
    return lower, upper, pvalue


def factor_eval(date_idx, company, score, measure, Q, owner=None):
    """lfmq_factor_eval: the per-date quantile backtest of the factor scores score [G,N] against the measures measure
    [M,N] (device fp64), with date_idx [N] in [0, D) and company [N] (device int32; D = date_idx.max() + 1).  Returns a
    dict of device tensors: n [G,D], bucket_n [G,D,Q] (int32), n_pair [G,M,D] (int32), ic [G,M,D], bucket_mean
    [G,M,D,Q], spread [G,M,D] and turnover [G,D] (fp64).  `owner` keeps the scratch."""
    date_idx, company = date_idx.contiguous(), company.contiguous()
    score, measure = score.contiguous(), measure.contiguous()
    n = date_idx.shape[0]
    G, M, Q = score.shape[0], measure.shape[0], int(Q)
    assert score.shape == (G, n) and measure.shape == (M, n) and company.shape == (n,), (
        tuple(score.shape), tuple(measure.shape), tuple(company.shape))
    assert score.dtype == measure.dtype == torch.float64 and date_idx.dtype == company.dtype == torch.int32
    D = int(date_idx.max().item()) + 1 if n else 0
    lib = N.load()
    dev = score.device
    work = _scratch(owner if owner is not None else _TopkScratch(dev), 'factor', lib.lfmq_factor_eval_work_bytes,
                    n, D, G, M, Q)
    i32 = dict(dtype=torch.int32, device=dev)
    f64 = dict(dtype=torch.float64, device=dev)
    out = dict(n=torch.empty(G, D, **i32), bucket_n=torch.empty(G, D, Q, **i32), n_pair=torch.empty(G, M, D, **i32),
               ic=torch.empty(G, M, D, **f64), bucket_mean=torch.empty(G, M, D, Q, **f64),
               spread=torch.empty(G, M, D, **f64), turnover=torch.empty(G, D, **f64))
    N.check(lib.lfmq_factor_eval(_ptr(date_idx), _ptr(company), n, D, _ptr(score), G, _ptr(measure), M, Q,
                                 _ptr(out['n']), _ptr(out['bucket_n']), _ptr(out['n_pair']), _ptr(out['ic']),
                                 _ptr(out['bucket_mean']), _ptr(out['spread']), _ptr(out['turnover']), _ptr(work),
                                 work.numel(), _stream()))
    return out


class _HandleEngine(object):
    """What every native handle offers whatever its model: parameter specs and views, weights in Keras order, the
    device share, the optimizer apply, the mask count, un-scaling and profiling."""

    def _read_specs(self):
        nt, ntr, ntot = C.c_int32(0), C.c_int64(0), C.c_int64(0)
        N.check(self.lib.lfmq_param_count(self.handle, C.byref(nt), C.byref(ntr), C.byref(ntot)))
        self.n_trainable, self.n_total = ntr.value, ntot.value
        self.specs = []
        for i in range(nt.value):
            name = C.create_string_buffer(96)
            ndim, off, tr = C.c_int32(0), C.c_int64(0), C.c_int32(0)
            shape = (C.c_int64 * 2)()
            N.check(self.lib.lfmq_param_spec(self.handle, i, name, 96, C.byref(ndim), shape, C.byref(off),
                                             C.byref(tr)))
            shp = (shape[0], shape[1]) if ndim.value == 2 else (shape[0],)
            self.specs.append((name.value.decode(), shp, off.value, bool(tr.value)))
        self.params = self._view('lfmq_params_ptr', self.n_total)
        self.grads = self._view('lfmq_grads_ptr', self.n_trainable + N.TAIL_LEN)

    def _view(self, fn, n):
        p = C.c_void_p(0)
        N.check(getattr(self.lib, fn)(self.handle, C.byref(p)))
        off = p.value - self.workspace.data_ptr()
        return self.workspace[off:off + 4 * n].view(torch.float32)

    def close(self):
        if getattr(self, 'handle', None) is not None and self.handle.value:
            self.lib.lfmq_destroy(self.handle)
            self.handle = C.c_void_p(0)

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_device_share(self, num, den):
        """The fraction num/den of the GPU's SMs a persistent launch of this handle may count on (lfmq_set_device_share):
        handles that run at the same time on one GPU each take a share, the shares summing to at most 1."""
        N.check(self.lib.lfmq_set_device_share(self.handle, int(num), int(den)))

    # ---- weights -------------------------------------------------------------------------------
    @property
    def trainable_specs(self):
        return [s for s in self.specs if s[3]]

    def set_flat(self, flat):
        flat = np.ascontiguousarray(flat, dtype=np.float32)
        assert flat.shape == (self.n_total,)
        N.check(self.lib.lfmq_set_params(self.handle, flat.ctypes.data_as(C.c_void_p), self.n_total, _stream()))

    def get_flat(self):
        out = np.empty(self.n_total, dtype=np.float32)
        N.check(self.lib.lfmq_get_params(self.handle, out.ctypes.data_as(C.c_void_p), self.n_total, _stream()))
        return out

    def set_weights(self, weights, bn_stats=None):
        """weights: arrays in Keras trainable_variables order; bn_stats: optional [(mean, var)] per layer."""
        flat = self.get_flat()
        tr = self.trainable_specs
        assert len(weights) == len(tr), (len(weights), len(tr))
        for w, (name, shp, off, _) in zip(weights, tr):
            w = np.asarray(w, dtype=np.float32)
            assert tuple(w.shape) == tuple(shp), (name, w.shape, shp)
            flat[off:off + w.size] = w.ravel()
        if bn_stats is not None:
            nontr = [s for s in self.specs if not s[3]]
            for l, (m, v) in enumerate(bn_stats):
                for arr, (name, shp, off, _) in zip((m, v), nontr[2 * l:2 * l + 2]):
                    flat[off:off + shp[0]] = np.asarray(arr, dtype=np.float32)
        self.set_flat(flat)

    def get_weights(self, trainable_only=True):
        flat = self.get_flat()
        out = []
        for name, shp, off, tr in self.specs:
            if trainable_only and not tr:
                continue
            out.append(flat[off:off + int(np.prod(shp))].reshape(shp).copy())
        return out

    def grads_list(self):
        g = self.grads.detach().cpu().numpy()
        return [g[off:off + int(np.prod(shp))].reshape(shp).copy() for name, shp, off, tr in self.specs if tr]

    # ---- compute -------------------------------------------------------------------------------
    def _check_x(self, x):
        assert x.is_cuda and x.dtype == torch.float32 and x.is_contiguous(), 'x must be a contiguous CUDA fp32 tensor'
        assert x.dim() == 3 and x.shape[1] == self.T and x.shape[2] == self.F, tuple(x.shape)
        return x.shape[0]

    def _influence_dims(self):
        """(D, J) of the training-window attributions: the head input's width (num_hidden, or T * F on a dense handle)
        and the explained outputs (2 on a uq handle)."""
        return (self.T * self.F if isinstance(self, DenseEngine) else self.H), (2 if self.uq else 1)

    def influence_features(self, x, y=None):
        """The features of the training-window attributions (lfmq_influence_*_features, DESIGN.md section 5i), with every
        dropout off: with targets y, the training features u [J,B,D+1]; without, the query features (a [B,D+1],
        s [J,B]).  fp32 / tf32 and dense engines; B is not bounded by max_batch."""
        B = self._check_x(x)
        D, J = self._influence_dims()
        work = _scratch(self, 'influence', self.lib.lfmq_influence_features_work_bytes, self.handle)
        if y is not None:
            y = y.contiguous()
            assert y.is_cuda and y.dtype == torch.float32 and y.shape[0] == B
            u = torch.empty(J, B, D + 1, dtype=torch.float32, device=x.device)
            N.check(self.lib.lfmq_influence_train_features(self.handle, _ptr(x), _ptr(y), B, _ptr(u), _ptr(work),
                                                           work.numel(), _stream()))
            return u
        a = torch.empty(B, D + 1, dtype=torch.float32, device=x.device)
        s = torch.empty(J, B, dtype=torch.float32, device=x.device)
        N.check(self.lib.lfmq_influence_query_features(self.handle, _ptr(x), B, _ptr(a), _ptr(s), _ptr(work),
                                                       work.numel(), _stream()))
        return a, s

    def influence(self, pool, queries, k):
        """Training-window attributions of the query windows: pool = [(x, y)] device batches of training windows, whose
        rows are numbered on in order; queries [N,T,F].  Returns influence_topk's tensors for the K = `k` windows that
        push each forecast up and down the most."""
        u = torch.cat([self.influence_features(x, y) for x, y in pool], dim=1)
        a, s = self.influence_features(queries)
        return influence_topk(a, u, s, k, owner=self)

    def unscale(self, arr, scale, center, log_squasher):
        """Train._unscale_preds (train.py:420-432) on the device: arr [..., O] fp32, scale / center fp64 CUDA tensors."""
        a = arr.contiguous()
        out = torch.empty_like(a)
        N.check(self.lib.lfmq_unscale(_ptr(a), _ptr(out), a.numel() // self.O, self.O, _ptr(scale), _ptr(center),
                                      1 if log_squasher else 0, _stream()))
        return out

    def mask_count(self, y):
        out = torch.empty(2, dtype=torch.float32, device=y.device)
        N.check(self.lib.lfmq_mask_count(self.handle, _ptr(y), y.shape[0], _ptr(out), _stream()))
        return out

    def set_row_weights(self, w):
        """Row weights of the training loss (lfmq_set_row_weights, DESIGN.md section 6d): w is a contiguous CUDA fp32
        tensor of at least max_batch entries, and row b of every later training batch weighs w[b]; None restores the
        unweighted step.  The handle keeps the pointer, so the engine keeps w alive and the caller may refill it in
        place between steps."""
        if w is not None:
            assert w.dtype == torch.float32 and w.is_cuda and w.is_contiguous(), 'row weights: a CUDA fp32 vector'
            assert w.numel() >= self.cfg.max_batch, (w.numel(), self.cfg.max_batch)
        N.check(self.lib.lfmq_set_row_weights(self.handle, _ptr(w)))
        self.row_weights = w

    def apply(self, lr, iteration):
        N.check(self.lib.lfmq_apply(self.handle, float(lr), int(iteration), _stream()))

    def loss(self, preds, y):
        out = torch.empty(2, dtype=torch.float32, device=preds.device)
        N.check(self.lib.lfmq_loss(self.handle, _ptr(preds.contiguous()), _ptr(y.contiguous()), preds.shape[0],
                                   _ptr(out), _stream()))
        return out

    def train_step(self, x, y, step, lr, out=None):
        """One training step of the point estimate (train.py:178-199) on this GPU; returns a device tensor
        {loss, mse_0} (no host sync).  uq engine: the uq range estimate's step (train.py:201-225),
        {uq_loss_last_tar, mse_0}."""
        B = self._check_x(x)
        if out is None:
            out = torch.empty(2, dtype=torch.float32, device=x.device)
        N.check(self.lib.lfmq_train_step(self.handle, _ptr(x), _ptr(y), B, 0, step, float(lr), _ptr(out), _stream()))
        return out

    def _train_step_dp_flat(self, x, y, step, lr, row0, denom_global):
        """The data-parallel step of a handle whose gradient and {loss, mse_0} tail are one contiguous vector: local
        backward with the global denominators, ONE all-reduce of grads[0 : n_trainable + 2], the replicated apply.
        x None (a rank without rows) joins with zeros.  Returns the global {loss, mse_0}."""
        import torch.distributed as dist
        from .dp import allreduce_flat_gradient
        loss_end = self.n_trainable + N.TAIL_MSE0 + 1
        if x is None:
            self.grads[:loss_end].zero_()
        else:
            self.backward(x, y, step=step, row0=row0, denom=denom_global)
        allreduce_flat_gradient(self.grads, self.n_trainable, dist)
        self.apply(lr, step)
        return self.grads[self.n_trainable:loss_end].clone()   # not a live view of the workspace tail

    REGIONS = ('fwd', 'head', 'bwd', 'wgrad', 'opt')

    def profile(self, enable=True):
        N.check(self.lib.lfmq_profile_enable(self.handle, 1 if enable else 0))

    def profile_read(self):
        """{region: (total_ms, count)} of the event-bracketed regions since profile(True)."""
        out = {}
        for r, name in enumerate(self.REGIONS):
            ms, n = C.c_float(0), C.c_int32(0)
            N.check(self.lib.lfmq_profile_read(self.handle, r, C.byref(ms), C.byref(n)))
            out[name] = (ms.value, n.value)
        return out

    @property
    def launch_count(self):
        return int(self.lib.lfmq_launch_count())


class ForecasterEngine(_HandleEngine):
    """fwd / loss / BPTT / clip / optimizer / MaxNorm for RNNPointEstimate on one GPU.

    Mirrors what the reference builds in RNNPointEstimate._build_model
    (scripts/models/point_estimate/rnn_point_estimate.py:40-107) plus the body of its training step
    (scripts/train.py:178-199).
    """

    def __init__(self, *, max_batch, seq_len, n_inputs, n_outputs, num_hidden, num_layers=1, target_idx=0,
                 train=True, precision='fp32', optimizer='Adadelta', dropout=0.0, recurrent_dropout=0.0,
                 target_lambda=0.5, rnn_lambda=0.7, max_grad_norm=50.0, max_norm=3.0, sgd_momentum=0.0,
                 seed=521, forward_only=False, device=None, rnn_cell='lstm', uq=False):
        if not torch.cuda.is_available():
            raise N.LfmqError('ForecasterEngine needs a CUDA device (no CPU fallback)')
        self.lib = N.load()
        self.device = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
        if optimizer not in N.OPTIMIZERS:
            raise ValueError("%s optimizer not found in tf.keras.optimizers" % optimizer)
        cfg = N.LfmqConfig()
        cfg.struct_size = C.sizeof(N.LfmqConfig)
        cfg.max_batch, cfg.seq_len, cfg.n_inputs, cfg.n_outputs = max_batch, seq_len, n_inputs, n_outputs
        cfg.num_hidden, cfg.num_layers, cfg.target_idx = num_hidden, num_layers, target_idx
        cfg.train = 1 if train else 0
        cfg.precision = PRECISIONS[precision]
        cfg.optimizer = N.OPTIMIZERS[optimizer]
        cfg.forward_only = 1 if forward_only else 0
        if rnn_cell not in N.CELLS:
            raise NotImplementedError('rnn_cell=%s (rnn_point_estimate.py:80-102 knows lstm and gru)' % rnn_cell)
        cfg.rnn_cell = N.CELLS[rnn_cell]
        cfg.uq = 1 if uq else 0
        self.uq = bool(uq)
        cfg.dropout, cfg.recurrent_dropout = dropout, recurrent_dropout
        cfg.target_lambda, cfg.rnn_lambda = target_lambda, rnn_lambda
        cfg.max_grad_norm, cfg.max_norm, cfg.sgd_momentum = max_grad_norm, max_norm, sgd_momentum
        cfg.bn_epsilon = 1e-3
        cfg.seed = seed
        self.cfg = cfg
        self.precision = precision
        self.T, self.F, self.O, self.H, self.L = seq_len, n_inputs, n_outputs, num_hidden, num_layers
        nbytes = C.c_uint64(0)
        N.check(self.lib.lfmq_workspace_bytes(C.byref(cfg), C.byref(nbytes)))
        with torch.cuda.device(self.device):
            self.workspace = torch.empty(nbytes.value, dtype=torch.uint8, device=self.device)
            self.handle = C.c_void_p(0)
            N.check(self.lib.lfmq_create(C.byref(cfg), _ptr(self.workspace), nbytes, C.byref(self.handle)))
        self._read_specs()
        self._denom = torch.zeros(2, dtype=torch.float32, device=self.device)
        self._dp = None

    def forward(self, x, step=0, row0=0, out=None):
        """preds [B,T,O]; on a uq engine the pair (preds, variance) -- model(inp)[0], model(inp)[1] of RNNUqRangeEstimate."""
        B = self._check_x(x)
        if self.uq:
            preds = torch.empty(B, self.T, self.O, dtype=torch.float32, device=x.device)
            var = torch.empty_like(preds)
            N.check(self.lib.lfmq_forward_uq(self.handle, _ptr(x), B, row0, step, _ptr(preds), _ptr(var), _stream()))
            return preds, var
        if out is None:
            out = torch.empty(B, self.T, self.O, dtype=torch.float32, device=x.device)
        N.check(self.lib.lfmq_forward(self.handle, _ptr(x), B, row0, step, _ptr(out), _stream()))
        return out

    def forward_mc(self, x, samples, step=0, row0=0):
        """`samples` Monte-Carlo dropout samples of every window in one call (lfmq_forward_uq_mc): the device tensors
        (mean_pred, mean_var, var_pred, var_var) [B,T,O] -- the sample means of the target predictions and of the
        variances, and their population variances.  Sample s of window b is row row0 + s * B + b; sample 0 is
        forward(x, step, row0).  uq engines only."""
        B = self._check_x(x)
        out = [torch.empty(B, self.T, self.O, dtype=torch.float32, device=x.device) for _ in range(4)]
        work = _scratch(self, 'mc', self.lib.lfmq_forward_uq_mc_work_bytes, self.handle, B, int(samples))
        N.check(self.lib.lfmq_forward_uq_mc(self.handle, _ptr(x), B, row0, step, samples, *[_ptr(t) for t in out],
                                            _ptr(work), work.numel(), _stream()))
        return tuple(out)

    def integrated_gradients(self, x, steps):
        """Integrated-gradients attributions of the point forecast pred[:, T-1, target_idx] in one call
        (lfmq_integrated_gradients): the device tensors (attr [B,T,F], f_x [B], f_base [B]) for the zero baseline and
        `steps` midpoint-rule interpolants; sum(attr[b]) approximates f_x[b] - f_base[b].  An fp32 or tf32 engine
        created with train=False, forward_only=False and uq=False; B and steps are not bounded by max_batch.  The
        engine's parameters, gradients and optimizer state are left as they were."""
        B = self._check_x(x)
        work = _scratch(self, 'ig', self.lib.lfmq_integrated_gradients_work_bytes, self.handle, B, int(steps))
        attr = torch.empty(B, self.T, self.F, dtype=torch.float32, device=x.device)
        f_x = torch.empty(B, dtype=torch.float32, device=x.device)
        f_base = torch.empty_like(f_x)
        N.check(self.lib.lfmq_integrated_gradients(self.handle, _ptr(x), B, int(steps), _ptr(attr), _ptr(f_x),
                                                   _ptr(f_base), _ptr(work), work.numel(), _stream()))
        return attr, f_x, f_base

    def loss_uq(self, preds, var, y):
        """Device tensor {uq_loss, uq_loss_last_tar, mse_0} (Losses.weight_adjusted_uq_loss, losses.py:137-284)."""
        out = torch.empty(3, dtype=torch.float32, device=preds.device)
        N.check(self.lib.lfmq_loss_uq(self.handle, _ptr(preds.contiguous()), _ptr(var.contiguous()), _ptr(y.contiguous()),
                                      preds.shape[0], _ptr(out), _stream()))
        return out

    def mask_count_uq(self, y):
        """Device {B, unmasked rows, unmasked last-step rows}: the denominators of the uq loss (losses.py:179-284)."""
        out = torch.empty(3, dtype=torch.float32, device=y.device)
        N.check(self.lib.lfmq_mask_count_uq(self.handle, _ptr(y), y.shape[0], _ptr(out), _stream()))
        return out

    def loss_counts(self, y):
        """The loss denominators of one batch that data parallelism all-reduces: mask_count_uq on a uq engine, else
        mask_count.  y None (a rank without rows): zeros of the same length."""
        if y is None:
            return torch.zeros(3 if self.uq else 2, dtype=torch.float32, device=self.device)
        return self.mask_count_uq(y) if self.uq else self.mask_count(y)

    def backward(self, x, y, step=0, row0=0, denom=None):
        B = self._check_x(x)
        assert y.is_cuda and y.dtype == torch.float32 and y.is_contiguous() and tuple(y.shape) == (B, self.T, self.O)
        N.check(self.lib.lfmq_backward(self.handle, _ptr(x), _ptr(y), B, row0, step, _ptr(denom), _stream()))

    def train_step_dp(self, x, y, step, lr, row0, denom_global):
        """Data-parallel step: local BPTT with global denominators, ONE NCCL all-reduce over the flat
        gradient (+ loss/mse tail), then the replicated clip + optimizer (SURVEY 8e).
        uq engine: the gradient and {uq_loss, mse_0, uq_loss_last_tar} travel as one packed vector (a chain of one
        stage, lfmq_chain_grad_pack).  x None (a rank without rows) joins the collective with zeros.  Returns the global
        {loss, mse_0}, uq engine {uq_loss_last_tar, mse_0}, as train_step."""
        import torch.distributed as dist
        if self.uq:
            if self._dp is None:
                self._dp = _PackedStep([self], [1.0])
            self._dp.step(lambda: self.backward(x, y, step=step, row0=row0, denom=denom_global), x is not None, dist)
            self.apply(lr, step)
            t = self.grads[self.n_trainable:]
            return torch.stack([t[N.TAIL_UQ_LOSS_LAST_TAR], t[N.TAIL_MSE0]])
        return self._train_step_dp_flat(x, y, step, lr, row0, denom_global)



class DenseEngine(_HandleEngine):
    """MLPLinearPointEstimate on one GPU (scripts/models/point_estimate/mlp_linear_point_estimate.py:66-77): one Dense(O)
    layer OUTPUT_1 over the flattened input window, its MLP-branch loss (model_utils/losses.py:69-75,100-115) with the
    Huber option, the clip and the optimizer -- a dense handle of include/lfmq.h (lfmq_dense_create).  x is the
    [B, T, F] batch or its [B, T*F] view; targets and predictions are [B, O]."""

    def __init__(self, *, max_batch, seq_len, n_inputs, n_outputs, target_idx=0, precision='fp32',
                 optimizer='Adadelta', target_lambda=0.5, max_grad_norm=50.0, sgd_momentum=0.0, huber_loss=False,
                 huber_delta=1.0, forward_only=False, device=None):
        if not torch.cuda.is_available():
            raise N.LfmqError('DenseEngine needs a CUDA device (no CPU fallback)')
        self.lib = N.load()
        self.device = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
        if optimizer not in N.OPTIMIZERS:
            raise ValueError("%s optimizer not found in tf.keras.optimizers" % optimizer)
        cfg = N.LfmqDenseConfig()
        cfg.struct_size = C.sizeof(N.LfmqDenseConfig)
        cfg.max_batch, cfg.seq_len, cfg.n_inputs, cfg.n_outputs = max_batch, seq_len, n_inputs, n_outputs
        cfg.target_idx = target_idx
        cfg.precision = PRECISIONS[precision]
        cfg.optimizer = N.OPTIMIZERS[optimizer]
        cfg.forward_only = 1 if forward_only else 0
        cfg.huber_loss = 1 if huber_loss else 0
        cfg.target_lambda, cfg.huber_delta = target_lambda, huber_delta
        cfg.max_grad_norm, cfg.sgd_momentum = max_grad_norm, sgd_momentum
        self.cfg = cfg
        self.precision = precision
        self.uq = False
        self.T, self.F, self.O = seq_len, n_inputs, n_outputs
        nbytes = C.c_uint64(0)
        N.check(self.lib.lfmq_dense_workspace_bytes(C.byref(cfg), C.byref(nbytes)))
        with torch.cuda.device(self.device):
            self.workspace = torch.empty(nbytes.value, dtype=torch.uint8, device=self.device)
            self.handle = C.c_void_p(0)
            N.check(self.lib.lfmq_dense_create(C.byref(cfg), _ptr(self.workspace), nbytes, C.byref(self.handle)))
        self._read_specs()

    def _check_x(self, x):
        assert x.is_cuda and x.dtype == torch.float32 and x.is_contiguous(), 'x must be a contiguous CUDA fp32 tensor'
        assert x.shape[0] * self.T * self.F == x.numel() and x.shape[1:] in ((self.T * self.F,), (self.T, self.F)), \
            tuple(x.shape)
        return x.shape[0]

    def _check_y(self, y, B):
        assert y.is_cuda and y.dtype == torch.float32 and y.is_contiguous() and tuple(y.shape) == (B, self.O), \
            'y must be a contiguous CUDA fp32 tensor [B, O]'

    def forward(self, x, step=0, row0=0, out=None):
        """model(inp) / model.predict(inp): preds [B, O].  step and row0 are accepted for the drivers' sake; the model
        has no dropout."""
        B = self._check_x(x)
        if out is None:
            out = torch.empty(B, self.O, dtype=torch.float32, device=x.device)
        N.check(self.lib.lfmq_forward(self.handle, _ptr(x), B, row0, step, _ptr(out), _stream()))
        return out

    def loss_counts(self, y):
        """{B, rows whose targets are not all zero}, the denominators data parallelism all-reduces; zeros for y None."""
        if y is None:
            return torch.zeros(2, dtype=torch.float32, device=self.device)
        return self.mask_count(y)

    def backward(self, x, y, step=0, row0=0, denom=None):
        B = self._check_x(x)
        self._check_y(y, B)
        N.check(self.lib.lfmq_backward(self.handle, _ptr(x), _ptr(y), B, row0, step, _ptr(denom), _stream()))

    def train_step(self, x, y, step, lr, out=None):
        self._check_y(y, self._check_x(x))
        return super(DenseEngine, self).train_step(x, y, step, lr, out)

    def train_step_dp(self, x, y, step, lr, row0, denom_global):
        """Data-parallel step (the point estimate's): local backward with the global {B, mask count}, ONE all-reduce
        of the flat gradient and its {loss, mse_0} tail, the replicated clip and optimizer."""
        return self._train_step_dp_flat(x, y, step, lr, row0, denom_global)


class _PackedStep(object):
    """The collective of a data-parallel step over the handles of a chain (or one uq handle): the backward fills every
    stage's gradient buffer, one launch packs them with their reduced loss tails into one contiguous vector, ONE SUM
    all-reduce, one launch scatters it back (and forms the weighted losses).  The apply then runs on every rank."""

    def __init__(self, engines, weights):
        e0 = engines[0]
        self.lib, self.S = e0.lib, len(engines)
        self.handles = (C.c_void_p * self.S)(*[e.handle.value for e in engines])
        self.w = (C.c_float * self.S)(*weights)
        n = C.c_int64(0)
        N.check(self.lib.lfmq_chain_grad_pack_size(self.handles, self.S, C.byref(n)))
        self.flat = torch.empty(n.value, dtype=torch.float32, device=e0.device)

    def step(self, backward, has_rows, dist, loss_out=None):
        from .dp import allreduce_packed
        if has_rows:
            backward()
            N.check(self.lib.lfmq_chain_grad_pack(self.handles, self.S, _ptr(self.flat), _stream()))
        else:
            self.flat.zero_()
        allreduce_packed(self.flat, dist)
        N.check(self.lib.lfmq_chain_grad_unpack(self.handles, self.S, _ptr(self.flat), self.w, _ptr(loss_out),
                                                _stream()))


class ForecastChainEngine(object):
    """The engine behind every model object: S >= 1 stages, list-valued throughout -- forward returns the Keras output
    list and the losses and steps take the list of S targets.

    S > 1 (scripts/models/point_estimate/rnn_point_estimate.py:109-150): stage 0 is the trunk, every further stage one
    more recurrent layer + BatchNormalization + Dropout + Dense on the shifted input window.  One ForecasterEngine (one
    C-ABI handle) per stage; the lfmq_chain_* entry points run the whole graph.
    uq=True: RNNUqRangeEstimate's graph (models/uq_range_estimate/rnn_uq_range_estimate.py:114-157), every stage with a
    target and a variance head and dropout always on; the next window is built from the target predictions.

    S == 1: every call goes to the one stage's own engine -- a ForecasterEngine, or the DenseEngine passed as
    ``stages=[engine]`` -- and its result is wrapped in a list.  A one-stage model so issues exactly its handle's library
    calls: lfmq_train_step as one call, bf16 / bf16x3 training handles (which the chain entry points refuse), and the
    handle's own data-parallel step.  Its step weights are [1.0] (losses.py:44-45) whatever ``weights`` holds."""

    def __init__(self, *, forecast_steps=1, weights=None, num_layers=1, uq=False, stages=None, **kw):
        if stages is None:
            assert forecast_steps >= 1
            stages = [ForecasterEngine(num_layers=num_layers if s == 0 else 1, uq=uq, **kw)
                      for s in range(forecast_steps)]
        self.stages = list(stages)
        self.S = len(self.stages)
        e0 = self.stages[0]
        self._one = e0 if self.S == 1 else None
        self.lib, self.device, self.cfg, self.precision, self.uq = e0.lib, e0.device, e0.cfg, e0.precision, e0.uq
        self.T, self.F, self.O = e0.T, e0.F, e0.O
        self.weights = [float(w) for w in weights] if self._one is None else [1.0]
        assert len(self.weights) == self.S, (self.weights, self.S)
        self._handles = (C.c_void_p * self.S)(*[e.handle.value for e in self.stages])
        self._w = (C.c_float * self.S)(*self.weights)
        self._work = None
        self._dp = None
        self.device_share = None
        # Keras names: the extra layer of stage s is lstm_{L+s} / batch_normalization_{L+s-1} / OUTPUT_{s+1}
        self.specs = []            # (stage, name, shape, offset in the stage's flat vector, trainable)
        cell = kw.get('rnn_cell', 'lstm')
        for s, e in enumerate(self.stages):
            for name, shp, off, tr in e.specs:
                if s > 0:
                    L = e0.L
                    name = name.replace('%s_1/' % cell, '%s_%d/' % (cell, L + s))
                    name = name.replace('batch_normalization/', 'batch_normalization_%d/' % (L + s - 1))
                    name = name.replace('OUTPUT_1/', 'OUTPUT_%d/' % (s + 1))
                    name = name.replace('OUTPUT_TARGET_1/', 'OUTPUT_TARGET_%d/' % (s + 1))
                    name = name.replace('OUTPUT_VARIANCE_1/', 'OUTPUT_VARIANCE_%d/' % (s + 1))
                self.specs.append((s, name, shp, off, tr))
        self.n_total = sum(e.n_total for e in self.stages)
        self.n_trainable = sum(e.n_trainable for e in self.stages)

    def set_device_share(self, num, den):
        """ForecasterEngine.set_device_share for every stage: the stages of a chain run one after another on one stream.
        The share is kept in ``device_share`` (None: the whole device), for engines that run beside this one's model."""
        for e in self.stages:
            e.set_device_share(num, den)
        self.device_share = (int(num), int(den))

    def set_row_weights(self, w):
        """_HandleEngine.set_row_weights for every stage: each stage's loss weighs row b of the batch by w[b]."""
        for e in self.stages:
            e.set_row_weights(w)

    def _ptrs(self, tensors):
        return (C.c_void_p * self.S)(*[t.data_ptr() for t in tensors])

    def _workbuf(self, B):
        n = self.S * B * self.T * self.F
        if self._work is None or self._work.numel() < n:
            self._work = torch.empty(n, dtype=torch.float32, device=self.device)
        return self._work

    def forward(self, x, step=0, row0=0):
        """model(inp) -> the Keras output list of device tensors [B,T,O] ([B,O] on a dense stage): [pred],
        [tar, var], [pred_1 .. pred_S] or, on a uq chain, [tar_1, var_1, .., tar_S, var_S]
        (rnn_uq_range_estimate.py:107-108,152-155)."""
        if self._one is not None:
            out = self._one.forward(x, step=step, row0=row0)
            return list(out) if self.uq else [out]
        B = self.stages[0]._check_x(x)
        preds = [torch.empty(B, self.T, self.O, dtype=torch.float32, device=x.device) for _ in range(self.S)]
        if self.uq:
            var = [torch.empty_like(p) for p in preds]
            N.check(self.lib.lfmq_chain_forward_uq(self._handles, self.S, _ptr(x), B, row0, step, self._ptrs(preds),
                                                   self._ptrs(var), _ptr(self._workbuf(B)), _stream()))
            return [t for pv in zip(preds, var) for t in pv]
        N.check(self.lib.lfmq_chain_forward(self._handles, self.S, _ptr(x), B, row0, step, self._ptrs(preds),
                                            _ptr(self._workbuf(B)), _stream()))
        return preds

    def forward_mc(self, x, samples, step=0, row0=0):
        """`samples` Monte-Carlo dropout samples of every window of a uq model in one call: per stage the device tensors
        (mean_pred, mean_var, var_pred, var_var) [B,T,O] (ForecasterEngine.forward_mc; a chain runs each sample's own
        trajectory, lfmq_chain_forward_uq_mc)."""
        if self._one is not None:
            return [self._one.forward_mc(x, samples, step=step, row0=row0)]
        B = self.stages[0]._check_x(x)
        out = [[torch.empty(B, self.T, self.O, dtype=torch.float32, device=x.device) for _ in range(self.S)]
               for _ in range(4)]
        work = _scratch(self, 'mc', self.lib.lfmq_chain_forward_uq_mc_work_bytes, self._handles, self.S, B,
                        int(samples))
        N.check(self.lib.lfmq_chain_forward_uq_mc(self._handles, self.S, _ptr(x), B, row0, step, samples,
                                                  *[self._ptrs(o) for o in out], _ptr(work), work.numel(), _stream()))
        return [tuple(o[s] for o in out) for s in range(self.S)]

    def forward_dist(self, x, samples, levels, ys=None, step=0, row0=0):
        """forward_mc's samples as each window's predictive mixture (lfmq_chain_forward_uq_dist, DESIGN.md section 5g):
        (moments, quantiles, scores) -- moments per stage forward_mc's (mean_pred, mean_var, var_pred, var_var) bit for
        bit, the device tensors quantiles [S,B,Q] at the host `levels` and, with ys (per stage targets [B,T,O]),
        scores [S,B,3] = {crps, nll, pit} of the target at [T-1, target_idx] (NaN where it is NaN), else None."""
        B = self.stages[0]._check_x(x)
        lv = np.ascontiguousarray(levels, dtype=np.float32)
        Q = int(lv.size)
        out = [[torch.empty(B, self.T, self.O, dtype=torch.float32, device=x.device) for _ in range(self.S)]
               for _ in range(4)]
        quantiles = torch.empty(self.S, B, max(Q, 1), dtype=torch.float32, device=x.device)
        scores = None
        y_arg = None
        if ys is not None:
            assert len(ys) == self.S
            ys = [y.contiguous() for y in ys]
            for y in ys:
                assert y.is_cuda and y.dtype == torch.float32 and y.shape == (B, self.T, self.O)
            scores = torch.empty(self.S, B, 3, dtype=torch.float32, device=x.device)
            y_arg = self._ptrs(ys)
        work = _scratch(self, 'dist', self.lib.lfmq_chain_forward_uq_dist_work_bytes, self._handles, self.S, B,
                        int(samples), Q)
        N.check(self.lib.lfmq_chain_forward_uq_dist(
            self._handles, self.S, _ptr(x), y_arg, B, row0, step, int(samples), lv.ctypes.data_as(C.c_void_p), Q,
            *[self._ptrs(o) for o in out], self._ptrs(quantiles), self._ptrs(scores) if scores is not None else None,
            _ptr(work), work.numel(), _stream()))
        return [tuple(o[s] for o in out) for s in range(self.S)], quantiles, scores

    def permutation_importance(self, x, ys, col_group, repeats, seed, step):
        """Permutation importance of the held-out set (x, ys) in one call (lfmq_chain_permutation_importance, DESIGN.md
        section 5e): the device tensor [1 + G * repeats, 3] of the model's loss on the unpermuted set (row 0) and on
        every copy with group g's columns shuffled across the windows (row 1 + g * repeats + r).  col_group [T*F] maps
        column t * F + f to its group; G = max(col_group) + 1.  Rows hold {loss, mse_0, 0}, on a uq model
        {uq_loss, uq_loss_last_tar, mse}.  Window i draws its dropout masks at (step, row i) in every copy.  N is not
        bounded by max_batch; the engine's parameters, gradients and optimizer state are left as they were."""
        B = self.stages[0]._check_x(x)
        assert len(ys) == self.S
        ys = [y.contiguous() for y in ys]
        for y in ys:
            assert y.is_cuda and y.dtype == torch.float32 and y.shape[0] == B
        cg = np.ascontiguousarray(col_group, dtype=np.int32)
        G = int(cg.max()) + 1
        work = _scratch(self, 'pi', self.lib.lfmq_chain_permutation_importance_work_bytes, self._handles, self.S, B)
        out = torch.empty(max(1 + G * int(repeats), 1), 3, dtype=torch.float32, device=self.device)
        N.check(self.lib.lfmq_chain_permutation_importance(
            self._handles, self.S, _ptr(x), self._ptrs(ys), self._w, B, cg.ctypes.data_as(C.c_void_p), G,
            int(repeats), int(seed), int(step), _ptr(out), _ptr(work), work.numel(), _stream()))
        return out

    def shapley(self, x, col_group, samples, seed, step):
        """Shapley attributions of every window's forecast in one call (lfmq_chain_shapley, DESIGN.md section 5f):
        device tensors (phi [N,K,G], f_x [N,K], f_bg [N,K]), sum_g phi = f_x - f_bg.  The K outputs are pred[:, T-1,
        target_idx] of every stage (tar_1, var_1, .., tar_S, var_S on a uq model; pred[:, target_idx] on a dense
        stage).  col_group [T*F] maps column t * F + f to its group; G = max(col_group) + 1.  `samples` orderings of the
        groups, in antithetic pairs, each against a donor window; a uq window draws its dropout masks at (step, row
        m * N + i) for sample m.  N is not bounded by max_batch; the engine's parameters, gradients and optimizer state
        are left as they were."""
        B = self.stages[0]._check_x(x)
        cg = np.ascontiguousarray(col_group, dtype=np.int32)
        G, M = int(cg.max()) + 1, int(samples)
        K = 1 if isinstance(self.stages[0], DenseEngine) else (2 * self.S if self.uq else self.S)
        work = _scratch(self, 'shapley', self.lib.lfmq_chain_shapley_work_bytes, self._handles, self.S, B, G, M)
        phi = torch.empty(B, K, G, dtype=torch.float32, device=self.device)
        f_x = torch.empty(B, K, dtype=torch.float32, device=self.device)
        f_bg = torch.empty(B, K, dtype=torch.float32, device=self.device)
        N.check(self.lib.lfmq_chain_shapley(
            self._handles, self.S, _ptr(x), B, cg.ctypes.data_as(C.c_void_p), G, M, int(seed), int(step), _ptr(phi),
            _ptr(f_x), _ptr(f_bg), _ptr(work), work.numel(), _stream()))
        return phi, f_x, f_bg

    def ale(self, x, cols, bins, step):
        """Accumulated local effects of single input columns in one call (lfmq_chain_ale, DESIGN.md section 5h): the
        device tensors (n_bins [G] int32, edges [G,K+1], counts [G,K] int32, ale [G,K+1,J], local_mean [G,K,J],
        local_sd [G,K,J]) of feature g = column cols[g] of the flattened window (t * F + f), with K = `bins` requested
        quantile bins and the J outputs shapley explains.  Both copies of window i draw its dropout masks at (step,
        row i).  N is not bounded by max_batch; the engine's parameters, gradients and optimizer state are left as they
        were."""
        B = self.stages[0]._check_x(x)
        cols = np.ascontiguousarray(cols, dtype=np.int32)
        G, K = int(cols.size), int(bins)
        J = 1 if isinstance(self.stages[0], DenseEngine) else (2 * self.S if self.uq else self.S)
        work = _scratch(self, 'ale', self.lib.lfmq_chain_ale_work_bytes, self._handles, self.S, B, G, K)
        n_bins = torch.empty(G, dtype=torch.int32, device=self.device)
        edges = torch.empty(G, K + 1, dtype=torch.float32, device=self.device)
        counts = torch.empty(G, K, dtype=torch.int32, device=self.device)
        ale = torch.empty(G, K + 1, J, dtype=torch.float32, device=self.device)
        local_mean = torch.empty(G, K, J, dtype=torch.float32, device=self.device)
        local_sd = torch.empty_like(local_mean)
        N.check(self.lib.lfmq_chain_ale(
            self._handles, self.S, _ptr(x), B, cols.ctypes.data_as(C.c_void_p), G, K, int(step), _ptr(n_bins),
            _ptr(edges), _ptr(counts), _ptr(ale), _ptr(local_mean), _ptr(local_sd), _ptr(work), work.numel(),
            _stream()))
        return n_bins, edges, counts, ale, local_mean, local_sd

    def loss(self, preds, ys):
        """Losses.weight_adjusted_mse(ys, preds): device tensor {loss, mse}."""
        if self._one is not None:
            return self._one.loss(preds[0], ys[0])
        out = torch.empty(2, dtype=torch.float32, device=preds[0].device)
        preds = [p.contiguous() for p in preds]
        ys = [y.contiguous() for y in ys]
        N.check(self.lib.lfmq_chain_loss(self._handles, self.S, self._ptrs(preds), self._ptrs(ys), self._w,
                                         preds[0].shape[0], _ptr(out), _stream()))
        return out

    def loss_uq(self, preds, var, ys):
        """Losses.weight_adjusted_uq_loss(ys, preds, var) (losses.py:137-178): device tensor
        {uq_loss, uq_loss_last_tar, mse}, each summed over the steps with forecast_steps_weights."""
        if self._one is not None:
            return self._one.loss_uq(preds[0], var[0], ys[0])
        out = torch.empty(3, dtype=torch.float32, device=preds[0].device)
        preds, var, ys = ([t.contiguous() for t in a] for a in (preds, var, ys))
        N.check(self.lib.lfmq_chain_loss_uq(self._handles, self.S, self._ptrs(preds), self._ptrs(var), self._ptrs(ys),
                                            self._w, preds[0].shape[0], _ptr(out), _stream()))
        return out

    def backward(self, x, ys, step=0, row0=0, out=None):
        B = self.stages[0]._check_x(x)
        assert len(ys) == self.S
        for y in ys:
            assert y.is_cuda and y.dtype == torch.float32 and y.is_contiguous() and tuple(y.shape) == (B, self.T, self.O)
        if out is None:
            out = torch.empty(3 if self.uq else 2, dtype=torch.float32, device=x.device)
        N.check(self.lib.lfmq_chain_backward(self._handles, self.S, _ptr(x), self._ptrs(ys), self._w, B, row0, step,
                                             _ptr(self._workbuf(B)), _ptr(out), _stream()))
        return out

    def apply(self, lr, iteration):
        if self._one is not None:
            return self._one.apply(lr, iteration)
        N.check(self.lib.lfmq_chain_apply(self._handles, self.S, float(lr), int(iteration), _stream()))

    # ---- data parallelism over the company-batch axis --------------------------------------------
    def mask_count(self, ys):
        """Device [S, 3]: every stage's {B, unmasked rows, unmasked last-step rows} (lfmq_chain_mask_count), the
        counts one batch all-reduces (dp.global_stage_counts).  ys None (a rank without rows): zeros."""
        if ys is None:
            return torch.zeros(self.S, 3, dtype=torch.float32, device=self.device)
        assert len(ys) == self.S
        out = torch.empty(self.S, 3, dtype=torch.float32, device=self.device)
        B = ys[0].shape[0]
        N.check(self.lib.lfmq_chain_mask_count(self._handles, self.S, self._ptrs([y.contiguous() for y in ys]), B,
                                               _ptr(out), _stream()))
        return out

    def loss_counts(self, ys):
        """The loss denominators of one batch that data parallelism all-reduces: the stage's own loss_counts, or
        mask_count of a chain.  ys None (a rank without rows): zeros."""
        if self._one is not None:
            return self._one.loss_counts(None if ys is None else ys[0])
        return self.mask_count(ys)

    def backward_dp(self, x, ys, denoms, step=0, row0=0, out=None):
        """backward with the global batch's stage counts (device [S, 3]) as the loss denominators; every stage's tail
        and `out` then hold this shard's contributions."""
        B = self.stages[0]._check_x(x)
        assert len(ys) == self.S and denoms.is_cuda and denoms.numel() == 3 * self.S
        for y in ys:
            assert y.is_cuda and y.dtype == torch.float32 and y.is_contiguous() and tuple(y.shape) == (B, self.T, self.O)
        if out is None:
            out = torch.empty(3 if self.uq else 2, dtype=torch.float32, device=x.device)
        N.check(self.lib.lfmq_chain_backward_dp(self._handles, self.S, _ptr(x), self._ptrs(ys), self._w, B, row0, step,
                                                _ptr(denoms.contiguous()), _ptr(self._workbuf(B)), _ptr(out),
                                                _stream()))
        return out

    def _packed(self):
        if self._dp is None:
            self._dp = _PackedStep(self.stages, self.weights)
        return self._dp

    @property
    def n_packed(self):
        """Length of the vector the step all-reduces: sum_s (n_trainable_s + 2), + 3 on a uq chain."""
        return self._packed().flat.numel()

    def pack(self, flat=None):
        """Every stage's gradients and reduced loss tail as one contiguous device vector (one launch)."""
        p = self._packed()
        flat = p.flat if flat is None else flat
        assert flat.is_cuda and flat.dtype == torch.float32 and flat.numel() == p.flat.numel() and flat.is_contiguous()
        N.check(self.lib.lfmq_chain_grad_pack(self._handles, self.S, _ptr(flat), _stream()))
        return flat

    def unpack(self, flat, out=None):
        """The inverse scatter; `out` (optional) receives the weighted losses, as backward's."""
        assert flat.is_cuda and flat.dtype == torch.float32 and flat.numel() == self.n_packed and flat.is_contiguous()
        N.check(self.lib.lfmq_chain_grad_unpack(self._handles, self.S, _ptr(flat), self._w, _ptr(out), _stream()))
        return out

    def train_step_dp(self, x, ys, step, lr, row0, denoms):
        """Data-parallel step of the whole graph: local BPTT of this rank's rows with the global stage counts, ONE
        all-reduce of the packed vector, then the joint clip, optimizer and MaxNorm on every rank.  x None joins the
        step without rows.  Returns the global {loss, mse}; uq chain {uq_loss_last_tar, mse}, as train_step.
        One stage: its own train_step_dp (a point or dense handle reduces its flat gradient in place)."""
        if self._one is not None:
            return self._one.train_step_dp(x, None if ys is None else ys[0], step, lr, row0, denoms)
        import torch.distributed as dist
        out = torch.empty(3 if self.uq else 2, dtype=torch.float32, device=self.device)
        self._packed().step(lambda: self.backward_dp(x, ys, denoms, step=step, row0=row0), x is not None, dist,
                            loss_out=out)
        self.apply(lr, step)
        return out[1:] if self.uq else out

    def train_step(self, x, ys, step, lr):
        """One training step (train.py:178-225) over the S-output model; device tensor {loss, mse}, on a uq model
        {uq_loss_last_tar, mse} (train.py:225), both weighted over the steps.  One stage: one lfmq_train_step."""
        if self._one is not None:
            return self._one.train_step(x, ys[0], step, lr)
        out = self.backward(x, ys, step=step)
        self.apply(lr, step)
        return out[1:] if self.uq else out

    def unscale(self, arr, scale, center, log_squasher):
        return self.stages[0].unscale(arr, scale, center, log_squasher)

    @property
    def launch_count(self):
        return self.stages[0].launch_count

    def grads_list(self):
        return [g for e in self.stages for g in e.grads_list()]

    def get_weights(self, trainable_only=True):
        return [w for e in self.stages for w in e.get_weights(trainable_only)]

    def set_weights(self, weights):
        """weights in trainable_variables order (the trunk's, then 7 per extra stage, 9 on a uq chain), or all of
        get_weights(trainable_only=False): every stage's trainable arrays followed by its BatchNormalization
        statistics."""
        full = len(weights) == len(self.specs)
        i = 0
        for e in self.stages:
            n = len(e.trainable_specs)
            bn = weights[i + n:i + len(e.specs)] if full else []
            e.set_weights(weights[i:i + n], list(zip(bn[0::2], bn[1::2])) if full else None)
            i += n + len(bn)
        assert i == len(weights), (i, len(weights))

    def named_arrays(self):
        out = {}
        flats = [e.get_flat() for e in self.stages]
        for s, name, shp, off, _ in self.specs:
            out[name] = flats[s][off:off + int(np.prod(shp))].reshape(shp).copy()
        return out

    def load_named(self, get):
        for s, e in enumerate(self.stages):
            flat = e.get_flat()
            for st, name, shp, off, _ in self.specs:
                if st != s:
                    continue
                w = np.asarray(get(name), dtype=np.float32)
                assert tuple(w.shape) == tuple(shp), (name, w.shape, shp)
                flat[off:off + w.size] = w.ravel()
            e.set_flat(flat)

    def close(self):
        for e in self.stages:
            e.close()


class HostBatchPipeline(object):
    """Feeds host-resident (pinned) batches to a ForecasterEngine with the H2D copy of step i+1 overlapped with the
    compute of step i (two device buffers, one copy stream) and an asynchronous D2H read of every step's
    {loss, mse_0}.  Each step still copies its own inputs host->device and its result device->host.

        pipe = HostBatchPipeline(engine, batch)
        for i, (x_pinned, y_pinned) in enumerate(batches):
            loss_mse = pipe.step(x_pinned, y_pinned, i, lr)     # host tensor of the PREVIOUS step (None at i=0)
        last = pipe.finish()

    Row weights (DESIGN.md section 6d): pass each batch's fp32 host weights as `w_host` (and as the third entry of
    `next_batch`); they are staged with the batch into a device vector of max_batch entries and set on the engine for
    the step that reads the batch.
    """

    def __init__(self, engine, batch, step_fn=None):
        self.eng = engine
        dev = engine.device
        self.copy_stream = torch.cuda.Stream(device=dev)
        self.x = [torch.empty(batch, engine.T, engine.F, dtype=torch.float32, device=dev) for _ in range(2)]
        self.y = [torch.empty(batch, engine.T, engine.O, dtype=torch.float32, device=dev) for _ in range(2)]
        self.copied = [torch.cuda.Event() for _ in range(2)]
        self.consumed = [torch.cuda.Event() for _ in range(2)]
        self.out_host = [torch.empty(2, dtype=torch.float32).pin_memory() for _ in range(2)]
        self.out_ready = [torch.cuda.Event() for _ in range(2)]
        self.w = [None, None]
        self.step_fn = step_fn or (lambda x, y, i, lr: engine.train_step(x, y, i, lr))
        self.n = 0
        self._staged = None

    def _stage(self, x_host, y_host, slot, w_host=None):
        with torch.cuda.stream(self.copy_stream):
            if self.n >= 2:
                self.copy_stream.wait_event(self.consumed[slot])      # the step that used this buffer is done
            self.x[slot].copy_(x_host, non_blocking=True)
            self.y[slot].copy_(y_host, non_blocking=True)
            if w_host is not None:
                if self.w[slot] is None:
                    self.w[slot] = torch.zeros(self.eng.cfg.max_batch, dtype=torch.float32, device=self.x[slot].device)
                self.w[slot][w_host.shape[0]:].zero_()
                self.w[slot][:w_host.shape[0]].copy_(w_host, non_blocking=True)
            self.copied[slot].record(self.copy_stream)

    def step(self, x_host, y_host, index, lr, next_batch=None, w_host=None):
        """Runs one step on (x_host, y_host[, row weights w_host]); `next_batch` (optional) is staged while it
        computes."""
        slot = self.n & 1
        if self._staged != self.n:
            self._stage(x_host, y_host, slot, w_host)
        cur = torch.cuda.current_stream()
        cur.wait_event(self.copied[slot])
        if w_host is not None:
            self.eng.set_row_weights(self.w[slot])
        out = self.step_fn(self.x[slot], self.y[slot], index, lr)
        self.consumed[slot].record(cur)
        self.out_host[slot].copy_(out, non_blocking=True)
        self.out_ready[slot].record(cur)
        self.n += 1
        if next_batch is not None:
            self._stage(next_batch[0], next_batch[1], self.n & 1, next_batch[2] if len(next_batch) > 2 else None)
            self._staged = self.n
        prev = None
        if self.n >= 2:
            self.out_ready[slot ^ 1].synchronize()
            prev = self.out_host[slot ^ 1]
        return prev

    def finish(self):
        slot = (self.n - 1) & 1
        self.out_ready[slot].synchronize()
        return self.out_host[slot]


def gather_batch(table, inp_idx, tar_idx, *, seq_len, stride, inp_cols, fin_cols, seq_norm_col, center, scale,
                 scale_flag, aux_flag, log_squasher=True, aux_masking=False):
    """Device batcher: Dataset.get_batch (scripts/data_processing.py:307-368) over a CUDA-resident fp64 table.

    All array arguments are CUDA tensors: table f64 [n_rows, n_cols]; inp_idx/tar_idx int32 [B,3];
    inp_cols/fin_cols int32; center/scale f64; scale_flag/aux_flag uint8 [F].
    Returns (x f32 [B,T,F], y f32 [B,T,O], seq_norm f64 [B]).
    """
    lib = N.load()
    B = inp_idx.shape[0]
    F, O = inp_cols.numel(), fin_cols.numel()
    dev = table.device
    x = torch.empty(B, seq_len, F, dtype=torch.float32, device=dev)
    y = torch.empty(B, seq_len, O, dtype=torch.float32, device=dev)
    sn = torch.empty(B, dtype=torch.float64, device=dev)
    a = N.LfmqGatherArgs()
    a.struct_size = C.sizeof(N.LfmqGatherArgs)
    a.n_rows, a.n_cols, a.B, a.T, a.F, a.O = table.shape[0], table.shape[1], B, seq_len, F, O
    a.stride = stride
    a.seq_norm_col = -1 if (seq_norm_col is None or int(seq_norm_col) < 0) else int(seq_norm_col)
    a.log_squasher, a.aux_masking = int(bool(log_squasher)), int(bool(aux_masking))
    for name, t, dt in (('table', table, torch.float64), ('inp_idx', inp_idx, torch.int32),
                        ('tar_idx', tar_idx, torch.int32), ('inp_cols', inp_cols, torch.int32),
                        ('fin_cols', fin_cols, torch.int32), ('center', center, torch.float64),
                        ('scale', scale, torch.float64), ('scale_flag', scale_flag, torch.uint8),
                        ('aux_flag', aux_flag, torch.uint8)):
        assert t.is_cuda and t.dtype == dt and t.is_contiguous(), name
        setattr(a, name, t.data_ptr())
    a.x, a.y, a.seq_norm = x.data_ptr(), y.data_ptr(), sn.data_ptr()
    N.check(lib.lfmq_gather_batch(C.byref(a), _stream()))
    return x, y, sn


def row_weights(table, inp_idx, *, weight_col, date_col, halflife, ref_month, out=None):
    """Device row weights of one training batch (lfmq_row_weights, DESIGN.md section 6d): table f64 [n_rows, n_cols] and
    inp_idx int32 [B, 3] CUDA tensors; weight_col < 0 turns the field source off, halflife = 0 the recency source.
    Returns fp32 [B] (or fills out[:B])."""
    for name, t, dt in (('table', table, torch.float64), ('inp_idx', inp_idx, torch.int32)):
        assert t.is_cuda and t.dtype == dt and t.is_contiguous(), name
    B = inp_idx.shape[0]
    w = torch.empty(B, dtype=torch.float32, device=table.device) if out is None else out
    N.check(N.load().lfmq_row_weights(_ptr(table), table.shape[0], table.shape[1], _ptr(inp_idx), B, int(weight_col),
                                      int(date_col), float(halflife), int(ref_month), _ptr(w), _stream()))
    return w


def window_index(key_codes, active, dates, *, train, stride, forecast_n, min_unrollings, max_unrollings, start_date,
                 end_date, last_train_date):
    """Device window index: Dataset._create_tf_dataset + _append_sequence_data (scripts/data_processing.py:170-305).

    key_codes int32 [n] (equal code <=> same gvkey), active uint8 [n], dates int32 [n] (yyyymmdd) -- CUDA tensors;
    the three date bounds are ints in the same encoding.  Returns (inp_idx int32 [N,3], tar_idx int32 [N,3],
    rows int32 [N]) as CUDA tensors, N = number of rows that yield a window, in row order.
    """
    lib = N.load()
    n = key_codes.numel()
    dev = key_codes.device
    for name, t, dt in (('key', key_codes, torch.int32), ('active', active, torch.uint8), ('date', dates, torch.int32)):
        assert t.is_cuda and t.dtype == dt and t.is_contiguous() and t.numel() == n, name
    inp = torch.empty(n, 3, dtype=torch.int32, device=dev)
    tar = torch.empty(n, 3, dtype=torch.int32, device=dev)
    rows = torch.empty(n, dtype=torch.int32, device=dev)
    count = torch.zeros(1, dtype=torch.int32, device=dev)
    work = torch.empty(4 * ((n + 1023) // 1024) + n, dtype=torch.int32, device=dev)
    a = N.LfmqWindowIndexArgs()
    a.struct_size = C.sizeof(N.LfmqWindowIndexArgs)
    a.n, a.train, a.stride, a.forecast_n = n, int(bool(train)), int(stride), int(forecast_n)
    a.min_unrollings, a.max_unrollings = int(min_unrollings), int(max_unrollings)
    a.start_date, a.end_date, a.last_train_date, a.cap = int(start_date), int(end_date), int(last_train_date), n
    a.key, a.active, a.date = key_codes.data_ptr(), active.data_ptr(), dates.data_ptr()
    a.inp_idx, a.tar_idx, a.rows, a.count, a.work = (inp.data_ptr(), tar.data_ptr(), rows.data_ptr(), count.data_ptr(),
                                                     work.data_ptr())
    N.check(lib.lfmq_window_index(C.byref(a), _stream()))
    k = int(count.item())
    return inp[:k], tar[:k], rows[:k]
