"""Thin Python owner of one native forecaster instance (one per process / GPU).

PyTorch is used for device allocation, streams and torch.distributed only; every piece of arithmetic
happens in lfm_quant_b200/_lfmq.so through the C-ABI of include/lfmq.h.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _native as N


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


class ForecasterEngine(object):
    """fwd / loss / BPTT / clip / optimizer / MaxNorm for RNNPointEstimate on one GPU.

    Mirrors what the reference builds in RNNPointEstimate._build_model
    (scripts/models/point_estimate/rnn_point_estimate.py:40-107) plus the step body of
    Train._train_step_point (scripts/train.py:178-199).
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
        cfg.precision = {'fp32': N.PREC_FP32, 'bf16': N.PREC_BF16, 'bf16x3': N.PREC_BF16X3}[precision]
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
        self.grads = self._view('lfmq_grads_ptr', self.n_trainable + 8)   # tail: loss, mse_0, grad_norm, clip_scale, uq_loss_last_tar
        self._denom = torch.zeros(2, dtype=torch.float32, device=self.device)

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

    def loss(self, preds, y):
        out = torch.empty(2, dtype=torch.float32, device=preds.device)
        N.check(self.lib.lfmq_loss(self.handle, _ptr(preds.contiguous()), _ptr(y.contiguous()), preds.shape[0],
                                   _ptr(out), _stream()))
        return out

    def loss_uq(self, preds, var, y):
        """Device tensor {uq_loss, uq_loss_last_tar, mse_0} (Losses.weight_adjusted_uq_loss, losses.py:137-284)."""
        out = torch.empty(3, dtype=torch.float32, device=preds.device)
        N.check(self.lib.lfmq_loss_uq(self.handle, _ptr(preds.contiguous()), _ptr(var.contiguous()), _ptr(y.contiguous()),
                                      preds.shape[0], _ptr(out), _stream()))
        return out

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

    def backward(self, x, y, step=0, row0=0, denom=None):
        B = self._check_x(x)
        assert y.is_cuda and y.dtype == torch.float32 and y.is_contiguous() and tuple(y.shape) == (B, self.T, self.O)
        N.check(self.lib.lfmq_backward(self.handle, _ptr(x), _ptr(y), B, row0, step, _ptr(denom), _stream()))

    def apply(self, lr, iteration):
        N.check(self.lib.lfmq_apply(self.handle, float(lr), int(iteration), _stream()))

    def train_step(self, x, y, step, lr, out=None):
        """One Train._train_step_point on this GPU; returns a device tensor {loss, mse_0} (no host sync).
        uq engine: one Train._train_step_uq_range, {uq_loss_last_tar, mse_0} (train.py:225)."""
        B = self._check_x(x)
        if out is None:
            out = torch.empty(2, dtype=torch.float32, device=x.device)
        N.check(self.lib.lfmq_train_step(self.handle, _ptr(x), _ptr(y), B, 0, step, float(lr), _ptr(out), _stream()))
        return out

    def train_step_dp(self, x, y, step, lr, row0, denom_global):
        """Data-parallel step: local BPTT with global denominators, ONE NCCL all-reduce over the flat
        gradient (+ loss/mse tail), then the replicated clip + optimizer (SURVEY 8e)."""
        import torch.distributed as dist
        from .dp import allreduce_flat_gradient
        self.backward(x, y, step=step, row0=row0, denom=denom_global)
        allreduce_flat_gradient(self.grads, self.n_trainable, dist)
        self.apply(lr, step)
        return self.grads[self.n_trainable:self.n_trainable + 2].clone()   # not a live view of the workspace tail

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


class ForecastChainEngine(object):
    """forecast_steps > 1 (scripts/models/point_estimate/rnn_point_estimate.py:109-150): stage 0 is the trunk, every
    further stage one more recurrent layer + BatchNormalization + Dropout + Dense on the shifted input window.  One
    ForecasterEngine (one C-ABI handle) per stage; the lfmq_chain_* entry points run the whole graph."""

    def __init__(self, *, forecast_steps, weights, num_layers, **kw):
        assert forecast_steps >= 1
        self.S = int(forecast_steps)
        self.stages = [ForecasterEngine(num_layers=num_layers if s == 0 else 1, **kw) for s in range(self.S)]
        e0 = self.stages[0]
        self.lib, self.device, self.cfg, self.precision = e0.lib, e0.device, e0.cfg, e0.precision
        self.T, self.F, self.O, self.H, self.L = e0.T, e0.F, e0.O, e0.H, e0.L
        self.weights = [float(w) for w in weights]
        assert len(self.weights) == self.S, (self.weights, self.S)
        self._handles = (C.c_void_p * self.S)(*[e.handle.value for e in self.stages])
        self._w = (C.c_float * self.S)(*self.weights)
        self._work = None
        # Keras names: the extra layer of stage s is lstm_{L+s} / batch_normalization_{L+s-1} / OUTPUT_{s+1}
        self.specs = []            # (stage, name, shape, offset in the stage's flat vector, trainable)
        cell = kw.get('rnn_cell', 'lstm')
        for s, e in enumerate(self.stages):
            for name, shp, off, tr in e.specs:
                if s > 0:
                    name = name.replace('%s_1/' % cell, '%s_%d/' % (cell, self.L + s))
                    name = name.replace('batch_normalization/', 'batch_normalization_%d/' % (self.L + s - 1))
                    name = name.replace('OUTPUT_1/', 'OUTPUT_%d/' % (s + 1))
                self.specs.append((s, name, shp, off, tr))
        self.n_total = sum(e.n_total for e in self.stages)
        self.n_trainable = sum(e.n_trainable for e in self.stages)

    def _ptrs(self, tensors):
        return (C.c_void_p * self.S)(*[t.data_ptr() for t in tensors])

    def _workbuf(self, B):
        n = self.S * B * self.T * self.F
        if self._work is None or self._work.numel() < n:
            self._work = torch.empty(n, dtype=torch.float32, device=self.device)
        return self._work

    def forward(self, x, step=0, row0=0):
        """model(inp) -> [pred_1 .. pred_S], device tensors [B,T,O]."""
        B = self.stages[0]._check_x(x)
        preds = [torch.empty(B, self.T, self.O, dtype=torch.float32, device=x.device) for _ in range(self.S)]
        N.check(self.lib.lfmq_chain_forward(self._handles, self.S, _ptr(x), B, row0, step, self._ptrs(preds),
                                            _ptr(self._workbuf(B)), _stream()))
        return preds

    def loss(self, preds, ys):
        """Losses.weight_adjusted_mse(ys, preds): device tensor {loss, mse}."""
        out = torch.empty(2, dtype=torch.float32, device=preds[0].device)
        preds = [p.contiguous() for p in preds]
        ys = [y.contiguous() for y in ys]
        N.check(self.lib.lfmq_chain_loss(self._handles, self.S, self._ptrs(preds), self._ptrs(ys), self._w,
                                         preds[0].shape[0], _ptr(out), _stream()))
        return out

    def backward(self, x, ys, step=0, row0=0, out=None):
        B = self.stages[0]._check_x(x)
        assert len(ys) == self.S
        for y in ys:
            assert y.is_cuda and y.dtype == torch.float32 and y.is_contiguous() and tuple(y.shape) == (B, self.T, self.O)
        if out is None:
            out = torch.empty(2, dtype=torch.float32, device=x.device)
        N.check(self.lib.lfmq_chain_backward(self._handles, self.S, _ptr(x), self._ptrs(ys), self._w, B, row0, step,
                                             _ptr(self._workbuf(B)), _ptr(out), _stream()))
        return out

    def apply(self, lr, iteration):
        N.check(self.lib.lfmq_chain_apply(self._handles, self.S, float(lr), int(iteration), _stream()))

    def train_step(self, x, ys, step, lr):
        """One Train._train_step_point over the S-output model; device tensor {loss, mse}."""
        out = self.backward(x, ys, step=step)
        self.apply(lr, step)
        return out

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
        """weights in trainable_variables order: the trunk's, then 7 per extra stage."""
        i = 0
        for e in self.stages:
            n = len(e.trainable_specs)
            e.set_weights(weights[i:i + n])
            i += n
        assert i == len(weights)

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
        self.step_fn = step_fn or (lambda x, y, i, lr: engine.train_step(x, y, i, lr))
        self.n = 0
        self._staged = None

    def _stage(self, x_host, y_host, slot):
        with torch.cuda.stream(self.copy_stream):
            if self.n >= 2:
                self.copy_stream.wait_event(self.consumed[slot])      # the step that used this buffer is done
            self.x[slot].copy_(x_host, non_blocking=True)
            self.y[slot].copy_(y_host, non_blocking=True)
            self.copied[slot].record(self.copy_stream)

    def step(self, x_host, y_host, index, lr, next_batch=None):
        """Runs one step on (x_host, y_host); `next_batch` (optional) is staged while it computes."""
        slot = self.n & 1
        if self._staged != self.n:
            self._stage(x_host, y_host, slot)
        cur = torch.cuda.current_stream()
        cur.wait_event(self.copied[slot])
        out = self.step_fn(self.x[slot], self.y[slot], index, lr)
        self.consumed[slot].record(cur)
        self.out_host[slot].copy_(out, non_blocking=True)
        self.out_ready[slot].record(cur)
        self.n += 1
        if next_batch is not None:
            self._stage(next_batch[0], next_batch[1], self.n & 1)
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
