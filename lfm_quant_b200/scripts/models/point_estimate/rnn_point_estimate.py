"""RNNPointEstimate (reference: scripts/models/point_estimate/rnn_point_estimate.py:17-154).

Same constructor ``RNNPointEstimate(config, dataset)`` and ``.model`` attribute; the Keras functional graph is
replaced by ``NativeForecaster``: n_layers x [LSTM -> BatchNormalization(inference affine) -> Dropout] -> Dense,
executed by hand-written sm_90a CUDA behind the C-ABI of include/lfmq.h.
"""
from __future__ import absolute_import, division, print_function

import os

import numpy as np

from ..model_base_class import BaseModelClass
from ...model_utils.initializers import Initializer
from ...model_utils.optimizers import Optimizers


class _Variable(object):
    """The slice of tf.Variable the drivers touch: name, shape, numpy()."""

    def __init__(self, model, index, name, shape):
        self._model, self._index, self.name, self.shape = model, index, name + ':0', tuple(shape)

    def numpy(self):
        return self._model.engine.get_weights()[self._index]


class NativeChainForecaster(object):
    """The model object for forecast_steps > 1 (reference :109-150): ``model(inp)`` and ``model.predict(inp)`` return
    the list [pred_1 .. pred_S]; ``train_step`` takes the list of S targets.  Every extra forecast step is one more
    recurrent layer + BatchNormalization + Dropout + Dense over the input window shifted by one, with
    [latest prediction's last time step, last available aux features] appended (models/model_base_class.py:18-51).
    Training-mode graphs run on the fp32 kernels; a forward-only graph (predict.py) may use any precision."""

    uq = False

    def __init__(self, config, seq_len, n_inputs, n_outputs, target_idx):
        from ....engine import ForecastChainEngine
        self.config = config
        if config.rnn_cell not in ('lstm', 'gru'):
            raise NotImplementedError                    # rnn_point_estimate.py:148-149
        precision = getattr(config, 'precision', 'fp32')
        if config.train and precision != 'fp32':
            raise NotImplementedError('forecast_steps > 1 trains on the fp32 kernels (precision=%s)' % precision)
        w = list(config.forecast_steps_weights)
        assert len(w) == config.forecast_steps, 'forecast_steps_weights needs one weight per forecast step'
        self.engine = ForecastChainEngine(
            forecast_steps=config.forecast_steps, weights=w,
            max_batch=config.batch_size, seq_len=seq_len, n_inputs=n_inputs, n_outputs=n_outputs,
            num_hidden=config.num_hidden, num_layers=config.num_layers, target_idx=target_idx,
            train=bool(config.train), precision=precision, optimizer=config.optimizer,
            dropout=config.dropout, recurrent_dropout=config.recurrent_dropout, target_lambda=config.target_lambda,
            rnn_lambda=config.rnn_lambda, max_grad_norm=config.max_grad_norm, max_norm=float(config.max_norm),
            sgd_momentum=config.sgd_momentum, seed=config.seed, forward_only=not config.train,
            rnn_cell=config.rnn_cell)
        specs = [(n, s) for (_, n, s, _, tr) in self.engine.specs if tr]
        self.engine.set_weights(Initializer(config).initial_weights(specs))
        self.trainable_variables = [_Variable(self, i, n, s) for i, (n, s) in enumerate(specs)]
        self._calls = 0

    def __call__(self, inp, training=None):
        self._calls += 1
        return self.engine.forward(self._to_device(inp), step=self._calls)

    def predict_device(self, inp):
        import torch
        x = self._to_device(inp)
        B, mb = x.shape[0], self.engine.cfg.max_batch
        self._calls += 1
        outs = [self.engine.forward(x[s:s + mb].contiguous(), step=self._calls, row0=s) for s in range(0, B, mb)]
        S = self.engine.S
        return [outs[0][k] if len(outs) == 1 else torch.cat([o[k] for o in outs], dim=0) for k in range(S)]

    def predict(self, inp, batch_size=None):
        """model.predict(inp) (train.py:289, predict.py:129): list of S ndarrays [B,T,O]."""
        return [p.cpu().numpy() for p in self.predict_device(inp)]

    def train_step(self, inp, targets, lr, iteration):
        """Train._train_step_point (train.py:178-199) over the S-output graph; device tensor {loss, mse}."""
        assert isinstance(targets, (list, tuple)), 'targets must be the list of forecast_steps targets (train.py:188)'
        return self.engine.train_step(self._to_device(inp), [self._to_device(t) for t in targets], iteration, lr)

    def reset_states(self):
        return None

    def count_params(self):
        return self.engine.n_total

    def summary(self):
        lines = ['Model: "RNNPointEstimate" (native sm_90a, forecast_steps=%d, precision=%s)' % (self.engine.S,
                                                                                                self.engine.precision),
                 '%-44s %-16s %10s' % ('Variable', 'Shape', 'Param #'), '=' * 72]
        for _, name, shape, _, tr in self.engine.specs:
            lines.append('%-44s %-16s %10d%s' % (name, str(tuple(shape)), int(np.prod(shape)), '' if tr else '  (non-trainable)'))
        lines += ['=' * 72, 'Total params: %d' % self.engine.n_total, 'Trainable params: %d' % self.engine.n_trainable]
        return '\n'.join(lines)

    def save_weights(self, prefix):
        from .... import tf_checkpoint
        arrs = self.engine.named_arrays()
        os.makedirs(os.path.dirname(os.path.abspath(prefix)), exist_ok=True)
        with open(prefix + '.lfmq.npz', 'wb') as fh:
            np.savez(fh, **arrs)
        tf_checkpoint.write_keras_checkpoint(prefix, arrs, construction_order=True)

    def load_weights(self, prefix):
        from .... import tf_checkpoint
        names = [n for _, n, _, _, _ in self.engine.specs]
        if os.path.isfile(prefix + '.lfmq.npz'):
            data = np.load(prefix + '.lfmq.npz')
        elif os.path.isfile(prefix + '.index'):
            data = tf_checkpoint.read_keras_checkpoint(prefix, names, {n: tuple(s_) for _, n, s_, _, _ in self.engine.specs},
                                                       construction_order=True)
        else:
            raise FileNotFoundError('no checkpoint at %s (.lfmq.npz or TensorFlow-format .index)' % prefix)
        self.engine.load_named(lambda name: data[name])

    def get_weights(self):
        return self.engine.get_weights(trainable_only=False)


class NativeForecaster(object):
    """Keras-subset model object (SURVEY 8b): __call__, predict, trainable_variables, save/load_weights,
    reset_states, summary -- plus ``train_step`` (the fused native Train._train_step_point)."""

    def __init__(self, config, seq_len, n_inputs, n_outputs, target_idx, uq=False):
        from ....engine import ForecasterEngine
        self.config = config
        self.uq = bool(uq)
        if config.rnn_cell not in ('lstm', 'gru'):
            raise NotImplementedError                    # rnn_point_estimate.py:101-102
        if config.forecast_steps != 1:
            raise NotImplementedError('forecast_steps > 1 is built by NativeChainForecaster (point estimates only)')
        self.engine = ForecasterEngine(
            max_batch=config.batch_size, seq_len=seq_len, n_inputs=n_inputs, n_outputs=n_outputs,
            num_hidden=config.num_hidden, num_layers=config.num_layers, target_idx=target_idx,
            train=bool(config.train), precision=getattr(config, 'precision', 'fp32'), optimizer=config.optimizer,
            dropout=config.dropout, recurrent_dropout=config.recurrent_dropout, target_lambda=config.target_lambda,
            rnn_lambda=config.rnn_lambda, max_grad_norm=config.max_grad_norm, max_norm=float(config.max_norm),
            sgd_momentum=config.sgd_momentum, seed=config.seed, forward_only=not config.train,
            rnn_cell=config.rnn_cell, uq=self.uq)
        specs = [(n, s) for (n, s, _, tr) in self.engine.specs if tr]
        self.engine.set_weights(Initializer(config).initial_weights(specs))
        self.trainable_variables = [_Variable(self, i, n, s) for i, (n, s) in enumerate(specs)]
        self._calls = 0

    # -- forward ---------------------------------------------------------------------------------------
    def _to_device(self, inp):
        import torch
        if isinstance(inp, torch.Tensor):
            return inp.to(self.engine.device, torch.float32).contiguous()
        return torch.from_numpy(np.ascontiguousarray(inp, dtype=np.float32)).to(self.engine.device)

    def __call__(self, inp, training=None):
        """model(inp) (train.py:182): preds [B,T,O] on the device; dropout follows config.train.
        uq model (train.py:204-206): the list [target_preds, variance_preds]; dropout is always on."""
        self._calls += 1
        out = self.engine.forward(self._to_device(inp), step=self._calls)
        return list(out) if self.uq else out

    def predict(self, inp, batch_size=None):
        """model.predict(inp) (train.py:289, predict.py:129): ndarray [B,T,O]."""
        x = self._to_device(inp)
        B = x.shape[0]
        mb = self.engine.cfg.max_batch
        if self.uq:       # every call draws fresh masks: MC dropout (rnn_uq_range_estimate.py:86,88)
            self._calls += 1
            outs = [self.engine.forward(x[s:s + mb].contiguous(), step=self._calls, row0=s) for s in range(0, B, mb)]
            return [np.concatenate([o[k].cpu().numpy() for o in outs], axis=0) for k in (0, 1)]
        # train-mode validation keeps dropout on (the literal training=config.train, rnn_point_estimate.py:87,89) and
        # draws fresh masks per call; rows of later chunks are keyed by their own global row (row0 = s)
        self._calls += 1
        outs = [self.engine.forward(x[s:s + mb].contiguous(), step=self._calls, row0=s).cpu().numpy()
                for s in range(0, B, mb)]
        return np.concatenate(outs, axis=0)

    def predict_device(self, inp):
        """model.predict(inp) without the host copy: a device tensor [B,T,O] (the validation pass keeps everything in
        HBM, train.py:284-336).  Same dropout semantics as predict()."""
        import torch
        assert not self.uq
        x = self._to_device(inp)
        B = x.shape[0]
        mb = self.engine.cfg.max_batch
        self._calls += 1
        outs = [self.engine.forward(x[s:s + mb].contiguous(), step=self._calls, row0=s) for s in range(0, B, mb)]
        return outs[0] if len(outs) == 1 else torch.cat(outs, dim=0)

    def train_step(self, inp, targets, lr, iteration):
        """Fused fwd + loss + BPTT + clip + optimizer + MaxNorm; returns a device tensor {loss, mse_0}."""
        return self.engine.train_step(self._to_device(inp), self._to_device(targets), iteration, lr)

    # -- Keras API surface -------------------------------------------------------------------------------
    def reset_states(self):
        return None                                      # layers are stateless (train.py:105, SURVEY App. B #6)

    def count_params(self):
        return self.engine.n_total

    def summary(self):
        lines = ['Model: "%s" (native sm_90a, precision=%s)' % ('RNNUqRangeEstimate' if self.uq else 'RNNPointEstimate',
                                                                   self.engine.precision),
                 '%-44s %-16s %10s' % ('Variable', 'Shape', 'Param #'), '=' * 72]
        for name, shape, _, tr in self.engine.specs:
            lines.append('%-44s %-16s %10d%s' % (name, str(tuple(shape)), int(np.prod(shape)), '' if tr else '  (non-trainable)'))
        lines += ['=' * 72, 'Total params: %d' % self.engine.n_total, 'Trainable params: %d' % self.engine.n_trainable]
        return '\n'.join(lines)

    @staticmethod
    def _weights_path(prefix):
        return prefix + '.lfmq.npz'

    def save_weights(self, prefix):
        """model.save_weights(<model_dir>/chkpts/chkpt) (train.py:99,171).  Two containers are written side by side:
        ``<prefix>.lfmq.npz`` (Keras-style names in one .npz, this package's native format) and the TF-format
        checkpoint the reference itself writes and reads -- ``<prefix>.index`` + ``<prefix>.data-00000-of-00001`` with
        Keras' object-graph variable keys (lfm_quant_b200/tf_checkpoint.py) -- so the reference's ``load_weights`` can
        address a model trained here."""
        from .... import tf_checkpoint
        flat = self.engine.get_flat()
        arrs = {name: flat[off:off + int(np.prod(shp))].reshape(shp) for name, shp, off, _ in self.engine.specs}
        os.makedirs(os.path.dirname(os.path.abspath(prefix)), exist_ok=True)
        with open(self._weights_path(prefix), 'wb') as fh:
            np.savez(fh, **arrs)
        tf_checkpoint.write_keras_checkpoint(prefix, arrs)

    def load_weights(self, prefix):
        """model.load_weights(prefix) (train.py:87, predict.py:93): the native ``<prefix>.lfmq.npz`` when present, else a
        TF-format checkpoint ``<prefix>.index`` (a model directory trained by the reference)."""
        from .... import tf_checkpoint
        path = self._weights_path(prefix)
        specs = self.engine.specs
        if os.path.isfile(path):
            data = np.load(path)
            get = lambda name: data[name]
        elif os.path.isfile(prefix + '.index'):
            data = tf_checkpoint.read_keras_checkpoint(prefix, [n for n, _, _, _ in specs],
                                                       {n: tuple(s_) for n, s_, _, _ in specs})
            get = lambda name: data[name]
        else:
            raise FileNotFoundError('no checkpoint at %s: neither the native %s nor a TensorFlow-format %s.index '
                                    '(Keras save_weights) exists' % (prefix, os.path.basename(path),
                                                                     os.path.basename(prefix)))
        flat = self.engine.get_flat()
        for name, shp, off, _ in specs:
            w = np.asarray(get(name), dtype=np.float32)
            assert tuple(w.shape) == tuple(shp), (name, w.shape, shp)
            flat[off:off + w.size] = w.ravel()
        self.engine.set_flat(flat)

    def get_weights(self):
        return self.engine.get_weights(trainable_only=False)

    def set_weights(self, weights):
        n_tr = len(self.trainable_variables)
        L = self.config.num_layers
        bn = [(weights[n_tr + 2 * l], weights[n_tr + 2 * l + 1]) for l in range(L)] if len(weights) > n_tr else None
        self.engine.set_weights(weights[:n_tr], bn)


NativeChainForecaster._to_device = NativeForecaster._to_device


class RNNPointEstimate(BaseModelClass):
    """Builds the native recurrent forecaster with the architecture defined in the configs."""

    def __init__(self, config, dataset):
        self.config = config
        self.dataset = dataset
        self.seq_len = self.dataset.seq_len
        self.n_inputs = self.dataset.n_inputs
        self.n_outputs = self.dataset.n_outputs
        self.forecast_steps = self.config.forecast_steps
        self.n_layers = self.config.num_layers
        self.n_hidden_units = self.config.num_hidden
        self.opt = Optimizers(self.config)
        self.initializer = Initializer(self.config)
        super(RNNPointEstimate, self).__init__(self.seq_len, self.n_inputs, self.n_outputs)
        self.model = self._build_model()

    def _build_model(self):
        if self.forecast_steps > 1:                      # reference :109-150
            return NativeChainForecaster(self.config, self.seq_len, self.n_inputs, self.n_outputs,
                                         self.dataset.target_index)
        return NativeForecaster(self.config, self.seq_len, self.n_inputs, self.n_outputs, self.dataset.target_index)
