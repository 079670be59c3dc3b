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

# Rows per launch of the model's wide engine (NativeForecaster._wide_engine), on which predict_mc,
# permutation_importance, shapley and ale run: the width at which one call of 32 samples at B = 256 ran 4x (fp32) to 10x
# (bf16x3) faster than a handle of B rows on an H100 (DESIGN.md section 5c).
MC_ROWS = 8192
# Rows per launch of NativeForecaster.attribute: the saved activations and gradients of the fp32 step grow with the rows
# (DESIGN.md section 5d gives the workspace and the times that chose it).
IG_ROWS = 4096


class _Variable(object):
    """The slice of tf.Variable the drivers touch: name, shape, numpy()."""

    def __init__(self, model, index, name, shape):
        self._model, self._index, self.name, self.shape = model, index, name + ':0', tuple(shape)

    def numpy(self):
        return self._model.engine.get_weights()[self._index]


def _to_device(engine, inp):
    """A tensor or ndarray as a contiguous fp32 tensor on the engine's device."""
    import torch
    if isinstance(inp, torch.Tensor):
        return inp.to(engine.device, torch.float32).contiguous()
    return torch.from_numpy(np.ascontiguousarray(inp, dtype=np.float32)).to(engine.device)


def _keras(outputs):
    """The Keras return convention of model(inp) and model.predict(inp): the output list, unwrapped when it holds one
    output -- a tensor / ndarray for a point model, [tar, var] for a uq model, lists for multi-step forecasts."""
    return outputs[0] if len(outputs) == 1 else outputs


def conformal_intervals(forecast, cal_batches, query_windows, query_forecast, query_targets, levels, knn=0,
                        knn_features=None, pool_batches=None):
    """Split-conformal intervals (DESIGN.md section 5j) of any model: forecast(inp) -> (pred [S,B], scale [S,B] or
    None), device fp32, gives the calibration windows' forecasts, query_forecast the query windows'.  The scores are
    those of engine.conformal_scores; the calibration set is cal_batches ([(inp, target)] with target [B] the normalised
    target field at the window's last step, which is norm_targets_s of every step s).  With knn = K > 0 the scale of a window x is d(x) + beta: d(x) the mean |y_t - pred_t| of
    the K windows of pool_batches nearest to x in knn_features(x) (engine.nearest_topk), beta 0.1 x the mean of
    |y_t - pred_t| over the pool (windows with a finite target only).  Returns the device tensors (n_cal [S], qhat
    [S,Q], lower, upper [S,N,Q], pvalue [S,N], scale [S,N]; scale 1 without one)."""
    import torch
    from ....engine import conformal_apply, conformal_calibrate, conformal_scores, nearest_topk
    pred_c, scale_c, y_c = [], [], []
    for x, y in cal_batches:
        p, sc = forecast(x)
        pred_c.append(p)
        scale_c.append(sc)
        y_c.append(y.to(torch.float32).unsqueeze(0).expand(p.shape[0], -1))
    pred_c, y_c = torch.cat(pred_c, dim=1), torch.cat(y_c, dim=1)
    scale_c = torch.cat(scale_c, dim=1) if scale_c[0] is not None else None
    pred_q, scale_q = query_forecast
    if knn > 0:
        feats, resid = [], []
        for x, y in pool_batches:
            p, _ = forecast(x)
            feats.append(knn_features(x))
            resid.append(conformal_scores(p, y.to(torch.float32).unsqueeze(0))[0])
        feats, resid = torch.cat(feats), torch.cat(resid)
        known = torch.isfinite(resid)
        feats, resid = feats[known].contiguous(), resid[known].contiguous()
        if resid.numel() == 0:
            raise ValueError('conformal: the kNN score needs training windows with known targets')
        beta = torch.tensor(0.1 * float(resid.double().mean()), dtype=torch.float32, device=resid.device)
        k = min(knn, resid.numel())

        def knn_scale(windows):
            return (nearest_topk(knn_features(windows), feats, k, value=resid)[2] + beta).unsqueeze(0).contiguous()
        scale_c = torch.cat([knn_scale(x) for x, _ in cal_batches], dim=1)
        scale_q = knn_scale(query_windows)
    cal = conformal_calibrate(pred_c, y_c, levels, scale=scale_c)
    lower, upper, pvalue = conformal_apply(pred_q, cal, y=query_targets, scale=scale_q)
    scale = scale_q if scale_q is not None else torch.ones_like(pred_q)
    return cal[0], cal[2], lower, upper, pvalue, scale


class NativeForecaster(object):
    """Keras-subset model object (SURVEY 8b) of every trained model kind: __call__, predict, trainable_variables,
    save/load_weights, reset_states, summary -- plus ``train_step`` / ``train_step_dp``, the fused native training step,
    which take the list of forecast_steps targets.

    The engine is a ForecastChainEngine of config.forecast_steps stages (reference :109-150): every extra forecast step
    is one more recurrent layer + BatchNormalization + Dropout + Dense over the input window shifted by one, with
    [latest prediction's last time step, last available aux features] appended (models/model_base_class.py:18-51).
    Multi-step training graphs run on the fp32 kernels (precision 'fp32' or 'tf32'); a forward-only graph (predict.py)
    may use any precision.
    uq=True: RNNUqRangeEstimate's graph (rnn_uq_range_estimate.py:66-110,114-157): the outputs are
    [tar_1, var_1, .., tar_S, var_S] and the step returns {uq_loss_last_tar, mse}."""

    def __init__(self, config, seq_len, n_inputs, n_outputs, target_idx, uq=False):
        self.config = config
        self.uq = bool(uq)
        self.engine = self._build_engine(config, seq_len, n_inputs, n_outputs, target_idx)
        specs = [(n, s) for (_, n, s, _, tr) in self.engine.specs if tr]
        self.trainable_variables = [_Variable(self, i, n, s) for i, (n, s) in enumerate(specs)]
        self._calls = 0
        self._side = {}          # role -> side engine: 'wide' (_wide_engine), 'ig' (_ig_rows_engine)
        self._stale = set()      # the roles whose side engine holds older weights than the model

    @property
    def title(self):
        return 'RNNUqRangeEstimate' if self.uq else 'RNNPointEstimate'

    def _build_engine(self, config, seq_len, n_inputs, n_outputs, target_idx):
        """The engine with its initial weights (Initializer, rnn_point_estimate.py:76-107)."""
        from ....engine import ForecastChainEngine
        if config.rnn_cell not in ('lstm', 'gru'):
            raise NotImplementedError                    # rnn_point_estimate.py:101-102,148-149
        precision = getattr(config, 'precision', 'fp32')
        if config.forecast_steps > 1 and config.train and precision not in ('fp32', 'tf32'):
            raise NotImplementedError('forecast_steps > 1 trains on the fp32 or tf32 kernels (precision=%s)' % precision)
        self._engine_kw = dict(
            forecast_steps=config.forecast_steps, weights=list(config.forecast_steps_weights),
            max_batch=config.batch_size, seq_len=seq_len, n_inputs=n_inputs, n_outputs=n_outputs,
            num_hidden=config.num_hidden, num_layers=config.num_layers, target_idx=target_idx,
            train=bool(config.train), precision=precision, optimizer=config.optimizer,
            dropout=config.dropout, recurrent_dropout=config.recurrent_dropout, target_lambda=config.target_lambda,
            rnn_lambda=config.rnn_lambda, max_grad_norm=config.max_grad_norm, max_norm=float(config.max_norm),
            sgd_momentum=config.sgd_momentum, seed=config.seed, forward_only=not config.train,
            rnn_cell=config.rnn_cell, uq=self.uq)
        engine = ForecastChainEngine(**self._engine_kw)
        engine.set_weights(Initializer(config).initial_weights([(n, s) for (_, n, s, _, tr) in engine.specs if tr]))
        return engine

    # -- forward ---------------------------------------------------------------------------------------
    def __call__(self, inp, training=None):
        """model(inp) (train.py:182,204-206) on the device; dropout follows config.train, on a uq model it is always
        on."""
        self._calls += 1
        return _keras(self.engine.forward(_to_device(self.engine, inp), step=self._calls))

    def predict_device(self, inp):
        """model.predict(inp) without the host copy: the output list of device tensors (the validation pass keeps
        everything in HBM, train.py:284-336).  Train-mode validation keeps dropout on (the literal training=config.train,
        rnn_point_estimate.py:87,89; MC dropout on a uq model, rnn_uq_range_estimate.py:86,88) and every call draws
        fresh masks; rows of later max_batch chunks are keyed by their own global row (row0 = s)."""
        import torch
        x = _to_device(self.engine, inp)
        B, mb = x.shape[0], self.engine.cfg.max_batch
        self._calls += 1
        outs = [self.engine.forward(x[s:s + mb].contiguous(), step=self._calls, row0=s) for s in range(0, B, mb)]
        return [outs[0][k] if len(outs) == 1 else torch.cat([o[k] for o in outs], dim=0) for k in range(len(outs[0]))]

    def predict_mc(self, inp, samples):
        """`samples` Monte-Carlo dropout samples of every window in one prediction, the in-process form of the
        reference's UQ ensemble (runtime/model_execution.py:201-241): per forecast step the device tensors
        (mean_pred, mean_var, var_pred, var_var) [B,T,O].  One step per call, as predict_device; sample 0 is what
        predict_device returns at that step, sample s of window b is keyed by row s * B + b.

        The samples run on an engine with room for min(samples * batch_size, MC_ROWS) rows per launch (_wide_engine),
        so that the samples of a batch share launches; the moments are the same bits on any launch size."""
        if not self.uq:
            raise ValueError('predict_mc needs a uq model (RNNUqRangeEstimate): a point estimate predicts with dropout '
                             'off (training=config.train), so every sample would be the same')
        if int(samples) < 1:
            raise ValueError('predict_mc: samples must be >= 1 (got %r)' % (samples,))
        self._calls += 1
        return self._wide_engine(int(samples) * self.config.batch_size).forward_mc(
            _to_device(self.engine, inp), int(samples), step=self._calls)

    def predict_dist(self, inp, samples, levels, targets=None):
        """predict_mc's samples as each window's predictive mixture (ForecastChainEngine.forward_dist, DESIGN.md
        section 5g): (moments, quantiles, scores) -- moments predict_mc's bit for bit, quantiles [S,B,Q] the mixture's
        quantiles at `levels` and, with targets (the list of forecast_steps targets [B,T,O]), scores [S,B,3] =
        {crps, nll, pit} of the target at the last step, else None.  One step per call, on the engine predict_mc
        uses."""
        if not self.uq:
            raise ValueError('predict_dist needs a uq model (RNNUqRangeEstimate): a point estimate predicts with dropout '
                             'off (training=config.train), so it has no predictive distribution')
        if int(samples) < 1:
            raise ValueError('predict_dist: samples must be >= 1 (got %r)' % (samples,))
        ys = None if targets is None else [_to_device(self.engine, t) for t in targets]
        self._calls += 1
        return self._wide_engine(int(samples) * self.config.batch_size).forward_dist(
            _to_device(self.engine, inp), int(samples), levels, ys=ys, step=self._calls)

    def permutation_importance(self, inp, targets, repeats):
        """Permutation importance of the held-out windows (inp, targets) (ForecastChainEngine.permutation_importance,
        DESIGN.md section 5e): the device tensors (fields [1 + F * repeats, 3], quarters [1 + T * repeats, 3]) of the
        model's loss on the windows as they are (row 0) and with one input field's whole trajectory (column f), or all
        fields of one quarter (t = 0 the oldest), shuffled across the windows, repeat r in row 1 + g * repeats + r.  Rows
        hold {loss, mse_0, 0}, on a uq model {uq_loss, uq_loss_last_tar, mse}.  Both tables use config.seed and one
        step, the model's next call, so row 0 is the same in both and a uq window draws the same dropout masks in
        every copy.  Runs on the wide engine of min(N, MC_ROWS) rows per launch."""
        if int(repeats) < 1:
            raise ValueError('permutation_importance: repeats must be >= 1 (got %r)' % (repeats,))
        x = _to_device(self.engine, inp)
        ys = [_to_device(self.engine, t) for t in targets]
        T, F = self.engine.T, self.engine.F
        self._calls += 1
        eng = self._wide_engine(x.shape[0])
        cols = np.arange(T * F)
        return tuple(eng.permutation_importance(x, ys, groups, int(repeats), self.config.seed, self._calls)
                     for groups in (cols % F, cols // F))

    def shapley(self, inp, samples):
        """Shapley attributions of every window's forecast (ForecastChainEngine.shapley, DESIGN.md section 5f): the
        device tensors (phi_fields [N,K,F], phi_quarters [N,K,T], f_x [N,K], f_bg [N,K]) that split each explained
        output, f_x - f_bg, over the input fields (column f of every quarter) and over the quarters (all fields of
        quarter t, t = 0 the oldest).  The K outputs are norm_preds_s at the last step, and norm_variance_s after each
        on a uq model (tar_1, var_1, ..).  Both partitions use config.seed and one step, the model's next call, so f_x
        and f_bg are the same bits in both; on a uq model f_x is the mean of `samples` Monte-Carlo dropout draws.  Runs
        on the wide engine of min(N, MC_ROWS) rows per launch."""
        if int(samples) < 1:
            raise ValueError('shapley: samples must be >= 1 (got %r)' % (samples,))
        x = _to_device(self.engine, inp)
        T, F = self.engine.T, self.engine.F
        self._calls += 1
        eng = self._wide_engine(x.shape[0])
        cols = np.arange(T * F)
        (phi_f, f_x, f_bg), (phi_q, _, _) = (eng.shapley(x, groups, int(samples), self.config.seed, self._calls)
                                             for groups in (cols % F, cols // F))
        return phi_f, phi_q, f_x, f_bg

    def ale(self, inp, bins):
        """Accumulated local effects of every input field's latest value (ForecastChainEngine.ale, DESIGN.md section
        5h): column (T-1) * F + f of the flattened window for field f, always real data as the batcher pads at the
        front.  The device tensors (n_bins [F], edges [F,K+1], counts [F,K], ale [F,K+1,J], local_mean [F,K,J],
        local_sd [F,K,J]) for K = `bins` requested quantile bins and the J outputs shapley explains.  One step, the
        model's next call, so a uq window draws the same dropout masks in both copies.  Runs on the wide engine of
        min(N, MC_ROWS) rows per launch."""
        if int(bins) < 1:
            raise ValueError('ale: bins must be >= 1 (got %r)' % (bins,))
        x = _to_device(self.engine, inp)
        T, F = self.engine.T, self.engine.F
        self._calls += 1
        eng = self._wide_engine(x.shape[0])
        return eng.ale(x, (T - 1) * F + np.arange(F), int(bins), self._calls)

    def _wide_engine(self, rows):
        """The forward-only engine that predict_mc, permutation_importance, shapley and ale run on: the model's own
        (batch_size rows) when it is as wide as `rows` or MC_ROWS, as at one sample, where a wider handle is slower
        (DESIGN.md section 5c).  Else a forward-only chain of the same stages and precision with max_batch =
        min(rows, MC_ROWS) and the model engine's device share, created at the first such call (again for a larger
        count) and owned by the model.  It holds a copy of the weights, renewed after set_weights, load_weights and the train steps."""
        rows = min(rows, MC_ROWS)
        if rows <= self.engine.cfg.max_batch:
            return self.engine
        return self._side_engine('wide', rows, self._new_wide_engine, share=True)

    def _new_wide_engine(self, rows):
        from ....engine import ForecastChainEngine
        return ForecastChainEngine(**dict(self._engine_kw, max_batch=rows, forward_only=True))

    def _side_engine(self, role, rows, new, share=False):
        """The side engine of `role` with room for `rows` rows per launch: new(rows), created at the first call (again
        for a larger count) and owned by the model, with the model engine's device share when `share`.  Its copy of the
        weights is renewed after _weights_changed."""
        eng = self._side.get(role)
        if eng is None or eng.cfg.max_batch < rows:
            if eng is not None:
                eng.close()
            eng = self._side[role] = new(rows)
            if share and self.engine.device_share is not None:
                eng.set_device_share(*self.engine.device_share)
            self._stale.add(role)
        if role in self._stale:
            for src, dst in zip(self.engine.stages, eng.stages):
                dst.set_flat(src.get_flat())
            self._stale.discard(role)
        return eng

    def _weights_changed(self):
        self._stale = set(self._side)

    # the wide side engine and the handle engine attribute runs on, None while they do not exist
    _mc_engine = property(lambda self: self._side.get('wide'))
    _ig_engine = property(lambda self: self._side['ig'].stages[0] if 'ig' in self._side else None)

    def attribute(self, inp, steps):
        """Integrated-gradients attributions of the point forecast norm_preds_1 = pred[:, T-1, target_idx] of every
        window, against the zero baseline with `steps` midpoint-rule interpolants (ForecasterEngine.integrated_gradients):
        the device tensors (attr [B,T,F], f_x [B], f_base [B]), sum(attr[b]) ~ f_x[b] - f_base[b].  Point estimates with
        forecast_steps = 1 only.  A tf32 model is explained through its tf32 arithmetic; every other precision,
        bf16 and bf16x3 included, through the fp32 arithmetic of the same weights (the bf16 paths form no input
        gradient), so f_x may differ from what model.predict returns by that precision's rounding."""
        if self.uq or self.config.forecast_steps != 1:
            raise ValueError('attribute explains a point estimate with forecast_steps = 1 (got %s, forecast_steps=%d)'
                             % (self.title, self.config.forecast_steps))
        if int(steps) < 1:
            raise ValueError('attribute: steps must be >= 1 (got %r)' % (steps,))
        return self._ig_rows_engine(int(steps)).integrated_gradients(_to_device(self.engine, inp), int(steps))

    def influence(self, pool_batches, query_windows, k):
        """Training-window attributions (_HandleEngine.influence, DESIGN.md section 5i): for every query window the K =
        `k` training windows of pool_batches ([(inp, targets)] device batches, numbered on in order) that push its
        norm_preds_1 (and a UQ model's norm_variance_1) up and down the most, and the summed influence of the whole
        pool, as the device tensors (pos_idx, pos_score, neg_idx, neg_score) [N,J,K] and total [N,J].  forecast_steps = 1
        only.  fp32, tf32 and linear models are explained through their own handle; bf16 and bf16x3 models through an
        fp32 handle with the same parameters (their forecasts may differ from it by that precision's rounding)."""
        if self.config.forecast_steps != 1:
            raise ValueError('influence explains models with forecast_steps = 1 (got %d)' % self.config.forecast_steps)
        eng = self._feature_engine()
        return eng.influence([(_to_device(eng, x), y.contiguous()) for x, y in pool_batches],
                             _to_device(eng, query_windows), int(k))

    def _feature_engine(self):
        """The handle engine of the head-input features (influence, the conformal kNN score): the model's own stage at
        fp32 and tf32 and on the linear model, else an fp32 handle with the same parameters."""
        eng = self.engine.stages[0]
        if getattr(eng, 'precision', 'fp32') not in ('fp32', 'tf32'):
            eng = self._side_engine('influence', self.config.batch_size, self._new_influence_engine).stages[0]
        return eng

    _flat_outputs = False         # model.predict returns [B,T,O] per output

    def conformal_forecast(self, inp):
        """The forecast and its conformal scale (DESIGN.md section 5j) of windows inp, as predict.py writes the
        forecast: (pred [S,B], scale [S,B] or None) device fp32, pred = norm_preds_s.  A point model's scale is None
        (the score is |y - pred|).  A uq model's is sigma: the one sample's at mc_samples = 1 (config.mc_samples),
        else sqrt(mean_var + var_pred) of predict_mc's moments, the mixture's total variance, with pred = mean_pred."""
        import torch
        tidx = self._engine_kw['target_idx']
        pick = (lambda t: t[:, tidx]) if self._flat_outputs else (lambda t: t[:, -1, tidx])      # noqa: E731
        if self.uq and self.config.mc_samples > 1:
            moments = self.predict_mc(inp, self.config.mc_samples)
            pred = [pick(m[0]) for m in moments]
            var = [pick(m[1] + m[2]) for m in moments]
        else:
            outs = self.predict_device(inp)
            pred = [pick(t) for t in (outs[0::2] if self.uq else outs)]
            var = [pick(t) for t in outs[1::2]] if self.uq else None
        pred = torch.stack(pred).contiguous()
        return pred, (torch.sqrt(torch.stack(var)).contiguous() if var is not None else None)

    def conformal(self, cal_batches, query_windows, levels, knn=0, query_forecast=None, query_targets=None,
                  pool_batches=None):
        """Split-conformal intervals (conformal_intervals, DESIGN.md section 5j) of the query windows, calibrated on
        cal_batches ([(inp, targets)] device batches).  query_forecast: the (pred, scale) conformal_forecast gave the
        query windows, when they are already predicted (a uq model draws new dropout masks at every call); else they
        are forecast here.  query_targets [S,N]: the normalised targets, for the p-values.  knn = K > 0 (point and
        linear models with forecast_steps = 1): the normalised score, with neighbours from pool_batches ([(inp, target)],
        the training split), in the head-input features of _feature_engine.  bf16 and bf16x3 models forecast at their own precision."""
        knn_features = None
        if int(knn) > 0:
            if self.uq or self.config.forecast_steps != 1:
                raise ValueError('conformal: the kNN score is for point and linear models with forecast_steps = 1')
            eng = self._feature_engine()
            knn_features = lambda x: eng.influence_features(_to_device(eng, x))[0]     # noqa: E731
        if query_forecast is None:
            query_forecast = self.conformal_forecast(query_windows)
        return conformal_intervals(self.conformal_forecast, cal_batches, query_windows, query_forecast, query_targets,
                                   levels, int(knn), knn_features, pool_batches)

    def _new_influence_engine(self, rows):
        from ....engine import ForecastChainEngine, ForecasterEngine
        kw = {k: v for k, v in self._engine_kw.items() if k not in ('forecast_steps', 'weights')}
        kw.update(max_batch=rows, train=False, forward_only=True, device=self.engine.device, precision='fp32')
        return ForecastChainEngine(stages=[ForecasterEngine(**kw)])

    def _ig_rows_engine(self, steps):
        """The engine attribute runs on: a trainable-mode handle with train = 0 (dropout off) of the model's stage,
        tf32 for a tf32 model and fp32 otherwise, with max_batch = min(steps * batch_size, IG_ROWS).  Created at the first
        call (again for a larger count) and owned by the model; its copy of the weights is renewed after set_weights,
        load_weights and the train steps."""
        return self._side_engine('ig', min(steps * self.config.batch_size, IG_ROWS), self._new_ig_engine).stages[0]

    def _new_ig_engine(self, rows):
        from ....engine import ForecastChainEngine, ForecasterEngine
        kw = {k: v for k, v in self._engine_kw.items() if k not in ('forecast_steps', 'weights')}
        kw.update(max_batch=rows, train=False, forward_only=False, device=self.engine.device,
                  precision='tf32' if kw['precision'] == 'tf32' else 'fp32')
        return ForecastChainEngine(stages=[ForecasterEngine(**kw)])

    def close(self):
        """Releases the device memory of the model's handles."""
        for eng in self._side.values():
            eng.close()
        self._side.clear()
        self.engine.close()

    def predict(self, inp, batch_size=None):
        """model.predict(inp) (train.py:289, predict.py:129): ndarrays [B,T,O], as model(inp) returns them."""
        return _keras([p.cpu().numpy() for p in self.predict_device(inp)])

    def train_step(self, inp, targets, lr, iteration):
        """Fused fwd + loss + BPTT + clip + optimizer + MaxNorm (train.py:178-225); returns the device tensor
        {loss, mse}, on a uq model {uq_loss_last_tar, mse}."""
        assert isinstance(targets, (list, tuple)), 'targets must be the list of forecast_steps targets (train.py:188)'
        self._weights_changed()
        return self.engine.train_step(_to_device(self.engine, inp), [_to_device(self.engine, t) for t in targets],
                                      iteration, lr)

    def train_step_dp(self, x, ys, step, lr, row0, denoms):
        """train_step under data parallelism: this rank's rows (x None: none) with the global loss denominators
        `denoms` (dp.global_denominators of engine.loss_counts), one all-reduce, the replicated apply; returns the global
        values train_step does."""
        if x is not None:
            assert isinstance(ys, (list, tuple)), 'ys must be the list of forecast_steps targets'
            x, ys = _to_device(self.engine, x), [_to_device(self.engine, t) for t in ys]
        self._weights_changed()
        return self.engine.train_step_dp(x, ys, step, lr, row0, denoms)

    # -- Keras API surface -------------------------------------------------------------------------------
    def reset_states(self):
        return None                                      # layers are stateless (train.py:105, SURVEY App. B #6)

    def count_params(self):
        return self.engine.n_total

    def summary(self):
        lines = ['Model: "%s" (native sm_90a, forecast_steps=%d, precision=%s)' % (self.title, self.engine.S,
                                                                                   self.engine.precision),
                 '%-44s %-16s %10s' % ('Variable', 'Shape', 'Param #'), '=' * 72]
        for _, name, shape, _, tr in self.engine.specs:
            lines.append('%-44s %-16s %10d%s' % (name, str(tuple(shape)), int(np.prod(shape)), '' if tr else '  (non-trainable)'))
        lines += ['=' * 72, 'Total params: %d' % self.engine.n_total, 'Trainable params: %d' % self.engine.n_trainable]
        return '\n'.join(lines)

    def save_weights(self, prefix):
        """model.save_weights(<model_dir>/chkpts/chkpt) (train.py:99,171).  Two containers are written side by side:
        ``<prefix>.lfmq.npz`` (Keras-style names in one .npz, this package's native format) and the TF-format
        checkpoint the reference itself writes and reads -- ``<prefix>.index`` + ``<prefix>.data-00000-of-00001`` with
        Keras' object-graph variable keys (lfm_quant_b200/tf_checkpoint.py) -- so the reference's ``load_weights`` can
        address a model trained here.  The layers are numbered in the order the specs list them, which for one stage is
        also the order keras_keys sorts them into."""
        from .... import tf_checkpoint
        arrs = self.engine.named_arrays()
        os.makedirs(os.path.dirname(os.path.abspath(prefix)), exist_ok=True)
        with open(prefix + '.lfmq.npz', 'wb') as fh:
            np.savez(fh, **arrs)
        tf_checkpoint.write_keras_checkpoint(prefix, arrs, construction_order=True)

    def load_weights(self, prefix):
        """model.load_weights(prefix) (train.py:87, predict.py:93): the native ``<prefix>.lfmq.npz`` when present, else a
        TF-format checkpoint ``<prefix>.index`` (a model directory trained by the reference)."""
        from .... import tf_checkpoint
        specs = self.engine.specs
        if os.path.isfile(prefix + '.lfmq.npz'):
            data = np.load(prefix + '.lfmq.npz')
        elif os.path.isfile(prefix + '.index'):
            data = tf_checkpoint.read_keras_checkpoint(prefix, [n for _, n, _, _, _ in specs],
                                                       {n: tuple(s_) for _, n, s_, _, _ in specs}, construction_order=True)
        else:
            raise FileNotFoundError('no checkpoint at %s: neither the native %s.lfmq.npz nor a TensorFlow-format '
                                    '%s.index (Keras save_weights) exists' % (prefix, os.path.basename(prefix),
                                                                              os.path.basename(prefix)))
        self.engine.load_named(lambda name: data[name])
        self._weights_changed()

    def get_weights(self):
        return self.engine.get_weights(trainable_only=False)

    def set_weights(self, weights):
        """The trainable arrays, optionally followed by the BatchNormalization statistics (get_weights' order)."""
        self.engine.set_weights(weights)
        self._weights_changed()


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
        return NativeForecaster(self.config, self.seq_len, self.n_inputs, self.n_outputs, self.dataset.target_index)
