"""Predict driver (reference: scripts/predict.py:27-300): load weights, forward every test batch, keep
``pred[:, -1, target_index]``, undo the scaling, write ``<model_dir>/pred/<preds_fname>`` with the reference's
column order (predict.py:113-126,148-157,174-182,214-259; SURVEY section 8b "Files")."""
from __future__ import absolute_import, division, print_function

import io
import os
import pathlib
from collections import defaultdict

import numpy as np
import pandas as pd

from .base_config import conformal_levels, pred_quantile_levels
from .model_utils.model import Model


class Predict(object):

    def __init__(self, config, dataset):
        self.config = config
        assert not self.config.train, 'Predict can only be instantiated when config.train is False'
        self.dataset = dataset
        self.dataset.generate_dataset()
        self.model = Model(self.config, self.dataset).get_model()
        self.target_index = self.dataset.target_index
        self.seq_len = self.dataset.seq_len
        self.n_inputs = self.dataset.n_inputs
        self.test_set = self.dataset.test_set.batch(batch_size=self.config.batch_size)
        self.model_dir = os.path.join(self.config.experiments_dir, self.config.model_dir)
        self.chkpts_dir = os.path.join(self.model_dir, 'chkpts')
        if not os.path.isdir(self.model_dir):
            os.mkdir(self.model_dir)
        print('creating preds directory')
        self.pred_dir = os.path.join(self.model_dir, 'pred')
        if 'Naive' not in self.config.nn_type:
            assert os.path.isdir(self.chkpts_dir), 'No checkpoint dir found to load the model'
        if not os.path.isdir(self.pred_dir):
            pathlib.Path(self.pred_dir).mkdir(parents=True, exist_ok=True)
        print("Creating batches ...")
        self._batches = [self.dataset.get_batch(*items) for items in self.test_set]

    def predict(self):
        if 'Naive' not in self.config.nn_type:            # predict.py:90-93: the naive forecast has no variables
            self.model.load_weights(os.path.join(self.chkpts_dir, "chkpt"))
        outputs = defaultdict(list)
        ig = defaultdict(list)
        held_out = []
        windows = []
        levels = pred_quantile_levels(getattr(self.config, 'pred_quantiles', None))
        dist = defaultdict(list)
        conf_levels = conformal_levels(getattr(self.config, 'conformal_levels', None))
        conf = defaultdict(list)          # the forecast and its variance that preds.dat holds, per step [B]
        factor_inp = []                   # the normalised inp_t0 of each window when preds.dat does not hold it
        for (inp_dev, target_dev, metadata) in self._batches:
            # one target window per input window: every forecast step is compared with it (Train._step_targets)
            inp, targets = inp_dev.cpu().numpy(), [target_dev.cpu().numpy()] * self.config.forecast_steps
            outputs['date'].append(np.expand_dims(metadata[:, 0].astype('int32'), -1))
            outputs['gvkey'].append(np.expand_dims(metadata[:, 1], -1))
            outputs['seq_norm'].append(np.expand_dims(metadata[:, 2].astype('float32'), -1))
            if self.config.write_inp_to_out_file:
                for i, t_step in enumerate(range(1 - self.seq_len, 1)):
                    outputs['inp_t' + str(t_step)].append(self._extract_inputs(inp, i))
            elif self._factor_q() > 0:      # qfm's current value, not written to preds.dat
                factor_inp.append(self._extract_inputs(inp, self.seq_len - 1))
            outputs['targets'].append(self._extract_targets(targets))
            if not self.config.UQ:      # predict.py:128-133: model.predict returns a list when forecast_steps > 1
                preds = self.model.predict(inp_dev)
                if self.config.forecast_steps == 1:
                    preds = [preds]
                variance = [np.zeros(x.shape) for x in preds]   # predict.py:133
            elif self.config.mc_samples > 1 or levels is not None:
                if levels is None:
                    moments = self.model.predict_mc(inp_dev, self.config.mc_samples)
                else:           # the same samples and moments, and each window's mixture (quantiles.dat)
                    moments, q, scores = self.model.predict_dist(inp_dev, self.config.mc_samples, levels,
                                                                 [target_dev] * self.config.forecast_steps)
                    dist['quantiles'].append(q.cpu().numpy())
                    dist['scores'].append(scores.cpu().numpy())
                moments = [[t.cpu().numpy() for t in m] for m in moments]
                preds = [m[0] for m in moments]
                conf_var = [m[1] + m[2] for m in moments]      # the mixture's total variance (DESIGN.md 5j)
                if self.config.mc_samples > 1:
                    # the reference's UQ ensemble in one prediction: the mean of the samples, and mean of the
                    # variances + variance of the variances (utils/post_processing.py:52-55); var_pred, the spread of
                    # the sampled predictions, is the one added column
                    variance = [m[1] + m[3] for m in moments]
                    outputs['norm_preds_var'].append(self._extract_preds([m[2] for m in moments]))
                else:           # one sample: its prediction and variance, the bits model.predict returns
                    variance = conf_var = [m[1] for m in moments]
            else:                       # predict.py:135-138: [tar_1, var_1, .., tar_S, var_S]
                model_preds = self.model.predict(inp_dev)
                preds, variance = model_preds[0::2], model_preds[1::2]
                conf_var = variance
            outputs['norm_preds'].append(self._extract_preds(preds))
            if conf_levels is not None:
                conf['pred'].append(np.concatenate(self._extract_preds(preds), axis=1).T)
                if self.config.UQ:
                    conf['var'].append(np.concatenate(self._extract_preds(conf_var), axis=1).T)
            outputs['norm_variance'].append(self._extract_preds(variance))
            if self.config.ig_steps > 0:
                for key, t in zip(('attr', 'f_x', 'f_base'), self.model.attribute(inp_dev, self.config.ig_steps)):
                    ig[key].append(t.cpu().numpy())
            if self.config.perm_importance > 0:
                held_out.append((inp_dev, target_dev))
            if (self.config.shapley_samples > 0 or self.config.ale_bins > 0 or self._influence_k() > 0
                    or (conf_levels is not None and getattr(self.config, 'conformal_knn', 0) > 0)):
                windows.append(inp_dev)
        if self.config.ig_steps > 0:
            self._write_attributions(outputs, ig)
        if self.config.perm_importance > 0:
            self._write_importance(held_out)
        if self.config.shapley_samples > 0:
            self._write_shapley(outputs, windows)
        if self.config.ale_bins > 0:
            self._write_ale(windows)
        if self._influence_k() > 0:
            self._write_influence(outputs, windows)

        single_outputs = ['date', 'gvkey', 'seq_norm'] + [x for x in outputs.keys() if 'inp_t' in x]
        for key in single_outputs:
            outputs[key] = np.vstack(outputs[key])
        for key in [k for k in ('targets', 'norm_preds', 'norm_variance', 'norm_preds_var') if k in outputs]:
            for i in range(self.config.forecast_steps):
                outputs[key + '_' + str(i + 1)] = np.vstack([x[i] for x in outputs[key]])
            outputs.pop(key)
        outputs = {k: v.flatten() for k, v in outputs.items()}

        df = pd.DataFrame.from_dict(outputs)
        try:
            df['date'] = pd.to_datetime(df['date'].astype(str), format="%Y%m%d")
        except ValueError:
            print("Input date is not in the '%Y%m%d' format")
            raise
        scale = self.dataset.scaling_params['scale'][self.target_index]
        center = self.dataset.scaling_params['center'][self.target_index]

        def unscale(col):
            """reverse centre/scale, log squash and seq_norm (predict.py:184-247)."""
            v = np.multiply(np.asarray(col, dtype=np.float64), scale) + center
            if self.config.log_squasher:
                v = self.dataset.reverse_log_squasher(v)
            return v * df['seq_norm'].values.astype(np.float64)

        tar_cols = [x for x in df.columns if 'targets' in x]
        for tar_c in tar_cols:
            step = tar_c.split('_')[-1]
            df['norm_' + tar_c] = df[tar_c]
            df['norm_squared_diff_' + step] = np.square(df['norm_' + tar_c] - df['norm_preds_' + step])
        for tar_c in tar_cols:
            df[tar_c] = unscale(df[tar_c])
        if self.config.write_inp_to_out_file:
            for c in [x for x in df.columns if 'inp_t' in x]:
                df[c] = unscale(df[c])
        preds_keys = [x for x in df.columns if 'norm_preds_' in x and 'norm_preds_var_' not in x]
        for pred_key in preds_keys:
            df['preds_' + pred_key.split('_')[-1]] = unscale(df[pred_key])
        for var_key in [x for x in df.columns if 'norm_variance_' in x]:
            df['variance_' + var_key.split('_')[-1]] = unscale(df[var_key])     # not zero: SURVEY App. B #8
        for o_key in [x.split('_')[-1] for x in preds_keys]:
            df['fcst_err_' + o_key] = ((df['targets_' + o_key] - df['preds_' + o_key]) / df['targets_' + o_key]).abs()
            df['abs_err_' + o_key] = (df['targets_' + o_key] - df['preds_' + o_key]).abs()
            df['unscaled_squared_err_' + o_key] = np.square(df['abs_err_' + o_key] / df['seq_norm'])

        df['gvkey'] = df['gvkey'].apply(lambda x: x.decode('utf-8') if isinstance(x, bytes) else str(x))
        df.to_csv(os.path.join(self.pred_dir, self.config.preds_fname), sep=' ', index=False, date_format="%Y%m%d")
        if levels is not None:
            self._write_quantiles(df, levels, np.concatenate(dist['quantiles'], axis=1),
                                  np.concatenate(dist['scores'], axis=1), unscale)
        if conf_levels is not None:
            self._write_conformal(df, conf_levels, conf, windows, unscale)
        if self._factor_q() > 0:
            self._write_factor(df, unscale(np.vstack(factor_inp).flatten()) if factor_inp else None)
        print("Unscaled MSE normalized by Seq_Norm (%s)" % self.config.model_dir.split('/')[-1])
        print(df[[x for x in df.columns if 'unscaled' in x]].mean())
        for i in range(self.config.forecast_steps):
            print("Scaled MSE for step %i: %1.4f" % (i + 1, df['norm_squared_diff_' + str(i + 1)].mean()))
        return df

    def _write_quantiles(self, df, levels, quantiles, scores, unscale):
        """<model_dir>/pred/quantiles.dat and calibration.dat (--pred_quantiles): the predictive quantiles and scores
        of every row of preds.dat (`df`, in its order) from NativeForecaster.predict_dist (quantiles [S,N,Q], scores
        [S,N,3]); quantile_table and calibration_table give the layouts."""
        targets = np.stack([df['norm_targets_%d' % (s + 1)].to_numpy() for s in range(len(quantiles))])
        quantile_table(df[['date', 'gvkey']], levels, quantiles, scores, unscale).to_csv(
            os.path.join(self.pred_dir, 'quantiles.dat'), sep=' ', index=False, date_format="%Y%m%d")
        calibration_table(levels, quantiles, scores, targets).to_csv(
            os.path.join(self.pred_dir, 'calibration.dat'), sep=' ', index=False)

    def _write_attributions(self, outputs, ig):
        """<model_dir>/pred/attributions.npz: the integrated-gradients attributions of norm_preds_1 (--ig_steps), one
        row per preds.dat row in its order -- date [N] (yyyymmdd), gvkey [N], fields [F] (the input fields in the
        Dataset's column order), attr [N,T,F], f_x [N] and f_base [N] (the forecast at the window and at the zero
        baseline)."""
        gvkey = np.vstack(outputs['gvkey']).flatten()
        np.savez(os.path.join(self.pred_dir, 'attributions.npz'),
                 date=np.vstack(outputs['date']).flatten().astype(np.int32),
                 gvkey=np.array([g.decode('utf-8') if isinstance(g, bytes) else str(g) for g in gvkey]),
                 fields=np.array(self.dataset.fin_col_names + self.dataset.aux_col_names),
                 **{k: np.concatenate(v).astype(np.float32) for k, v in ig.items()})

    def _write_importance(self, held_out):
        """<model_dir>/pred/importance.dat (--perm_importance R): the permutation importance of every input field and
        quarter on the predicted windows (NativeForecaster.permutation_importance over all batches at once, seeded by
        config.seed), one row per group (importance_table).  Only the windows whose targets are all known count: the
        batcher fills the targets that lie past the data with NaN, and one NaN makes the loss NaN."""
        import torch
        x = torch.cat([b[0] for b in held_out])
        y = torch.cat([b[1] for b in held_out])
        known = torch.isfinite(y.reshape(y.shape[0], -1)).all(dim=1)
        if not bool(known.any()):
            raise ValueError('--perm_importance: no predicted window has known targets, so there is no loss to measure')
        x, y = x[known].contiguous(), y[known].contiguous()
        R = self.config.perm_importance
        fields, quarters = self.model.permutation_importance(x, [y] * self.config.forecast_steps, R)
        df = importance_table(fields.cpu().numpy(), quarters.cpu().numpy(), R,
                              self.dataset.fin_col_names + self.dataset.aux_col_names, self.config.UQ)
        df.to_csv(os.path.join(self.pred_dir, 'importance.dat'), sep=' ', index=False)

    def _write_shapley(self, outputs, windows):
        """<model_dir>/pred/shapley.npz (--shapley_samples M): the Shapley attributions of every predicted window, known
        targets or not, in preds.dat's row order (NativeForecaster.shapley over all batches at once, seeded by
        config.seed; write_shapley gives the layout)."""
        import torch
        phi_f, phi_q, f_x, f_bg = (t.cpu().numpy() for t in
                                   self.model.shapley(torch.cat(windows), self.config.shapley_samples))
        write_shapley(os.path.join(self.pred_dir, 'shapley.npz'), np.vstack(outputs['date']).flatten(),
                      np.vstack(outputs['gvkey']).flatten(), self.dataset.fin_col_names + self.dataset.aux_col_names,
                      shapley_output_names(self.config.forecast_steps, self.config.UQ), phi_f, phi_q, f_x, f_bg)

    def _write_ale(self, windows):
        """<model_dir>/pred/ale.dat (--ale_bins K): the accumulated local effects of every input field's latest value
        over every predicted window, known targets or not (NativeForecaster.ale over all batches at once; ale_table
        gives the layout)."""
        import torch
        out = [t.cpu().numpy() for t in self.model.ale(torch.cat(windows), self.config.ale_bins)]
        ale_table(self.dataset.fin_col_names + self.dataset.aux_col_names,
                  shapley_output_names(self.config.forecast_steps, self.config.UQ), *out).to_csv(
            os.path.join(self.pred_dir, 'ale.dat'), sep=' ', index=False)

    def _influence_k(self):
        return int(getattr(self.config, 'influence_top_k', 0))

    def _write_influence(self, outputs, windows):
        """<model_dir>/pred/influence.npz (--influence_top_k K): for every predicted window, known targets or not, the K
        windows of the training split that push its forecast up and down the most (NativeForecaster.influence).  The
        pool is the training split a --train=True run with this run's flags draws, with this model's scales.dat; in a
        walk-forward run the origin's own (pool_dates).  write_influence gives the layout."""
        import torch
        pool = self._training_draw()
        batches = [pool.get_batch(*items) for items in pool.train_set.batch(batch_size=self.config.batch_size)]
        meta = np.concatenate([m for _, _, m in batches])
        tgt = torch.cat([(y if y.dim() == 2 else y[:, -1]) for _, y, _ in batches])[:, self.target_index]
        res = self.model.influence([(x, y) for x, y, _ in batches], torch.cat(windows), self._influence_k())
        write_influence(os.path.join(self.pred_dir, 'influence.npz'), np.vstack(outputs['date']).flatten(),
                        np.vstack(outputs['gvkey']).flatten(),
                        shapley_output_names(1, self.config.UQ), meta[:, 0].astype('int32'), meta[:, 1],
                        tgt.cpu().numpy(), *[t.cpu().numpy() for t in res])

    def _training_draw(self):
        """The Dataset a --train=True run with this run's flags draws (its training and validation splits), with this
        model's scales.dat; in a walk-forward run the origin's own (pool_dates)."""
        import copy
        cfg = copy.deepcopy(self.config)
        cfg.train = True
        if getattr(self.config, 'pool_dates', None):
            cfg.start_date, cfg.end_date = self.config.pool_dates
        pool = type(self.dataset)(cfg)
        pool.generate_dataset()
        return pool

    def _target_batches(self, index_set, pool):
        """[(inp, target [B])] device batches of an IndexSet of `pool`, with each window's normalised target field at
        its last step (norm_targets_s), and the windows' metadata."""
        batches = [pool.get_batch(*items) for items in index_set.batch(batch_size=self.config.batch_size)]
        pairs = [(x, (y if y.dim() == 2 else y[:, -1])[:, self.target_index].contiguous()) for x, y, _ in batches]
        meta = np.concatenate([m for _, _, m in batches]) if batches else np.zeros((0, 3), dtype=object)
        return pairs, meta

    def _write_conformal(self, df, levels, conf, windows, unscale):
        """<model_dir>/pred/intervals.dat and coverage.dat (--conformal_levels): split-conformal intervals of every
        row of preds.dat (`df`), calibrated on the validation split of _training_draw (NativeForecaster.conformal,
        DESIGN.md section 5j); interval_table and coverage_table give the layouts."""
        import torch
        pool = self._training_draw()
        cal, cal_meta = self._target_batches(pool.valid_set, pool)
        if not cal:
            raise ValueError('--conformal_levels: the validation split of the training draw has no windows to '
                             'calibrate on (validation_size = %s)' % self.config.validation_size)
        knn = int(getattr(self.config, 'conformal_knn', 0))
        train = self._target_batches(pool.train_set, pool)[0] if knn > 0 else None
        dev = cal[0][0].device
        pred = torch.from_numpy(np.concatenate(conf['pred'], axis=1)).to(dev)
        scale = (torch.sqrt(torch.from_numpy(np.concatenate(conf['var'], axis=1)).to(dev))
                 if self.config.UQ else None)
        S = pred.shape[0]
        targets = np.stack([df['norm_targets_%d' % (s + 1)].to_numpy(dtype=np.float32) for s in range(S)])
        n_cal, qhat, lower, upper, pvalue, scale = (t.cpu().numpy() for t in self.model.conformal(
            cal, torch.cat(windows) if knn > 0 else None, levels, knn=knn, query_forecast=(pred, scale),
            query_targets=torch.from_numpy(targets).to(dev), pool_batches=train))
        seq_norm = df['seq_norm'].to_numpy(dtype=np.float64)
        interval_table(df[['date', 'gvkey']], levels, lower, upper, scale, pvalue, seq_norm, unscale).to_csv(
            os.path.join(self.pred_dir, 'intervals.dat'), sep=' ', index=False, date_format="%Y%m%d")
        date = np.asarray([int(d.strftime('%Y%m%d')) for d in df['date']], dtype=np.int64)
        gvkey = df['gvkey'].astype(str).to_numpy()
        subset = conformal_subsets(date, gvkey, cal_meta[:, 0].astype(np.int64),
                                   [g.decode('utf-8') if isinstance(g, bytes) else str(g) for g in cal_meta[:, 1]],
                                   set(str(g) for g in pool._train_gvkeys), int(pool.config.end_date))
        coverage_table(levels, subset, n_cal, qhat, pred.cpu().numpy(), targets, scale, lower, upper, seq_norm,
                       unscale).to_csv(os.path.join(self.pred_dir, 'coverage.dat'), sep=' ', index=False)

    def _factor_q(self):
        return int(getattr(self.config, 'factor_quantiles', 0))

    def _write_factor(self, df, inp_t0):
        """<model_dir>/pred/factor_dates.dat and factor.dat (--factor_quantiles Q): the lookahead factor backtest of
        the rows of preds.dat (`df`; inp_t0 the fundamentals-unit inp_t0 when df does not hold it); factor_tables,
        factor_dates_table and factor_summary give the layouts."""
        per_date, summary = factor_tables(df, self.config, inp_t0)
        per_date.to_csv(os.path.join(self.pred_dir, 'factor_dates.dat'), sep=' ', index=False)
        summary.to_csv(os.path.join(self.pred_dir, 'factor.dat'), sep=' ', index=False)

    def _flat(self):
        """MLP* / Naive* batches are 2-D: targets [B, O], inputs [B, T*F] (predict.py:275-300)."""
        return 'MLP' in self.config.nn_type or 'Naive' in self.config.nn_type

    def _extract_targets(self, targets):
        if self._flat():
            return [np.expand_dims(x[:, self.target_index], -1) for x in targets]
        return [np.expand_dims(x[:, -1, self.target_index], -1) for x in targets]

    def _extract_preds(self, preds):
        if self._flat():
            return [np.expand_dims(x[:, self.target_index], -1) for x in preds]
        return [np.expand_dims(x[:, -1, self.target_index], -1) for x in preds]

    def _extract_inputs(self, inp, i):
        if self._flat():                                 # step i of the target field: column i * F + target_index
            return np.expand_dims(inp[:, i * self.n_inputs + self.target_index], -1)
        return np.expand_dims(inp[:, i, self.target_index], -1)


def importance_table(fields, quarters, repeats, field_names, uq):
    """The rows of importance.dat from the two outputs of NativeForecaster.permutation_importance (fields
    [1 + F * repeats, 3], quarters [1 + T * repeats, 3]): the fields in Dataset order, then the quarters from the oldest
    (group 1 - T, as inp_t<k> numbers them) to the latest (0).  base_* is the unpermuted row, perm_* the mean over the
    repeats (perm_loss_std their population standard deviation) and delta_* = perm_* - base_*.  The loss is column 0
    (uq_loss on a uq model) and the mse column 1, column 2 on a uq model."""
    mse = 2 if uq else 1
    frames = []
    for kind, out, names in (('field', fields, list(field_names)),
                             ('quarter', quarters, list(range(1 - (len(quarters) - 1) // repeats, 1)))):
        out = np.asarray(out, dtype=np.float64)
        perm = out[1:].reshape(len(names), repeats, 3)
        base_loss, base_mse = out[0, 0], out[0, mse]
        perm_loss, perm_mse = perm[:, :, 0].mean(axis=1), perm[:, :, mse].mean(axis=1)
        frames.append(pd.DataFrame({'kind': kind, 'group': names, 'base_loss': base_loss, 'perm_loss': perm_loss,
                                    'perm_loss_std': perm[:, :, 0].std(axis=1), 'delta_loss': perm_loss - base_loss,
                                    'base_mse': base_mse, 'perm_mse': perm_mse, 'delta_mse': perm_mse - base_mse}))
    return pd.concat(frames, ignore_index=True)


def shapley_output_names(forecast_steps, uq):
    """The outputs NativeForecaster.shapley explains, as preds.dat names their normalised columns: norm_preds_s, and
    on a uq model norm_variance_s after each."""
    kinds = ('norm_preds', 'norm_variance') if uq else ('norm_preds',)
    return ['%s_%d' % (k, s) for s in range(1, forecast_steps + 1) for k in kinds]


def write_shapley(path, date, gvkey, field_names, outputs, phi_field, phi_quarter, f_x, f_bg):
    """shapley.npz: date [N] (yyyymmdd), gvkey [N], fields [F] (Dataset order), quarters [T] (1 - T .. 0, as inp_t<k>
    numbers them), outputs [K] (shapley_output_names), phi_field [N,K,F], phi_quarter [N,K,T], f_x [N,K] and f_bg
    [N,K], in normalised units: phi_field[i, k].sum() and phi_quarter[i, k].sum() are each f_x[i, k] - f_bg[i, k]."""
    T = np.shape(phi_quarter)[2]
    np.savez(path, date=np.asarray(date).astype(np.int32),
             gvkey=np.array([g.decode('utf-8') if isinstance(g, bytes) else str(g) for g in gvkey]),
             fields=np.array(list(field_names)), quarters=np.arange(1 - T, 1, dtype=np.int32),
             outputs=np.array(list(outputs)), phi_field=np.asarray(phi_field, dtype=np.float32),
             phi_quarter=np.asarray(phi_quarter, dtype=np.float32), f_x=np.asarray(f_x, dtype=np.float32),
             f_bg=np.asarray(f_bg, dtype=np.float32))


def write_influence(path, date, gvkey, outputs, train_date, train_gvkey, train_target, pos_idx, pos_score, neg_idx,
                    neg_score, total):
    """influence.npz: date [N], gvkey [N] (preds.dat row order), outputs [J] (shapley_output_names), train_date [Nt]
    (the last input date of each training window), train_gvkey [Nt], train_target [Nt] (its normalised target of the
    target field at the last step), pos_idx / pos_score / neg_idx / neg_score [N,J,K] (indices into the train_* arrays,
    -1 with score 0 where fewer windows have that sign) and total [N,J], the summed influence of the whole pool."""
    np.savez(path, date=np.asarray(date, dtype=np.int32), gvkey=np.asarray(gvkey, dtype=str),
             outputs=np.asarray(outputs, dtype=str), train_date=np.asarray(train_date, dtype=np.int32),
             train_gvkey=np.asarray(train_gvkey, dtype=str), train_target=np.asarray(train_target, dtype=np.float32),
             pos_idx=np.asarray(pos_idx, dtype=np.int32), pos_score=np.asarray(pos_score, dtype=np.float32),
             neg_idx=np.asarray(neg_idx, dtype=np.int32), neg_score=np.asarray(neg_score, dtype=np.float32),
             total=np.asarray(total, dtype=np.float32))


def ale_table(field_names, outputs, n_bins, edges, counts, ale, local_mean, local_sd):
    """The rows of ale.dat from NativeForecaster.ale's outputs (n_bins [F], edges [F,K+1], counts [F,K],
    ale [F,K+1,J], local_mean and local_sd [F,K,J]): one row per field, in Dataset order, and edge k = 0..K_f, with the
    edge in normalised input units and n the windows in the bin that ends at it (0 at k = 0); then per explained output
    <out> (shapley_output_names) ale_<out>, the centred accumulated effect at the edge, and local_<out> and
    local_sd_<out>, the mean and standard deviation of the bin's local effects (NaN at k = 0).  A field with fewer than
    two distinct values (K_f = 0) has no rows."""
    cols = {'field': [], 'edge_idx': [], 'edge': [], 'n': []}
    for o in outputs:
        cols.update({'ale_' + o: [], 'local_' + o: [], 'local_sd_' + o: []})
    for f, name in enumerate(field_names):
        kf = int(n_bins[f])
        if kf == 0:
            continue
        cols['field'] += [name] * (kf + 1)
        cols['edge_idx'] += list(range(kf + 1))
        cols['edge'] += list(np.asarray(edges[f][:kf + 1], dtype=np.float64))
        cols['n'] += [0] + [int(c) for c in counts[f][:kf]]
        for j, o in enumerate(outputs):
            cols['ale_' + o] += list(np.asarray(ale[f][:kf + 1, j], dtype=np.float64))
            cols['local_' + o] += [np.nan] + list(np.asarray(local_mean[f][:kf, j], dtype=np.float64))
            cols['local_sd_' + o] += [np.nan] + list(np.asarray(local_sd[f][:kf, j], dtype=np.float64))
    return pd.DataFrame(cols)


def quantile_name(level):
    """q<100 tau> of a level, as %g formats it: 0.05 -> q5, 0.5 -> q50, 0.125 -> q12.5."""
    return 'q%g' % (100.0 * level)


def quantile_table(keys, levels, quantiles, scores, unscale):
    """The rows of quantiles.dat: `keys` (date, gvkey of preds.dat), then per forecast step s the mixture quantiles
    norm_q<100 tau>_s (normalised units), q<100 tau>_s = unscale(norm_q<100 tau>_s) (the fundamentals' units: quantiles
    pass through the increasing map of centre, scale, expm1 and seq_norm unchanged wherever seq_norm > 0, and their
    order reverses where seq_norm < 0), and crps_s, nll_s and pit_s of the normalised target (NaN where it is unknown).
    quantiles [S,N,Q] and scores [S,N,3] as NativeForecaster.predict_dist returns them."""
    df = keys.reset_index(drop=True).copy()
    for s in range(len(quantiles)):
        for k, level in enumerate(levels):
            df['norm_%s_%d' % (quantile_name(level), s + 1)] = quantiles[s][:, k]
        for k, level in enumerate(levels):
            df['%s_%d' % (quantile_name(level), s + 1)] = unscale(quantiles[s][:, k])
        for j, name in enumerate(('crps', 'nll', 'pit')):
            df['%s_%d' % (name, s + 1)] = scores[s][:, j]
    return df


def pit_ks(pit):
    """The Kolmogorov-Smirnov distance sup |F_n(u) - u| of the PIT values from U(0, 1); NaN when there are none."""
    p = np.sort(np.asarray(pit, dtype=np.float64))
    n = len(p)
    if n == 0:
        return np.nan
    i = np.arange(1, n + 1)
    return float(max(np.max(i / n - p), np.max(p - (i - 1) / n)))


def calibration_table(levels, quantiles, scores, targets):
    """The rows of calibration.dat, one per (forecast step, level): frac_below, the share of the n_known windows with a
    known normalised target (targets [S,N]) whose target lies below norm_q<100 tau> -- close to the level when the
    forecast is calibrated -- and, repeated on every row of a step, the mean CRPS and log score of those windows and
    pit_ks, the Kolmogorov-Smirnov distance of their PIT values from U(0, 1)."""
    rows = []
    for s in range(len(quantiles)):
        y = np.asarray(targets[s], dtype=np.float64)
        known = np.isfinite(y)
        n = int(known.sum())
        sc = np.asarray(scores[s], dtype=np.float64)[known]
        mean_crps, mean_nll = (float(sc[:, 0].mean()), float(sc[:, 1].mean())) if n else (np.nan, np.nan)
        ks = pit_ks(sc[:, 2])
        for k, level in enumerate(levels):
            below = float(np.mean(y[known] < np.asarray(quantiles[s])[known, k])) if n else np.nan
            rows.append({'step': s + 1, 'level': level, 'frac_below': below, 'n_known': n, 'mean_crps': mean_crps,
                         'mean_nll': mean_nll, 'pit_ks': ks})
    return pd.DataFrame(rows, columns=['step', 'level', 'frac_below', 'n_known', 'mean_crps', 'mean_nll', 'pit_ks'])


def conformal_level_name(level):
    """A coverage level as intervals.dat names it: quantile_name without its q (0.9 -> 90, 0.125 -> 12.5)."""
    return quantile_name(level)[1:]


def _unscaled_bounds(lo, hi, seq_norm, unscale):
    """The fundamentals-unit bounds of normalised bounds: unscale of each, swapped where seq_norm < 0 (where unscale
    reverses the order), so that lower <= upper."""
    a, b = unscale(lo), unscale(hi)
    flip = np.asarray(seq_norm) < 0
    return np.where(flip, b, a), np.where(flip, a, b)


def interval_table(keys, levels, lower, upper, scale, pvalue, seq_norm, unscale):
    """The rows of intervals.dat: `keys` (date, gvkey of preds.dat), then per forecast step s and level l (named by
    conformal_level_name, e.g. 90) norm_lo90_s and norm_hi90_s (normalised units), lo90_s and hi90_s (the fundamentals'
    units: unscale of the bounds, as preds_s, swapped where seq_norm < 0), then scale_s (the window's scale: 1, sigma
    or d(x) + beta) and pvalue_s (its conformal p-value, NaN where the target is unknown).  lower / upper [S,N,Q],
    scale and pvalue [S,N] as NativeForecaster.conformal returns them."""
    df = keys.reset_index(drop=True).copy()
    cols = {}
    for s in range(len(lower)):
        for k, level in enumerate(levels):
            name = '%s_%d' % (conformal_level_name(level), s + 1)
            cols['norm_lo' + name] = lower[s][:, k]
            cols['norm_hi' + name] = upper[s][:, k]
            cols['lo' + name], cols['hi' + name] = _unscaled_bounds(lower[s][:, k], upper[s][:, k], seq_norm, unscale)
        cols['scale_%d' % (s + 1)] = scale[s]
        cols['pvalue_%d' % (s + 1)] = pvalue[s]
    return pd.concat([df, pd.DataFrame(cols)], axis=1)


def conformal_subsets(date, gvkey, cal_date, cal_gvkey, train_gvkeys, end_date):
    """The coverage.dat subset of every window (date yyyymmdd, gvkey): 'calibration' when (date, gvkey) is a
    calibration window, 'training' when its company is in the training split and its date is in or before end_date
    (YYYYMM) of the training draw, else 'out_of_sample'."""
    cal = set(zip((int(d) for d in cal_date), (str(g) for g in cal_gvkey)))
    out = []
    for d, g in zip(date, gvkey):
        if (int(d), str(g)) in cal:
            out.append('calibration')
        elif str(g) in train_gvkeys and int(d) // 100 <= end_date:
            out.append('training')
        else:
            out.append('out_of_sample')
    return np.asarray(out)


def coverage_table(levels, subset, n_cal, qhat, pred, targets, scale, lower, upper, seq_norm, unscale):
    """The rows of coverage.dat, one per forecast step, level and subset (calibration, training, out_of_sample, all):
    n_cal and qhat of the step and level, n (the subset's windows with a known target), coverage (the share of them
    whose score |y - pred| / scale, in float32 as the library forms it, is at most qhat: whose target lies in the
    interval) and the mean normalised and fundamentals-unit interval widths over those n windows."""
    rows = []
    for s in range(len(lower)):
        y = np.asarray(targets[s], dtype=np.float32)
        r = np.abs(y - np.asarray(pred[s], dtype=np.float32)) / np.asarray(scale[s], dtype=np.float32)
        known = np.isfinite(y)
        for k, level in enumerate(levels):
            lo, hi = np.asarray(lower[s][:, k], dtype=np.float64), np.asarray(upper[s][:, k], dtype=np.float64)
            ulo, uhi = _unscaled_bounds(lo, hi, seq_norm, unscale)
            for name in ('calibration', 'training', 'out_of_sample', 'all'):
                m = known & ((subset == name) if name != 'all' else True)
                n = int(m.sum())
                with np.errstate(invalid='ignore'):
                    rows.append({'step': s + 1, 'level': level, 'subset': name, 'n_cal': int(n_cal[s]),
                                 'qhat': float(qhat[s][k]), 'n': n,
                                 'coverage': float(np.mean(r[m] <= qhat[s][k])) if n else np.nan,
                                 'mean_norm_width': float(np.mean(hi[m] - lo[m])) if n else np.nan,
                                 'mean_width': float(np.mean(uhi[m] - ulo[m])) if n else np.nan})
    return pd.DataFrame(rows, columns=['step', 'level', 'subset', 'n_cal', 'qhat', 'n', 'coverage', 'mean_norm_width',
                                       'mean_width'])


# ---- lookahead factor backtests (--factor_quantiles, DESIGN.md section 5k) ---------------------------------------------
FACTOR_MAX_SCORES = 8       # lfmq_factor_eval's caps on the factors and the measures
FACTOR_MAX_MEASURES = 4


def factor_names(forecast_steps, uq):
    """The factors of a run: lfm_s (forecast yield) per step, qfm (current yield), and on a UQ model lfm_risk_s."""
    return (['lfm_%d' % s for s in range(1, forecast_steps + 1)] + ['qfm']
            + (['lfm_risk_%d' % s for s in range(1, forecast_steps + 1)] if uq else []))


def factor_scores(df, forecast_steps, uq, inp_t0=None):
    """(names, scores [G,N] fp64) of the rows of a preds.dat frame: lfm_s = preds_s / seq_norm, qfm = inp_t0 / seq_norm
    (inp_t0 the frame's column unless given) and, on a UQ model, lfm_risk_s = pred_var_s / seq_norm with pred_var_s =
    preds_s / sqrt(variance_s) as ensemble_uq_estimate forms it; NaN where variance_s is not finite or not > 0."""
    seq_norm = df['seq_norm'].to_numpy(dtype=np.float64)
    col = lambda c: df[c].to_numpy(dtype=np.float64)        # noqa: E731
    inp = col('inp_t0') if inp_t0 is None else np.asarray(inp_t0, dtype=np.float64)
    with np.errstate(divide='ignore', invalid='ignore'):
        scores = [col('preds_%d' % s) / seq_norm for s in range(1, forecast_steps + 1)] + [inp / seq_norm]
        if uq:
            for s in range(1, forecast_steps + 1):
                v = col('variance_%d' % s)
                ok = np.isfinite(v) & (v > 0)
                scores.append(np.where(ok, col('preds_%d' % s) / np.sqrt(np.where(ok, v, 1.0)), np.nan) / seq_norm)
    return factor_names(forecast_steps, uq), np.stack(scores)


def _yyyymmdd(dates):
    """The dates of a frame column (datetime or yyyymmdd / yyyymm integers) as int64."""
    d = pd.Series(dates)
    if np.issubdtype(d.dtype, np.datetime64):
        return (d.dt.year * 10000 + d.dt.month * 100 + d.dt.day).to_numpy(dtype=np.int64)
    return d.astype(np.int64).to_numpy()


def month_index(dates):
    """The calendar month (12 * year + month - 1) of yyyymmdd or yyyymm integer dates."""
    d = np.asarray(dates, dtype=np.int64)
    ym = np.where(d >= 10 ** 7, d // 100, d)
    return (ym // 100) * 12 + ym % 100 - 1


def forward_returns(data, field, date, gvkey, horizon):
    """ret of rows (date, gvkey): prod_{k=1..H} (1 + r_{c, t+k}) - 1, with r the raw column `field` of the datafile
    frame `data` (date, gvkey, field) and t+k the company's row exactly k calendar months after the row's date; NaN
    when any of those rows is missing or its r is not finite."""
    months = month_index(_yyyymmdd(data['date']))
    r = pd.Series(data[field].to_numpy(dtype=np.float64),
                  index=pd.MultiIndex.from_arrays([data['gvkey'].astype(str).to_numpy(), months]))
    if not r.index.is_unique:
        raise ValueError('--factor_return_field %s: the datafile has two rows for one company in one month' % field)
    g, t = np.asarray(gvkey).astype(str), month_index(date)
    prod, ok = np.ones(len(g)), np.ones(len(g), dtype=bool)
    for k in range(1, int(horizon) + 1):
        rk = r.reindex(pd.MultiIndex.from_arrays([g, t + k])).to_numpy(dtype=np.float64)
        ok &= np.isfinite(rk)
        prod *= np.where(np.isfinite(rk), 1.0 + rk, 1.0)
    return np.where(ok, prod - 1.0, np.nan)


def factor_codes(date, gvkey):
    """(dates [D] ascending, date_idx [N], company [N]) int codes of the rows; two rows of one (date, gvkey) raise."""
    dates, date_idx = np.unique(np.asarray(date, dtype=np.int64), return_inverse=True)
    _, company = np.unique(np.asarray(gvkey).astype(str), return_inverse=True)
    pairs = date_idx.astype(np.int64) * (int(company.max()) + 1 if len(company) else 1) + company
    if len(np.unique(pairs)) != len(pairs):
        raise ValueError('--factor_quantiles: the frame has two rows for one (date, gvkey); a factor ranks each '
                         'company once per date')
    return dates, date_idx.astype(np.int32), company.astype(np.int32)


def factor_dates_table(dates, factors, measures, out, Q):
    """The rows of factor_dates.dat, one per (date, factor, measure) in that order: date factor measure n n_pair ic
    q1..qQ (the bucket means, bucket Q the highest scores) spread turnover, from lfmq_factor_eval's outputs `out`
    (NumPy arrays as engine.factor_eval names them)."""
    D, G, M = len(dates), len(factors), len(measures)
    d, g, m = (a.ravel() for a in np.meshgrid(np.arange(D), np.arange(G), np.arange(M), indexing='ij'))
    cols = {'date': np.asarray(dates)[d], 'factor': np.asarray(factors)[g], 'measure': np.asarray(measures)[m],
            'n': out['n'][g, d], 'n_pair': out['n_pair'][g, m, d], 'ic': out['ic'][g, m, d]}
    for q in range(Q):
        cols['q%d' % (q + 1)] = out['bucket_mean'][g, m, d, q]
    cols['spread'] = out['spread'][g, m, d]
    cols['turnover'] = out['turnover'][g, d]
    return pd.DataFrame(cols)


def newey_west_t(x, lag):
    """x̄ / sqrt(var / n) of the finite entries of x (consecutive ones adjacent), var = γ0 + 2 Σ_{k=1..L} (1 - k/(L+1))
    γk with Bartlett weights; NaN when n < 2 or var <= 0."""
    x = np.asarray(x, dtype=np.float64)
    x = x[np.isfinite(x)]
    n = len(x)
    if n < 2:
        return np.nan
    xc = x - x.mean()
    var = xc @ xc / n
    for k in range(1, min(int(lag), n - 1) + 1):
        var += 2.0 * (1.0 - k / (lag + 1.0)) * (xc[k:] @ xc[:-k]) / n
    return float(x.mean() / np.sqrt(var / n)) if var > 0 else np.nan


def newey_west_lag(dates, horizon):
    """L = max(0, ceil(h / spacing) - 1), spacing the smallest gap in months between consecutive dates (0 for one
    date): overlapping h-month outcomes are correlated over L dates."""
    months = np.unique(month_index(dates))
    if len(months) < 2:
        return 0
    return max(0, int(np.ceil(horizon / float(np.diff(months).min()))) - 1)


def _finite_stats(x):
    """(n, mean, sd with ddof 1) of the finite entries of x (NaN where undefined)."""
    x = np.asarray(x, dtype=np.float64)
    x = x[np.isfinite(x)]
    return len(x), (float(x.mean()) if len(x) else np.nan), (float(x.std(ddof=1)) if len(x) > 1 else np.nan)


def factor_summary(dates, factors, measures, out, Q, horizons):
    """The rows of factor.dat, one per (factor, measure): n_dates (dates with a finite ic), mean_ic, sd_ic, ir =
    mean_ic / sd_ic, hit (share of those dates with ic > 0), t_ic, mean_q1..mean_qQ (means over dates of each bucket's
    mean), mean_spread, sd_spread, t_spread, mean_turnover and nw_lag, the Newey-West lag of the t-statistics for the
    measure's horizon in months (horizons [M])."""
    rows = []
    for g, f in enumerate(factors):
        for m, meas in enumerate(measures):
            lag = newey_west_lag(dates, horizons[m])
            ic = out['ic'][g, m]
            n, mean_ic, sd_ic = _finite_stats(ic)
            _, mean_sp, sd_sp = _finite_stats(out['spread'][g, m])
            row = {'factor': f, 'measure': meas, 'n_dates': n, 'mean_ic': mean_ic, 'sd_ic': sd_ic,
                   'ir': mean_ic / sd_ic if sd_ic > 0 else np.nan,
                   'hit': float(np.mean(ic[np.isfinite(ic)] > 0)) if n else np.nan,
                   't_ic': newey_west_t(ic, lag)}
            for q in range(Q):
                row['mean_q%d' % (q + 1)] = _finite_stats(out['bucket_mean'][g, m, :, q])[1]
            row.update({'mean_spread': mean_sp, 'sd_spread': sd_sp, 't_spread': newey_west_t(out['spread'][g, m], lag),
                        'mean_turnover': _finite_stats(out['turnover'][g])[1], 'nw_lag': lag})
            rows.append(row)
    return pd.DataFrame(rows)


def factor_measures(df, forecast_n, returns=None, horizon=1):
    """(names, measures [M,N], horizons [M] in months): yield = targets_1 / seq_norm over forecast_n months, and with
    `returns` (forward_returns of the rows) ret over `horizon` months."""
    with np.errstate(divide='ignore', invalid='ignore'):
        y = df['targets_1'].to_numpy(dtype=np.float64) / df['seq_norm'].to_numpy(dtype=np.float64)
    if returns is None:
        return ['yield'], y[None, :], [int(forecast_n)]
    return ['yield', 'ret'], np.stack([y, np.asarray(returns, dtype=np.float64)]), [int(forecast_n), int(horizon)]


def factor_tables(df, config, inp_t0=None):
    """(factor_dates.dat, factor.dat) frames of a preds.dat frame `df` (or walk_forward_preds.dat's) for the run's
    --factor_quantiles Q: the factors (factor_scores), the measures (factor_measures, ret read from the datafile with
    --factor_return_field), one lfmq_factor_eval call on the GPU, and the summary on the host."""
    import torch
    from ..engine import factor_eval
    Q = int(config.factor_quantiles)
    date = _yyyymmdd(df['date'])
    gvkey = df['gvkey'].astype(str).to_numpy()
    # the values as preds.dat holds them: a float32 column (seq_norm) is written in its shortest decimal form, so a
    # fixed_dates run and a walk-forward run, which reads its frame back from the files, rank the same numbers
    cols = [c for c in df.columns if c in ('seq_norm', 'inp_t0') or c.startswith(('preds_', 'targets_', 'variance_'))]
    df = pd.read_csv(io.StringIO(df[cols].to_csv(sep=' ', index=False)), sep=' ', float_precision='round_trip')
    factors, score = factor_scores(df, config.forecast_steps, config.UQ, inp_t0)
    field = getattr(config, 'factor_return_field', None)
    returns = None
    if field:
        data = pd.read_csv(os.path.join(config.data_dir, config.datafile), sep=' ', usecols=['date', 'gvkey', field],
                           dtype={'gvkey': str})
        returns = forward_returns(data, field, date, gvkey, config.factor_horizon)
    measures, measure, horizons = factor_measures(df, config.forecast_n, returns, config.factor_horizon)
    dates, date_idx, company = factor_codes(date, gvkey)
    cu = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()      # noqa: E731
    out = {k: v.cpu().numpy() for k, v in factor_eval(cu(date_idx), cu(company), cu(score), cu(measure), Q).items()}
    return (factor_dates_table(dates, factors, measures, out, Q),
            factor_summary(dates, factors, measures, out, Q, horizons))
