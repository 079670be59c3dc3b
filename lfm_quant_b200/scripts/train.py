"""Train driver (reference: scripts/train.py:27-432).

Same life cycle -- build model/optimizer/losses, materialise every batch up front (train.py:64-80), epoch loop
with shuffled batch order, CSV logs (train.py:133-147,156-167,227-238), save-best / early-stop
(train.py:240-266) -- but the step body of every model (``_train_step``, train.py:178-225) is ONE native call
(fwd + loss + BPTT + clip + optimizer + MaxNorm on the GPU) and the per-step ``mse.numpy()`` host sync of the
reference (train.py:199) is deferred: device scalars are read back only when a log line is due.
"""
from __future__ import absolute_import, division, print_function

import copy
import os
import pathlib
import random
import time
from collections import defaultdict

import numpy as np
import pandas as pd

from .model_utils.losses import Losses
from .model_utils.model import Model
from .model_utils.optimizers import Optimizers


class Train(object):

    def __init__(self, config, dataset):
        self.config = config
        self.dataset = dataset
        self.dataset.generate_dataset()
        # Data parallelism over the company-batch axis (SURVEY 8e): under torchrun every rank walks the same seeded
        # batch sequence, gathers only its rows of each global batch and all-reduces the flat gradient once per step.
        # The process group / device is chosen before the model (and its workspace) is created on that device.
        from .. import dp as _dp
        self.rank, self.world = _dp.init_from_env()
        self.model = Model(self.config, self.dataset).get_model()
        if self.world > 1:                       # one set of initial weights: rank 0's, for every forecast stage
            import torch
            import torch.distributed as dist
            for eng in self.model.engine.stages:
                flat = torch.from_numpy(eng.get_flat()).to(eng.device)
                dist.broadcast(flat, 0)
                eng.set_flat(flat.cpu().numpy())
        self.target_index = self.dataset.target_index
        self.optimizer = Optimizers(self.config).get_optimizer()
        self.optimizer.bind(self.model)
        self.losses = Losses(self.config, self.target_index, engine=self.model.engine)

        self.train_set = self.dataset.train_set
        self.valid_set = self.dataset.valid_set
        self.train_set = self.train_set.shuffle(buffer_size=10000, seed=self.config.seed)
        self.train_set = self.train_set.batch(batch_size=self.config.batch_size)
        self.valid_set = self.valid_set.batch(batch_size=self.config.batch_size)

        self.model_dir = os.path.join(self.config.experiments_dir, self.config.model_dir)
        self.chkpts_dir = os.path.join(self.model_dir, 'chkpts')
        self.train_log_dir = os.path.join(self.model_dir, 'train_log')
        train_dirs = [self.model_dir, self.chkpts_dir, self.train_log_dir]
        print(train_dirs)
        for dirname in train_dirs:
            if not os.path.isdir(dirname):
                print("Creating dir %s" % dirname)
                pathlib.Path(dirname).mkdir(parents=True, exist_ok=True)

        self.min_valid_mse = np.inf
        self.min_valid_uq_loss = np.inf
        self._grad_norm = 1.0

        print("Creating batches ...")
        self._batches = [self._build_train_batch(items) for items in self.train_set]
        self._valid_batches = [self.dataset.get_batch(*items) for items in self.valid_set]

    def _build_train_batch(self, items):
        """(inp, target, metadata[, row0, global denominators][, row weights]) of one global batch; the shard of this
        rank under DP.  The denominators: {B, mask count} of the point estimate; the uq loss's {B, mask count, last-step
        mask count}; with forecast_steps > 1 those three per forecast stage -- their weighted sums with row weights
        (--sample_weight_field / --recency_halflife, DESIGN.md section 6d), a device vector of the batch's weights,
        zero-padded to the engine's max_batch."""
        eng = self.model.engine
        weighted = self.dataset.row_weighted
        if self.world == 1:
            batch = self.dataset.get_batch(*items)
            if not weighted:
                return batch
            return tuple(batch) + (0, None, self.dataset.row_weights(items[0], eng.cfg.max_batch))
        import torch.distributed as dist
        from .. import dp as _dp
        inp_idx, tar_idx, meta, row0 = _dp.shard_batch_indices(items[0], items[1], items[2], self.rank, self.world)
        x = y = md = w = None
        if len(inp_idx) > 0:                     # else fewer windows than ranks: this rank only joins the collectives
            x, y, md = self.dataset.get_batch(inp_idx, tar_idx, meta)
        if weighted:                             # the counts below read the handles' weights
            w = self.dataset.row_weights(inp_idx, eng.cfg.max_batch)
            eng.set_row_weights(w)
        # loss denominators are global (losses.py:87,90,131-135); a rank without rows adds zeros
        denom = _dp.global_denominators(eng.loss_counts(None if y is None else self._step_targets(y)), dist)
        return (x, y, md, row0, denom) + ((w,) if weighted else ())

    def train(self):
        if self.config.load_saved_weights:
            self.model.load_weights(os.path.join(self.chkpts_dir, "chkpt"))
        print("Training in progress ...")
        epochs = self.config.max_epoch
        checkpoint_prefix = os.path.join(self.chkpts_dir, "chkpt")
        train_logs_batch = defaultdict(list)
        train_logs_epoch = defaultdict(list)
        if self.rank == 0:
            self.model.save_weights(checkpoint_prefix)
        valid_mse = None
        start = time.time()
        for epoch in range(epochs):
            self.model.reset_states()
            mse_steps, uq_loss_steps = [], []
            # The reference's other unseeded draw, the seeds of ensemble members k > 0 (model_execution.py:187-188), comes
            # from random.Random(config.seed) here (runtime/model_execution.member_configs).
            if self.world == 1 and not os.environ.get('LFMQ_SEEDED_SHUFFLE'):
                random.shuffle(self._batches)                   # train.py:115 (unseeded in the reference)
            else:                                               # every rank must walk the same batch order
                random.Random(self.config.seed + epoch).shuffle(self._batches)
            for (batch_n, cur_batch) in enumerate(self._batches):
                uq_loss, mse = self._train_step(cur_batch)      # device scalars, no host sync here
                mse_steps.append(mse)
                uq_loss_steps.append(uq_loss)
                if batch_n % self.config.logging_interval == 0:
                    train_logs_batch['batch_n'].append(batch_n)
                    train_logs_batch['time'].append(time.time() - start)
                    train_logs_batch['mse'].append(self._mean(mse_steps))
                    train_logs_batch['uq_loss'].append(self._mean(uq_loss_steps) if self.config.UQ else None)
                    train_logs_batch['valid_mse'].append(None)
                    train_logs_batch['valid_uq_loss'].append(None)
                    self._write_train_logs(train_logs_batch, 'train-logs-batch')

            if epoch % self.config.epoch_logging_interval == 0:
                if self.config.UQ:
                    valid_uq_loss, valid_mse, valid_mse_fcst = self._validation_metrics_uq_range_estimate()
                else:
                    valid_uq_loss, valid_mse, valid_mse_fcst = self._validation_metrics_point_estimate()
                train_logs_epoch['epoch'].append(epoch)
                train_logs_epoch['time'].append(time.time() - start)
                train_logs_epoch['mse'].append(self._mean(mse_steps))
                train_logs_epoch['uq_loss'].append(self._mean(uq_loss_steps) if self.config.UQ else None)
                train_logs_epoch['valid_mse'].append(valid_mse)
                train_logs_epoch['valid_uq_loss'].append(valid_uq_loss)
                train_logs_epoch['valid_mse_fcst'].append(valid_mse_fcst)
                self._write_train_logs(train_logs_epoch, 'train-logs-epoch')
                if self._save_criteria(train_logs_epoch) and self.rank == 0:
                    self.model.save_weights(checkpoint_prefix)
                if self._stop_criteria(train_logs_epoch):
                    break
        return valid_mse

    @staticmethod
    def _mean(device_scalars):
        import torch
        return float(torch.stack(list(device_scalars)).mean().item())

    def _train_step(self, cur_batch):
        """One training step of any model (train.py:178-225) as one fused native step; returns
        (uq_loss_last_tar or None, mse) as device scalars, weighted over the forecast steps.  Under torchrun: local BPTT
        of this rank's rows with the global denominators, ONE all-reduce, the replicated clip + optimizer + MaxNorm; a
        rank without rows joins with zeros.  Same trajectory as one GPU."""
        inp = cur_batch[0]
        ys = None if inp is None else self._step_targets(cur_batch[1])
        lr, it = self.optimizer.current_lr(), self.optimizer.iterations
        if len(cur_batch) > 5:                  # row weights: the batch's own vector for this step
            self.model.engine.set_row_weights(cur_batch[5])
        if self.world > 1:
            out = self.model.train_step_dp(inp, ys, it, lr, cur_batch[3], cur_batch[4])
        else:
            out = self.model.train_step(inp, ys, lr, it)
        self.optimizer.iterations += 1
        return (out[0] if self.config.UQ else None), out[1]

    def _step_targets(self, targets):
        """The list of forecast_steps targets of one batch.  The dataset materialises one target window per input window
        (forecast_n ahead); every forecast step of a multi-step graph is scored against it."""
        if isinstance(targets, (list, tuple)):
            return targets
        return [targets] * self.config.forecast_steps

    def _write_train_logs(self, train_logs, name):
        if self.rank != 0:
            return
        df = pd.DataFrame.from_dict(train_logs)
        fname = os.path.join(self.train_log_dir, self.config.name + '-' + name + '.csv')
        df.to_csv(fname, sep=',', index=False)

    def _save_criteria(self, train_logs_epoch):
        assert len(train_logs_epoch['valid_mse']) > 0, 'Error in computing valid_mse or incorrect train log dict passed'
        if train_logs_epoch['valid_mse'][-1] < self.min_valid_mse:
            self.min_valid_mse = train_logs_epoch['valid_mse'][-1]
            return True
        return False

    def _stop_criteria(self, train_logs_epoch):
        """train.py:253-266, including its off-by-one (SURVEY App. B #3)."""
        assert len(train_logs_epoch['valid_mse']) > 0, \
            'Error in computing valid_mse or incorrect train log dict passed'
        valid_mse = np.array(train_logs_epoch['valid_mse'])
        return bool(valid_mse.shape[0] - np.argmin(valid_mse) + 1 >= self.config.early_stop)

    def _validation_metrics_point_estimate(self):
        """train.py:268-336: predict every validation batch, loss over the stacked arrays, scaled and un-scaled -- all on
        the device: the validation batches are resident (built once in __init__), predictions stay in HBM
        (predict_device), un-scaling is lfmq_unscale, both losses are lfmq_loss; the only host traffic per epoch is the
        two result scalars."""
        import torch
        if not self._valid_batches:
            return None, float('nan'), float('nan')
        preds = [self.model.predict_device(cur_batch[0]) for cur_batch in self._valid_batches]    # lists of S
        targets = [self._step_targets(cur_batch[1]) for cur_batch in self._valid_batches]
        scale, center = self._scaling_dev()
        eng = self.model.engine
        S = self.config.forecast_steps
        pred_all = [torch.cat([p[i] for p in preds], dim=0) for i in range(S)]            # train.py:316-320
        target_all = [torch.cat([t[i] for t in targets], dim=0) for i in range(S)]
        pred_unscaled = [eng.unscale(p, scale, center, self.config.log_squasher) for p in pred_all]
        target_unscaled = [eng.unscale(t, scale, center, self.config.log_squasher) for t in target_all]
        _, valid_mse = self.losses.weight_adjusted_mse(target_all, pred_all, True)
        _, valid_mse_fcst = self.losses.weight_adjusted_mse(target_unscaled, pred_unscaled, True)
        both = torch.stack([valid_mse._t, valid_mse_fcst._t]).cpu().numpy()      # the epoch's single D2H
        return None, float(both[0]), float(both[1])

    def _scaling_dev(self):
        import torch
        if getattr(self, '_scale_dev', None) is None:
            n = self.dataset.n_outputs
            dev = self.model.engine.device
            self._scale_dev = torch.from_numpy(np.ascontiguousarray(self.dataset.scaling_params['scale'][:n],
                                                                    dtype=np.float64)).to(dev)
            self._center_dev = torch.from_numpy(np.ascontiguousarray(self.dataset.scaling_params['center'][:n],
                                                                     dtype=np.float64)).to(dev)
        return self._scale_dev, self._center_dev

    def _validation_metrics_uq_range_estimate(self):
        """train.py:338-416: predict every validation batch (dropout stays on), uq loss over the stacked arrays, MSE of
        the un-scaled target predictions: every forecast step's arrays, the losses weighted over the steps
        (train.py:387-416)."""
        S = self.config.forecast_steps
        preds, var, targets = [], [], []
        for cur_batch in self._valid_batches:
            batch_pred = self.model.predict(cur_batch[0])
            preds.append(batch_pred[0::2])
            var.append(batch_pred[1::2])
            targets.append([t.cpu().numpy() for t in self._step_targets(cur_batch[1])])
        if not preds:
            return float('nan'), float('nan'), float('nan')
        pred_all, var_all, target_all = ([np.vstack([b[i] for b in a]).astype('float32') for i in range(S)]
                                         for a in (preds, var, targets))
        pred_unscaled = [self._unscale_preds(copy.deepcopy(p)) for p in pred_all]
        target_unscaled = [self._unscale_preds(copy.deepcopy(t)) for t in target_all]
        _, valid_uq_loss, valid_mse = self.losses.weight_adjusted_uq_loss(target_all, pred_all, var_all)
        _, valid_mse_fcst = self.losses.weight_adjusted_mse(target_unscaled, pred_unscaled)
        return valid_uq_loss.numpy(), valid_mse.numpy(), valid_mse_fcst.numpy()

    def _unscale_preds(self, arr):
        """train.py:420-432."""
        arr = np.multiply(arr, self.dataset.scaling_params['scale'][:self.dataset.n_outputs]) + \
            self.dataset.scaling_params['center'][:self.dataset.n_outputs]
        if self.config.log_squasher:
            arr = self.dataset.reverse_log_squasher(arr)
        return arr
