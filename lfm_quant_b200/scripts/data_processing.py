"""Dataset: the reference's sliding-window batcher interface (scripts/data_processing.py:23-619) over a
device-resident table.

Host side (this file, NumPy/pandas): file parsing, date filter, key split, column-range parsing, window index
generation (vectorised restatement of the per-row Python loop at data_processing.py:209-237) and scaler fitting.
Device side (lfmq_gather_batch, csrc/kernels_simt.cu): ``get_batch`` -- strided row gather, zero padding,
seq-norm, log-squash, centre/scale, aux masking, fp64 arithmetic then fp32 cast (data_processing.py:307-368).

Divergences from the reference, all deliberate:
  * batches come back as CUDA torch tensors (the reference returns tf tensors, :367);
  * ``pre_metadata`` is kept aligned per split (the reference zips ONE metadata array over all splits with the
    per-split index arrays, :451-474, so training metadata is misaligned there; it is only consumed in predict
    mode, where both agree);
  * the 30 % scaler sample (:550-553) is drawn from a RandomState seeded with config.seed -- the reference uses
    the unseeded global ``random`` module and is not reproducible against itself;
  * ``CDRSInferenceData`` (:630-759) needs the private ``cdrs`` package and is not provided.
"""
from __future__ import absolute_import, division, print_function

import os
import pathlib
import pickle

import numpy as np
import pandas as pd

_MIN_SEQ_NORM = 10


class IndexSet(object):
    """The slice of tf.data.Dataset the drivers use (train.py:42-44, predict.py:43): zip of window index
    triples + metadata supporting ``shuffle(buffer_size, seed)``, ``batch(batch_size)`` and iteration."""

    def __init__(self, inp_idx, tar_idx, meta, batch_size=None):
        self.inp_idx, self.tar_idx, self.meta, self.batch_size = inp_idx, tar_idx, meta, batch_size

    def __len__(self):
        n = self.inp_idx.shape[0]
        return n if self.batch_size is None else (n + self.batch_size - 1) // self.batch_size

    def shuffle(self, buffer_size, seed=None):
        """Streaming buffer shuffle (the algorithm of tf.data's shuffle; its RNG stream is not reproducible)."""
        n = self.inp_idx.shape[0]
        rng = np.random.RandomState(seed)
        order = np.empty(n, dtype=np.int64)
        buf = list(range(min(buffer_size, n)))
        nxt = len(buf)
        for k in range(n):
            j = rng.randint(len(buf))
            order[k] = buf[j]
            if nxt < n:
                buf[j] = nxt
                nxt += 1
            else:
                buf[j] = buf[-1]
                buf.pop()
        return IndexSet(self.inp_idx[order], self.tar_idx[order], self.meta[order], self.batch_size)

    def batch(self, batch_size):
        return IndexSet(self.inp_idx, self.tar_idx, self.meta, batch_size)

    def __iter__(self):
        n = self.inp_idx.shape[0]
        if self.batch_size is None:
            for i in range(n):
                yield self.inp_idx[i], self.tar_idx[i], self.meta[i]
        else:
            for s in range(0, n, self.batch_size):
                e = min(n, s + self.batch_size)
                yield self.inp_idx[s:e], self.tar_idx[s:e], self.meta[s:e]


class Dataset(object):
    """Same constructor, attributes and methods as the reference Dataset (data_processing.py:23-134)."""

    def __init__(self, config):
        self.config = config
        self._data_path = os.path.join(self.config.data_dir, self.config.datafile)
        self.is_train = self.config.train
        self.seq_len = self.config.max_unrollings

        # data_processing.py:40-57: read, parse dates (%Y%m%d then %Y%m), filter the date range
        self.data = pd.read_csv(self._data_path, sep=' ', dtype={'gvkey': str})
        try:
            self.data['date'] = pd.to_datetime(self.data['date'].astype(str), format="%Y%m%d")
            self.start_date = pd.to_datetime(str(self.config.start_date), format="%Y%m%d")
            self.end_date = pd.to_datetime(str(self.config.end_date), format="%Y%m%d")
        except ValueError:
            self.data['date'] = pd.to_datetime(self.data['date'].astype(str), format="%Y%m")
            self.start_date = pd.to_datetime(str(self.config.start_date), format="%Y%m")
            self.end_date = pd.to_datetime(str(self.config.end_date), format="%Y%m")
        self._date_offset_from_end = pd.DateOffset(months=self.config.stride)
        self._date_offset_from_start = pd.DateOffset(years=self.config.max_unrollings)
        self.data = self.data[(self.data['date'] >= self.start_date - self._date_offset_from_start) &
                              (self.data['date'] <= self.end_date + self._date_offset_from_end)]
        self.data = self.data.reset_index(drop=True)

        # data_processing.py:60-64
        self.gvkeys = self._get_gvkeys()
        self._train_gvkeys, self._valid_gvkeys, self._test_gvkeys = self.train_test_split(
            self.gvkeys, self.config.validation_size, self.config.seed, self.is_train)

        print("Start Date: %s" % self.start_date.strftime('%Y-%m-%d'))
        print("End Date: %s" % self.end_date.strftime('%Y-%m-%d'))
        print("Loading dataset %s complete" % self.config.datafile)
        print("Total number of records: %i" % self.data.shape[0])
        if self.config.train:
            print("Run type: Training")
            print("Number of training entities: %i" % len(self._train_gvkeys))
            print("Number of validation entities: %i" % len(self._valid_gvkeys))
        else:
            print("Run type: Prediction")
            print("Number of test entities: %i" % len(self._test_gvkeys))

        # data_processing.py:78-119
        _, self.fin_col_names = self.get_cols_from_colnames(self.config.financial_fields)
        _, self.aux_col_names = self.get_cols_from_colnames(self.config.aux_fields)
        _, self.dont_scale_col_names = self.get_cols_from_colnames(self.config.dont_scale_fields)
        self.n_inputs = len(self.fin_col_names) + len(self.aux_col_names)
        self.n_outputs = len(self.fin_col_names)
        self.target_index = self.fin_col_names.index(self.config.target_field)
        self._cols = ['date', 'gvkey', 'active'] + self.fin_col_names + self.aux_col_names
        self._cols_offset = 3
        if self.config.scale_field in self.data.columns and self.config.scale_field not in self._cols:
            self._cols.append(self.config.scale_field)
        # row weights of the training loss (DESIGN.md section 6d); ignored at prediction
        wfield = getattr(self.config, 'sample_weight_field', '') if self.config.train else ''
        self.recency_halflife = float(getattr(self.config, 'recency_halflife', 0.0)) if self.config.train else 0.0
        if self.recency_halflife < 0:
            raise ValueError('--recency_halflife %g: the half-life is in years, > 0 (0 = off)' % self.recency_halflife)
        if wfield:
            if wfield not in self.data.columns or wfield in ('date', 'gvkey'):
                raise ValueError('--sample_weight_field %s: not a numeric column of %s' % (wfield, self.config.datafile))
            vals = self.data[wfield].values.astype(np.float64)
            bad = np.flatnonzero((vals < 0) | np.isinf(vals))
            if bad.size:
                r = bad[0]
                raise ValueError('--sample_weight_field %s: %g at date %s, gvkey %s; weights must be >= 0 and finite '
                                 '(NaN counts as 0)' % (wfield, vals[r], self.data['date'].iloc[r].strftime('%Y%m%d'),
                                                       self.data['gvkey'].iloc[r]))
            if wfield not in self._cols:
                self._cols.append(wfield)
        self.data = self.data[self._cols]
        self._weight_col = self._cols.index(wfield) if wfield else -1
        self.ref_month = None
        self._gvkey_idx = self._cols.index(self.config.key_field)
        self._date_idx = self._cols.index(self.config.date_field)
        self._active_idx = self._cols.index(self.config.active_field)
        self.fin_col_ids = [self._cols.index(x) for x in self.fin_col_names]
        self.aux_col_ids = [self._cols.index(x) for x in self.aux_col_names]
        self.dont_scale_col_ids = [self._cols.index(x) for x in self.dont_scale_col_names]
        self.inp_col_ids = self.fin_col_ids + self.aux_col_ids
        self.scale_inp_col_ids = [x - self._cols_offset for x in self.inp_col_ids if x not in self.dont_scale_col_ids]
        self._aux_col_ids_seq = [x - self._cols_offset for x in self.aux_col_ids]
        self._seq_norm_idx = self._cols.index(self.config.scale_field) if self.config.scale_field in self._cols else None

        # numeric float64 view of data_values (:122); date/key columns are never read arithmetically
        num = self.data.copy()
        num['date'] = num['date'].dt.strftime('%Y%m%d').astype(np.float64)
        num['gvkey'] = 0.0
        self.table = np.ascontiguousarray(num.values.astype(np.float64))
        self._keys = np.asarray([str(k) for k in self.data['gvkey'].tolist()], dtype=str)   # plain numpy '<U' array
        self._dates = self.data['date'].values
        self._dataset = {k: None for k in ('train_X', 'train_Y', 'valid_X', 'valid_Y', 'test_X', 'test_Y')}
        self._meta = {'train': None, 'valid': None, 'test': None}
        self.model_dir = None
        self.scaling_params = None
        self._dev = None

    # ------------------------------------------------------------------------------------------------
    def generate_dataset(self):
        """data_processing.py:136-165: window indices + scaling params (fit or load ``scales.dat``)."""
        self._create_index()
        self.model_dir = os.path.join(self.config.experiments_dir, self.config.model_dir)
        if not os.path.isdir(self.model_dir):
            pathlib.Path(self.model_dir).mkdir(parents=True, exist_ok=True)
        scales_path = self.config.scalesfile if self.config.scalesfile else os.path.join(self.model_dir, 'scales.dat')
        if self.config.train:
            try:
                self.scaling_params = pickle.load(open(scales_path, 'rb'))
            except FileNotFoundError:
                self.scaling_params = self.get_scaling_params()
                pickle.dump(self.scaling_params, open(scales_path, 'wb'))
        else:
            assert os.path.isfile(scales_path), "scalesfile not provided. Ensure to use the same scalesfile as used " \
                                                "during training "
            self.scaling_params = pickle.load(open(scales_path, 'rb'))
        if self.recency_halflife > 0:
            # the recency reference: the latest last-input month of this run's training windows (so per walk-forward
            # origin, whose run ends at its own origin)
            self.ref_month = int(np.max(self._months(self._dataset['train_X'][:, 1]))) \
                if len(self._dataset['train_X']) else 0
        self._dev = None

    # ---- row weights of the training loss (DESIGN.md section 6d) --------------------------------------------------
    @property
    def row_weighted(self):
        return self._weight_col >= 0 or self.recency_halflife > 0

    def _months(self, rows):
        ymd = self.table[rows, self._date_idx].astype(np.int64)
        return (ymd // 10000) * 12 + (ymd // 100) % 100

    def row_weights_host(self, inp_indices):
        """The NumPy form of lfmq_row_weights: fp32 [B] weights of the windows inp_indices [B, 3], computed in fp64 --
        the sample_weight_field value at the window's last input row (NaN -> 0) times 2^(-months / (12 Y))."""
        rows = np.asarray(inp_indices)[:, 1].astype(np.int64)
        v = np.ones(rows.size, dtype=np.float64)
        if self._weight_col >= 0:
            v = self.table[rows, self._weight_col].copy()
            v[np.isnan(v)] = 0.0
        if self.recency_halflife > 0:
            months = (self.ref_month - self._months(rows)).astype(np.float64)
            v = v * np.exp2(-months / (12.0 * self.recency_halflife))
        return v.astype(np.float32)

    def row_weights(self, inp_indices, length=None):
        """The same weights computed on the GPU from the resident table (lfmq_row_weights): a CUDA fp32 vector of
        max(B, length) entries, zero beyond B."""
        import torch
        from ..engine import row_weights
        d = self._device_state()
        B = len(inp_indices)
        out = torch.zeros(max(B, length or 0), dtype=torch.float32, device=d['table'].device)
        if B:
            inp_idx = torch.from_numpy(np.ascontiguousarray(inp_indices, dtype=np.int32)).cuda()
            row_weights(d['table'], inp_idx, weight_col=self._weight_col, date_col=self._date_idx,
                        halflife=self.recency_halflife, ref_month=self.ref_month or 0, out=out)
        return out

    def _create_index(self):
        """Vectorised data_processing.py:170-305 (_create_tf_dataset + _append_sequence_data)."""
        cfg = self.config
        n = self.table.shape[0]
        stride, fn = cfg.stride, cfg.forecast_n
        min_steps = stride * (cfg.min_unrollings - 1) + 1
        max_steps = stride * (cfg.max_unrollings - 1) + 1
        keys = self._keys
        idx = np.arange(n)
        new_run = np.ones(n, dtype=bool)
        new_run[1:] = keys[1:] != keys[:-1]
        run_start = np.maximum.accumulate(np.where(new_run, idx, 0))
        cur_len = idx - run_start + 1                                   # :218-219,227
        active = self.table[:, self._active_idx].astype(np.int64) != 0  # :211
        tar_key = np.full(n, '', dtype=keys.dtype)
        if fn < n:
            tar_key[:n - fn] = keys[fn:]                                # :213-216
        dates = pd.DatetimeIndex(self._dates)
        last = self.end_date - pd.DateOffset(months=stride)             # :222
        dev_idx = self._create_index_device(keys, active, dates, last) if self._use_device_index() else None
        if dev_idx is not None:
            inp, tar, sel = dev_idx
        else:
            if cfg.train:                                                   # :221-225
                ok = (cur_len >= min_steps) & active & (dates >= self.start_date) & (dates <= last) & (tar_key == keys)
            else:                                                           # :231-234
                ok = (cur_len >= min_steps) & active & (dates >= self.start_date) & (dates <= self.end_date)
            sel = idx[ok]
            cl = cur_len[sel]
            seq_len = np.minimum(cl - (cl - 1) % stride, max_steps)        # :263
            pad = (max_steps - seq_len) // stride                           # :264
            inp = np.stack([sel - seq_len + 1, sel, pad], axis=1).astype(np.int32)
            same = tar_key[sel] == keys[sel]
            tar_end = np.where(same, sel + fn, sel)                         # :270-279
            tar = np.stack([sel - seq_len + 1 + fn, tar_end, pad], axis=1).astype(np.int32)
        meta = np.stack([dates[sel].strftime('%Y%m%d').values.astype('S'), keys[sel].astype('S'),
                         tar_key[sel].astype('S')], axis=1)
        in_train = np.isin(keys[sel], np.asarray(self._train_gvkeys, dtype=keys.dtype))
        in_valid = np.isin(keys[sel], np.asarray(self._valid_gvkeys, dtype=keys.dtype))
        in_test = np.isin(keys[sel], np.asarray(self._test_gvkeys, dtype=keys.dtype))
        if cfg.train:
            if not np.all(in_train | in_valid):                         # :297-298
                raise ValueError("Mismatch between gvkey category (train/valid/test set) and run type (train/ pred)")
            for name, m in (('train', in_train), ('valid', in_valid & ~in_train)):
                self._dataset[name + '_X'], self._dataset[name + '_Y'], self._meta[name] = inp[m], tar[m], meta[m]
        else:
            if not np.all(in_test):
                raise ValueError("Mismatch between gvkey category (train/valid/test set) and run type (train/ pred)")
            self._dataset['test_X'], self._dataset['test_Y'], self._meta['test'] = inp, tar, meta

    @staticmethod
    def _use_device_index():
        """The window index is built by the CUDA kernels (lfmq_window_index) whenever a GPU is present; the vectorised
        NumPy form above serves GPU-less tooling and the CPU tests (LFMQ_HOST_INDEX=1 forces it)."""
        if os.environ.get('LFMQ_HOST_INDEX') == '1':
            return False
        try:
            import torch
            return torch.cuda.is_available()
        except Exception:
            return False

    def _create_index_device(self, keys, active, dates, last_train_date):
        """data_processing.py:170-305 on the device.  String keys become integer codes (equal code <=> equal gvkey), dates
        yyyymmdd ints; the triples come back once, at start-up."""
        import torch
        from ..engine import window_index
        cfg = self.config
        codes = np.unique(keys, return_inverse=True)[1].astype(np.int32)
        ymd = (dates.year.values * 10000 + dates.month.values * 100 + dates.day.values).astype(np.int32)
        as_int = lambda ts: int(pd.Timestamp(ts).strftime('%Y%m%d'))
        cu = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
        inp, tar, rows = window_index(cu(codes), cu(active.astype(np.uint8)), cu(ymd), train=bool(cfg.train),
                                      stride=cfg.stride, forecast_n=cfg.forecast_n, min_unrollings=cfg.min_unrollings,
                                      max_unrollings=cfg.max_unrollings, start_date=as_int(self.start_date),
                                      end_date=as_int(self.end_date), last_train_date=as_int(last_train_date))
        return inp.cpu().numpy(), tar.cpu().numpy(), rows.cpu().numpy().astype(np.int64)

    # ---- the tf.data-like views (data_processing.py:451-474) ------------------------------------------
    @property
    def train_set(self):
        assert self.config.train, 'config.train is not True. train_set is only available during training'
        return IndexSet(self._dataset['train_X'], self._dataset['train_Y'], self._meta['train'])

    @property
    def valid_set(self):
        assert self.config.train, "config.train is not True. valid_set is only available during training"
        return IndexSet(self._dataset['valid_X'], self._dataset['valid_Y'], self._meta['valid'])

    @property
    def test_set(self):
        assert not self.config.train, "config.train is not False. test_set is only available during prediction"
        return IndexSet(self._dataset['test_X'], self._dataset['test_Y'], self._meta['test'])

    # ---- device batcher --------------------------------------------------------------------------------
    def _device_state(self):
        import torch
        if self._dev is None:
            F = len(self.inp_col_ids)
            sflag = np.zeros(F, dtype=np.uint8)
            sflag[self.scale_inp_col_ids] = 1
            aflag = np.zeros(F, dtype=np.uint8)
            aflag[self._aux_col_ids_seq] = 1
            center = np.zeros(F, dtype=np.float64)
            scale = np.ones(F, dtype=np.float64)
            c = np.asarray(self.scaling_params['center'], dtype=np.float64)
            s = np.asarray(self.scaling_params['scale'], dtype=np.float64)
            center[:min(F, c.size)] = c[:F]
            scale[:min(F, s.size)] = s[:F]
            cu = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
            self._dev = dict(table=cu(self.table), inp_cols=cu(np.asarray(self.inp_col_ids, dtype=np.int32)),
                             fin_cols=cu(np.asarray(self.fin_col_ids, dtype=np.int32)), center=cu(center),
                             scale=cu(scale), scale_flag=cu(sflag), aux_flag=cu(aflag))
        return self._dev

    def get_batch(self, inp_indices, tar_indices, pre_metadata):
        """data_processing.py:307-368 -> (inp f32 [B,T,F], tar f32 [B,T,O], metadata [B,3]) on the GPU."""
        import torch
        from ..engine import gather_batch
        d = self._device_state()
        inp_idx = torch.from_numpy(np.ascontiguousarray(inp_indices, dtype=np.int32)).cuda()
        tar_idx = torch.from_numpy(np.ascontiguousarray(tar_indices, dtype=np.int32)).cuda()
        x, y, sn = gather_batch(d['table'], inp_idx, tar_idx, seq_len=self.seq_len, stride=self.config.stride,
                                inp_cols=d['inp_cols'], fin_cols=d['fin_cols'],
                                seq_norm_col=self._seq_norm_idx if self._seq_norm_idx else None,   # `if self._seq_norm_idx:` (:393,444)
                                center=d['center'], scale=d['scale'], scale_flag=d['scale_flag'],
                                aux_flag=d['aux_flag'], log_squasher=self.config.log_squasher,
                                aux_masking=self.config.aux_masking)
        metadata = np.array(pre_metadata, dtype=object)
        metadata[:, 2] = sn.cpu().numpy()              # :349 overwrite tar_key with seq_norm
        if 'MLP' in self.config.nn_type or 'Naive' in self.config.nn_type:
            # :363-365: the window flattened to [B, T*F] (a view of the gathered batch), the targets of the last step
            x = x.view(x.shape[0], self.seq_len * x.shape[2])
            y = y[:, -1, :].contiguous()
        return x, y, metadata

    # ---- helpers kept from the reference ------------------------------------------------------------------
    def get_cols_from_colnames(self, columns):
        """'f1-f5,f7' -> indices and names, ranges follow file column order (data_processing.py:476-503)."""
        colidxs, col_names = [], []
        if columns:
            data_cols = self.data.columns.tolist()
            for col in columns.split(','):
                rng = col.split('-')
                if len(rng) == 1:
                    colidxs.append(data_cols.index(rng[0]))
                    col_names.append(rng[0])
                elif len(rng) == 2:
                    s, e = data_cols.index(rng[0]), data_cols.index(rng[1])
                    assert 0 <= s <= e
                    colidxs.extend(range(s, e + 1))
                    col_names += data_cols[s:e + 1]
        return colidxs, col_names

    def _get_gvkeys(self):
        g = self.data[['date', 'gvkey']]
        return np.asarray([str(k) for k in g[g['date'] <= self.end_date]['gvkey'].unique()], dtype=str)

    @staticmethod
    def train_test_split(keys, validation_size, seed, is_train):
        """data_processing.py:515-537.  The reference seeds the global NumPy generator and draws from it; a generator of
        its own draws the same keys and lets the members of an ensemble build their datasets on concurrent threads."""
        if is_train:
            rng = np.random.RandomState(seed)
            valid_keys = rng.choice(keys, size=int(len(keys) * validation_size), replace=False)
            train_keys = list(set(keys) - set(valid_keys))
            test_keys = []
        else:
            train_keys, valid_keys, test_keys = [], [], keys
        return sorted(train_keys), sorted(valid_keys), sorted(test_keys)

    def get_scaling_params(self):
        """data_processing.py:539-572: fit the sklearn scaler on one random step of a 30 % sample of windows."""
        from sklearn import preprocessing as sk_pre
        assert self.config.train, "scaling params are only calculated during training"
        idx = self._dataset['train_X']
        rng = np.random.RandomState(self.config.seed)
        pick = rng.choice(idx.shape[0], size=int(0.3 * idx.shape[0]), replace=False)
        sample = []
        for start_idx, end_idx, _ in idx[pick]:
            step = rng.randint(self.config.min_unrollings)
            cur_idx = start_idx + step * self.config.stride
            sample.append(np.append(self.get_feature_vector(cur_idx, end_idx), self.get_aux_vector(cur_idx)))
        scaler_class = self.config.data_scaler
        if not hasattr(sk_pre, scaler_class):
            raise RuntimeError("Unknown scaler = %s" % scaler_class)
        scaler = getattr(sk_pre, scaler_class)()
        scaler.fit(np.asarray(sample, dtype=np.float64))
        return {'center': scaler.center_ if hasattr(scaler, 'center_') else scaler.mean_, 'scale': scaler.scale_}

    def get_feature_vector(self, cur_idx, end_idx):
        x = self.table[cur_idx, self.fin_col_ids]
        normalizer = max(self.table[end_idx, self._seq_norm_idx], _MIN_SEQ_NORM) if self._seq_norm_idx else 1.
        x = x / normalizer
        if self.config.log_squasher:
            x = np.sign(x) * np.log1p(np.abs(x))
        return x

    def get_aux_vector(self, cur_idx):
        return self.table[cur_idx, self.aux_col_ids]

    def log_squasher(self, x):
        if self.config.log_squasher:
            x = np.multiply(np.sign(x), np.log1p(np.absolute(x).astype(float)))
        return x

    def reverse_log_squasher(self, x):
        if self.config.log_squasher:
            x = np.multiply(np.sign(x), np.expm1(np.fabs(x)))
        return x

    def print_dataset_stats(self):
        print("[samples, sequence_length, features]")
        for k, v in self._dataset.items():
            print("%s : %s" % (k, None if v is None else (v.shape,)))


class CDRSInferenceData(Dataset):
    """data_processing.py:630-759 depends on the private ``cdrs`` feed (runtime/cdrs_data.py:6); out of scope."""

    def __init__(self, config):
        raise NotImplementedError('CDRSInferenceData needs the proprietary cdrs package; not part of the hot path')
