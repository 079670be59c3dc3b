"""Wall time of a walk-forward backtest (training_type iterative, DESIGN.md section 6c) with its W origins trained and
predicted side by side (NPE = W) against one after another (NPE = 1), in one command, on the synthetic dataset.

Default size: W = 5 origins (split_date 199912, stride 12, end_date 200412), 1000 companies over 35 years, the
reference's default window (min/max_unrollings 5) and layers (2), num_hidden 256, batch_size 256, fp32, 1 epoch.  The
two modes alternate (--repeats times each, default once), both with the seeded batch order, and their stitched
walk_forward_preds.dat must be identical.

    python tools/bench_walk_forward.py [--origins 5] [--n_keys 1000] [--num_hidden 256] [--batch_size 256]
                                       [--max_epoch 1] [--precision fp32] [--repeats 1] [--out FILE]

Prints one JSON line per run: wall seconds of the whole backtest (train every origin, then predict every origin) and
each origin's mean epoch seconds (from its train_log), with the GPU's name and power limit read in the same command.
Everything it writes goes to a temporary directory, removed at the end; --out FILE also writes the JSON lines there.
Without a CUDA device it builds the dataset, the backtest's config and the origins' directories and configs, prints
them, and exits with an error.
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CONF = """--name wf-bench
--datafile open-dataset.dat
--data_dir {data_dir}
--experiments_dir {experiments_dir}
--nn_type RNNPointEstimate
--rnn_cell lstm
--financial_fields saleq_ttm-ltq_mrq
--aux_fields rel_mom1m-rel_mom9m
--target_field oiadpq_ttm
--scale_field mrkcap
--num_layers 2
--min_unrollings 5
--max_unrollings 5
--stride 12
--forecast_n 12
--start_date 197501
--end_date 200412
--training_type iterative
--early_stop 10
--optimizer Adadelta
--learning_rate 0.6
--logging_interval 100
--seed 521
"""


def gpu_info():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else 'unknown'


def backtest_argv(a, conf, model_dir, npe):
    from lfm_quant_b200.scripts.runtime.model_execution import add_months
    return ['--config=' + conf, '--model_dir', model_dir, '--NPE', str(npe), '--train=True',
            '--split_date', str(add_months(200412, -12 * a.origins)), '--num_hidden', str(a.num_hidden),
            '--batch_size', str(a.batch_size), '--max_epoch', str(a.max_epoch), '--precision', a.precision]


def config(argv):
    from lfm_quant_b200.scripts import configs, lfm_quant
    configs.reset()
    return lfm_quant.get_configs(argv)


def epoch_seconds(train_cfg):
    """Mean seconds per epoch of one origin, from the times its epoch log records at the end of each epoch."""
    import numpy as np
    import pandas as pd
    log = pd.read_csv(os.path.join(train_cfg.model_dir, 'train_log', train_cfg.name + '-train-logs-epoch.csv'))
    return float(np.diff(np.concatenate([[0.0], log['time'].to_numpy()])).mean())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--origins', type=int, default=5)
    ap.add_argument('--n_keys', type=int, default=1000)
    ap.add_argument('--num_hidden', type=int, default=256)
    ap.add_argument('--batch_size', type=int, default=256)
    ap.add_argument('--max_epoch', type=int, default=1)
    ap.add_argument('--precision', default='fp32')
    ap.add_argument('--repeats', type=int, default=1)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    from lfm_quant_b200.scripts.runtime.model_execution import ModelExecution, check_walk_forward, origin_configs
    from lfm_quant_b200.scripts.synthetic import write_open_dataset
    os.environ['LFMQ_SEEDED_SHUFFLE'] = '1'          # both modes walk the same batch order: the same work, the same bits
    work = tempfile.mkdtemp(prefix='bench_wf_')
    try:
        os.environ.setdefault('LFM_QUANT_ROOT', work)
        rows = write_open_dataset(os.path.join(work, 'datasets', 'open-dataset.dat'), n_keys=a.n_keys, n_months=420,
                                  seed=521)
        conf = os.path.join(work, 'bench.conf')
        os.makedirs(os.path.join(work, 'experiments'))
        with open(conf, 'w') as fh:
            fh.write(CONF.format(data_dir=os.path.join(work, 'datasets'),
                                 experiments_dir=os.path.join(work, 'experiments')))
        modes = [('side_by_side', a.origins), ('one_after_another', 1)]
        runs = [(name, npe, r) for r in range(a.repeats) for name, npe in modes]
        plans = {}
        for name, npe, r in runs:
            c = config(backtest_argv(a, conf, '%s-%d' % (name, r), npe))
            check_walk_forward(c)
            _, origins = origin_configs(c)
            plans[(name, r)] = (c, origins)
        c0, origins0 = plans[runs[0][0], 0]
        print('dataset: %d rows, %d companies; origins %s; predictions %s' % (
            rows, a.n_keys, [o for o, _, _ in origins0], [(p.start_date, p.end_date) for _, _, p in origins0]),
            flush=True)
        for o, t, _ in origins0:
            print('  origin %d: %s (training %d-%d)' % (o, t.model_dir, t.start_date, t.end_date), flush=True)

        import torch
        if not torch.cuda.is_available():
            raise SystemExit('bench_walk_forward needs a CUDA GPU')
        torch.cuda.set_device(0)
        gpu = gpu_info()
        lines, stitched = [], {}
        for name, npe, r in runs:
            c, origins = plans[(name, r)]
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ModelExecution(c)()
            torch.cuda.synchronize()
            wall = time.perf_counter() - t0
            path = os.path.join(c.experiments_dir, c.model_dir, 'walk_forward_preds.dat')
            stitched[(name, r)] = open(path, 'rb').read()
            res = {'mode': name, 'repeat': r, 'NPE': npe, 'origins': len(origins), 'wall_s': wall,
                   'epoch_s': {str(o): epoch_seconds(t) for o, t, _ in origins},
                   'shape': {'n_keys': a.n_keys, 'T': c.max_unrollings, 'H': c.num_hidden, 'L': c.num_layers,
                             'B': c.batch_size, 'max_epoch': c.max_epoch, 'precision': c.precision},
                   'identical_to_first': stitched[(name, r)] == stitched[(runs[0][0], 0)], 'gpu': gpu}
            print(json.dumps(res), flush=True)
            lines.append(res)
        if a.out:
            os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
            with open(a.out, 'w') as f:
                for res in lines:
                    f.write(json.dumps(res) + '\n')
    finally:
        shutil.rmtree(work, ignore_errors=True)


if __name__ == '__main__':
    main()
