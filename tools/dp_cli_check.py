"""Data parallelism through the CLI (scripts/train.py under torchrun): trains the system-test configuration on 1 GPU and on
2 GPUs (one model, the company-batch axis sharded) and compares the epoch logs and the final weights.

    python tools/dp_cli_check.py [--precision fp32]        (needs 2 GPUs)
"""
import argparse
import os
import subprocess
import sys
import tempfile

import numpy as np
import pandas as pd

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from lfm_quant_b200.scripts.synthetic import write_open_dataset, write_system_test_conf  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--precision', default='fp32')
    a = ap.parse_args()
    d = tempfile.mkdtemp(prefix='dpcli')
    write_open_dataset(os.path.join(d, 'datasets', 'open-dataset.dat'), n_keys=30, n_months=420, seed=9)
    conf = os.path.join(d, 'config', 'system-test.conf')
    write_system_test_conf(conf, os.path.join(d, 'datasets'), os.path.join(d, 'experiments'))
    # the reference shuffles the batch ORDER of an epoch with an unseeded random.shuffle (train.py:115); data-parallel runs
    # must seed it (all ranks walk the same order).  LFMQ_SEEDED_SHUFFLE=1 makes the 1-GPU run walk that order too, so the
    # two trajectories are comparable step by step.
    env = dict(os.environ, LFM_QUANT_ROOT=d, LFMQ_SEEDED_SHUFFLE='1',
               PYTHONPATH=ROOT + os.pathsep + os.environ.get('PYTHONPATH', ''))
    common = ['-m', 'lfm_quant_b200.scripts.lfm_quant', '--config=' + conf, '--train=True', '--precision', a.precision]
    subprocess.run([sys.executable] + common + ['--model_dir', 'one'], check=True, env=env, cwd=ROOT)
    subprocess.run([sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node', '2', '--master-addr',
                    '127.0.0.1', '--master-port', '29533'] + common + ['--model_dir', 'two'], check=True, env=env, cwd=ROOT)
    e1 = pd.read_csv(os.path.join(d, 'experiments', 'one', 'train_log', 'system-test-train-logs-epoch.csv'))
    e2 = pd.read_csv(os.path.join(d, 'experiments', 'two', 'train_log', 'system-test-train-logs-epoch.csv'))
    w1 = np.load(os.path.join(d, 'experiments', 'one', 'chkpts', 'chkpt.lfmq.npz'))
    w2 = np.load(os.path.join(d, 'experiments', 'two', 'chkpts', 'chkpt.lfmq.npz'))
    print('epoch mse 1 GPU :', e1['mse'].tolist(), 'valid', e1['valid_mse'].tolist())
    print('epoch mse 2 GPUs:', e2['mse'].tolist(), 'valid', e2['valid_mse'].tolist())
    worst = max(float(np.abs(w1[k] - w2[k]).max() / max(np.abs(w1[k]).max(), 1e-30)) for k in w1.files)
    rel = float(np.max(np.abs(e1['mse'].values - e2['mse'].values) / np.abs(e1['mse'].values)))
    print('max rel diff of epoch mse %.3e, of saved weights %.3e' % (rel, worst))
    tol = 1e-3 if a.precision == 'fp32' else 3e-2
    assert np.isfinite(e2['mse']).all() and e2['mse'].iloc[-1] < e2['mse'].iloc[0]
    assert rel < tol and worst < 10 * tol, (rel, worst)
    print('OK')


if __name__ == '__main__':
    main()
