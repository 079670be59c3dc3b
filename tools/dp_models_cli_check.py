"""Data parallelism of RNNUqRangeEstimate and of multi-step forecasts through the CLI (scripts/train.py under torchrun):
trains the system-test configuration on 1 GPU and on 2 GPUs (one model, the company-batch axis sharded), once with
--UQ=True and once with --forecast_steps 2 --forecast_steps_weights 1.0-0.5, and compares the train logs and the saved
weights of the two runs.

    python tools/dp_models_cli_check.py        (needs 2 GPUs)
"""
import os
import subprocess
import sys
import tempfile

import numpy as np
import pandas as pd

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from lfm_quant_b200.scripts.synthetic import write_open_dataset, write_system_test_conf  # noqa: E402

CASES = {
    'uq': ['--nn_type', 'RNNUqRangeEstimate', '--UQ=True', '--dropout', '0.1'],
    'forecast2': ['--forecast_steps', '2', '--forecast_steps_weights', '1.0-0.5'],
}
TOL = 1e-3          # fp32: the two runs differ only in the order of the gradient sums


def _rel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(np.max(np.abs(a - b) / np.maximum(np.abs(b), 1e-30)))


def main():
    d = tempfile.mkdtemp(prefix='dpmodels')
    write_open_dataset(os.path.join(d, 'datasets', 'open-dataset.dat'), n_keys=30, n_months=420, seed=9)
    conf = os.path.join(d, 'config', 'system-test.conf')
    write_system_test_conf(conf, os.path.join(d, 'datasets'), os.path.join(d, 'experiments'))
    # LFMQ_SEEDED_SHUFFLE=1: the 1-GPU run walks the batch order every data-parallel rank walks
    env = dict(os.environ, LFM_QUANT_ROOT=d, LFMQ_SEEDED_SHUFFLE='1',
               PYTHONPATH=ROOT + os.pathsep + os.environ.get('PYTHONPATH', ''))
    ok = True
    for name, extra in CASES.items():
        common = ['-m', 'lfm_quant_b200.scripts.lfm_quant', '--config=' + conf, '--train=True'] + extra
        subprocess.run([sys.executable] + common + ['--model_dir', name + '-one'], check=True, env=env, cwd=ROOT)
        subprocess.run([sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node', '2',
                        '--master-addr', '127.0.0.1', '--master-port', '29534'] + common + ['--model_dir', name + '-two'],
                       check=True, env=env, cwd=ROOT)
        ex = os.path.join(d, 'experiments')
        logs = [pd.read_csv(os.path.join(ex, name + m, 'train_log', 'system-test-train-logs-%s.csv' % kind))
                for m in ('-one', '-two') for kind in ('batch', 'epoch')]
        w1, w2 = (np.load(os.path.join(ex, name + m, 'chkpts', 'chkpt.lfmq.npz')) for m in ('-one', '-two'))
        cols = ['mse', 'uq_loss'] if '--UQ=True' in extra else ['mse']
        rel = max(_rel(logs[i + 2][c], logs[i][c]) for i in (0, 1) for c in cols)
        worst = max(float(np.abs(w1[k] - w2[k]).max() / max(np.abs(w1[k]).max(), 1e-30)) for k in w1.files)
        print('%s: epoch %s 1 GPU %s, 2 GPUs %s' % (name, cols, logs[1][cols].values.tolist(),
                                                   logs[3][cols].values.tolist()))
        print('%s: max rel diff of the logged losses %.3e, of the saved weights %.3e' % (name, rel, worst))
        good = (set(w1.files) == set(w2.files) and np.isfinite(logs[3]['mse']).all() and rel < TOL
                and worst < 10 * TOL)
        print('%s: %s' % (name, 'OK' if good else 'FAILED'))
        ok &= good
    sys.exit(0 if ok else 1)


if __name__ == '__main__':
    main()
