"""A point-estimate ensemble over two GPUs through the CLI: trains and predicts the system-test configuration with
--num_procs 4 --NPE 4 --num_gpu 2 (members 0 and 2 on GPU 0, 1 and 3 on GPU 1, each with half its GPU), checks every
member's files, checks ensemble_preds.dat against the reference's aggregation, and checks that each member predicts
alone from its model-k.conf what it predicted in the ensemble.

    python tools/ensemble_two_gpu_check.py        (needs 2 GPUs)
"""
import os
import subprocess
import sys
import tempfile

import numpy as np
import pandas as pd

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
from ensemble_checker import expected_ensemble_frame  # noqa: E402
from lfm_quant_b200.scripts.synthetic import write_open_dataset, write_system_test_conf  # noqa: E402


def main():
    import torch
    if torch.cuda.device_count() < 2:
        raise SystemExit('needs 2 GPUs, %d visible' % torch.cuda.device_count())
    d = tempfile.mkdtemp(prefix='ens2gpu')
    write_open_dataset(os.path.join(d, 'datasets', 'open-dataset.dat'), n_keys=30, n_months=420, seed=9)
    conf = os.path.join(d, 'config', 'system-test.conf')
    write_system_test_conf(conf, os.path.join(d, 'datasets'), os.path.join(d, 'experiments'))
    os.makedirs(os.path.join(d, 'experiments'))
    env =dict(os.environ, LFM_QUANT_ROOT=d, PYTHONPATH=ROOT + os.pathsep + os.environ.get('PYTHONPATH', ''))
    cli = [sys.executable, '-m', 'lfm_quant_b200.scripts.lfm_quant']
    ens = ['--config=' + conf, '--num_procs', '4', '--NPE', '4', '--num_gpu', '2', '--model_dir', 'ens']
    for train in ('True', 'False'):
        subprocess.run(cli + ens + ['--train=' + train], check=True, env=env, cwd=ROOT)
    edir = os.path.join(d, 'experiments', 'ens')
    mdirs = [os.path.join(edir, 'system-test-%d' % k) for k in range(4)]
    ok = True
    for k, m in enumerate(mdirs):
        conf_k = os.path.join(m, 'model-%d.conf' % k)
        gpu = [l for l in open(conf_k) if l.startswith('--default_gpu')][0].split()[1]
        files = ['chkpts/chkpt.lfmq.npz', 'train_log/system-test-train-logs-epoch.csv', 'pred/preds.dat']
        good = gpu == '/gpu:%d' % (k % 2) and all(os.path.isfile(os.path.join(m, f)) for f in files)
        subprocess.run(cli + ['--config=' + conf_k, '--train=False', '--preds_fname', 'alone.dat'], check=True, env=env,
                       cwd=ROOT)
        a, b = (pd.read_csv(os.path.join(m, 'pred', f), sep=' ', dtype={'gvkey': str}) for f in ('alone.dat', 'preds.dat'))
        good &= a.equals(b)
        print('member %d on %s: files %s, alone == in the ensemble: %s' % (k, gpu, 'present' if good else 'CHECK',
                                                                          a.equals(b)))
        ok &= good
    members = [pd.read_csv(os.path.join(m, 'pred', 'preds.dat'), sep=' ', dtype={'gvkey': str}) for m in mdirs]
    written = pd.read_csv(os.path.join(edir, 'ensemble_preds.dat'), sep=' ', dtype={'gvkey': str})
    want = expected_ensemble_frame(members, 1)
    agg = bool(np.allclose(written['norm_preds_1'], want['norm_preds_1'], rtol=1e-12, atol=0) and
               list(written.columns) == list(want.columns))
    print('ensemble_preds.dat equals the independent checker: %s' % agg)
    ok &= agg
    print('OK' if ok else 'FAILED')
    sys.exit(0 if ok else 1)


if __name__ == '__main__':
    main()
