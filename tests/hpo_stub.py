"""Stand-in for training a hyper-parameter search candidate: reads the candidate's model.conf and writes the files the
search reads back, with losses that are a fixed function of the config.  Used by tests/golden/make_reference_hpo.py
(in place of the reference's ``os.system("python lfm_quant.py --config=...")``) and by tests/test_hpo_host.py (in place
of training on the GPU), so that both searches see the same objective for the same candidate.

The candidate with member_id FAIL_ID writes nothing, as a candidate whose run failed: the search scores it inf.
"""
import os
import zlib

FAIL_ID = 3
# bookkeeping flags that differ between candidates of the same config, and the project's own `precision` flag (the
# reference has no such flag): left out of the objective
_NOT_HASHED = ('member_id', 'model_dir', 'default_gpu', 'precision')


def read_conf(path):
    """{flag: value as written} of a model.conf file (list values keep their '-' joins)."""
    flags, name = {}, None
    for token in open(path).read().split():
        if token.startswith('--'):
            name = token[2:]
            flags[name] = ''
        else:
            flags[name] = (flags[name] + ' ' + token).strip()
    return flags


def objective(flags):
    key = '\n'.join('%s=%s' % (k, flags[k]) for k in sorted(flags) if k not in _NOT_HASHED)
    return 0.5 + (zlib.crc32(key.encode()) % 10007) / 1000.0


def train_candidate(conf_path):
    """Writes <experiments_dir>/<model_dir>/train_log/<name>-train-logs-epoch.csv (train=True; two epochs, the second
    the better one) or pred/<preds_fname> (train=False) for the candidate of `conf_path`."""
    flags = read_conf(conf_path)
    if int(flags['member_id']) == FAIL_ID:
        return
    mse = objective(flags)
    model_dir = os.path.join(flags['experiments_dir'], flags['model_dir'])
    if flags.get('train', 'True') == 'True':
        os.makedirs(os.path.join(model_dir, 'train_log'), exist_ok=True)
        with open(os.path.join(model_dir, 'train_log', flags['name'] + '-train-logs-epoch.csv'), 'w') as fh:
            fh.write('epoch,valid_mse,valid_mse_fcst,valid_uq_loss\n')
            fh.write('0,%r,%r,%r\n' % (mse + 0.5, 2 * mse, 3 * mse))
            fh.write('1,%r,%r,%r\n' % (mse, 2 * mse + 0.125, 3 * mse + 0.25))
    else:
        os.makedirs(os.path.join(model_dir, 'pred'), exist_ok=True)
        with open(os.path.join(model_dir, 'pred', flags.get('preds_fname', 'preds.dat')), 'w') as fh:
            fh.write('date gvkey norm_squared_diff_1\n')
            fh.write('200001 001000 %r\n200001 001001 %r\n' % (mse, mse + 0.25))
