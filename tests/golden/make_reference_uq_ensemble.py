"""Generates tests/golden/reference_uq_ensemble.npz by running the UNMODIFIED reference post-processing
(/root/reference/scripts/utils/post_processing.py: PredictionsPostProcessing(...).aggregate_uq_estimate([0.5])) on
seeded synthetic UQ prediction frames, one frame per call, as the project's Monte-Carlo prediction writes them.

What is replaced, and nothing else: ``from base_config import get_configs`` (the reference's flag parser, which
post_processing only imports for its __main__ block) by a module whose get_configs is never called.  The config is a
namespace with the two attributes the class reads, UQ = True and forecast_steps.  scikit-learn is the installed one.

Each frame is written as preds.dat is (sep=' ', the column order of the project's Predict with --mc_samples, including
the norm_preds_var_<k> columns) and read back as ModelExecution.read_results reads it.  The reference is given that
frame without its norm_preds_var_<k> columns.  Recorded per case:
- ``<case>/in_csv``: the preds.dat text;
- ``<case>/out_csv``: the returned frame, written with to_csv(sep=' ', index=False);
- ``<case>/stdout``: what the call printed;
- ``<case>/freq`` [100, fields] and ``<case>/z`` [fields]: the coverage of each prediction field over the 100 z-scores
  (the reference's _get_frequency) and IsotonicRegression().fit(freq[:, i], z_score).predict([0.5]).
Cases: one and two forecast steps with some NaN targets, every target NaN, five rows (tied coverage frequencies), and a
second step whose intervals never cover half the targets (the level outside the fitted range: NaN lower bounds).
``iso/<name>/{freq,level,out}`` hold a few direct isotonic cases: a single distinct frequency, levels on and beside
the fitted points, levels below and above the range.

Only runs where /root/reference exists; the .npz it writes is what travels.

usage: python tests/golden/make_reference_uq_ensemble.py
"""
import contextlib
import io
import os
import sys
import types

import numpy as np
import pandas as pd

HERE = os.path.dirname(os.path.abspath(__file__))
REF = '/root/reference/scripts/utils'


def preds_frame(n, steps, seed, nan_frac=0.0, tight_steps=()):
    """A preds.dat of a UQ prediction with Monte-Carlo samples: the moments of the scaled forecast, un-scaled with a
    centre, a scale and seq_norm.  Steps in `tight_steps` get variances far below their errors."""
    rng = np.random.RandomState(seed)
    scale, center = 1.7, 0.05
    d = {'date': rng.choice([19991231, 20000331, 20000630, 20000930], n),
         'gvkey': ['%06d' % k for k in rng.randint(1000, 99999, n)],
         'seq_norm': rng.uniform(1.0, 10.0, n)}
    nt = rng.normal(size=n)
    nt[rng.rand(n) < nan_frac] = np.nan
    cols = {}
    for s in range(1, steps + 1):
        cols['targets_%d' % s] = nt
        cols['norm_preds_%d' % s] = np.where(np.isnan(nt), rng.normal(size=n), nt) + rng.normal(0, 0.4 * s, n)
        v = np.exp(rng.normal(-1.5, 0.5, n))
        cols['norm_variance_%d' % s] = v * 1e-2 if s in tight_steps else v
        cols['norm_preds_var_%d' % s] = np.exp(rng.normal(-3.0, 0.5, n))
    for key in ('targets', 'norm_preds', 'norm_variance', 'norm_preds_var'):
        for s in range(1, steps + 1):
            d['%s_%d' % (key, s)] = cols['%s_%d' % (key, s)]
    df = pd.DataFrame(d)

    def unscale(a):
        return (np.asarray(a) * scale + center) * df['seq_norm'].values

    for s in range(1, steps + 1):
        df['norm_targets_%d' % s] = df['targets_%d' % s]
        df['norm_squared_diff_%d' % s] = np.square(df['norm_targets_%d' % s] - df['norm_preds_%d' % s])
    for s in range(1, steps + 1):
        df['targets_%d' % s] = unscale(df['targets_%d' % s])
    for s in range(1, steps + 1):
        df['preds_%d' % s] = unscale(df['norm_preds_%d' % s])
    for s in range(1, steps + 1):
        df['variance_%d' % s] = (df['norm_variance_%d' % s] * scale) * df['seq_norm'].values
    for s in range(1, steps + 1):
        df['fcst_err_%d' % s] = ((df['targets_%d' % s] - df['preds_%d' % s]) / df['targets_%d' % s]).abs()
        df['abs_err_%d' % s] = (df['targets_%d' % s] - df['preds_%d' % s]).abs()
        df['unscaled_squared_err_%d' % s] = np.square(df['abs_err_%d' % s] / df['seq_norm'])
    buf = io.StringIO()
    df.to_csv(buf, sep=' ', index=False)
    return buf.getvalue()


CASES = {
    'one_step': dict(n=160, steps=1, seed=1, nan_frac=0.05),
    'two_steps': dict(n=120, steps=2, seed=2, nan_frac=0.08),
    'all_nan': dict(n=40, steps=1, seed=3, nan_frac=1.0),
    'few_rows': dict(n=5, steps=1, seed=4),
    'out_of_range': dict(n=100, steps=2, seed=5, nan_frac=0.03, tight_steps=(2,)),
}

ISO = {
    # every interval holds the same share of the targets: one distinct frequency, a constant fit
    'single_frequency': (np.zeros(100), 0.5),
    'below_range': (np.linspace(0.6, 1.0, 100), 0.5),
    'above_range': (np.linspace(0.0, 0.4, 100), 0.5),
    'on_a_point': (np.repeat(np.linspace(0.0, 1.0, 11), [20, 5, 5, 10, 10, 10, 10, 10, 10, 5, 5]), 0.5),
    'decreasing_run': (np.concatenate([np.linspace(0.0, 0.7, 60), np.linspace(0.6, 0.2, 20), np.ones(20)]), 0.5),
}


def main():
    sys.path.insert(0, REF)
    sys.modules['base_config'] = types.SimpleNamespace(get_configs=None)
    import scipy.stats as st
    from post_processing import PredictionsPostProcessing
    from sklearn.isotonic import IsotonicRegression
    z_score = st.norm.ppf(np.linspace(0.0001, 0.999999, 100))     # post_processing.py:109-110
    out = {}
    for name, case in CASES.items():
        text = preds_frame(**case)
        frame = pd.read_csv(io.StringIO(text), sep=' ', dtype={'gvkey': str})
        frame = frame.drop(columns=[c for c in frame.columns if c.startswith('norm_preds_var_')])
        config = types.SimpleNamespace(UQ=True, forecast_steps=case['steps'])
        pp = PredictionsPostProcessing([frame], config)
        freq = np.array([pp._get_frequency(z, frame) for z in z_score])
        printed = io.StringIO()
        with contextlib.redirect_stdout(printed):
            agg = PredictionsPostProcessing([frame.copy()], config).aggregate_uq_estimate([0.5])
        buf = io.StringIO()
        agg.to_csv(buf, sep=' ', index=False)
        out[name + '/in_csv'] = np.array(text)
        out[name + '/out_csv'] = np.array(buf.getvalue())
        out[name + '/stdout'] = np.array(printed.getvalue())
        out[name + '/freq'] = freq
        if name != 'all_nan':
            out[name + '/z'] = np.array([IsotonicRegression().fit(freq[:, i], z_score).predict([0.5])[0]
                                         for i in range(freq.shape[1])])
        print(name, agg.shape, list(agg.columns)[-4:], printed.getvalue().strip().replace('\n', ' | '))
    for name, (freq, level) in ISO.items():
        out['iso/%s/freq' % name] = freq
        out['iso/%s/level' % name] = np.array(level)
        out['iso/%s/out' % name] = IsotonicRegression().fit(freq, z_score).predict([level])
        print('iso', name, out['iso/%s/out' % name])
    np.savez_compressed(os.path.join(HERE, 'reference_uq_ensemble.npz'), **out)


if __name__ == '__main__':
    main()
