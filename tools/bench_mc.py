"""Times Monte-Carlo dropout prediction of RNNUqRangeEstimate on one GPU: `samples` samples of every window in one
call (ForecastChainEngine.forward_mc, lfmq_forward_uq_mc) against `samples` back-to-back predictions, each
ForecasterEngine.forward at the keys of one sample, the way a caller would draw them one model.predict at a time.

Shapes: H = 256, T = 48, F = 32, O = 16, one layer, dropout 0.2 and recurrent dropout 0.15, at B = 256 (the
reference's prediction batch_size) and B = 65536, samples 1 / 8 / 32, at fp32, bf16 and bf16x3.  Both sides are device
time over CUDA events after a warm-up call; the loop's predictions stay on the device and its moments are not
combined, so it is the loop's lower bound.  Prints one JSON line per case and the card it ran on.

--model: the model object's route instead, NativeForecaster.predict_mc at batch_size B, on the engine of
min(S * B, MC_ROWS) rows it creates ("after") against the batch_size handle it used before ("before": MC_ROWS = 1
keeps it there), same weights and shapes, device time over CUDA events.
--cli: `lfm_quant.py --train=False --mc_samples S` wall time on a synthetic dataset (--keys companies, trained for one
epoch first), after and before alternated, and the time of the ensemble_preds.dat aggregation of its preds.dat.

usage: python tools/bench_mc.py [--out FILE] [--reps N] [--model | --cli]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from lfm_quant_b200.engine import ForecastChainEngine  # noqa: E402
from lfm_quant_b200.scripts.models.point_estimate import rnn_point_estimate as rpe  # noqa: E402

H, T, F, O = 256, 48, 32, 16


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()


def timed(fn, reps):
    fn()                                              # warm-up: module load, first launches of this shape
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def _flags(argv):
    from lfm_quant_b200.scripts import base_config, configs
    configs.reset()
    return base_config.get_configs(argv)


def bench_model(a, gpu):
    """predict_mc of the model object, after (wide engine) and before (batch_size handle)."""
    rows = []
    for prec in a.precisions.split(','):
        for B in [int(v) for v in a.batches.split(',')]:
            m = rpe.NativeForecaster(_flags(['--num_hidden', str(H), '--num_layers', '1', '--batch_size', str(B),
                                             '--dropout', '0.2',
                                             '--recurrent_dropout', '0.15', '--precision', prec, '--train=False',
                                             '--nn_type', 'RNNUqRangeEstimate', '--UQ=True', '--seed', '7']),
                                     T, F, O, 0, uq=True)
            rng = np.random.RandomState(0)
            m.set_weights([w + rng.normal(size=w.shape).astype(np.float32) * 0.05 if w.ndim == 2 else w
                           for w in m.get_weights()])
            x = torch.randn(B, T, F, generator=torch.Generator(device='cuda').manual_seed(0), device='cuda')
            for S in [int(v) for v in a.samples.split(',')]:
                after = timed(lambda: m.predict_mc(x, S), a.reps)
                mc_rows = rpe.MC_ROWS
                rpe.MC_ROWS = 1
                try:
                    before = timed(lambda: m.predict_mc(x, S), a.reps)
                finally:
                    rpe.MC_ROWS = mc_rows
                r = dict(route='predict_mc', precision=prec, B=B, samples=S, before_ms=round(before, 3),
                         after_ms=round(after, 3), speedup=round(before / after, 3),
                         rows_per_launch=min(S * B, mc_rows), card=gpu)
                print(json.dumps(r), flush=True)
                rows.append(r)
            m.close()
            del m, x
            torch.cuda.empty_cache()
    return rows


def bench_cli(a, gpu):
    """lfm_quant.py prediction with --mc_samples, after and before, and the aggregation step."""
    from lfm_quant_b200.scripts import configs
    from lfm_quant_b200.scripts import lfm_quant as cli
    from lfm_quant_b200.scripts.runtime.model_execution import ModelExecution, ensemble_uq_estimate
    from lfm_quant_b200.scripts.synthetic import write_open_dataset, write_system_test_conf
    rows = []
    with tempfile.TemporaryDirectory() as d:
        write_open_dataset(os.path.join(d, 'datasets', 'open-dataset.dat'), n_keys=a.keys, n_months=420, seed=9)
        conf = os.path.join(d, 'system-test.conf')
        write_system_test_conf(conf, os.path.join(d, 'datasets'), os.path.join(d, 'experiments'))
        os.makedirs(os.path.join(d, 'experiments'))
        os.environ.setdefault('LFM_QUANT_ROOT', d)
        base = ['--config=' + conf, '--nn_type', 'RNNUqRangeEstimate', '--UQ=True', '--num_hidden', str(H),
                '--batch_size', '256', '--dropout', '0.2', '--recurrent_dropout', '0.15', '--max_epoch', '1']
        configs.reset()
        cli.main(base + ['--train=True'])
        for prec in a.precisions.split(','):
            argv = base + ['--train=False', '--precision', prec]
            for S in [int(v) for v in a.samples.split(',')]:
                times = {'after': [], 'before': []}
                for rep in range(a.reps + 1):               # rep 0 warms up both
                    for name in ('after', 'before'):
                        mc_rows = rpe.MC_ROWS
                        rpe.MC_ROWS = mc_rows if name == 'after' else 1
                        try:
                            configs.reset()
                            t0 = time.perf_counter()
                            cli.main(argv + ['--mc_samples', str(S)])
                            torch.cuda.synchronize()
                            dt = time.perf_counter() - t0
                        finally:
                            rpe.MC_ROWS = mc_rows
                        if rep:
                            times[name].append(dt)
                c = _flags(argv + ['--mc_samples', str(S)])
                frame = ModelExecution.read_results(c)[2]
                t0 = time.perf_counter()
                ensemble_uq_estimate(frame, c.forecast_steps)
                agg = time.perf_counter() - t0
                r = dict(route='cli', precision=prec, samples=S, windows=len(frame),
                         before_s=round(min(times['before']), 3), after_s=round(min(times['after']), 3),
                         speedup=round(min(times['before']) / min(times['after']), 3),
                         aggregation_ms=round(agg * 1e3, 2), card=gpu)
                print(json.dumps(r), flush=True)
                rows.append(r)
        configs.reset()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--precisions', default='fp32,bf16,bf16x3')
    ap.add_argument('--batches', default='256,65536')
    ap.add_argument('--samples', default='1,8,32')
    ap.add_argument('--model', action='store_true')
    ap.add_argument('--cli', action='store_true')
    ap.add_argument('--keys', type=int, default=400)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_mc.py needs a CUDA GPU')
    gpu = card()
    print('card: %s' % gpu)
    if a.model or a.cli:
        rows = bench_model(a, gpu) if a.model else bench_cli(a, gpu)
        if a.out:
            os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
            with open(a.out, 'w') as f:
                json.dump(rows, f, indent=1)
        return
    rows = []
    g = torch.Generator(device='cuda').manual_seed(0)
    for prec in a.precisions.split(','):
        for B in [int(v) for v in a.batches.split(',')]:
            eng = ForecastChainEngine(max_batch=B, seq_len=T, n_inputs=F, n_outputs=O, num_hidden=H, num_layers=1,
                                      uq=True, precision=prec, train=False, forward_only=True, dropout=0.2,
                                      recurrent_dropout=0.15, seed=7)
            flat = torch.randn(eng.stages[0].n_total, generator=g, device='cuda') * 0.05
            flat[-H:] = 1.0                           # BN moving variance
            eng.stages[0].set_flat(flat.cpu().numpy())
            x = torch.randn(B, T, F, generator=g, device='cuda')
            one = eng.stages[0]
            # the same weights on a handle with room for every sample of the batch in one launch (max_batch = B * the
            # largest sample count, up to 65536 rows): only there do the samples share a launch
            wide_mb = min(B * max(int(v) for v in a.samples.split(',')), 65536)
            wide = None
            if wide_mb > B:
                wide = ForecastChainEngine(max_batch=wide_mb, seq_len=T, n_inputs=F, n_outputs=O, num_hidden=H,
                                           num_layers=1, uq=True, precision=prec, train=False, forward_only=True,
                                           dropout=0.2, recurrent_dropout=0.15, seed=7)
                wide.stages[0].set_flat(flat.cpu().numpy())
            for S in [int(v) for v in a.samples.split(',')]:
                reps = max(1, a.reps if B * S <= 65536 * 8 else 1)
                mc = timed(lambda: eng.forward_mc(x, S, step=1), reps)
                loop = timed(lambda: [one.forward(x, step=1, row0=s * B) for s in range(S)], reps)
                r = dict(precision=prec, B=B, samples=S, mc_ms=round(mc, 3), loop_ms=round(loop, 3),
                         speedup=round(loop / mc, 3), mc_window_samples_per_s=round(B * S / mc * 1e3),
                         loop_window_samples_per_s=round(B * S / loop * 1e3), card=gpu)
                if wide is not None:
                    got, ref = wide.forward_mc(x, S, step=1), eng.forward_mc(x, S, step=1)
                    assert all(torch.equal(u, v) for u, v in zip(got[0], ref[0])), 'wide launches changed the bits'
                    mcw = timed(lambda: wide.forward_mc(x, S, step=1), reps)
                    r.update(wide_max_batch=wide_mb, mc_wide_ms=round(mcw, 3), speedup_wide=round(loop / mcw, 3))
                print(json.dumps(r), flush=True)
                rows.append(r)
            eng.close()
            if wide is not None:
                wide.close()
            del eng, wide, x
            torch.cuda.empty_cache()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(rows, f, indent=1)


if __name__ == '__main__':
    main()
