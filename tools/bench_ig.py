"""Times integrated-gradients attributions of the point forecast on one GPU (ForecasterEngine.integrated_gradients,
lfmq_integrated_gradients) against a loop of M forward + backward calls through the public API (lfmq_forward +
lfmq_backward on a handle of B rows, the work a caller pays per interpolant today; it forms parameter gradients and no
input gradient, so it is the loop's lower bound).

Shapes: T = 48, F = 32, O = 16 at B = 256 and 4096, H = 256 / L = 1 and BASELINE configs[2] (H = 512, L = 2), M = 1, 8
and 32, at fp32 and tf32.  The attribution runs on a handle of min(M * B, --rows) rows, as NativeForecaster.attribute
does (IG_ROWS).  Device time over CUDA events after a warm-up call; the card's name and power limit are read in the
same run.  Prints one JSON line per case.

The switch that skips the parameter-gradient GEMMs is measured by running this tool on the library built with
-DLFMQ_IG_PARAM_GRADS (`make alt ALT_FLAGS=-DLFMQ_IG_PARAM_GRADS`, then LFMQ_LIB_PATH=lfm_quant_b200/_lfmq_alt.so):
its attribution column is then the call with the parameter gradients formed.
--sweep: the attribution at B = 256, M = 32, H = 256 on handles of 2048, 4096 and 8192 rows, and their workspaces.

usage: python tools/bench_ig.py [--out FILE] [--rows N] [--no-loop] [--sweep]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from lfm_quant_b200 import _native as N  # noqa: E402
from lfm_quant_b200.engine import ForecasterEngine  # noqa: E402

T, F, O = 48, 32, 16
SHAPES = {'H256-L1': (256, 1), 'configs2': (512, 2)}


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


def engine(rows, H, L, prec):
    rng = np.random.RandomState(0)
    e = ForecasterEngine(max_batch=rows, seq_len=T, n_inputs=F, n_outputs=O, num_hidden=H, num_layers=L, target_idx=3,
                         precision=prec, train=False, forward_only=False, dropout=0.2, recurrent_dropout=0.15)
    e.set_weights([rng.uniform(-0.1, 0.1, size=s[1]) for s in e.trainable_specs])
    return e


def workspace_gb(e):
    return e.workspace.numel() / 1e9


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    ap.add_argument('--rows', type=int, default=4096)
    ap.add_argument('--no-loop', action='store_true')
    ap.add_argument('--sweep', action='store_true')
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_ig: no CUDA device')
    gpu = card()
    lib = N.lib_path()
    out = open(a.out, 'a') if a.out else None
    rng = np.random.RandomState(1)

    def emit(rec):
        rec.update(gpu=gpu, lib=os.path.basename(lib))
        line = json.dumps(rec)
        print(line, flush=True)
        if out:
            out.write(line + '\n')
            out.flush()

    if a.sweep:
        H, L = SHAPES['H256-L1']
        x = torch.from_numpy(rng.normal(size=(256, T, F)).astype(np.float32)).cuda()
        for prec in ('fp32', 'tf32'):
            for rows in (2048, 4096, 8192):
                e = engine(rows, H, L, prec)
                ms = timed(lambda: e.integrated_gradients(x, 32), 3)
                emit(dict(mode='sweep', prec=prec, B=256, M=32, rows=rows, shape='H256-L1', ig_ms=round(ms, 3),
                          workspace_gb=round(workspace_gb(e), 3)))
                e.close()
                torch.cuda.empty_cache()
        return
    for shape, (H, L) in SHAPES.items():
        for prec in ('fp32', 'tf32'):
            for B in (256, 4096):
                x = torch.from_numpy(rng.normal(size=(B, T, F)).astype(np.float32)).cuda()
                y = torch.from_numpy(rng.normal(size=(B, T, O)).astype(np.float32)).cuda()
                loop_eng = None if a.no_loop else engine(B, H, L, prec)
                for M in (1, 8, 32):
                    rows = min(M * B, a.rows)
                    e = engine(rows, H, L, prec)
                    reps = 3 if M * B * H * L <= 8192 * 256 else 1
                    ig = timed(lambda: e.integrated_gradients(x, M), reps)
                    rec = dict(mode='ig', shape=shape, prec=prec, B=B, M=M, rows=rows, ig_ms=round(ig, 3),
                               workspace_gb=round(workspace_gb(e), 3))
                    e.close()
                    if loop_eng is not None:
                        def loop():
                            for _ in range(M):
                                loop_eng.forward(x)
                                loop_eng.backward(x, y)
                        lp = timed(loop, reps)
                        rec.update(loop_ms=round(lp, 3), loop_over_ig=round(lp / ig, 3))
                    emit(rec)
                    torch.cuda.empty_cache()
                if loop_eng is not None:
                    loop_eng.close()


if __name__ == '__main__':
    main()
