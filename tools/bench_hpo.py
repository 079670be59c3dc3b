"""Wall time of one hyper-parameter search generation: 8 candidates (a grid over 8 learning rates) trained for one
epoch on a synthetic dataset through runtime.model_execution.run_candidates, one after another (NPE 1) against side by
side (NPE 8).  Dataset building, training, validation and the files each candidate writes are all inside the timed
region: it is what one generation of hyper_param_opt.py costs.

Shapes: the reference's default (B=256, T=5, H=64, L=2; stride 12) and BASELINE configs[1] (B=4096, T=48, H=256, L=1;
stride 1), each at fp32 and bf16.

    python tools/bench_hpo.py [--cases ref_fp32,ref_bf16,cfg1_fp32,cfg1_bf16] [--repeat 1] [--out FILE]

Prints one JSON line per case with the GPU's name and power limit.  Everything it writes goes to a temporary directory.
"""
import argparse
import json
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench_ensemble import gpu_info  # noqa: E402  (tools/ is this script's directory)

LRS = ['0.1', '0.2', '0.3', '0.4', '0.5', '0.6', '0.7', '0.8']
SHAPES = {
    'ref': dict(keys=100, argv=['--batch_size', '256', '--min_unrollings', '5', '--max_unrollings', '5', '--stride',
                                '12', '--num_hidden', '64', '--num_layers', '2']),
    'cfg1': dict(keys=150, argv=['--batch_size', '4096', '--min_unrollings', '48', '--max_unrollings', '48',
                                 '--stride', '1', '--num_hidden', '256', '--num_layers', '1']),
}


def generation(work, shape, precision):
    """model.conf paths of the 8 candidates and the search object that wrote them."""
    from lfm_quant_b200.scripts import hyper_param_opt
    from lfm_quant_b200.scripts.param_search.grid_search import GridSearch
    argv = ['--name', '%s_%s' % (shape, precision), '--search_algorithm', 'grid_search', '--NPE', '8',
            '--experiments_dir', os.path.join(work, 'experiments'), '--datafile', 'ds-%s.dat' % shape,
            '--recurrent_dropout', '0.0', '--max_epoch', '1', '--end_date', '200412', '--logging_interval', '100000',
            '--precision', precision, '--learning_rate'] + LRS + SHAPES[shape]['argv']
    search = GridSearch(hyper_param_opt.get_configs(argv))
    pop = search._get_gen(0)
    for m in pop:
        search._prepare(m)
    return search, pop, [search._write_conf(m) for m in pop]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--cases', default='ref_fp32,ref_bf16,cfg1_fp32,cfg1_bf16')
    ap.add_argument('--repeat', type=int, default=1)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('bench_hpo needs a CUDA GPU')
    from lfm_quant_b200.scripts.runtime.model_execution import run_candidates
    from lfm_quant_b200.scripts.synthetic import write_open_dataset
    gpu = gpu_info()
    lines = []
    with tempfile.TemporaryDirectory() as work:
        os.environ['LFM_QUANT_ROOT'] = work
        os.environ['LFMQ_SEEDED_SHUFFLE'] = '1'
        os.makedirs(os.path.join(work, 'experiments'))
        for shape, s in SHAPES.items():
            write_open_dataset(os.path.join(work, 'datasets', 'ds-%s.dat' % shape), n_keys=s['keys'], n_months=420,
                               seed=5)
        for case in a.cases.split(','):
            shape, precision = case.split('_')
            search, pop, paths = generation(work, shape, precision)
            run_candidates(paths[:1], 1)                # warm-up: module loads, first launches
            times = {1: [], 8: []}
            objectives = {}
            for _ in range(a.repeat):
                for npe in (1, 8):                      # alternated, so that drift on the host hits both
                    t0 = time.perf_counter()
                    errors = run_candidates(paths, npe)
                    torch.cuda.synchronize()
                    times[npe].append(time.perf_counter() - t0)
                    assert not any(errors), errors
                    objectives[npe] = [float(search._read_results(m)[1]) for m in pop]
            res = {'case': case, 'candidates': len(paths), 'shape': SHAPES[shape]['argv'], 'precision': precision,
                   'npe1_s_per_generation': min(times[1]), 'npe8_s_per_generation': min(times[8]),
                   'all_s': {str(k): v for k, v in times.items()}, 'speedup': min(times[1]) / min(times[8]),
                   'same_objectives': objectives[1] == objectives[8], 'gpu': gpu}
            print(json.dumps(res), flush=True)
            lines.append(res)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            for r in lines:
                f.write(json.dumps(r) + '\n')


if __name__ == '__main__':
    main()
