"""Generates tests/golden/reference_hpo.json by running the UNMODIFIED reference hyper-parameter search
(/root/reference/scripts/hyper_param_opt.py and param_search/) with candidate training stubbed out.

What is replaced, and nothing else:
- ``import tensorflow`` (imported, never used by param_search) by an empty module;
- ``np.bool``, which the reference's isinstance checks name, by ``bool`` where it is missing (NumPy 1.24 to 1.26
  removed it; NumPy 2 has it again, as an alias of ``np.bool_``);
- ``multiprocessing.Pool`` by a serial map in this process;
- ``os.system("... lfm_quant.py --config=<model.conf>")`` by tests/hpo_stub.py, which writes the train log (or
  preds.dat) that the reference then reads, with losses that are a fixed function of the candidate's model.conf; the
  candidate with member_id hpo_stub.FAIL_ID writes nothing, so the reference scores it inf.

Each case runs in a subprocess of its own (the reference's flag parser is module-global) in an empty directory, with
DEEP_QUANT_ROOT=/lfmq-root.  Recorded per case: the argv, the input files, every generation's member configs as they
enter training, and every model.conf and opt_hist.csv the search wrote (paths relative to the directory).  Only runs
where /root/reference exists; the JSON it writes is what travels.

usage: python tests/golden/make_reference_hpo.py
"""
import json
import os
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
TESTS = os.path.dirname(HERE)
REF = '/root/reference/scripts'
DATA_ROOT = '/lfmq-root'

CASES = {
    # 3 generations x 6 members over 3 tunable flags, members round robin over 2 GPUs
    'genetic': dict(argv=['--name', 'ga', '--search_algorithm', 'genetic', '--generations', '3', '--pop_size', '6',
                          '--NPE', '3', '--num_gpu', '2', '--mutate_rate', '0.5', '--rnn_cell', 'lstm', 'gru',
                          '--num_hidden', '32', '64', '128', '--learning_rate', '0.1', '0.3', '0.6'],
                    files={}),
    # the initial population read from a DOE file: NPE = pop_size = its 4 rows (read as strings)
    'genetic_doe': dict(argv=['--name', 'gadoe', '--search_algorithm', 'genetic', '--generations', '2',
                              '--doe_file', 'ga_doe.csv', '--num_hidden', '32', '64',
                              '--learning_rate', '0.1', '0.3', '0.6'],
                        files={'ga_doe.csv': 'num_hidden,learning_rate\n32,0.1\n64,0.3\n32,0.6\n64,0.6\n'}),
    # 2 x 3 x 2 = 12 combinations, NPE 5: two generations, the last 2 combinations dropped
    'grid_search': dict(argv=['--name', 'grid', '--search_algorithm', 'grid_search', '--NPE', '5',
                              '--num_hidden', '32', '64', '--learning_rate', '0.1', '0.3', '0.6',
                              '--num_layers', '1', '2'],
                        files={}),
    # 5 rows with their own member_id, model_dir and train, NPE 2: three generations; row 4 is scored from preds.dat
    'doe': dict(argv=['--name', 'doe', '--search_algorithm', 'doe', '--NPE', '2', '--doe_file', 'doe.csv'],
                files={'doe.csv': 'member_id,model_dir,num_hidden,learning_rate,train\n'
                                  '1,doe/run-1,32,0.1,True\n2,doe/run-2,64,0.3,True\n3,doe/run-3,32,0.6,True\n'
                                  '4,doe/run-4,64,0.1,False\n5,doe/run-5,128,0.3,True\n'}),
}

CHILD = r'''
import json, multiprocessing, os, sys, types
sys.path[:0] = [%(ref)r, %(tests)r]
import numpy as np
if not hasattr(np, 'bool'):
    np.bool = bool
sys.modules['tensorflow'] = types.ModuleType('tensorflow')


class SerialPool(object):
    def __init__(self, processes=None):
        pass

    def map(self, fn, items):
        return [fn(x) for x in items]


multiprocessing.Pool = SerialPool
import hpo_stub


def system(cmd):
    hpo_stub.train_candidate(cmd.split('--config=')[1].strip())
    return 0


os.system = system
case = json.loads(%(case)r)
for name, text in case['files'].items():
    open(name, 'w').write(text)
sys.argv = ['hyper_param_opt.py'] + case['argv']
os.environ['DEEP_QUANT_ROOT'] = %(root)r
import hyper_param_opt
from param_search import doe, genetic_algorithm, grid_search
generations = []


def record(cls):
    train = cls._train_population

    def recorded(self, gen):
        generations.append([[[k, v] for k, v in json.loads(json.dumps(list(m.__dict__['__configs'].items()),
                                                                        default=str))]
                            for m in self._cur_pop])
        return train(self, gen)
    cls._train_population = recorded


for cls in (genetic_algorithm.GeneticAlgorithm, grid_search.GridSearch, doe.DOE):
    record(cls)
hyper_param_opt.HPOptimization(hyper_param_opt.get_configs())()
files = {}
for d, _, names in os.walk('.'):
    for n in names:
        if n in ('model.conf', 'opt_hist.csv'):
            p = os.path.relpath(os.path.join(d, n))
            files[p] = open(p).read()
print('@@' + json.dumps(dict(generations=generations, outputs=files)))
'''


def main():
    out = {}
    for name, case in CASES.items():
        with tempfile.TemporaryDirectory() as work:
            src = CHILD % dict(ref=REF, tests=TESTS, case=json.dumps(case), root=DATA_ROOT)
            r = subprocess.run([sys.executable, '-c', src], cwd=work, capture_output=True, text=True)
            if r.returncode != 0:
                raise SystemExit('%s: %s' % (name, r.stderr))
            rec = json.loads([l for l in r.stdout.splitlines() if l.startswith('@@')][-1][2:])
        out[name] = dict(argv=case['argv'], files=case['files'], **rec)
        print(name, '%d generations, %d files' % (len(rec['generations']), len(rec['outputs'])))
    out['data_root'] = DATA_ROOT
    json.dump(out, open(os.path.join(HERE, 'reference_hpo.json'), 'w'), indent=1, sort_keys=True)


if __name__ == '__main__':
    main()
