"""Generates tests/golden/reference_mlp_losses.npz by running the UNMODIFIED reference loss code
(/root/reference/scripts/model_utils/losses.py: Losses.weight_adjusted_mse, MLP branch :100-115) on fixed inputs.

The import shim is make_reference_losses.py's: each TensorFlow primitive the module uses maps to its NumPy equivalent
(float32 arithmetic, like the reference's tensors), so the masking, slicing, weighting and denominators that run are the
reference's own lines.  Here the shim's keras.losses.Huber also carries Keras' formula (0.5 r^2 for |r| <= delta, else
delta (|r| - delta / 2), averaged over all elements), so the Huber cases (keys ``huber_*``) are RESTATED, NOT PINNED:
they check the branch's wiring around a Huber written here, not Keras' Huber itself.
Cases: rows whose targets are all zero, target_lambda in {0, 0.5, 1}, O = 1 and O > 1, training and validation.
Only runs where /root/reference exists; the .npz is what travels.

usage: python tests/golden/make_reference_mlp_losses.py
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))

CHILD = r'''
import sys, types
import numpy as np

tf = types.ModuleType('tensorflow')
tf.float32 = np.float32
tf.constant = lambda v, dtype=None: np.asarray(v, dtype=dtype)
tf.equal = np.equal
tf.reduce_all = lambda a, axis=None: np.all(a, axis=axis)
tf.cast = lambda a, dtype=None: np.asarray(a).astype(dtype)
tf.multiply = np.multiply
tf.divide = np.divide
tf.expand_dims = np.expand_dims
tf.reduce_mean = lambda a, axis=None: np.mean(a, axis=axis, dtype=np.asarray(a).dtype)
tf.reduce_sum = lambda a, axis=None: np.sum(a, axis=axis, dtype=np.asarray(a).dtype)
tf.math = types.SimpleNamespace(log=np.log)
py = types.ModuleType('tensorflow.python'); fw = types.ModuleType('tensorflow.python.framework')
opsm = types.ModuleType('tensorflow.python.framework.ops'); opsm.convert_to_tensor = lambda a: np.asarray(a)
pops = types.ModuleType('tensorflow.python.ops'); mo = types.ModuleType('tensorflow.python.ops.math_ops')
mo.squared_difference = lambda a, b: np.square(np.subtract(a, b))
mo.cast = lambda a, dtype: np.asarray(a).astype(dtype)
keras = types.ModuleType('tensorflow.keras'); kl = types.ModuleType('tensorflow.keras.losses')


class Huber(object):
    """keras.losses.Huber(delta) with the default sum-over-batch-size reduction, restated."""

    def __init__(self, delta=1.0):
        self.delta = np.float32(delta)

    def __call__(self, y_true, y_pred):
        r = np.abs(np.subtract(y_pred, y_true, dtype=np.float32))
        e = np.where(r <= self.delta, np.float32(0.5) * r * r, self.delta * r - np.float32(0.5) * self.delta ** 2)
        return np.mean(e, dtype=np.float32)


kl.Huber = Huber
fw.ops = opsm; pops.math_ops = mo; py.framework = fw; py.ops = pops; keras.losses = kl; tf.python = py; tf.keras = keras
for name, mod in (('tensorflow', tf), ('tensorflow.python', py), ('tensorflow.python.framework', fw),
                  ('tensorflow.python.framework.ops', opsm), ('tensorflow.python.ops', pops),
                  ('tensorflow.python.ops.math_ops', mo), ('tensorflow.keras', keras), ('tensorflow.keras.losses', kl)):
    sys.modules[name] = mod

OUT = sys.argv[1]
sys.path.insert(0, '/root/reference/scripts')
sys.path.insert(0, '/root/reference/scripts/model_utils')
sys.argv = ['x']
import losses as ref
import base_config
c = base_config.get_configs()
c.nn_type = 'MLPLinearPointEstimate'
c.forecast_steps = 1
c.forecast_steps_weights = [1.0]
out = {}
rng = np.random.RandomState(11)
cases = []
for B, O, tidx in ((9, 1, 0), (12, 5, 3), (16, 16, 7)):
    y = rng.normal(size=(B, O)).astype(np.float32)
    y[1] = 0.0                                   # rows whose targets are all zero
    y[B - 2] = 0.0
    p = (y + rng.normal(scale=1.5, size=(B, O))).astype(np.float32)
    for lam in (0.0, 0.5, 1.0):
        cases.append((B, O, tidx, lam, y, p))
for k, (B, O, tidx, lam, y, p) in enumerate(cases):
    c.target_lambda = lam
    c.huber_loss = False
    l, m = ref.Losses(c, tidx).weight_adjusted_mse([y], [p])
    out['mse_%d_y' % k], out['mse_%d_p' % k] = y, p
    out['mse_%d' % k] = np.array([tidx, lam, float(l), float(m)])
    c.huber_loss, c.huber_delta = True, 0.8
    l, m = ref.Losses(c, tidx).weight_adjusted_mse([y], [p])
    lv, mv = ref.Losses(c, tidx).weight_adjusted_mse([y], [p], True)     # validation: the MSE form
    out['huber_%d' % k] = np.array([tidx, lam, 0.8, float(l), float(m), float(lv), float(mv)])
out['n_cases'] = np.int64(len(cases))
np.savez_compressed(OUT, **out)
print('ok', len(cases), 'cases')
'''


def main():
    dst = os.path.join(HERE, 'reference_mlp_losses.npz')
    r = subprocess.run([sys.executable, '-c', CHILD, dst], capture_output=True, text=True)
    print(r.returncode)
    print((r.stdout.strip().splitlines() or [''])[-1][:1500])
    if r.returncode != 0:
        print('\n'.join(r.stderr.strip().splitlines()[-12:]))


if __name__ == '__main__':
    main()
