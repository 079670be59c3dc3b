"""The rounding oracle of LFMQ_PREC_TF32: the fp64 oracles (lfm_oracle, uq_chain_oracle) with both operands of every
matrix product rounded to tf32 the way tf32_gemm.cu rounds them.

A tf32 handle runs the fp32 step with only its GEMMs changed: each GEMM loads its operand tiles, rounds every element
with cvt.rna.tf32.f32 (the float32 value to 10 mantissa bits, nearest, ties away from zero) and accumulates the exact
products in fp32.  Every matrix product in the oracles is one of those GEMMs (the recurrent and input products of each
step and their backward, the weight gradients, the heads), and nothing else in the oracles is, so the restatement is
the oracles themselves with `@` rounding its operands first:

    with rounding():                  # or rounding(False): the same machinery with nothing rounded
        preds, fc = call(orc.forward, P, x, num_layers=L, ...)

Inside `rounding()` the oracle modules see a numpy whose array constructors return `Tf32Array`, an ndarray whose
`@` rounds both sides; `call` views its array arguments (and lists of them) the same way and returns plain arrays.
The accumulation stays in fp64: what remains between the kernels and this oracle is fp32 accumulation and the fp32
pointwise arithmetic, the differences an fp32 handle has against lfm_oracle.
"""
from __future__ import annotations

import contextlib

import numpy as np

import lfm_oracle as orc
import uq_chain_oracle as uco


def round_tf32(a):
    """float32(a) rounded to tf32 (cvt.rna.tf32.f32), as float64.  Sign-magnitude bits: adding half an ulp of tf32 to
    the magnitude and truncating rounds ties away from zero; a carry into the exponent is the correct result."""
    b = np.asarray(a, dtype=np.float32).view(np.uint32).astype(np.uint64)
    b = ((b + 0x1000) & 0xFFFFE000).astype(np.uint32)
    return b.view(np.float32).astype(np.float64)


_ENABLED = [True]


def _r(a):
    return round_tf32(a) if _ENABLED[0] else np.asarray(a, dtype=np.float64)


class Tf32Array(np.ndarray):
    """An ndarray whose matrix product rounds both operands to tf32 (when rounding is on) and then multiplies in fp64.
    The priority makes it win over plain arrays in concatenations, and Python tries a subclass's reflected operator
    first, so `plain @ Tf32Array` rounds as well."""
    __array_priority__ = 10.0

    def __matmul__(self, other):
        return np.matmul(_r(self), _r(other)).view(Tf32Array)

    def __rmatmul__(self, other):
        return np.matmul(_r(other), _r(self)).view(Tf32Array)


def _wrap_ctor(fn):
    def ctor(*a, **k):
        out = fn(*a, **k)
        return out.view(Tf32Array) if isinstance(out, np.ndarray) else out
    return ctor


class _Numpy(object):
    """numpy as the oracle modules see it inside `rounding()`: every array they build is a Tf32Array."""
    _CTORS = ('empty', 'zeros', 'ones', 'full', 'zeros_like', 'ones_like', 'empty_like', 'full_like', 'concatenate',
              'stack', 'where', 'asarray', 'array')

    def __getattr__(self, name):
        fn = getattr(np, name)
        return _wrap_ctor(fn) if name in self._CTORS else fn


@contextlib.contextmanager
def rounding(enabled=True):
    """Run lfm_oracle / uq_chain_oracle with every matrix product's operands rounded to tf32 (enabled=False: the same
    arrays, nothing rounded, which must give lfm_oracle's own results)."""
    saved = orc.np, uco.np, _ENABLED[0]
    orc.np = uco.np = _Numpy()
    _ENABLED[0] = enabled
    try:
        yield
    finally:
        orc.np, uco.np, _ENABLED[0] = saved


def _to(a):
    if isinstance(a, np.ndarray):
        return np.asarray(a).view(Tf32Array)
    if isinstance(a, list):
        return [_to(v) for v in a]
    if isinstance(a, tuple):
        return tuple(_to(v) for v in a)
    return a


def _back(a):
    if isinstance(a, np.ndarray):
        return np.asarray(a).view(np.ndarray)
    if isinstance(a, list):
        return [_back(v) for v in a]
    if isinstance(a, tuple):
        return tuple(_back(v) for v in a)
    return a


def call(fn, *args, **kw):
    """fn(*args, **kw) of an oracle function with its array arguments as Tf32Array; call inside `rounding()`.
    Caches (forward results fed to a backward) stay Tf32Array inside; the returned arrays are plain."""
    return _back(fn(*_to(list(args)), **{k: _to(v) for k, v in kw.items()}))
