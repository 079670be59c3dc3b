"""CPU-side checks of the drop-in boundary: the C-ABI library loads and exports exactly what
include/lfmq.h declares; argument validation works without a GPU."""
import ctypes as C
import os
import re

import pytest

from lfm_quant_b200 import _native as N

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_symbols():
    src = open(os.path.join(ROOT, 'include', 'lfmq.h')).read()
    src = re.sub(r'/\*.*?\*/', '', src, flags=re.S)
    return set(re.findall(r'\b(lfmq_[a-z_]+)\s*\(', src))


def test_library_exports_every_declared_symbol():
    lib = N.load()
    declared = _header_symbols()
    assert declared == set(N.SYMBOLS), declared ^ set(N.SYMBOLS)
    for name in declared:
        assert hasattr(lib, name), name
    assert lib.lfmq_abi_version() == N.ABI_VERSION == 4


def test_gradient_tail_slots_match_header():
    """The engine reads the loss and its parts from the gradient vector's tail by position: _native's TAIL_* must be
    the header's LFMQ_TAIL_*."""
    src = open(os.path.join(ROOT, 'include', 'lfmq.h')).read()
    header = {k: int(v) for k, v in re.findall(r'\bLFMQ_TAIL_(\w+)\s*=\s*(\d+)', src)}
    mirror = {k[len('TAIL_'):]: v for k, v in vars(N).items() if k.startswith('TAIL_')}
    assert header == mirror and header['LEN'] == 8, (header, mirror)


def test_struct_sizes_match_header_layout():
    # 12 int32 + 8 float + uint64, naturally aligned
    assert C.sizeof(N.LfmqConfig) == 14 * 4 + 8 * 4 + 8
    assert C.sizeof(N.LfmqGatherArgs) == 11 * 4 + 4 + 12 * 8


def _cfg(**kw):
    c = N.LfmqConfig()
    c.struct_size = C.sizeof(N.LfmqConfig)
    c.max_batch, c.seq_len, c.n_inputs, c.n_outputs, c.num_hidden, c.num_layers = 32, 20, 32, 16, 64, 1
    c.target_idx = 3
    c.bn_epsilon = 1e-3
    for k, v in kw.items():
        setattr(c, k, v)
    return c


def test_workspace_bytes_and_validation_without_gpu():
    lib = N.load()
    n = C.c_uint64(0)
    assert lib.lfmq_workspace_bytes(C.byref(_cfg()), C.byref(n)) == 0
    small = n.value
    assert small > 32 * 20 * 64 * 4
    assert lib.lfmq_workspace_bytes(C.byref(_cfg(max_batch=64)), C.byref(n)) == 0
    assert n.value > small
    fo = C.c_uint64(0)
    assert lib.lfmq_workspace_bytes(C.byref(_cfg(forward_only=1)), C.byref(fo)) == 0
    assert fo.value < small
    for bad in (dict(struct_size=4), dict(num_hidden=0), dict(num_hidden=66), dict(target_idx=16),
                dict(optimizer=9), dict(dropout=1.0), dict(precision=7)):
        rc = lib.lfmq_workspace_bytes(C.byref(_cfg(**bad)), C.byref(n))
        assert rc != 0, bad
        assert len(lib.lfmq_last_error()) > 0
    with pytest.raises(N.LfmqError):
        N.check(lib.lfmq_workspace_bytes(C.byref(_cfg(num_layers=0)), C.byref(n)))


def test_tensor_core_workspace_leaves_out_fp32_activations():
    """A bf16 handle carves only its own path's buffers, not the fp32 path's per-layer h, c, y (at B=65536, T=48, H=256
    those alone are 3*B*T*H*4 bytes = 9.7 GB)."""
    lib = N.load()

    def ws(precision, max_batch=4096, forward_only=0):
        n = C.c_uint64(0)
        cfg = _cfg(max_batch=max_batch, seq_len=48, num_hidden=256, precision=precision, forward_only=forward_only)
        N.check(lib.lfmq_workspace_bytes(C.byref(cfg), C.byref(n)))
        return n.value

    assert ws(N.PREC_BF16) < ws(N.PREC_FP32)
    assert ws(N.PREC_BF16, 65536, 1) < ws(N.PREC_FP32, 65536, 1)


def test_cluster_path_carves_dropout_head_buffers_only_with_dropout():
    """A bf16 training handle without dropout runs the tensor-core head, fused with the backward recurrence: it carves
    neither the dropout head's dLoss/dh (bf16 [tiles*128][T][H]) nor its fp32 dLoss/dpred ([B*T][16])."""
    lib = N.load()
    B, T, F, O, H = 4096, 48, 32, 16, 256

    def ws(dropout):
        n = C.c_uint64(0)
        cfg = _cfg(max_batch=B, seq_len=T, n_inputs=F, n_outputs=O, num_hidden=H, target_idx=O - 1,
                   precision=N.PREC_BF16, train=1, dropout=dropout)
        N.check(lib.lfmq_workspace_bytes(C.byref(cfg), C.byref(n)))
        return n.value

    dhout = (B + 127) // 128 * 128 * T * H * 2
    dpred = B * T * 16 * 4
    assert ws(0.0) + dhout + dpred <= ws(0.2)


def test_engine_refuses_to_run_without_cuda():
    import torch
    if torch.cuda.is_available():
        pytest.skip('CUDA present')
    from lfm_quant_b200.engine import ForecasterEngine
    with pytest.raises(N.LfmqError):
        ForecasterEngine(max_batch=4, seq_len=4, n_inputs=4, n_outputs=2, num_hidden=8)
