"""CPU checks of tensor-core inference for the GRU cell and RNNUqRangeEstimate (no GPU needed): what forward-only GRU /
uq handles carve on the general path, and what ptxas reports for their kernels (skipped without nvcc)."""
import ctypes as C
import os
import re
import shutil
import subprocess
import tempfile

import pytest

from lfm_quant_b200 import _native as N

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _ws(**kw):
    c = N.LfmqConfig()
    c.struct_size = C.sizeof(N.LfmqConfig)
    c.max_batch, c.seq_len, c.n_inputs, c.n_outputs, c.num_hidden, c.num_layers = 4096, 48, 32, 16, 256, 1
    c.target_idx = 3
    c.bn_epsilon = 1e-3
    c.train, c.forward_only = 0, 1
    for k, v in kw.items():
        setattr(c, k, v)
    n = C.c_uint64(0)
    N.check(N.load().lfmq_workspace_bytes(C.byref(c), C.byref(n)))
    return n.value


def test_forward_only_gru_bf16_handle_is_smaller_than_fp32():
    gru = N.CELLS['gru']
    assert _ws(max_batch=65536, rnn_cell=gru, precision=N.PREC_BF16) < _ws(max_batch=65536, rnn_cell=gru,
                                                                          precision=N.PREC_FP32)


@pytest.mark.parametrize('cell', ['lstm', 'gru'])
def test_forward_only_uq_handle_carves_the_masked_h_only_with_recurrent_dropout(cell):
    """MC dropout: a uq handle keeps recurrent dropout on at prediction time, so it needs the masked copy of h (hmseq,
    bf16 [T+1][Bp][H] per layer) and at bf16x3 its low halves as well; without recurrent dropout it carves neither."""
    B, T, H, L = 4096, 48, 256, 2
    hm = (T + 1) * B * H * 2
    for precision, copies in ((N.PREC_BF16, 1), (N.PREC_BF16X3, 2)):
        kw = dict(max_batch=B, seq_len=T, num_hidden=H, num_layers=L, rnn_cell=N.CELLS[cell], uq=1, precision=precision,
                  dropout=0.2)
        assert _ws(recurrent_dropout=0.1, **kw) - _ws(recurrent_dropout=0.0, **kw) == L * copies * hm, precision
    # a point-estimate predict handle runs without dropout: the rate does not change what it carves
    kw = dict(max_batch=B, seq_len=T, num_hidden=H, rnn_cell=N.CELLS[cell], precision=N.PREC_BF16X3)
    assert _ws(recurrent_dropout=0.1, **kw) == _ws(recurrent_dropout=0.0, **kw)


# ---- ptxas ---------------------------------------------------------------------------------------------------------
EPI_FWD, EPI_FWD_ACC, EPI_GRU_FWD, EPI_GRU_FWD_ACC, EPI_HEAD_UQ = 0, 3, 5, 6, 7


@pytest.fixture(scope='module')
def rnn_tc_spills():
    """{(BN, EPI): (spill store bytes, spill load bytes)} of tile_gemm_kernel from one cross-compile of rnn_tc.cu with the
    Makefile's command."""
    nvcc = shutil.which('nvcc') or ('/usr/local/cuda/bin/nvcc' if os.path.exists('/usr/local/cuda/bin/nvcc') else None)
    if nvcc is None or shutil.which('make') is None:
        pytest.skip('nvcc or make not found')
    r = subprocess.run(['make', '-n', '-B', '-C', ROOT, 'NVCC=' + nvcc, 'all'], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    cmd = [line for line in r.stdout.splitlines() if line.startswith(nvcc + ' ') and 'rnn_tc.cu' in line]
    assert len(cmd) == 1, r.stdout
    import shlex
    cmd = shlex.split(cmd[0])
    with tempfile.TemporaryDirectory() as tmp:
        cmd[cmd.index('-o') + 1] = os.path.join(tmp, 'rnn_tc.o')
        r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
    out, cur = {}, None
    for line in (r.stdout + r.stderr).splitlines():
        m = re.search(r"Compiling entry function '_ZN4lfmq16tile_gemm_kernelILi(\d+)ELi(\d+)EE\w*'", line)
        if m:
            cur = (int(m.group(1)), int(m.group(2)))
            continue
        if "Compiling entry function" in line:
            cur = None
            continue
        m = re.search(r'(\d+) bytes spill stores, (\d+) bytes spill loads', line)
        if m and cur:
            out[cur] = (int(m.group(1)), int(m.group(2)))
            cur = None
    return out


@pytest.mark.parametrize('gru,lstm', [(EPI_GRU_FWD, EPI_FWD), (EPI_GRU_FWD_ACC, EPI_FWD_ACC)])
def test_gru_forward_step_spills_no_more_than_the_lstm_step(rnn_tc_spills, gru, lstm):
    g, l = rnn_tc_spills[(256, gru)], rnn_tc_spills[(256, lstm)]
    assert g[0] <= l[0] and g[1] <= l[1], (g, l)


def test_uq_head_gemm_does_not_spill(rnn_tc_spills):
    assert rnn_tc_spills[(32, EPI_HEAD_UQ)] == (0, 0)
