"""How the bf16 LSTM recurrences move their saved state, read from the sm_90a SASS (no GPU needed; skipped without nvcc).

Training runs lstm_fwd_tc_kernel<SAVE=true, ROWS>, whose saved gates and cell states feed the backward recurrence.  The
forward keeps the post-activation gates of its cell update for the saved state rather than evaluating them a second
time, and stores gates and cell states in accumulator-fragment order as 16- and 8-byte vectors; the FUSED backward reads
them back the same way.  Neither shows in any result, only in the length of each step's dependency chain, so this reads
the instructions: for both tile heights,
  - <true, ROWS> has exactly the MUFU.TANH count of the forward-only <false, ROWS>;
  - its 32-bit STG count equals <false, ROWS>'s (the h_t stores), so every saved-state store is a vector;
  - lstm_bwd_tc_kernel<true, ROWS> issues only 64- and 128-bit LDGs.
lstm_tc.cu is compiled with exactly the command the Makefile runs for it (see test_ptxas_report.py).
"""
import os
import re
import shutil
import subprocess
import tempfile

import pytest

from test_ptxas_report import ROOT, ROWS, _compile_commands, _instantiations, _nvcc


@pytest.fixture(scope='module')
def sass():
    """{mangled kernel name: [SASS instruction lines]} of lstm_tc.cu."""
    nvcc = _nvcc()
    if nvcc is None or shutil.which('make') is None:
        pytest.skip('nvcc or make not found')
    cuobjdump = shutil.which('cuobjdump') or os.path.join(os.path.dirname(nvcc), 'cuobjdump')
    if not os.path.exists(cuobjdump):
        pytest.skip('cuobjdump not found')
    cmd = [c for c in _compile_commands(nvcc) if os.path.basename(c[c.index('-c') + 1]) == 'lstm_tc.cu']
    assert len(cmd) == 1
    cmd = list(cmd[0])
    with tempfile.TemporaryDirectory() as tmp:
        cmd[cmd.index('-o') + 1] = os.path.join(tmp, 'lstm_tc.o')
        r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
        r = subprocess.run([cuobjdump, '-sass', os.path.join(tmp, 'lstm_tc.o')], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
    funcs, cur = {}, None
    for line in r.stdout.splitlines():
        m = re.search(r'Function : (\w+)', line)
        if m:
            cur = m.group(1)
            funcs[cur] = []
        elif cur and re.search(r'/\*[0-9a-f]{4,}\*/', line):
            funcs[cur].append(line)
    return funcs


def _pair(funcs, kernel, rows):
    """(<false, rows>, <true, rows>) instruction lists of a recurrence."""
    names = _instantiations(funcs, kernel, rows)
    return tuple(funcs[next(k for k in names if 'ILb%dE' % flag in k)] for flag in (0, 1))


def _widths(lines, op):
    """Access width in bits of every `op` (STG / LDG) instruction."""
    out = []
    for line in lines:
        m = re.search(r'\b%s(\.\S+)?\s' % op, line)
        if m:
            mods = (m.group(1) or '').split('.')
            out.append(128 if '128' in mods else 64 if '64' in mods else 32)
    return out


@pytest.mark.parametrize('rows', ROWS)
def test_forward_saves_gates_without_evaluating_them_again(sass, rows):
    predict, train = _pair(sass, 'lstm_fwd_tc_kernel', rows)
    n_pred, n_train = (sum('MUFU.TANH' in l for l in f) for f in (predict, train))
    assert n_pred > 0
    assert n_train == n_pred, 'SAVE=true: %d MUFU.TANH, forward-only: %d' % (n_train, n_pred)


@pytest.mark.parametrize('rows', ROWS)
def test_forward_saved_state_stores_are_vectors(sass, rows):
    predict, train = _pair(sass, 'lstm_fwd_tc_kernel', rows)
    wp, wt = _widths(predict, 'STG'), _widths(train, 'STG')
    assert wp and all(w == 32 for w in wp)                 # h_t, one bf16 pair per store
    assert wt.count(32) == len(wp), 'SAVE=true: %d 32-bit STG, forward-only: %d' % (wt.count(32), len(wp))
    assert wt.count(128) > 0 and wt.count(64) > 0          # gate vectors, cell-state vectors


@pytest.mark.parametrize('rows', ROWS)
def test_fused_backward_loads_saved_state_as_vectors(sass, rows):
    _, fused = _pair(sass, 'lstm_bwd_tc_kernel', rows)
    widths = _widths(fused, 'LDG')
    assert widths.count(128) > 0 and widths.count(64) > 0
    assert widths.count(32) == 0, '%d 32-bit LDG in lstm_bwd_tc_kernel<true, %d>' % (widths.count(32), rows)
