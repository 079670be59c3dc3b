"""What ptxas reports for the library's sm_90a kernels (no GPU needed; skipped without nvcc).

The persistent LSTM recurrences are latency-bound: a wgmma pipeline that ptxas serialises, or spill traffic inside the
step loop, costs time on every one of the T steps without changing any result, so no numerical test notices.  This
compiles every library source with exactly the commands the Makefile runs (`make -n -B`, objects redirected to a
temporary directory) and reads `-Xptxas -v`:
  - no kernel may have its wgmma serialised (C7510-C7520 "Potential Performance Loss ... serialized");
  - lstm_fwd_tc_kernel<SAVE, ROWS> and lstm_bwd_tc_kernel<FUSED, ROWS>, all four instantiations each (128-row tiles
    and 64-row half tiles), must not spill: 0 bytes of spill stores and loads, and no local-memory load or store
    (LDL / STL) anywhere in their SASS.
"""
import os
import re
import shlex
import shutil
import subprocess
import tempfile
from concurrent.futures import ThreadPoolExecutor

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RECURRENCES = ('lstm_fwd_tc_kernel', 'lstm_bwd_tc_kernel')
ROWS = (128, 64)                   # tiles, half tiles


def _nvcc():
    found = shutil.which('nvcc')
    if found:
        return found
    cand = '/usr/local/cuda/bin/nvcc'
    return cand if os.path.exists(cand) else None


def _compile_commands(nvcc):
    """The Makefile's object compile commands, as argument lists (compiler replaced by the nvcc found)."""
    r = subprocess.run(['make', '-n', '-B', '-C', ROOT, 'NVCC=' + nvcc, 'all'], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    cmds = [shlex.split(line) for line in r.stdout.splitlines() if line.startswith(nvcc + ' ') and ' -c ' in line]
    assert cmds, r.stdout
    return cmds


@pytest.fixture(scope='module')
def build():
    """(ptxas log of all sources, {source: object path}) for one cross-compile of the library."""
    nvcc = _nvcc()
    if nvcc is None or shutil.which('make') is None:
        pytest.skip('nvcc or make not found')
    cmds = _compile_commands(nvcc)
    with tempfile.TemporaryDirectory() as tmp:
        objs = {}

        def compile_one(cmd):
            cmd = list(cmd)
            src = cmd[cmd.index('-c') + 1]
            obj = os.path.join(tmp, os.path.basename(src) + '.o')
            cmd[cmd.index('-o') + 1] = obj
            objs[os.path.basename(src)] = obj
            r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True)
            assert r.returncode == 0, r.stdout + r.stderr
            return r.stdout + r.stderr

        with ThreadPoolExecutor(len(cmds)) as ex:
            log = '\n'.join(ex.map(compile_one, cmds))
        sass = None
        cuobjdump = shutil.which('cuobjdump') or os.path.join(os.path.dirname(nvcc), 'cuobjdump')
        if os.path.exists(cuobjdump) and 'lstm_tc.cu' in objs:
            r = subprocess.run([cuobjdump, '-sass', objs['lstm_tc.cu']], capture_output=True, text=True)
            assert r.returncode == 0, r.stderr
            sass = r.stdout
        yield log, sass


def _spills(log):
    """{mangled kernel name: (spill store bytes, spill load bytes)} for every entry function in the log."""
    out = {}
    cur = None
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            cur = m.group(1)
            continue
        m = re.search(r'(\d+) bytes spill stores, (\d+) bytes spill loads', line)
        if m and cur:
            out[cur] = (int(m.group(1)), int(m.group(2)))
            cur = None
    return out


def _instantiations(names, name, rows):
    """The mangled names of the <false, rows> and <true, rows> instantiations of a recurrence, after checking that all
    four <flag, ROWS> instantiations (flag false / true, ROWS 128 / 64) are there."""
    found = [k for k in names if re.match(r'_ZN4lfmq%d%sILb[01]ELi(128|64)EEEv' % (len(name), name), k)]
    assert len(found) == 4, (name, sorted(names))
    return [k for k in found if 'ELi%dEE' % rows in k]


def test_no_serialised_wgmma(build):
    log, _ = build
    bad = [line for line in log.splitlines() if re.search(r'\(C75\d\d\).*serialized', line)]
    assert not bad, '\n'.join(bad)


@pytest.mark.parametrize('rows', ROWS)
@pytest.mark.parametrize('kernel', RECURRENCES)
def test_recurrence_does_not_spill(build, kernel, rows):
    log, _ = build
    spills = _spills(log)
    for k in _instantiations(spills, kernel, rows):
        assert spills[k] == (0, 0), '%s: %d B spill stores, %d B spill loads' % ((k,) + spills[k])


@pytest.mark.parametrize('rows', ROWS)
@pytest.mark.parametrize('kernel', RECURRENCES)
def test_recurrence_sass_has_no_local_memory_access(build, kernel, rows):
    _, sass = build
    if sass is None:
        pytest.skip('cuobjdump not found')
    funcs = {}
    cur = None
    for line in sass.splitlines():
        m = re.search(r'Function : (\w+)', line)
        if m:
            cur = m.group(1)
            funcs[cur] = []
        elif cur:
            funcs[cur].append(line)
    for k in _instantiations(funcs, kernel, rows):
        local = [l.strip() for l in funcs[k] if re.search(r'\b(LDL|STL)\b', l)]
        assert not local, '%s: %d local-memory instructions, e.g. %s' % (k, len(local), local[:3])
