"""Register budget of the persistent decode kernel (CPU only: needs nvcc, no GPU).

decode_group_kernel runs 512 threads per CTA, so ptxas may give it at most 128 registers a thread.  What does not fit
goes to local memory, and with the maximum shared-memory carve-out an SM keeps only ~28 KB of L1 for it: reloads that
miss there wait on L2 in the middle of a latency-bound step.  This compiles csrc/decode_group.cu alone with the flags of
build.py and reads ptxas's report for the production instantiation (kStamps = false; the clock64-stamped one serves
tools/decode_phases.py only).

The remaining frame is 13 words: per-thread shared-memory offsets and row indices formed once before the step loop and
reloaded by a few phases.  The bound below is what the kernel compiles to; it used to be a 248-byte frame with 440 bytes
of spill stores and 596 of spill loads.
"""
import os
import re
import shutil
import subprocess

import pytest

from opentransformer_b200 import build

MAX_STACK, MAX_SPILL_STORES, MAX_SPILL_LOADS = 56, 52, 96


def _nvcc():
    try:
        nvcc = build._nvcc()
    except RuntimeError:
        return None
    return nvcc if os.path.isabs(nvcc) and os.path.exists(nvcc) else shutil.which(nvcc)


def _ptxas_report(tmp_path):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip('nvcc is not available')
    cmd = [nvcc] + build.NVCC_FLAGS + ['-c', os.path.join(build.CSRC, 'decode_group.cu'), '-o', str(tmp_path / 'decode_group.o')]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, cwd=str(tmp_path))
    assert r.returncode == 0, r.stdout
    return r.stdout


def _properties(report, mangled):
    """(stack frame, spill stores, spill loads, registers) of one entry function in a ptxas -v report."""
    m = re.search(r"Function properties for " + re.escape(mangled) + r"\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                  r"(\d+) bytes spill loads\s*\n.*?Used (\d+) registers", report)
    assert m, f'no ptxas report for {mangled}:\n{report}'
    return tuple(int(x) for x in m.groups())


def test_production_decode_kernel_spills(tmp_path):
    report = _ptxas_report(tmp_path)
    stack, st, ld, regs = _properties(report, '_ZN3otb19decode_group_kernelILb0EEEvNS_8DgParamsE')
    assert regs <= 128, f'{regs} registers: 512 threads per CTA allow 128'
    assert stack <= MAX_STACK and st <= MAX_SPILL_STORES and ld <= MAX_SPILL_LOADS, (
        f'decode_group_kernel<false>: {stack} bytes stack frame, {st} bytes spill stores, {ld} bytes spill loads '
        f'(at most {MAX_STACK} / {MAX_SPILL_STORES} / {MAX_SPILL_LOADS})')
    # the stamped instantiation exists for otb_debug_decode_timing
    _properties(report, '_ZN3otb19decode_group_kernelILb1EEEvNS_8DgParamsE')
