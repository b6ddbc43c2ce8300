"""Build libotb200.so (the C-ABI CUDA library) in-tree with nvcc for sm_90a (H100).

    python -m opentransformer_b200.build [--force]

The .so lands next to this file (git-ignored; build() recreates it from a clean checkout).
cudart is linked statically and libcuda is resolved at run time through
cudaGetDriverEntryPoint, so the library also *loads* on a machine without a GPU driver.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
LIB = os.path.join(HERE, 'libotb200.so')
SOURCES = ['gemm_tc.cu', 'attn_tc.cu', 'attn_bwd.cu', 'backward.cu', 'ops_simt.cu', 'beam.cu', 'decode_group.cu', 'loss.cu', 'ctc.cu', 'fbank.cu', 'capi.cu']
HEADERS = ['otb_internal.h', 'ptx.cuh', 'beam_common.cuh', 'launch.cuh', os.path.join('..', '..', 'include', 'otb200.h')]
NVCC_FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-std=c++17', '-lineinfo',
              '-Xcompiler', '-fPIC', '-Xptxas', '-v', '--expt-relaxed-constexpr']


def _nvcc():
    for c in (os.environ.get('NVCC'), '/usr/local/cuda/bin/nvcc', 'nvcc'):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    raise RuntimeError('nvcc not found')


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, s) for s in SOURCES + HEADERS] + [os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    if not force and not needs_build():
        return LIB
    objs = []
    os.makedirs(os.path.join(HERE, 'build'), exist_ok=True)
    procs = []
    for s in SOURCES:
        o = os.path.join(HERE, 'build', s.replace('.cu', '.o'))
        cmd = [_nvcc()] + NVCC_FLAGS + ['-c', os.path.join(CSRC, s), '-o', o]
        procs.append((s, o, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    log = []
    for s, o, p in procs:
        out, _ = p.communicate()
        log.append(f'==== {s}\n{out}')
        if p.returncode != 0:
            raise RuntimeError(f'nvcc failed on {s}:\n{out}')
        objs.append(o)
    cmd = [_nvcc(), '-shared', '-o', LIB] + objs + ['-gencode', 'arch=compute_90a,code=sm_90a', '-cudart', 'static']
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError('link failed:\n' + r.stdout)
    with open(os.path.join(HERE, 'build', 'ptxas.log'), 'w') as f:
        f.write('\n'.join(log))
    if verbose:
        print('\n'.join(log))
    return LIB


if __name__ == '__main__':
    print(build(force='--force' in sys.argv, verbose='-v' in sys.argv))
