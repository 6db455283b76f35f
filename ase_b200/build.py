"""Builds ase_b200/csrc/libase_b200.so for sm_90a (H100) with nvcc (cross-compiles without a GPU).
Every .cu is compiled to its own object (in parallel, rebuilt only when it or a header changed), then linked."""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

CSRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'csrc')
LIB = os.path.join(CSRC, 'libase_b200.so')
OBJ = os.path.join(CSRC, 'build')
SOURCES = ['api.cu', 'obs_kernels.cu', 'rms_kernels.cu', 'rollout_kernels.cu', 'gemm_simt.cu', 'gemm_tc.cu',
           'loss_kernels.cu', 'learner.cu', 'motion_kernels.cu', 'reset_kernels.cu', 'player_kernels.cu', 'comm.cu', 'peer.cu']
HEADERS = ['common.cuh', 'kernels.h', 'tc_common.cuh', 'philox.cuh', 'motion_common.cuh', os.path.join('..', '..', 'include', 'ase_b200.h')]
NVCC_FLAGS = ['-O3', '-std=c++17', '-gencode', 'arch=compute_90a,code=sm_90a', '-lineinfo', '-Xcompiler', '-fPIC']


def _nccl_include():
    """nccl.h of the NCCL build PyTorch ships (comm.cu resolves the library itself at run time with dlopen)."""
    import importlib.util
    for cand in ([os.path.join(os.path.dirname(os.path.dirname(importlib.util.find_spec('torch').origin)), 'nvidia', 'nccl', 'include')]
                 if importlib.util.find_spec('torch') else []) + ['/usr/include']:
        if os.path.exists(os.path.join(cand, 'nccl.h')):
            return cand
    return None


def _nvcc():
    for c in (os.environ.get('NVCC'), '/usr/local/cuda/bin/nvcc', 'nvcc'):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    return 'nvcc'


def _sources():
    return [s for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]


def _headers():
    return [h for h in HEADERS if os.path.exists(os.path.join(CSRC, h))]


def _obj(src):
    return os.path.join(OBJ, src[:-3] + '.o')


def _stale(src):
    o = _obj(src)
    if not os.path.exists(o):
        return True
    t = os.path.getmtime(o)
    return any(os.path.getmtime(os.path.join(CSRC, f)) > t for f in [src] + _headers())


def up_to_date():
    if not os.path.exists(LIB):
        return False
    t = os.path.getmtime(LIB)
    return all(os.path.getmtime(os.path.join(CSRC, f)) <= t for f in _sources() + _headers())


def build(force=False, verbose=False):
    if not force and up_to_date():
        return LIB
    os.makedirs(OBJ, exist_ok=True)
    todo = [s for s in _sources() if force or _stale(s)]

    def compile_one(src):
        inc = ['-I', _nccl_include()] if (src == 'comm.cu' and _nccl_include()) else []
        cmd = [_nvcc()] + NVCC_FLAGS + inc + (['-Xptxas', '-v'] if verbose else []) + ['-c', '-o', _obj(src), src]
        return src, subprocess.run(cmd, cwd=CSRC, capture_output=True, text=True)

    with ThreadPoolExecutor(max_workers=max(1, min(len(todo), os.cpu_count() or 1))) as ex:
        results = list(ex.map(compile_one, todo))
    for src, r in results:
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError(f'nvcc failed compiling {src}')
        if verbose:
            print(f'==== {src}\n{r.stderr}')
    r = subprocess.run([_nvcc(), '-shared', '-o', LIB] + [_obj(s) for s in _sources()] + ['-ldl'], cwd=CSRC, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError('nvcc failed linking libase_b200.so')
    return LIB


if __name__ == '__main__':
    print(build(force='--force' in sys.argv, verbose='-v' in sys.argv))
