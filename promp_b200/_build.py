"""Build promp_b200/libpromp_b200.so (sm_90a) in-tree with nvcc.  No torch dependency: the library
is plain CUDA runtime + the C ABI of include/promp_b200.h; nvcc cross-compiles without a GPU."""
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

PKG = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG)
CSRC = os.path.join(PKG, 'csrc')
OBJ = os.path.join(ROOT, 'build', 'obj')
LIB = os.path.join(PKG, 'libpromp_b200.so')
SOURCES = ('common.cu', 'rollout.cu', 'process.cu', 'policy.cu', 'policy_relu.cu', 'policy_otanh.cu', 'policy_relu_otanh.cu', 'comm.cu',
           'trpo.cu', 'paths.cu', 'env_module.cu')
NVCC_FLAGS = ['-std=c++17', '-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-lineinfo',
              '-Xcompiler', '-fPIC', '-Xptxas', '-v']


def _nvcc():
    for cand in (shutil.which('nvcc'), '/usr/local/cuda/bin/nvcc'):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: cannot build libpromp_b200.so")


def _deps():
    files = [os.path.join(CSRC, f) for f in os.listdir(CSRC)]
    files.append(os.path.join(ROOT, 'include', 'promp_b200.h'))
    return files


def is_stale():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(f) > t for f in _deps())


def build(force=False, verbose=False):
    """Compile every .cu for sm_90a and link the shared library.  Returns the library path."""
    if not force and not is_stale():
        return LIB
    nvcc = _nvcc()
    os.makedirs(OBJ, exist_ok=True)

    def compile_one(src):
        obj = os.path.join(OBJ, src.replace('.cu', '.o'))
        cmd = [nvcc] + NVCC_FLAGS + ['-c', os.path.join(CSRC, src), '-o', obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (src, r.stdout, r.stderr))
        with open(obj + '.ptxas.log', 'w') as f:      # register / spill report (-Xptxas -v)
            f.write(r.stderr)
        if verbose:
            sys.stderr.write(r.stderr)
        return obj

    with ThreadPoolExecutor(max_workers=len(SOURCES)) as ex:
        objs = list(ex.map(compile_one, SOURCES))
    cmd = [nvcc, '-shared', '-o', LIB] + objs      # static cudart (nvcc default): self-contained .so
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("link failed:\n%s\n%s" % (r.stdout, r.stderr))
    return LIB


if __name__ == '__main__':
    print(build(force='--force' in sys.argv, verbose='-v' in sys.argv))
