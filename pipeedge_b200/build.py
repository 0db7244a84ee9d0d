"""Build `libpipeedge_b200.so` (the C-ABI library) in-tree with nvcc for sm_90a (H100).

`python -m pipeedge_b200.build` or `__graft_entry__.build()`. The `.so` and the objects are git-ignored build
products; nothing is JIT-compiled at import time.
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG_DIR, 'csrc')
OBJ_DIR = os.path.join(CSRC, 'build')
LIB_PATH = os.path.join(PKG_DIR, 'libpipeedge_b200.so')
SOURCES = ['api.cu', 'gemm_wgmma.cu', 'layernorm.cu', 'attention.cu', 'attention_wgmma.cu', 'quant.cu', 'stage.cu', 'edges.cu', 'hop.cu', 'link.cu', 'hostring.cu', 'pipe.cu']
NVCC = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
# -fmad=false is NOT set globally: the quantisation kernels use explicit _rn intrinsics where bit-exactness
# matters, everything else may contract.
FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-std=c++17', '-lineinfo',
         '-Xcompiler', '-fPIC', '-Xcompiler', '-Wall', '--expt-relaxed-constexpr']


def _newer(src: str, dst: str) -> bool:
    if not os.path.exists(dst):
        return True
    deps = [src, os.path.join(PKG_DIR, '..', 'include', 'pipeedge_b200.h')] + \
        [os.path.join(CSRC, h) for h in os.listdir(CSRC) if h.endswith('.cuh')]
    return any(os.path.getmtime(d) > os.path.getmtime(dst) for d in deps)


def _compile(name: str, verbose: bool) -> str:
    src = os.path.join(CSRC, name)
    obj = os.path.join(OBJ_DIR, name.replace('.cu', '.o'))
    if _newer(src, obj):
        cmd = [NVCC, *FLAGS, '-c', src, '-o', obj] + (['-Xptxas', '-v'] if verbose else [])
        res = subprocess.run(cmd, capture_output=True, text=True, check=False)
        if res.returncode != 0:
            raise RuntimeError(f"nvcc failed for {name}:\n{res.stdout}\n{res.stderr}")
        if verbose:
            print(res.stderr)
    return obj


def build(verbose: bool = False, force: bool = False) -> str:
    """Compile every CUDA source for sm_90a and link the shared library; returns its path."""
    os.makedirs(OBJ_DIR, exist_ok=True)
    sources = [s for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]
    if force:
        for s in sources:
            obj = os.path.join(OBJ_DIR, s.replace('.cu', '.o'))
            if os.path.exists(obj):
                os.remove(obj)
    with ThreadPoolExecutor(max_workers=min(8, len(sources))) as pool:
        objs = list(pool.map(lambda s: _compile(s, verbose), sources))
    if force or not os.path.exists(LIB_PATH) or any(os.path.getmtime(o) > os.path.getmtime(LIB_PATH) for o in objs):
        cmd = [NVCC, '-shared', '-o', LIB_PATH, *objs, '-gencode', 'arch=compute_90a,code=sm_90a', '-lcudart_static',
               '-ldl', '-lpthread', '-lrt']
        res = subprocess.run(cmd, capture_output=True, text=True, check=False)
        if res.returncode != 0:
            raise RuntimeError(f"link failed:\n{res.stdout}\n{res.stderr}")
    return LIB_PATH


if __name__ == '__main__':
    print(build(verbose='-v' in sys.argv, force='-f' in sys.argv))
