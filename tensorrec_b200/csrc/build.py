"""Builds libtensorrec_b200.so (the C-ABI library of include/tensorrec_b200.h) in-tree with nvcc for sm_90a (H100).

    python -m tensorrec_b200.csrc.build [--force] [--verbose]

nvcc cross-compiles without a GPU.  Objects are cached next to the sources (git-ignored) and rebuilt when a source
or header is newer.  The CUDA runtime is linked statically, so the library loads (and exports its symbols) on a
machine without a driver; cuTensorMapEncodeTiled is resolved at run time through cudaGetDriverEntryPoint.
"""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
SOURCES = ['api.cu', 'csr_gather.cu', 'score_simt.cu', 'rank_full.cu', 'topk_merge.cu', 'score_topk_tc.cu',
           'score_filter_tc.cu', 'score_wide_tc.cu', 'rescore_topk.cu', 'rescore_wide.cu', 'similar_items.cu',
           'wmrb_step.cu', 'relu_layer.cu']
HEADERS = [os.path.join(HERE, 'common.cuh'), os.path.join(HERE, 'filter_tc.cuh'),
           os.path.join(ROOT, 'include', 'tensorrec_b200.h')]
LIB_PATH = os.path.join(os.path.dirname(HERE), 'libtensorrec_b200.so')

NVCC_FLAGS = [
    '-gencode', 'arch=compute_90a,code=sm_90a',
    '-O3', '-std=c++17', '-lineinfo',
    '-Xcompiler', '-fPIC',
    '--expt-relaxed-constexpr',
]


def find_nvcc():
    nvcc = shutil.which('nvcc') or '/usr/local/cuda/bin/nvcc'
    if not os.path.exists(nvcc):
        raise RuntimeError('nvcc not found; tensorrec_b200 needs the CUDA 12.9 toolkit to build its kernels')
    return nvcc


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False, defines=(), out_dir=None):
    """Builds the library; returns its path.  `defines` (e.g. ['TRK_FILTER_CYCLES']) are passed to every translation
    unit as -D flags; such a build belongs in its own `out_dir` (objects and library), which leaves the in-tree build
    alone."""
    nvcc = find_nvcc()
    obj_dir = out_dir or HERE
    lib_path = os.path.join(out_dir, 'libtensorrec_b200.so') if out_dir else LIB_PATH
    dflags = ['-D' + d for d in defines]
    objs = []
    for src in SOURCES:
        src_path = os.path.join(HERE, src)
        obj = os.path.join(obj_dir, src.replace('.cu', '.o'))
        objs.append(obj)
        if force or _stale(obj, [src_path] + HEADERS):
            cmd = [nvcc] + NVCC_FLAGS + dflags + (['-Xptxas', '-v'] if verbose else []) + ['-c', src_path, '-o', obj]
            if verbose:
                print(' '.join(cmd), flush=True)
            subprocess.run(cmd, check=True)
    if force or _stale(lib_path, objs):
        cmd = [nvcc, '-shared', '-gencode', 'arch=compute_90a,code=sm_90a', '-o', lib_path] + objs
        if verbose:
            print(' '.join(cmd), flush=True)
        subprocess.run(cmd, check=True)
    return lib_path


if __name__ == '__main__':
    path = build(force='--force' in sys.argv, verbose='--verbose' in sys.argv)
    print(path)
