"""In-tree ahead-of-time build of the native runtime (``tutel_b200/_C*.so``) for sm_90a.

The reference compiles its kernels at run time by fork/exec of nvcc (tutel/custom/custom_kernel.cpp:94-125) and
builds one C++ extension through setuptools (setup.py:123-130).  Here every kernel is compiled ahead of time with
``-gencode arch=compute_90a,code=sm_90a -lineinfo`` (cross-compiles without a GPU) and linked into a single
extension that lives next to the Python sources, so it travels to the GPU box with the snapshot.

Usage:  python -m tutel_b200._build [--force] [--verbose]
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
import sysconfig
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'csrc')
BUILD = os.path.join(ROOT, 'build', 'obj')
EXT_SUFFIX = sysconfig.get_config_var('EXT_SUFFIX') or '.so'
TARGET = os.path.join(ROOT, 'tutel_b200', '_C' + EXT_SUFFIX)

CUDA_SOURCES = ['gemm_sm90.cu', 'gemm_mx.cu', 'gemm_block_fp8.cu', 'moe_kernels.cu', 'gate_route.cu', 'p2p_kernels.cu', 'skinny_gemm.cu', 'gemm_w4a16.cu']
CPP_SOURCES = ['bindings.cpp', 'cpu_kernels.cpp', 'symm_heap.cpp', 'jit_nvrtc.cpp']

NVCC_FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-lineinfo', '-O3', '-std=c++17',
              '--expt-relaxed-constexpr', '-Xcompiler', '-fPIC', '-DTORCH_EXTENSION_NAME=_C']


def _cuda_home():
    for c in (os.environ.get('CUDA_HOME'), os.environ.get('CUDA_PATH'), '/usr/local/cuda'):
        if c and os.path.exists(os.path.join(c, 'bin', 'nvcc')):
            return c
    nvcc = shutil.which('nvcc')
    if nvcc:
        return os.path.dirname(os.path.dirname(nvcc))
    raise RuntimeError('nvcc not found: tutel_b200 needs the CUDA toolkit to build its sm_90a kernels')


def _digest(paths, extra=''):
    h = hashlib.sha256(extra.encode())
    for p in sorted(paths):
        with open(p, 'rb') as f:
            h.update(p.encode())
            h.update(f.read())
    return h.hexdigest()


def _run(cmd, verbose):
    if verbose:
        print(' '.join(cmd), flush=True)
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError('build step failed:\n%s\n%s\n%s' % (' '.join(cmd), r.stdout, r.stderr))
    if verbose and (r.stdout or r.stderr):
        print(r.stdout, r.stderr)


def build(force=False, verbose=False):
    """Compile (if stale) and return the path of the extension."""
    import torch
    from torch.utils import cpp_extension as ce

    cuda_home = _cuda_home()
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(('.h', '.cuh'))]
    os.makedirs(BUILD, exist_ok=True)
    torch_inc = ce.include_paths()
    inc = ['-I' + CSRC, '-I' + os.path.join(cuda_home, 'include'), '-I' + sysconfig.get_paths()['include']]
    inc += ['-I' + p for p in torch_inc]
    abi = int(getattr(torch._C, '_GLIBCXX_USE_CXX11_ABI', True))
    cxx_flags = ['-O2', '-std=c++17', '-fPIC', '-DTORCH_EXTENSION_NAME=_C', '-DTORCH_API_INCLUDE_EXTENSION_H',
                 '-D_GLIBCXX_USE_CXX11_ABI=%d' % abi, '-Wno-deprecated-declarations']

    jobs, objs = [], []
    for src in CUDA_SOURCES + CPP_SOURCES:
        path = os.path.join(CSRC, src)
        obj = os.path.join(BUILD, src + '.o')
        stamp = obj + '.sha'
        is_cu = src.endswith('.cu')
        flags = NVCC_FLAGS if is_cu else cxx_flags
        dig = _digest([path] + headers, ' '.join(flags) + torch.__version__)
        objs.append(obj)
        if not force and os.path.exists(obj) and os.path.exists(stamp) and open(stamp).read() == dig:
            continue
        if is_cu:
            cmd = [os.path.join(cuda_home, 'bin', 'nvcc')] + NVCC_FLAGS + ['-I' + CSRC, '-c', path, '-o', obj]
        else:
            cmd = [os.environ.get('CXX', 'g++')] + cxx_flags + inc + ['-c', path, '-o', obj]
        jobs.append((cmd, stamp, dig))

    def _do(job):
        cmd, stamp, dig = job
        _run(cmd, verbose)
        with open(stamp, 'w') as f:
            f.write(dig)

    if jobs:
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            list(ex.map(_do, jobs))

    if jobs or not os.path.exists(TARGET):
        torch_lib = os.path.join(os.path.dirname(torch.__file__), 'lib')
        cudart_dirs = [torch_lib, os.path.join(cuda_home, 'lib64')]
        try:
            import nvidia.cuda_runtime
            cudart_dirs.insert(0, os.path.join(list(nvidia.cuda_runtime.__path__)[0], 'lib'))
        except Exception:
            pass
        link = [os.environ.get('CXX', 'g++'), '-shared', '-o', TARGET] + objs
        for d in cudart_dirs:
            link += ['-L' + d, '-Wl,-rpath,' + d]
        link += ['-lc10', '-ltorch', '-ltorch_cpu', '-ltorch_python', '-lc10_cuda', '-ltorch_cuda', '-ldl']
        cudart = None
        for d in cudart_dirs:
            for name in ('libcudart.so.12', 'libcudart.so'):
                if os.path.exists(os.path.join(d, name)):
                    cudart = os.path.join(d, name)
                    break
            if cudart:
                break
        link += [cudart] if cudart else ['-lcudart']
        _run(link, verbose)
    return TARGET


if __name__ == '__main__':
    out = build(force='--force' in sys.argv, verbose='--verbose' in sys.argv)
    print(out)
