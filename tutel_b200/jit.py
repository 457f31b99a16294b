"""Run-time CUDA kernel creation (mirrors tutel/jit.py:4, tutel/impls/jit_compiler.py:24-55).

The source is compiled with NVRTC for the device's architecture (``sm_90a`` on H100) inside the native runtime
(csrc/jit_nvrtc.cpp); launch extents come from ``// [thread_extent] blockIdx.x = N`` comments exactly like the
reference's kernel strings, and ``@key@`` placeholders are substituted from ``keyword_dict``.
"""
from .ops import backend


class JitCompiler:
    @staticmethod
    def create_raw(source):
        C = backend.require_ext()
        handle = C.jit_inject_source(source)

        def func(*inputs, extra=(), blocks=()):
            C.jit_invoke(list(inputs), [int(v) for v in extra], [int(v) for v in blocks], handle)
        return func

    @staticmethod
    def generate_kernel(keyword_dict, template):
        for key, value in keyword_dict.items():
            template = template.replace('@%s@' % key, str(value))
        return JitCompiler.create_raw(template)


def create_cuda_kernel(source, keyword_dict=None):
    return JitCompiler.generate_kernel(keyword_dict or {}, source)
