"""MX block-scaled fp8 (OCP Microscaling: e4m3 elements, one UE8M0 power-of-two scale per 32 consecutive K elements).

The scales are applied to the fp32 partial sum of every 32-element K block (one e4m3 ``wgmma`` each, csrc/gemm_mx.cu), so the
finer granularity costs no epilogue work.  The reference has no reduced-precision expert path (its experts run
``torch.matmul`` in the model dtype, tutel/experts/ffn.py); the framework's fused engine uses the row-scaled e4m3 GEMM of
csrc/gemm_sm90.cu, this module is the finer-grained alternative for GEMMs whose rows carry outliers.

Everything here also has a pure PyTorch definition (``*_reference``) that runs on CPU: the tests compare the kernels
against it, and it documents the number format:

* block exponent   ``e = ceil(log2(amax / 448))`` clamped to [-126, 126] for a block with a non-zero element, where
  ``amax`` is the largest magnitude that is not NaN; ``e = -127`` (scale byte 0) for a block whose ``amax`` is 0
* elements         ``q = e4m3_rn_satfinite(x * 2**-e)`` (+-inf saturate to +-448, NaN stays NaN)
* scale byte       ``e + 127``; byte 0 decodes to a scale of 0, not 2**-127 (the GEMM kernel and :func:`mx_dequantize`)
* scale storage    ``sf[g][k // 128][r // 128][(r % 32) * 16 + ((r % 128) // 32) * 4 + (k % 128) // 32]`` - 512-byte
  atoms in the order the tensor core reads them from tensor memory (rows padded to a multiple of 128 with byte 0).
"""
from __future__ import annotations

from typing import Any, Optional, Tuple

import torch

from . import backend

BLOCK = 32
E4M3_MAX = 448.0


def _check_k(K: int):
    if K % 128 != 0:
        raise ValueError('MX operands need K %% 128 == 0 (got %d)' % K)


def block_exponents_reference(x: torch.Tensor) -> torch.Tensor:
    """Shared exponents [.., K / 32] (int32) of the 32-element blocks along the last dim."""
    a = x.float().abs()
    # NaN takes no part in the maximum (the kernels' fmaxf): the block's other elements keep their scale
    a = torch.where(torch.isnan(a), torch.zeros_like(a), a)
    amax = a.reshape(*x.shape[:-1], x.shape[-1] // BLOCK, BLOCK).amax(-1)
    # ceil(log2(v)) from the float representation: exponent field (+1 when the mantissa is non-zero), as the kernel does.
    # Below 448 * 2^-126, v is an fp32 subnormal and this gives -126; only amax == 0 gives -127.
    v = (amax * (1.0 / E4M3_MAX)).contiguous()
    bits = v.view(torch.int32)
    e = ((bits >> 23) & 0xFF) - 127 + ((bits & 0x7FFFFF) != 0).to(torch.int32)
    return e.clamp_(-127, 126)


def pack_scales(e: torch.Tensor) -> torch.Tensor:
    """Block exponents [G, R, K / 32] -> scale bytes in tile order (uint8, flat)."""
    G, R, KB32 = e.shape
    K = KB32 * BLOCK
    _check_k(K)
    RT = (R + 127) // 128
    b = torch.zeros(G, RT * 128, KB32, dtype=torch.uint8, device=e.device)
    b[:, :R] = (e + 127).to(torch.uint8)
    # [G, rt, c(4), l(32), kb, j(4)] -> [G, kb, rt, l, c, j]
    b = b.view(G, RT, 4, 32, K // 128, 4).permute(0, 4, 1, 3, 2, 5)
    return b.contiguous().view(-1)


def unpack_scales(sf: torch.Tensor, G: int, R: int, K: int) -> torch.Tensor:
    """Inverse of :func:`pack_scales`: block exponents [G, R, K / 32] (int32)."""
    _check_k(K)
    RT = (R + 127) // 128
    b = sf.view(G, K // 128, RT, 32, 4, 4).permute(0, 2, 4, 3, 1, 5).contiguous().view(G, RT * 128, K // BLOCK)
    return b[:, :R].to(torch.int32) - 127


def mx_quantize_reference(x: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """x [G, R, K] -> (q e4m3 [G, R, K], sf uint8) in pure PyTorch (any device)."""
    G, R, K = x.shape
    _check_k(K)
    e = block_exponents_reference(x)
    inv = torch.exp2(-e.float()).unsqueeze(-1)
    q = (x.float().view(G, R, K // BLOCK, BLOCK) * inv).clamp_(-E4M3_MAX, E4M3_MAX).view(G, R, K).to(torch.float8_e4m3fn)
    return q, pack_scales(e)


def mx_dequantize(q: torch.Tensor, sf: torch.Tensor) -> torch.Tensor:
    """fp32 values of an MX operand (pure PyTorch).  Scale byte 0 (e = -127, only all-zero blocks and padded rows) is
    a scale of 0, as in the GEMM kernel."""
    G, R, K = q.shape
    e = unpack_scales(sf, G, R, K)
    s = torch.where(e == -127, torch.zeros_like(e, dtype=torch.float32), torch.exp2(e.float()))
    return (q.float().view(G, R, K // BLOCK, BLOCK) * s.unsqueeze(-1)).view(G, R, K)


def mx_quantize(x: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """x [G, R, K] (or [R, K]) bf16 / fp16 -> (q, sf).  One launch of ``mx_quantize_kernel`` on a GPU."""
    squeeze = x.dim() == 2
    x3 = x.unsqueeze(0) if squeeze else x
    _check_k(x3.shape[-1])
    if x3.is_cuda and x3.element_size() == 2 and backend.has_ext():
        backend.count_launch()
        q, sf = backend.require_ext().mx_quantize(x3.contiguous())
    else:
        if x3.is_cuda and not backend.allow_fallback():
            raise RuntimeError('mx_quantize: 16-bit CUDA input and the native extension are required on a GPU')
        q, sf = mx_quantize_reference(x3)
    return (q[0] if squeeze else q), sf


EPI_NONE, EPI_RELU, EPI_RELU_BWD = 0, 1, 2


def mx_quantize_transpose(x: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """x [G, R, K] -> MX copy of ``x^T`` ([G, K, R], quantised along R) without a 16-bit transpose (one launch)."""
    G, R, K = x.shape
    if x.is_cuda and x.element_size() == 2 and backend.has_ext() and R % 128 == 0 and K % 64 == 0:
        backend.count_launch()
        q, sf = backend.require_ext().mx_quantize_transpose(x.contiguous())
        return q, sf
    return mx_quantize(x.transpose(1, 2).contiguous())


def mx_gemm(a: torch.Tensor, sfa: torch.Tensor, b: torch.Tensor, sfb: torch.Tensor, bias: Optional[torch.Tensor] = None,
            aux: Optional[torch.Tensor] = None, epilogue: int = EPI_NONE, block_n: int = 0, cta_group: int = 0,
            max_ctas: int = 0) -> torch.Tensor:
    """``epilogue(a [G, M, K] @ b [G, N, K]^T + bias [G, N])`` -> bf16 [G, M, N]; operands from :func:`mx_quantize`.
    ``EPI_RELU``: max(., 0);  ``EPI_RELU_BWD``: keep the result where ``aux`` (the forward activation) is positive."""
    if a.is_cuda and backend.has_ext():
        backend.count_launch()
        if bias is not None:
            bias = bias.reshape(a.size(0), b.size(1)).to(torch.bfloat16).contiguous()
        if aux is not None:
            aux = aux.to(torch.bfloat16).contiguous()
        return backend.require_ext().mx_gemm(a, sfa, b, sfb, bias, aux, int(epilogue), int(block_n), int(cta_group), int(max_ctas))
    if a.is_cuda and not backend.allow_fallback():
        raise RuntimeError('mx_gemm: the native extension is required on a GPU')
    y = torch.matmul(mx_dequantize(a, sfa), mx_dequantize(b, sfb).transpose(1, 2))
    if bias is not None:
        y = y + bias.float().reshape(a.size(0), 1, b.size(1))
    if epilogue == EPI_RELU:
        y = torch.relu(y)
    elif epilogue == EPI_RELU_BWD:
        y = torch.where(aux.float() > 0, y, torch.zeros_like(y))
    return y.to(torch.bfloat16)


_MX_WEIGHT_CACHE = {}


def mx_weight(w: torch.Tensor, transpose: bool = False):
    """MX copy of a weight [G, N, K] (or of ``w^T`` when ``transpose``), cached like ``ops.gemm.fp8_operand``: valid until
    the next optimizer step or in-place modification."""
    import weakref
    from . import gemm as _gemm
    _gemm._ensure_step_hook()
    anchor = w._base if w._base is not None else w
    key = (id(anchor), w.data_ptr(), bool(transpose), tuple(w.shape), tuple(w.stride()))
    stamp = (w._version, _gemm._FP8_STEP[0])
    hit = _MX_WEIGHT_CACHE.get(key)
    if hit is not None and hit[0] == stamp and hit[3]() is anchor:
        return hit[1], hit[2]
    src = w.detach()
    q, sf = mx_quantize_transpose(src.contiguous()) if transpose else mx_quantize(src.contiguous())
    if len(_MX_WEIGHT_CACHE) > 256:
        for k in [k for k, v in _MX_WEIGHT_CACHE.items() if v[3]() is None]:
            del _MX_WEIGHT_CACHE[k]
    _MX_WEIGHT_CACHE[key] = (stamp, q, sf, weakref.ref(anchor))
    return q, sf


def mx_linear(x: torch.Tensor, w: torch.Tensor, w_layout: str = 'nk', bias: Optional[torch.Tensor] = None,
              epilogue: int = EPI_NONE, aux: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``epilogue(x [G, R, K] @ W + bias)`` with both operands quantised to MX fp8 on the fly (weights cached); W is
    [G, N, K] ('nk') or [G, K, N] ('kn')."""
    xq, xs = mx_quantize(x)
    wq, ws = mx_weight(w, transpose=(w_layout == 'kn'))
    return mx_gemm(xq, xs, wq, ws, bias=bias, aux=aux, epilogue=epilogue)


def can_use_mx(x: torch.Tensor, w1: torch.Tensor, w2: torch.Tensor) -> bool:
    """bf16 tensors on a GPU, every GEMM dimension a multiple of 128 (K steps and scale atoms are 128 wide)."""
    return (x.is_cuda and backend.has_ext() and x.dtype == torch.bfloat16 and w1.dtype == torch.bfloat16 and w2.dtype == torch.bfloat16
            and x.dim() == 3 and x.size(-1) % 128 == 0 and w1.size(1) % 128 == 0 and w2.size(2) % 128 == 0)


class FusedReluFFNMx(torch.autograd.Function):
    """ReLU expert FFN ``relu(x @ w1^T + b1) @ w2 + b2`` (x [E, C, M], w1 [E, H, M], w2 [E, H, Mo]: the layout of
    models/experts/ffn.py) with MX fp8 forward and data-gradient GEMMs - scales applied by the tensor core - and 16-bit
    weight-gradient GEMMs on the master weights.  Same structure as ``ops.gemm.FusedReluFFNFp8`` (row scales)."""

    @staticmethod
    def forward(ctx: Any, x, w1, b1, w2, b2):
        act = mx_linear(x, w1, 'nk', b1, EPI_RELU)
        y = mx_linear(act, w2, 'kn', b2)
        ctx.save_for_backward(x, w1, w2, act)
        ctx.has_b1, ctx.has_b2 = b1 is not None, b2 is not None
        return y

    @staticmethod
    def backward(ctx: Any, dy: torch.Tensor):
        from . import gemm as _gemm
        x, w1, w2, act = ctx.saved_tensors
        dy = dy.contiguous()
        dh = mx_linear(dy, w2, 'nk', None, EPI_RELU_BWD, aux=act)       # dy @ W2^T: W2 [H, Mo] is K-major for it
        dw2 = _gemm.raw_gemm(act, dy, a_mn=True, b_mn=True) if ctx.needs_input_grad[3] else None
        db2 = _gemm.column_sums(dy) if ctx.has_b2 and ctx.needs_input_grad[4] else None
        dx = mx_linear(dh, w1, 'kn') if ctx.needs_input_grad[0] else None   # dh @ W1: W1^T [M, H] K-major
        dw1 = _gemm.raw_gemm(dh, x, a_mn=True, b_mn=True) if ctx.needs_input_grad[1] else None
        db1 = _gemm.column_sums(dh) if ctx.has_b1 and ctx.needs_input_grad[2] else None
        return dx, dw1, db1, dw2, db2


def fused_relu_ffn_mx(x, w1, b1, w2, b2):
    b1 = None if b1 is None else b1.reshape(w1.size(0), -1)
    b2 = None if b2 is None else b2.reshape(w2.size(0), -1)
    return FusedReluFFNMx.apply(x, w1, b1, w2, b2)


def mx_ffn(x: torch.Tensor, w1: torch.Tensor, w2: torch.Tensor) -> torch.Tensor:
    """Bias-free shorthand of :func:`fused_relu_ffn_mx`."""
    return fused_relu_ffn_mx(x, w1, None, w2, None)
