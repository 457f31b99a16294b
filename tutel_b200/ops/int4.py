"""Group-32 int4 expert weights (W4A16): the routed-expert format of Kimi-K2-Thinking (compressed-tensors
``pack-quantized``, symmetric, one bf16 scale per 32 input elements) and a common quantisation of Mixtral- and
Qwen-MoE-style models.  Inference only; the activations stay bf16.

The format, which the pure PyTorch definitions below (``*_reference``) spell out and the tests check the kernels against:

* values           ``w = q * s`` with ``q`` a signed int4 in [-8, 7] and ``s`` a bf16 scale shared by 32 consecutive
                   elements along the input (K) dimension of one output row.  Checkpoint orientation ``[N, K]``: gate /
                   up ``[E, H, M]``, down ``[E, M, H]``.  Group size 32 only, no zero points.
* nibble packing   byte ``j`` of a row holds element ``2j`` in bits 0-3 and ``2j + 1`` in bits 4-7, each as ``u = q + 8``
                   (offset binary).  A 16-byte load is one whole group: word ``i`` holds elements ``8i .. 8i + 7``,
                   element ``8i + e`` in bits ``4e .. 4e + 3``.
* scales           ``[E, N, K / 32]`` bf16, row-major: the checkpoint's own layout, one copy for both kernels.  The
                   decode kernel reads a row along K, a group's scale beside its 16 bytes of nibbles.  In the prefill
                   GEMM each expanding thread reads its row's scale of a K step straight from global memory (L2), so
                   no TMA box of scales is needed (a row has 4 bytes per K step, under TMA's 16-byte minimum).
* stored copy      ``W_gate_up [E, 2H, M / 2]`` uint8 with gate and up rows interleaved every 64 (rows ``128 t + j`` = gate
                   unit ``64 t + j``, rows ``128 t + 64 + j`` = its up partner, the convention of ``fp8_block``) and
                   ``W_gate_up_scale [E, 2H, M / 32]`` interleaved the same way; ``W_down [E, M, H / 2]`` uint8 and
                   ``W_down_scale [E, M, H / 32]`` in the checkpoint orientation.  0.5625 bytes per weight.
* quantiser        (``export_int4_weights``, this project's rule): per group, ``amax`` = the largest magnitude that is not
                   NaN, ``s = max(bf16_rn(amax / 7), 2^-126)`` (the smallest normal bf16) and ``s = 1`` when ``amax == 0``;
                   ``q = clamp(rn(w / s), -8, 7)`` with the stored ``s``, rn = round half to even, NaN -> 0.
* compressed-tensors int32 packing (``unpack_int32``): ``weight_packed [N, K / 8]`` int32, element ``i`` of a word in bits
                   ``4i .. 4i + 3`` as ``q + 8``.  This is the convention we understand compressed-tensors to use; it
                   could not be checked against a real checkpoint here, so verify a first load against the model's
                   reference output.

Kernels (a GPU runs these; the CPU runs the references):

* decode           ``skinny_glu_ffn_int4`` (``skinny_glu_ffn_int4_kernel``, csrc/skinny_gemm.cu): the whole SwiGLU expert
                   in one launch driven by device row counts, reading every active expert's bytes once per 4 rows;
                   ``acc += s * sum(q * x)`` per 32-term group in fp32.
* prefill          ``glu_ffn_int4``: two launches of the mixed-input wgmma GEMM ``w4a16_gemm_kernel``
                   (csrc/gemm_w4a16.cu), which TMA-loads the nibbles and expands them in shared memory to
                   ``bf16_rn(q * s)`` (exact product, one rounding) for bf16 tensor-core MMAs with fp32 accumulation:
                   the GLU GEMM (h = act(g) * u in the epilogue) and the down GEMM, with the device row counts of
                   dropless prefill.  No bf16 copy of the weights is ever written to memory.
"""
from __future__ import annotations

from typing import Optional

import torch

from . import backend
from . import block_fp8 as BF8

GROUP = 32
BF16_MIN_NORMAL = 2.0 ** -126
ACT_CODES = BF8.ACT_CODES


def _check(ok: bool, msg: str):
    if not ok:
        raise ValueError(msg)


# ------------------------------------------------------------------------------------------------------------------
# definitions
# ------------------------------------------------------------------------------------------------------------------
def pack_reference(q: torch.Tensor) -> torch.Tensor:
    """int8 values in [-8, 7], ``[..., K]`` (K even) -> uint8 ``[..., K / 2]``: byte j = (q[2j] + 8) | (q[2j + 1] + 8) << 4."""
    u = (q.to(torch.int16) + 8).to(torch.uint8)
    return u[..., 0::2] | (u[..., 1::2] << 4)


def unpack_reference(packed: torch.Tensor) -> torch.Tensor:
    """uint8 ``[..., K / 2]`` -> int8 ``[..., K]``, the inverse of ``pack_reference``."""
    lo = (packed & 0xF).to(torch.int8) - 8
    hi = (packed >> 4).to(torch.int8) - 8
    return torch.stack([lo, hi], dim=-1).reshape(*packed.shape[:-1], packed.size(-1) * 2)


def unpack_int32(packed: torch.Tensor, k: int) -> torch.Tensor:
    """compressed-tensors ``weight_packed`` int32 ``[..., K / 8]`` -> int8 ``[..., k]``: element i of a word is bits
    4i .. 4i + 3, stored as q + 8 (see the module doc: not verified against a real checkpoint)."""
    _check(packed.dtype == torch.int32, 'unpack_int32: int32 packed weights expected (got %s)' % (packed.dtype,))
    _check(k % 8 == 0 and packed.size(-1) == k // 8, 'unpack_int32: [..., %d] int32 expected for k=%d (got %s)'
           % (k // 8, k, tuple(packed.shape)))
    shifts = torch.arange(8, device=packed.device, dtype=torch.int32) * 4
    u = (packed.unsqueeze(-1) >> shifts) & 0xF                    # arithmetic shift: the mask drops the sign bits
    return (u - 8).to(torch.int8).reshape(*packed.shape[:-1], k)


def quantize_reference(w: torch.Tensor):
    """w ``[..., K]`` (K % 32 == 0) -> (q int8 ``[..., K]``, s bf16 ``[..., K / 32]``) by the quantiser rule of the module
    doc."""
    _check(w.size(-1) % GROUP == 0, 'int4 quantiser: K must be a multiple of 32 (got %d)' % w.size(-1))
    wg = w.double().reshape(*w.shape[:-1], w.size(-1) // GROUP, GROUP)
    amax = torch.nan_to_num(wg.abs(), nan=0.0).amax(dim=-1)
    s = torch.clamp((amax / 7).to(torch.bfloat16).double(), min=BF16_MIN_NORMAL)
    s = torch.where(amax == 0, torch.ones_like(s), s).to(torch.bfloat16)
    q = torch.nan_to_num(torch.round(wg / s.double().unsqueeze(-1)), nan=0.0).clamp(-8, 7)
    return q.to(torch.int8).reshape(w.shape), s


def dequantize_reference(q: torch.Tensor, s: torch.Tensor, dtype=torch.float64) -> torch.Tensor:
    """int8 q ``[..., K]`` and bf16 s ``[..., K / 32]`` -> q * s (exact in fp32 and fp64; bf16 rounds once)."""
    v = q.double().reshape(*q.shape[:-1], -1, GROUP) * s.double().unsqueeze(-1)
    return v.reshape(q.shape).to(dtype)


def stored_values(packed: torch.Tensor, s: torch.Tensor, dtype=torch.float64) -> torch.Tensor:
    """A stored operand (nibbles ``[..., K / 2]``, scales ``[..., K / 32]``) -> q * s in ``dtype``."""
    return dequantize_reference(unpack_reference(packed), s, dtype)


def export_glu_weights(w1: torch.Tensor, w2: torch.Tensor, w3: torch.Tensor):
    """bf16 SwiGLU weights in the ``llama_ffn`` layout (w1, w2 [E, M, H], w3 [E, H, M]) -> the six checkpoint tensors
    (gate int8 [E, H, M], gate_scale bf16 [E, H, M / 32], up, up_scale, down int8 [E, M, H], down_scale [E, M, H / 32])."""
    for name, w in (('w1', w1), ('w2', w2), ('w3', w3)):
        _check(w.dtype == torch.bfloat16 and w.dim() == 3, 'export_int4_weights: %s must be a bf16 [E, *, *] tensor '
               '(got %s %s)' % (name, w.dtype, tuple(w.shape)))
    _check(w1.shape == w2.shape and w3.shape == (w1.size(0), w1.size(2), w1.size(1)),
           'export_int4_weights: w1, w2 [E, M, H] and w3 [E, H, M] expected (got %s, %s, %s)'
           % (tuple(w1.shape), tuple(w2.shape), tuple(w3.shape)))
    gate, gate_s = quantize_reference(w1.detach().transpose(1, 2))
    up, up_s = quantize_reference(w2.detach().transpose(1, 2))
    down, down_s = quantize_reference(w3.detach().transpose(1, 2))
    return gate, gate_s, up, up_s, down, down_s


def load_glu_weights(gate, gate_scale, up, up_scale, down, down_scale):
    """The six checkpoint tensors (see ``export_glu_weights``) -> the stored layout (qglu, sglu, q3t, s3t) on gate's
    device.  Shapes, dtypes and the value range are checked; packing and interleaving are one-time torch ops."""
    def expect(t, dtype, shape, name):
        _check(isinstance(t, torch.Tensor) and t.dtype == dtype and tuple(t.shape) == tuple(shape),
               'load_int4_weights: %s must be %s %s (got %s %s)' % (
                   name, dtype, tuple(shape), getattr(t, 'dtype', type(t)), tuple(getattr(t, 'shape', ()))))
    _check(isinstance(gate, torch.Tensor) and gate.dim() == 3, 'load_int4_weights: gate must be int8 [E, H, M]')
    E, H, M = gate.shape
    _check(H % 128 == 0 and M % 128 == 0, 'load_int4_weights: H and M must be multiples of 128 (got %d, %d)' % (H, M))
    for name, t, shape in (('gate', gate, (E, H, M)), ('up', up, (E, H, M)), ('down', down, (E, M, H))):
        expect(t, torch.int8, shape, name)
        _check(not bool(((t < -8) | (t > 7)).any()), 'load_int4_weights: %s holds values outside the int4 range [-8, 7]'
               % name)
    expect(gate_scale, torch.bfloat16, (E, H, M // GROUP), 'gate_scale')
    expect(up_scale, torch.bfloat16, (E, H, M // GROUP), 'up_scale')
    expect(down_scale, torch.bfloat16, (E, M, H // GROUP), 'down_scale')
    dev = gate.device
    qglu = BF8.interleave_glu_reference(pack_reference(gate), pack_reference(up.to(dev)))
    sglu = BF8.interleave_glu_reference(gate_scale.to(dev), up_scale.to(dev))
    return qglu.contiguous(), sglu.contiguous(), pack_reference(down.to(dev)).contiguous(), down_scale.to(dev).contiguous()


# ------------------------------------------------------------------------------------------------------------------
# kernels
# ------------------------------------------------------------------------------------------------------------------
def can_use_stored_glu(x: torch.Tensor) -> bool:
    """Inputs the int4 SwiGLU expert runs on: bf16 [E, rows, M].  Nothing is cast: other dtypes are refused."""
    return x.dtype == torch.bfloat16 and x.dim() == 3


def can_use_skinny_glu_ffn_int4(x: torch.Tensor) -> bool:
    """``skinny_glu_ffn_int4`` covers up to 64 rows per expert and M up to 12544 (the shared memory of fp8_block's)."""
    return can_use_stored_glu(x) and x.size(1) <= 64 and 8 * x.size(2) + 2048 <= BF8.SKINNY_SMEM_LIMIT


def _split_glu(w: torch.Tensor):
    """[E, 2H, *] rows interleaved every 64 -> gate [E, H, *], up [E, H, *]."""
    E, H2 = w.shape[:2]
    t = w.reshape(E, H2 // 128, 2, 64, *w.shape[2:])
    return t[:, :, 0].reshape(E, H2 // 2, *w.shape[2:]), t[:, :, 1].reshape(E, H2 // 2, *w.shape[2:])


def skinny_glu_ffn_int4_reference(x, qglu, sglu, q3t, s3t, row_counts, act='silu'):
    """fp32 composition on the exact stored values q * s; rows past the counts are zero.  The CPU path of the kernel."""
    wg, wu = _split_glu(stored_values(qglu, sglu, torch.float32))
    w3 = stored_values(q3t, s3t, torch.float32)
    xf = x.float()
    h = BF8._act(xf @ wg.transpose(1, 2), act)[0] * (xf @ wu.transpose(1, 2))
    y = h @ w3.transpose(1, 2)
    if row_counts is not None:
        y = BF8.zero_rows_past(y, row_counts)
    return y.to(x.dtype)


def skinny_glu_ffn_int4(x, qglu, sglu, q3t, s3t, row_counts, act='silu'):
    """y[g, r] = (act(x @ W1) * (x @ W2)) @ W3 for r < row_counts[g] (other rows zero) on the stored int4 weights, in one
    weight-streaming launch of ``skinny_glu_ffn_int4_kernel`` on a GPU (x stays bf16)."""
    if BF8._native(x, 'int4.skinny_glu_ffn_int4'):
        backend.count_launch(2)          # zero-fill of the fp32 accumulator + the kernel
        y = backend.require_ext().skinny_glu_ffn_int4(x.contiguous(), qglu, sglu, q3t, s3t, row_counts, ACT_CODES[act])
        return y.to(x.dtype)
    return skinny_glu_ffn_int4_reference(x, qglu, sglu, q3t, s3t, row_counts, act)


def w4a16_gemm_reference(a, q, s, act=None, row_counts=None):
    """The CPU definition of ``w4a16_gemm``: a [G, M, K] bf16 times bf16_rn(q * s)^T with fp32 products, bf16 out; with
    ``act`` the GLU epilogue on the interleaved gate / up operand (h = act(gate) * up)."""
    w = stored_values(q, s, torch.bfloat16).float()
    if act is None:
        y = a.float() @ w.transpose(1, 2)
    else:
        wg, wu = _split_glu(w)
        af = a.float()
        y = BF8._act(af @ wg.transpose(1, 2), act)[0] * (af @ wu.transpose(1, 2))
    y = y.to(torch.bfloat16)
    return y if row_counts is None else BF8.zero_rows_past(y, row_counts)


def w4a16_gemm(a, q, s, act=None, row_counts=None):
    """Mixed-input grouped GEMM (``w4a16_gemm_kernel``, csrc/gemm_w4a16.cu): bf16 a [G, M, K] times the stored int4
    operand (nibbles [G, N, K / 2], scales [G, N, K / 32]) expanded on chip to bf16_rn(q * s); fp32 accumulation, bf16
    out [G, M, N].  ``act``: the GLU epilogue on the interleaved gate / up operand, h = act(gate) * up, [G, M, N / 2].
    Rows at or past ``row_counts`` are zero."""
    if BF8._native(a, 'int4.w4a16_gemm'):
        backend.count_launch()
        return backend.require_ext().w4a16_gemm(a.contiguous(), q, s, row_counts, 0 if act is None else 1,
                                                0 if act is None else ACT_CODES[act])
    return w4a16_gemm_reference(a, q, s, act, row_counts)


def glu_ffn_int4(x, qglu, sglu, q3t, s3t, act='silu', row_counts=None):
    """Inference forward of the int4 experts on the mixed-input GEMM: the GLU launch (h = act(x Wg) * (x Wu), h in bf16)
    and the down launch, with the device row counts of dropless prefill when given (rows past them are zero)."""
    h = w4a16_gemm(x, qglu, sglu, act, row_counts)
    return w4a16_gemm(h, q3t, s3t, None, row_counts)
