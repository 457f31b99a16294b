"""Block-scaled fp8 expert GEMMs, the DeepSeek-V3 recipe (also that of DeepGEMM and of the block-scaled fp8 checkpoints
DeepSeek-V3, Kimi-K2, GLM-4.5 and Moonlight ship with, ``weight_scale_inv`` per 128 x 128 block):

* activations ``[G, R, K]``: e4m3 with one fp32 scale per row and 128-element K tile (1 x 128);
* weights ``[G, N, K]``: e4m3 with one fp32 scale per 128 x 128 block;
* the GEMM (csrc/gemm_block_fp8.cu) runs each 128-deep K step as four e4m3 ``wgmma`` into a scratch fragment and promotes
  it into the fp32 accumulator with the step's two scales: ``acc += scratch * (sa[row] * sb)``.

A 128 x 128 block is the same block in ``W`` and ``W^T``, so the data-gradient copy of a weight is the forward copy
transposed, scales included; one launch writes both.

Everything here also has a pure PyTorch definition (``*_reference``) that runs on CPU: the tests compare the kernels
against it, and it documents the format:

* block scale      ``amax`` = the largest magnitude in the block that is not NaN,
                   ``s = max(amax * (1 / 448), FLT_MIN)`` if ``amax > 0`` else ``1`` (fp32 arithmetic, the rule of
                   ``quantize_rows_kernel``, csrc/moe_kernels.cu)
* elements         ``q = e4m3_rn_satfinite(x * (1 / s))`` (+-inf saturate to +-448, NaN stays NaN)
* activation scales ``[G, K / 128, roundup(R, 128)]`` fp32, MN-major (one K step of a 128-row tile is 512 contiguous
                   bytes); pad rows have scale 0
* weight scales    ``[G, N / 128, K / 128]`` fp32
* SwiGLU gate / up ``w1, w2 [G, M, H]``: the data-gradient operand is ``[W1 W2]`` ``[G, M, 2H]`` with scales
                   ``[G, M / 128, 2H / 128]``; the forward operand is ``W1^T`` and ``W2^T`` interleaved every 64 rows,
                   ``[G, 2H, M]`` (rows ``128 t + j`` = gate column ``64 t + j``, rows ``128 t + 64 + j`` = up column
                   ``64 t + j``) with one scale per 64 rows, ``[G, 2H / 64, M / 128]``, so that one 128-wide N tile holds
                   a gate column and its up partner in the same thread and the GLU epilogue stays in registers.
* column-wise activations (weight gradients, ``fp8_wgrad``): ``x [G, R, K]`` transposed to ``qT [G, K, Rp]`` e4m3,
                   ``Rp = roundup(R, 128)``, with one scale per column of ``x`` and 128-row block (128 x 1 tiles), stored
                   ``sT [G, Rp / 128, K]``; rows ``R..Rp-1`` are zero bytes and take no part in the scale.  One launch
                   (``quantize_act_dual``) writes it together with the row-wise operand above.
* weight-gradient GEMM ``D[g] = A[g] B[g]^T`` over the padded token dimension: A ``[G, Ma, Rp]`` and B ``[G, N, Rp]``
                   are both column-wise operands, so both have one scale per row and 128-deep K step, and each step is
                   promoted as ``acc = fma(part, sa[m] * sb[n], acc)``.
* expert-packed layout (ops/packed.py; dropless training on one GPU): every packed buffer ``[R, K]`` is one group.  The
                   GEMM runs block-mapped (``b_group_map``: row tile ``m`` takes expert ``block_expert[m]``'s weights,
                   ``row_counts`` = ``block_rows``), the weight-gradient GEMM with ragged K (``k_offsets`` = ``seg_off``:
                   expert ``e`` reduces over its own segment) and the quantisers stop at ``live_rows`` = ``seg_off[E]``.
                   Segments start on 128-row boundaries and padding rows are zero, so every 1 x 128 and 128 x 1 tile an
                   expert sees is the one it sees in the padded layout.

Every GEMM dimension but the token count must be a multiple of 128; the operands are bf16.
"""
from __future__ import annotations

from typing import Any, Optional, Tuple

import torch

from . import backend

TILE = 128
E4M3_MAX = 448.0
FLT_MIN = 2.0 ** -126
EPI_NONE, EPI_RELU, EPI_RELU_BWD, EPI_GLU, EPI_GLU_BWD = 0, 1, 2, 3, 4
ACT_CODES = {'relu': 1, 'gelu': 2, 'silu': 3}


def _f32(v: float, like: torch.Tensor) -> torch.Tensor:
    return torch.tensor(v, dtype=torch.float32, device=like.device)


# ------------------------------------------------------------------------------------------------------------------
# number format (pure PyTorch)
# ------------------------------------------------------------------------------------------------------------------
def block_scale_reference(amax: torch.Tensor) -> torch.Tensor:
    """fp32 scales of blocks whose largest non-NaN magnitude is ``amax`` (fp32)."""
    s = torch.maximum(amax * _f32(1.0 / E4M3_MAX, amax), _f32(FLT_MIN, amax))
    return torch.where(amax > 0, s, torch.ones_like(s))


def _nan_abs(x: torch.Tensor) -> torch.Tensor:
    a = x.float().abs()
    return torch.where(torch.isnan(a), torch.zeros_like(a), a)


def _e4m3(v: torch.Tensor) -> torch.Tensor:
    return v.clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn)


def quantize_act_reference(x: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """x [G, R, K] -> (q e4m3 [G, R, K], s fp32 [G, K / 128, roundup(R, 128)])."""
    G, R, K = x.shape
    _check(K % TILE == 0, 'block fp8 activations need K %% 128 == 0 (got %d)' % K)
    KT, Rp = K // TILE, -(-R // TILE) * TILE
    xf = x.float().view(G, R, KT, TILE)
    s = block_scale_reference(_nan_abs(xf).amax(-1))                                  # [G, R, KT]
    q = _e4m3(xf * (1.0 / s).unsqueeze(-1)).view(G, R, K)
    st = torch.zeros(G, KT, Rp, dtype=torch.float32, device=x.device)
    st[:, :, :R] = s.transpose(1, 2)
    return q, st


def quantize_act_dual_reference(x: torch.Tensor, rowwise: bool = True):
    """x [G, R, K] -> (q, s, qT [G, K, Rp], sT [G, Rp / 128, K]); q, s as ``quantize_act_reference`` (None unless
    ``rowwise``)."""
    G, R, K = x.shape
    _check(K % TILE == 0, 'block fp8 activations need K %% 128 == 0 (got %d)' % K)
    Rp = -(-R // TILE) * TILE
    xp = torch.zeros(G, Rp, K, dtype=torch.float32, device=x.device)
    xp[:, :R] = x.float()
    blocks = xp.view(G, Rp // TILE, TILE, K)
    sT = block_scale_reference(_nan_abs(blocks).amax(2))                              # [G, Rp / 128, K]
    qT = _e4m3(blocks * (1.0 / sT).unsqueeze(2)).view(G, Rp, K).transpose(1, 2).contiguous()
    q, s = quantize_act_reference(x) if rowwise else (None, None)
    return q, s, qT, sT


def quantize_weight_reference(w: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]:
    """w [G, R, C] -> (q [G, R, C], s [G, R / 128, C / 128], qT [G, C, R], sT [G, C / 128, R / 128])."""
    G, R, C = w.shape
    _check(R % TILE == 0 and C % TILE == 0, 'block fp8 weights need both dims %% 128 == 0 (got %s)' % (tuple(w.shape),))
    wf = w.float().view(G, R // TILE, TILE, C // TILE, TILE)
    s = block_scale_reference(_nan_abs(wf).amax(dim=(2, 4)))                         # [G, RB, CB]
    q = _e4m3(wf * (1.0 / s)[:, :, None, :, None]).view(G, R, C)
    return q, s, q.transpose(1, 2).contiguous(), s.transpose(1, 2).contiguous()


def interleave_glu_reference(t1: torch.Tensor, t2: torch.Tensor, rows_per: int = 64) -> torch.Tensor:
    """[G, H, *] gate and up rows -> [G, 2H, *]: blocks of ``rows_per`` rows, gate then up."""
    G, H = t1.shape[:2]
    pair = torch.stack([t1.reshape(G, H // rows_per, rows_per, -1), t2.reshape(G, H // rows_per, rows_per, -1)], dim=2)
    return pair.reshape(G, 2 * H, *t1.shape[2:])


def quantize_glu_weight_reference(w1: torch.Tensor, w2: torch.Tensor):
    """Gate / up weights w1, w2 [G, M, H] -> (qcat [G, M, 2H], scat [G, M / 128, 2H / 128], qglu [G, 2H, M],
    sglu [G, 2H / 64, M / 128])."""
    q1, s1, q1t, s1t = quantize_weight_reference(w1)
    q2, s2, q2t, s2t = quantize_weight_reference(w2)
    qcat, scat = torch.cat([q1, q2], dim=2), torch.cat([s1, s2], dim=2)
    # one scale per 64 interleaved rows: each 128-row scale block of W^T covers two of them
    qglu = interleave_glu_reference(q1t.view(torch.uint8), q2t.view(torch.uint8)).view(torch.float8_e4m3fn)
    sglu = interleave_glu_reference(s1t.repeat_interleave(2, dim=1), s2t.repeat_interleave(2, dim=1), rows_per=1)
    return qcat, scat, qglu, sglu


def dequantize_act(q: torch.Tensor, s: torch.Tensor) -> torch.Tensor:
    """fp32 values of an activation operand."""
    G, R, K = q.shape
    return (q.float().view(G, R, K // TILE, TILE) * s[:, :, :R].transpose(1, 2).unsqueeze(-1)).view(G, R, K)


def dequantize_weight(q: torch.Tensor, s: torch.Tensor) -> torch.Tensor:
    """fp32 values of a weight operand [G, N, K] with one scale per 128 x 128 block (or per 64 x 128, GLU layout)."""
    G, N, K = q.shape
    rows = N // s.size(1)
    return (q.float().view(G, s.size(1), rows, K // TILE, TILE) * s[:, :, None, :, None]).view(G, N, K)


def _act(g: torch.Tensor, act: str) -> Tuple[torch.Tensor, torch.Tensor]:
    if act == 'relu':
        return g.clamp_min(0), (g > 0).to(g.dtype)
    if act == 'gelu':
        cdf = 0.5 * (1 + torch.erf(g * 0.70710678118654752))
        return g * cdf, cdf + g * 0.3989422804014327 * torch.exp(-0.5 * g * g)
    sg = torch.sigmoid(g)
    return g * sg, sg * (1 + g * (1 - sg))


def block_fp8_gemm_reference(a, sa, b, sb, bias=None, aux=None, aux2=None, epilogue=EPI_NONE, act='silu'):
    """fp32 emulation of one ``block_fp8_gemm`` launch, in the kernel's order: one fresh fp32 sum per 128-deep K step,
    promoted with a single rounding, ``acc = fma(part, sa * sb, acc)``; then the epilogue in fp32 and one bf16 rounding.
    Returns what the binding returns (a list)."""
    G, M, K = a.shape
    N = b.size(1)
    rows_b = N // sb.size(1)
    acc = torch.zeros(G, M, N, dtype=torch.float32, device=a.device)
    af, bf = a.float(), b.float()
    for kb in range(K // TILE):
        k = slice(kb * TILE, (kb + 1) * TILE)
        part = af[:, :, k] @ bf[:, :, k].transpose(1, 2)
        sab = sa[:, kb, :M].unsqueeze(-1) * sb[:, :, kb].repeat_interleave(rows_b, dim=1).unsqueeze(1)   # fp32 product
        acc = (part.double() * sab.double() + acc.double()).float()
    if epilogue == EPI_GLU:
        H = N // 2
        t = acc.view(G, M, H // 64, 2, 64)
        g, u = t[:, :, :, 0].reshape(G, M, H), t[:, :, :, 1].reshape(G, M, H)
        h = _act(g, act)[0] * u
        return [h.bfloat16(), g.bfloat16(), u.bfloat16()]
    if epilogue == EPI_GLU_BWD:
        a_, da = _act(aux.float(), act)
        return [torch.cat([acc * aux2.float() * da, acc * a_], dim=2).bfloat16()]
    if bias is not None:
        acc = acc + bias.float().reshape(G, 1, N)
    if epilogue == EPI_RELU:
        acc = acc.clamp_min(0)
    elif epilogue == EPI_RELU_BWD:
        acc = torch.where(aux.float() > 0, acc, torch.zeros_like(acc))
    return [acc.bfloat16()]


def wgrad_gemm_reference(aT, saT, bT, sbT, split: Optional[int] = None):
    """fp32 emulation of one ``wgrad_gemm`` launch in the kernel's order: a fresh fp32 sum per 128-deep K step, promoted
    with ``acc = fma(part, sa[m] * sb[n], acc)`` (the scale product rounded to fp32), then one bf16 rounding."""
    G, M, K = aT.shape
    N = bT.size(1)
    acc = torch.zeros(G, M, N, dtype=torch.float32, device=aT.device)
    af, bf = aT.float(), bT.float()
    for kb in range(K // TILE):
        k = slice(kb * TILE, (kb + 1) * TILE)
        part = af[:, :, k] @ bf[:, :, k].transpose(1, 2)
        sab = saT[:, kb, :, None] * sbT[:, kb, None, :]                                # fp32 product
        acc = (part.double() * sab.double() + acc.double()).float()
    d = acc.bfloat16()
    return [d] if not split else [d[..., :split].contiguous(), d[..., split:].contiguous()]


# ------------------------------------------------------------------------------------------------------------------
# expert-packed launch modes (pure PyTorch): the references above, applied per segment.  What the kernels leave
# unwritten (rows past ``live_rows``, tiles with no live rows) is zero here.
# ------------------------------------------------------------------------------------------------------------------
def _host_int(t: torch.Tensor) -> int:
    return int(t.reshape(-1)[0])


def quantize_act_bounded_reference(x: torch.Tensor, live_rows: torch.Tensor):
    """x [1, R, K] -> (q, s) of ``quantize_act_reference`` for the rows below ``live_rows``; zero past it."""
    _, R, K = x.shape
    n = max(0, min(_host_int(live_rows), R))
    q = torch.zeros(1, R, K, dtype=torch.float8_e4m3fn, device=x.device)
    s = torch.zeros(1, K // TILE, -(-R // TILE) * TILE, dtype=torch.float32, device=x.device)
    qn, sn = quantize_act_reference(x[:, :n])
    q[:, :n], s[:, :, :sn.size(2)] = qn, sn
    return q, s


def quantize_act_dual_bounded_reference(x: torch.Tensor, live_rows: torch.Tensor, rowwise: bool = True):
    """x [1, R, K] -> (q, s, qT, sT) of ``quantize_act_dual_reference`` for the 128-row tiles below ``live_rows``;
    zero past it."""
    _, R, K = x.shape
    Rp = -(-R // TILE) * TILE
    n = max(0, min(_host_int(live_rows), R))
    _, _, qTn, sTn = quantize_act_dual_reference(x[:, :n], rowwise=False)
    qT = torch.zeros(1, K, Rp, dtype=torch.float8_e4m3fn, device=x.device)
    sT = torch.zeros(1, Rp // TILE, K, dtype=torch.float32, device=x.device)
    qT[:, :, :qTn.size(2)], sT[:, :sTn.size(1)] = qTn, sTn
    q, s = quantize_act_bounded_reference(x, live_rows) if rowwise else (None, None)
    return q, s, qT, sT


def block_fp8_gemm_packed_reference(a, sa, b, sb, bias=None, aux=None, aux2=None, epilogue=EPI_NONE, act='silu', *,
                                    row_counts, b_group_map):
    """One block-mapped ``block_fp8_gemm`` launch: a [R, K] (sa [1, K / 128, R]); the row tiles of expert e are the
    reference GEMM on expert e's operand, rows at or past a tile's ``row_counts`` are zero.  Results (and aux) are
    [R, *]."""
    R = a.size(0)
    rc, bm = row_counts.cpu().long(), b_group_map.cpu().long()
    N = b.size(1)
    widths = [N // 2] * 3 if epilogue == EPI_GLU else [2 * N] if epilogue == EPI_GLU_BWD else [N]
    outs = [torch.zeros(R, w, dtype=torch.bfloat16, device=a.device) for w in widths]
    zero = torch.zeros((), dtype=torch.bfloat16, device=a.device)
    for e in sorted(set(bm[rc > 0].tolist())):
        tiles = torch.nonzero((bm == e) & (rc > 0)).flatten()
        rows = (tiles.view(-1, 1) * TILE + torch.arange(TILE)).flatten().to(a.device)
        side = None if aux is None else aux.reshape(R, -1)[rows].unsqueeze(0)
        side2 = None if aux2 is None else aux2.reshape(R, -1)[rows].unsqueeze(0)
        res = block_fp8_gemm_reference(a[rows].unsqueeze(0), sa[:, :, rows], b[e:e + 1], sb[e:e + 1],
                                       None if bias is None else bias.reshape(b.size(0), -1)[e:e + 1],
                                       side, side2, epilogue, act)
        live = (torch.arange(TILE).view(1, -1) < rc[tiles].view(-1, 1)).flatten().to(a.device)
        for o, t in zip(outs, res):
            o[rows] = torch.where(live.view(-1, 1), t[0], zero)
    return outs


def wgrad_gemm_ragged_reference(aT, saT, bT, sbT, k_offsets, split: Optional[int] = None):
    """One ragged-K ``wgrad_gemm`` launch: aT [1, M, R], bT [1, N, R] (scales [1, R / 128, *]); expert e is the
    reference weight-gradient GEMM over the tokens from k_offsets[e] to k_offsets[e + 1] (zeros if none), [E, M, N]."""
    ko = [int(v) for v in k_offsets.cpu().tolist()]
    M, N = aT.size(1), bT.size(1)
    d = torch.zeros(len(ko) - 1, M, N, dtype=torch.bfloat16, device=aT.device)
    for e, (k0, k1) in enumerate(zip(ko[:-1], ko[1:])):
        if k1 > k0:
            kb = slice(k0 // TILE, k1 // TILE)
            d[e] = wgrad_gemm_reference(aT[:, :, k0:k1], saT[:, kb], bT[:, :, k0:k1], sbT[:, kb])[0][0]
    return [d] if not split else [d[..., :split].contiguous(), d[..., split:].contiguous()]


def _check(ok: bool, msg: str):
    if not ok:
        raise ValueError(msg)


# ------------------------------------------------------------------------------------------------------------------
# kernels
# ------------------------------------------------------------------------------------------------------------------
def _native(x: torch.Tensor, what: str) -> bool:
    if x.is_cuda and backend.has_ext():
        return True
    if x.is_cuda and not backend.allow_fallback():
        raise RuntimeError('%s: the native extension is required on a GPU' % what)
    return False


def quantize_act(x: torch.Tensor, live_rows: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """x [G, R, K] bf16 -> (q, s).  One launch of ``block_fp8_quantize_act_kernel`` on a GPU.
    ``live_rows`` (one-element device int32, the packed layout's ``used_rows``): x is one packed buffer ([R, K] or
    [1, R, K]); rows at or past the bound are neither read nor written, and the result is [1, R, K]."""
    if live_rows is not None:
        x = x.reshape(1, -1, x.size(-1))
    if _native(x, 'block_fp8.quantize_act'):
        backend.count_launch()
        if live_rows is None:
            return backend.require_ext().block_fp8_quantize_act(x.contiguous())
        return backend.require_ext().block_fp8_quantize_act(x.contiguous(), live_rows.to(torch.int32))
    return quantize_act_reference(x) if live_rows is None else quantize_act_bounded_reference(x, live_rows)


def quantize_act_dual(x: torch.Tensor, rowwise: bool = True, live_rows: Optional[torch.Tensor] = None):
    """x [G, R, K] bf16 -> (q, s, qT, sT): the row-wise operand of ``quantize_act`` (bit for bit; None, None unless
    ``rowwise``) and the column-wise operand of the weight-gradient GEMM, from one launch of
    ``block_fp8_quantize_dual_kernel`` on a GPU.  ``live_rows``: as for ``quantize_act``, a multiple of 128 (the
    128-row tiles at or past it are skipped)."""
    if live_rows is not None:
        x = x.reshape(1, -1, x.size(-1))
    if _native(x, 'block_fp8.quantize_act_dual'):
        backend.count_launch()
        ext = backend.require_ext()
        out = (ext.block_fp8_quantize_act_dual(x.contiguous(), bool(rowwise)) if live_rows is None else
               ext.block_fp8_quantize_act_dual(x.contiguous(), bool(rowwise), live_rows.to(torch.int32)))
        return tuple(out) if rowwise else (None, None, out[0], out[1])
    if live_rows is not None:
        return quantize_act_dual_bounded_reference(x, live_rows, rowwise)
    return quantize_act_dual_reference(x, rowwise)


def wgrad_gemm(aT, saT, bT, sbT, split: Optional[int] = None, max_ctas: int = 0,
               k_offsets: Optional[torch.Tensor] = None):
    """``aT [G, M, Kp] @ bT [G, N, Kp]^T`` over the padded token dimension, both operands column-wise (scales
    ``[G, Kp / 128, rows]``) -> ``[d bf16 [G, M, N]]``, or with ``split = H`` (N = 2H) ``[d[..., :H], d[..., H:]]`` as two
    contiguous tensors written by the one launch.
    ``k_offsets`` (device int32 [E + 1], the packed layout's ``seg_off``): ragged K over single packed operands
    ``[1, *, R]``; ``d[e]`` reduces over the tokens ``k_offsets[e]`` to ``k_offsets[e + 1]`` (zero if there are none)."""
    if _native(aT, 'block_fp8.wgrad_gemm'):
        backend.count_launch()
        if k_offsets is None:
            return backend.require_ext().block_fp8_wgrad_gemm(aT, saT, bT, sbT, int(split or 0), int(max_ctas))
        return backend.require_ext().block_fp8_wgrad_gemm(aT, saT, bT, sbT, int(split or 0), int(max_ctas),
                                                          k_offsets.to(torch.int32).contiguous())
    if k_offsets is not None:
        return wgrad_gemm_ragged_reference(aT, saT, bT, sbT, k_offsets, split)
    return wgrad_gemm_reference(aT, saT, bT, sbT, split)


def quantize_weight(w: torch.Tensor):
    """w [G, R, C] bf16 -> (q, s, qT, sT), both orientations from one launch."""
    if _native(w, 'block_fp8.quantize_weight'):
        backend.count_launch()
        return tuple(backend.require_ext().block_fp8_quantize_weight(w.contiguous()))
    return quantize_weight_reference(w)


def quantize_glu_weight(w1: torch.Tensor, w2: torch.Tensor):
    """Gate / up weights [G, M, H] bf16 -> (qcat, scat, qglu, sglu) from one launch."""
    if _native(w1, 'block_fp8.quantize_glu_weight'):
        backend.count_launch()
        return tuple(backend.require_ext().block_fp8_quantize_glu_weight(w1.contiguous(), w2.contiguous()))
    return quantize_glu_weight_reference(w1, w2)


def zero_rows_past(t: torch.Tensor, row_counts: torch.Tensor) -> torch.Tensor:
    """t [G, R, ...] with rows r >= row_counts[g] of group g set to zero (whatever they held, NaN included)."""
    live = torch.arange(t.size(1), device=t.device).view(1, -1) < row_counts.to(t.device).view(-1, 1).long()
    return torch.where(live.view(*live.shape, *([1] * (t.dim() - 2))), t, torch.zeros((), dtype=t.dtype, device=t.device))


def block_fp8_gemm(a, sa, b, sb, bias=None, aux=None, aux2=None, epilogue: int = EPI_NONE, act: str = 'silu',
                   max_ctas: int = 0, row_counts: Optional[torch.Tensor] = None,
                   b_group_map: Optional[torch.Tensor] = None):
    """``epilogue(a [G, M, K] @ b [G, N, K]^T)`` -> a list of bf16 results (see csrc/bindings.cpp: block_fp8_gemm).
    ``row_counts`` (device int32 [G], optional): rows r >= row_counts[g] of every result are zero, and the kernel skips
    the tiles that start at or past the count (dropless prefill).
    ``b_group_map`` (device int32 [R / 128], the packed layout's ``block_expert``, with ``row_counts`` = ``block_rows``):
    ``a`` is one packed buffer ([R, K] or [1, R, K], scales [1, K / 128, R]) whose row tile m is multiplied by expert
    ``b_group_map[m]``'s operand, scales and bias; ``aux``, ``aux2`` and the results are [R, *].  Rows of a tile at or
    past its count are zero; tiles with no live rows are neither read nor written."""
    if b_group_map is not None:
        _check(row_counts is not None, "block_fp8_gemm: a block-mapped launch needs the row tiles' row_counts")
        a = a.reshape(-1, a.size(-1))
        aux = None if aux is None else aux.reshape(a.size(0), -1)
        aux2 = None if aux2 is None else aux2.reshape(a.size(0), -1)
    if _native(a, 'block_fp8_gemm'):
        backend.count_launch()
        if bias is not None:
            bias = bias.reshape(b.size(0), b.size(1)).to(torch.bfloat16).contiguous()
        args = (a, sa, b, sb, bias, aux, aux2, int(epilogue), ACT_CODES[act], int(max_ctas))
        if row_counts is None:
            return backend.require_ext().block_fp8_gemm(*args)
        if b_group_map is None:
            return backend.require_ext().block_fp8_gemm(*args, row_counts.to(torch.int32).contiguous())
        return backend.require_ext().block_fp8_gemm(*args, row_counts.to(torch.int32).contiguous(),
                                                    b_group_map.to(torch.int32).contiguous())
    if b_group_map is not None:
        return block_fp8_gemm_packed_reference(a, sa, b, sb, bias, aux, aux2, epilogue, act, row_counts=row_counts,
                                               b_group_map=b_group_map)
    out = block_fp8_gemm_reference(a, sa, b, sb, bias, aux, aux2, epilogue, act)
    return out if row_counts is None else [zero_rows_past(t, row_counts) for t in out]


_WEIGHT_CACHE = {}


def _cached(tensors, make):
    """``make()`` cached like ``ops.mx.mx_weight``: valid until the next optimizer step or in-place change of any of
    ``tensors`` (stamp ``(w._version, gemm._FP8_STEP)``, weakly anchored to the parameter)."""
    import weakref
    from . import gemm as _gemm
    _gemm._ensure_step_hook()
    anchors = tuple(w._base if w._base is not None else w for w in tensors)
    key = tuple((id(a), w.data_ptr(), tuple(w.shape), tuple(w.stride())) for a, w in zip(anchors, tensors))
    stamp = (tuple(w._version for w in tensors), _gemm._FP8_STEP[0])
    hit = _WEIGHT_CACHE.get(key)
    if hit is not None and hit[0] == stamp and all(r() is a for r, a in zip(hit[2], anchors)):
        return hit[1]
    val = make()
    if len(_WEIGHT_CACHE) > 256:
        for k in [k for k, v in _WEIGHT_CACHE.items() if any(r() is None for r in v[2])]:
            del _WEIGHT_CACHE[k]
    _WEIGHT_CACHE[key] = (stamp, val, tuple(weakref.ref(a) for a in anchors))
    return val


def weight(w: torch.Tensor):
    """Cached (q, s, qT, sT) of a weight [G, R, C]."""
    return _cached((w,), lambda: quantize_weight(w.detach()))


def glu_weight(w1: torch.Tensor, w2: torch.Tensor):
    """Cached (qcat, scat, qglu, sglu) of the gate / up weights [G, M, H]."""
    return _cached((w1, w2), lambda: quantize_glu_weight(w1.detach(), w2.detach()))


# ------------------------------------------------------------------------------------------------------------------
# expert FFNs
# ------------------------------------------------------------------------------------------------------------------
def can_use_block_fp8(x: torch.Tensor, *weights: torch.Tensor) -> bool:
    """bf16 tensors on a GPU with the native extension, and every weight dimension a multiple of 128."""
    return (x.is_cuda and backend.has_ext() and x.dtype == torch.bfloat16 and x.dim() == 3 and x.size(-1) % TILE == 0 and
            all(w.dtype == torch.bfloat16 and w.dim() == 3 and w.size(1) % TILE == 0 and w.size(2) % TILE == 0 for w in weights))


class FusedReluFFNBlockFp8(torch.autograd.Function):
    """ReLU expert FFN ``relu(x @ w1^T + b1) @ w2 + b2`` (x [E, C, M], w1 [E, H, M], w2 [E, H, Mo]: the layout of
    models/experts/ffn.py) with block-scaled e4m3 forward and data-gradient GEMMs.  The weight-gradient GEMMs are 16-bit on
    the master weights, or with ``wgrad`` block-scaled e4m3 on column-wise operands: the forward then saves ``x^T`` in
    e4m3 instead of bf16 ``x``, the backward quantises ``dy`` and ``dh`` in both orientations from one read each and
    ``act^T`` column-wise only (``act`` stays bf16 for the ReLU-backward epilogue).  Same structure as
    ``ops.mx.FusedReluFFNMx``.

    ``layout`` (:class:`tutel_b200.ops.packed.PackedLayout`): ``x [R, M]`` is an expert-packed buffer and so is the
    result.  Every GEMM then runs block-mapped, every quantiser stops at ``used_rows``, the weight gradients reduce over
    each expert's segment (ragged K: the block GEMM with ``wgrad``, the 16-bit one otherwise) and the bias gradients are
    segmented column sums.  ``dy``'s padding rows must be zero, as the packed decode's backward leaves them."""

    @staticmethod
    def forward(ctx: Any, x, w1, b1, w2, b2, wgrad: bool = False, layout=None):
        pk, qk = _packed_kwargs(layout)
        q1, s1, _, _ = weight(w1)
        _, _, q2t, s2t = weight(w2)                                     # y = act @ W2: W2^T [Mo, H] K-major
        if wgrad:
            xq, xs, xqT, xsT = quantize_act_dual(x, **qk)
        else:
            xq, xs = quantize_act(x, **qk)
        act = block_fp8_gemm(xq, xs, q1, s1, bias=b1, epilogue=EPI_RELU, **pk)[0]
        y = block_fp8_gemm(*quantize_act(act, **qk), q2t, s2t, bias=b2, **pk)[0]
        ctx.save_for_backward(*((xqT, xsT) if wgrad else (x,)), w1, w2, act)
        ctx.has_b1, ctx.has_b2, ctx.wgrad, ctx.layout = b1 is not None, b2 is not None, wgrad, layout
        return y

    @staticmethod
    def backward(ctx: Any, dy: torch.Tensor):
        from . import gemm as _gemm
        if ctx.wgrad:
            xqT, xsT, w1, w2, act = ctx.saved_tensors
        else:
            x, w1, w2, act = ctx.saved_tensors
        layout = ctx.layout
        pk, qk = _packed_kwargs(layout)
        wk = {} if layout is None else dict(k_offsets=layout.seg_off)  # weight gradients: one K range per expert
        dy = dy.contiguous()
        q2, s2, _, _ = weight(w2)                                       # dh = dy @ W2^T: W2 [H, Mo] is K-major for it
        if ctx.wgrad:
            dq, ds, dqT, dsT = quantize_act_dual(dy, **qk)
        else:
            dq, ds = quantize_act(dy, **qk)
        dh = block_fp8_gemm(dq, ds, q2, s2, aux=act, epilogue=EPI_RELU_BWD, **pk)[0]
        dw2 = None
        if ctx.needs_input_grad[3]:                                     # dW2 = act^T dy: [H, C] [C, Mo]
            dw2 = (wgrad_gemm(*quantize_act_dual(act, rowwise=False, **qk)[2:], dqT, dsT, **wk)[0] if ctx.wgrad else
                   _gemm.raw_gemm(act, dy, a_mn=True, b_mn=True, **wk))
        if ctx.wgrad:
            del dqT, dsT                                                # lower the backward's peak memory
        db2 = _column_sums(dy, layout) if ctx.has_b2 and ctx.needs_input_grad[4] else None
        dx = dw1 = None
        if ctx.wgrad and (ctx.needs_input_grad[0] or ctx.needs_input_grad[1]):
            hq, hs, hqT, hsT = quantize_act_dual(dh, rowwise=ctx.needs_input_grad[0], **qk)
        elif ctx.needs_input_grad[0]:
            hq, hs = quantize_act(dh, **qk)
        if ctx.needs_input_grad[0]:
            _, _, q1t, s1t = weight(w1)                                 # dx = dh @ W1: W1^T [M, H] K-major
            dx = block_fp8_gemm(hq, hs, q1t, s1t, **pk)[0]
        if ctx.needs_input_grad[1]:                                     # dW1 = dh^T x: [H, C] [C, M]
            dw1 = (wgrad_gemm(hqT, hsT, xqT, xsT, **wk)[0] if ctx.wgrad else
                   _gemm.raw_gemm(dh, x, a_mn=True, b_mn=True, **wk))
        db1 = _column_sums(dh, layout) if ctx.has_b1 and ctx.needs_input_grad[2] else None
        return dx, dw1, db1, dw2, db2, None, None


def _packed_kwargs(layout):
    """Keyword arguments of the packed launch modes (block-mapped GEMMs, bounded quantisers), or two empty dicts."""
    if layout is None:
        return {}, {}
    return dict(row_counts=layout.block_rows, b_group_map=layout.block_expert), dict(live_rows=layout.used_rows)


def _column_sums(t: torch.Tensor, layout) -> torch.Tensor:
    """Bias gradient: [G, T, N] -> [G, N] column sums, or per expert segment of a packed [R, N]."""
    from . import gemm as _gemm
    if layout is None:
        return _gemm.column_sums(t)
    from .packed import segment_colsum
    return segment_colsum(t, layout)


def fused_relu_ffn_block_fp8(x, w1, b1, w2, b2, wgrad: bool = False, layout=None):
    b1 = None if b1 is None else b1.reshape(w1.size(0), -1)
    b2 = None if b2 is None else b2.reshape(w2.size(0), -1)
    return FusedReluFFNBlockFp8.apply(x, w1, b1, w2, b2, wgrad, layout)


class FusedGLUFFNBlockFp8(torch.autograd.Function):
    """SwiGLU expert ``(act(x @ W1) * (x @ W2)) @ W3`` (w1, w2 [E, M, H], w3 [E, H, Mo]: the layout of
    models/experts/llama_ffn.py) with block-scaled e4m3 forward and data-gradient GEMMs:

    * forward: one GLU launch on the interleaved gate / up copy writes h and the 16-bit g and u; then the down projection;
    * backward: ``dy @ W3^T`` with the GLU-backward epilogue writes ``[dg du]`` side by side into one ``[E, C, 2H]``
      buffer, and ``dx = [dg du] @ [W1 W2]^T`` is one GEMM with K = 2H on the same quantised blocks as the forward;
      ``dW1``, ``dW2`` and ``dW3`` are 16-bit GEMMs on the master weights;
    * with ``wgrad`` the weight gradients are block-scaled e4m3 GEMMs on column-wise operands: the forward quantises x and
      h in both orientations and saves ``x^T`` and ``h^T`` in e4m3 instead of bf16 ``x`` and ``h``; the backward does
      the same for dy and ``[dg du]``, and ``[dW1 | dW2] = x^T [dg du]`` is one launch writing both gradients;
    * ``layout`` (a ``PackedLayout``): ``x [R, M]`` and the result are expert-packed buffers, and the launches run in the
      packed modes, as in :class:`FusedReluFFNBlockFp8`."""

    @staticmethod
    def forward(ctx: Any, x, w1, w2, w3, act: str, wgrad: bool = False, layout=None):
        pk, qk = _packed_kwargs(layout)
        _, _, qglu, sglu = glu_weight(w1, w2)
        _, _, q3t, s3t = weight(w3)
        quant = quantize_act_dual if wgrad else quantize_act
        xs = quant(x, **qk)
        h, g, u = block_fp8_gemm(xs[0], xs[1], qglu, sglu, epilogue=EPI_GLU, act=act, **pk)
        hs = quant(h, **qk)
        y = block_fp8_gemm(hs[0], hs[1], q3t, s3t, **pk)[0]
        ctx.act, ctx.wgrad, ctx.layout = act, wgrad, layout
        if wgrad:
            ctx.save_for_backward(xs[2], xs[3], w1, w2, w3, g, u, hs[2], hs[3])
        else:
            ctx.save_for_backward(x, w1, w2, w3, g, u, h)
        return y

    @staticmethod
    def backward(ctx: Any, dy: torch.Tensor):
        from . import gemm as _gemm
        if ctx.wgrad:
            xqT, xsT, w1, w2, w3, g, u, hqT, hsT = ctx.saved_tensors
        else:
            x, w1, w2, w3, g, u, h = ctx.saved_tensors
        layout = ctx.layout
        pk, qk = _packed_kwargs(layout)
        wk = {} if layout is None else dict(k_offsets=layout.seg_off)  # weight gradients: one K range per expert
        dy = dy.contiguous()
        H = g.size(-1)
        q3, s3, _, _ = weight(w3)                                       # dh = dy @ W3^T: W3 [H, Mo] is K-major for it
        ds = quantize_act_dual(dy, **qk) if ctx.wgrad else quantize_act(dy, **qk)
        dgu = block_fp8_gemm(ds[0], ds[1], q3, s3, aux=g, aux2=u, epilogue=EPI_GLU_BWD, act=ctx.act, **pk)[0]
        dx = dw1 = dw2 = dw3 = None
        if ctx.wgrad:
            if ctx.needs_input_grad[3]:                                 # dW3 = h^T dy: [H, C] [C, Mo]
                dw3 = wgrad_gemm(hqT, hsT, ds[2], ds[3], **wk)[0]
            del ds, hqT, hsT                                            # lower the backward's peak memory
            need_w12 = ctx.needs_input_grad[1] or ctx.needs_input_grad[2]
            gs = None
            if ctx.needs_input_grad[0] or need_w12:
                gs = quantize_act_dual(dgu, rowwise=ctx.needs_input_grad[0], **qk)
            if need_w12:                                                # [dW1 | dW2] = x^T [dg du]: [M, C] [C, 2H]
                dw1, dw2 = wgrad_gemm(xqT, xsT, gs[2], gs[3], split=H, **wk)
                dw1 = dw1 if ctx.needs_input_grad[1] else None
                dw2 = dw2 if ctx.needs_input_grad[2] else None
            if ctx.needs_input_grad[0]:
                qcat, scat, _, _ = glu_weight(w1, w2)
                dx = block_fp8_gemm(gs[0], gs[1], qcat, scat, **pk)[0]
            return dx, dw1, dw2, dw3, None, None, None
        dg, du = dgu[..., :H], dgu[..., H:]
        dw3 = _gemm.raw_gemm(h, dy, a_mn=True, b_mn=True, **wk) if ctx.needs_input_grad[3] else None
        dw1 = _gemm.raw_gemm(x, dg, a_mn=True, b_mn=True, **wk) if ctx.needs_input_grad[1] else None
        dw2 = _gemm.raw_gemm(x, du, a_mn=True, b_mn=True, **wk) if ctx.needs_input_grad[2] else None
        if ctx.needs_input_grad[0]:
            qcat, scat, _, _ = glu_weight(w1, w2)
            dx = block_fp8_gemm(*quantize_act(dgu, **qk), qcat, scat, **pk)[0]
        return dx, dw1, dw2, dw3, None, None, None


def fused_glu_ffn_block_fp8(x, w1, w2, w3, act='silu', wgrad: bool = False, layout=None):
    return FusedGLUFFNBlockFp8.apply(x, w1, w2, w3, act, wgrad, layout)


# ------------------------------------------------------------------------------------------------------------------
# stored block-fp8 experts (no 16-bit master weights): the checkpoint format of DeepSeek-V3, Kimi-K2, GLM-4.5, Moonlight
# and Qwen3-FP8, and inference on it
# ------------------------------------------------------------------------------------------------------------------
# Checkpoint orientation, stacked over E local experts (HF ``{gate,up,down}_proj.weight`` / ``.weight_scale_inv``,
# ``w ~= q * s`` per 128 x 128 block): gate, up e4m3 [E, H, M] + [E, H / 128, M / 128]; down e4m3 [E, M, H] +
# [E, M / 128, H / 128].  Stored layout (what the block GEMM's forward reads): qglu [E, 2H, M] + sglu [E, 2H / 64, M / 128]
# (gate / up interleaved every 64 rows, as ``quantize_glu_weight`` writes them) and q3t = down, s3t = down's scales.
def export_glu_weights(w1: torch.Tensor, w2: torch.Tensor, w3: torch.Tensor):
    """bf16 SwiGLU weights in the ``llama_ffn`` layout (w1, w2 [E, M, H], w3 [E, H, M]) -> the six checkpoint tensors
    (gate, gate_scale, up, up_scale, down, down_scale), quantised per 128 x 128 block by ``quantize_weight``.  A block is
    the same block in W and W^T, so ``load_glu_weights`` of the result is bit for bit the forward copy ``glu_weight(w1,
    w2)[2:]`` and ``weight(w3)[2:]`` that a ``fp8='block'`` layer of these weights reads."""
    for name, w in (('w1', w1), ('w2', w2), ('w3', w3)):
        _check(w.dtype == torch.bfloat16 and w.dim() == 3, 'export_glu_weights: %s must be a bf16 [E, *, *] tensor (got %s %s)'
               % (name, w.dtype, tuple(w.shape)))
    _check(w1.shape == w2.shape and w3.shape == (w1.size(0), w1.size(2), w1.size(1)),
           'export_glu_weights: w1, w2 [E, M, H] and w3 [E, H, M] expected (got %s, %s, %s)'
           % (tuple(w1.shape), tuple(w2.shape), tuple(w3.shape)))
    _, _, gate, gate_s = quantize_weight(w1.detach())
    _, _, up, up_s = quantize_weight(w2.detach())
    _, _, down, down_s = quantize_weight(w3.detach())
    return gate, gate_s, up, up_s, down, down_s


def load_glu_weights(gate, gate_scale, up, up_scale, down, down_scale):
    """The six checkpoint tensors (see ``export_glu_weights``) -> the stored layout (qglu, sglu, q3t, s3t) on gate's device.
    Shapes and dtypes are checked; the interleave is one-time torch indexing."""
    def expect(t, dtype, shape, name):
        _check(isinstance(t, torch.Tensor) and t.dtype == dtype and tuple(t.shape) == tuple(shape),
               'load_fp8_block_weights: %s must be %s %s (got %s %s)' % (
                   name, dtype, tuple(shape), getattr(t, 'dtype', type(t)), tuple(getattr(t, 'shape', ()))))
    _check(isinstance(gate, torch.Tensor) and gate.dim() == 3, 'load_fp8_block_weights: gate must be e4m3 [E, H, M]')
    E, H, M = gate.shape
    _check(H % TILE == 0 and M % TILE == 0, 'load_fp8_block_weights: H and M must be multiples of 128 (got %d, %d)' % (H, M))
    e4m3 = torch.float8_e4m3fn
    expect(gate, e4m3, (E, H, M), 'gate')
    expect(up, e4m3, (E, H, M), 'up')
    expect(down, e4m3, (E, M, H), 'down')
    expect(gate_scale, torch.float32, (E, H // TILE, M // TILE), 'gate_scale')
    expect(up_scale, torch.float32, (E, H // TILE, M // TILE), 'up_scale')
    expect(down_scale, torch.float32, (E, M // TILE, H // TILE), 'down_scale')
    dev = gate.device
    qglu = interleave_glu_reference(gate.view(torch.uint8), up.to(dev).view(torch.uint8)).view(e4m3)
    sglu = interleave_glu_reference(gate_scale.to(dev).repeat_interleave(2, dim=1),
                                    up_scale.to(dev).repeat_interleave(2, dim=1), rows_per=1)
    return qglu.contiguous(), sglu.contiguous(), down.to(dev).contiguous(), down_scale.to(dev).contiguous()


def can_use_stored_glu(x: torch.Tensor) -> bool:
    """Inputs the stored block-fp8 SwiGLU expert runs on: bf16 [E, rows, M] (on a GPU or, through the references, on
    CPU).  Nothing is cast: other dtypes are refused by the caller."""
    return x.dtype == torch.bfloat16 and x.dim() == 3


SKINNY_SMEM_LIMIT = 100 * 1024       # staged bf16 x rows (8 M bytes) + the 2 KB hidden slice: two blocks per SM


def can_use_skinny_glu_ffn_block_fp8(x: torch.Tensor) -> bool:
    """``skinny_glu_ffn_block_fp8`` covers up to 64 rows per expert and M up to 12544 (csrc/skinny_gemm.cu)."""
    return can_use_stored_glu(x) and x.size(1) <= 64 and 8 * x.size(2) + 2048 <= SKINNY_SMEM_LIMIT


def skinny_glu_ffn_block_fp8_reference(x, qglu, sglu, q3t, s3t, row_counts, act='silu'):
    """fp32 composition on the dequantised stored weights; rows past the counts are zero.  The CPU path of the kernel."""
    G, R, _ = x.shape
    H = qglu.size(1) // 2
    t = (x.float() @ dequantize_weight(qglu, sglu).transpose(1, 2)).view(G, R, H // 64, 2, 64)
    g, u = t[:, :, :, 0].reshape(G, R, H), t[:, :, :, 1].reshape(G, R, H)
    y = (_act(g, act)[0] * u) @ dequantize_weight(q3t, s3t).transpose(1, 2)
    if row_counts is not None:
        y = zero_rows_past(y, row_counts)
    return y.to(x.dtype)


def skinny_glu_ffn_block_fp8(x, qglu, sglu, q3t, s3t, row_counts, act='silu'):
    """y[g, r] = (act(x @ W1) * (x @ W2)) @ W3 for r < row_counts[g] (other rows zero) on the stored block-scaled e4m3
    weights, in one weight-streaming launch of ``skinny_glu_ffn_block_fp8_kernel`` on a GPU (x stays bf16)."""
    if _native(x, 'block_fp8.skinny_glu_ffn_block_fp8'):
        backend.count_launch(2)          # zero-fill of the fp32 accumulator + the kernel
        y = backend.require_ext().skinny_glu_ffn_block_fp8(x.contiguous(), qglu, sglu, q3t, s3t, row_counts, ACT_CODES[act])
        return y.to(x.dtype)
    return skinny_glu_ffn_block_fp8_reference(x, qglu, sglu, q3t, s3t, row_counts, act)


def glu_ffn_block_fp8_stored(x, qglu, sglu, q3t, s3t, act='silu', row_counts=None):
    """Inference forward of the stored experts: the launches of ``FusedGLUFFNBlockFp8.forward`` on the stored bytes (GLU
    GEMM, then the down projection), with the device row counts of dropless prefill when given."""
    h = block_fp8_gemm(*quantize_act(x.contiguous()), qglu, sglu, epilogue=EPI_GLU, act=act, row_counts=row_counts)[0]
    return block_fp8_gemm(*quantize_act(h), q3t, s3t, row_counts=row_counts)[0]
