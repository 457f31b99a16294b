"""References with per-element error bounds for the MX block-scaled fp8 kernels (csrc/gemm_mx.cu: mx_quantize_kernel,
mx_quantize_transpose_kernel, mx_gemm_kernel).  Plain torch: runs on the CPU or the GPU.

Quantiser (exact).  Written from the number format, not from the kernel's bit trick:

* a block's exponent e is the smallest integer with ``amax <= 448 * 2^e``, found exactly in fp64, then clamped to
  [-126, 126]; a block whose largest non-NaN magnitude is 0 gets e = -127 (scale byte 0).  NaN elements do not take
  part in the maximum, so a NaN leaves its 31 neighbours their own scale;
* elements ``q = e4m3_rn_satfinite(x * 2^-e)``: +-inf saturate to +-448, NaN stays NaN;
* scale bytes ``e + 127`` at ``sf[g][k // 128][r // 128][(r % 32) * 16 + ((r % 128) // 32) * 4 + (k % 128) // 32]``
  (csrc/gemm_mx.h), computed here by index arithmetic; padded rows get byte 0.

GEMM (bounded).  ``ref_gemm`` computes ``epi(sum_k deq(a) deq(b) + bias)`` in fp64 from exactly the e4m3 bytes and scale
bytes the kernel read, with scale byte 0 decoded as 0 (what ``ue8m0_to_float`` does).  The kernel issues one fresh
``wgmma m64n128k32`` (scale-d = 0) per 32-element K block and folds it with ``fmaf(part, sa * sb, acc)``:

* each block's MMA error is the single-MMA e4m3 case: ``C_ACC[e4m3] * 2^-24 * S_kb`` (tests/gemm_reference.py) with
  S_kb = sum over the block of |a_k b_k| 2^(ea + eb);
* ``sa * sb`` is exact (a power of two in fp32's normal range, which gemm_mx.h requires), and each fold rounds once:
  at most 2^-24 * S per block, K / 32 in all, plus 2 for the second-order terms;
* bias: one more fp32 rounding, 2^-24 * |acc + bias|; ReLU is 1-Lipschitz and needs no term of its own;
* fp32 subnormals: one subnormal spacing per fold, (K / 32 + 1) * 2^-149;
* the bf16 rounding of the output: half an ulp at |ref| + the rest of the bound (the fp32 value may sit one binade up).

So ``|d - ref| <= half_ulp_bf16 + (C_ACC[e4m3] + K/32 + 2) * 2^-24 * S + 2^-24 |pre| + (K/32 + 1) * 2^-149``.  The
ReLU-backward mask comes from ``aux`` and is checked exactly: the output is exactly 0 wherever ``aux > 0`` is false
(+-0 and NaN included).

C_ACC[e4m3] = 32768 is not loose for this kernel.  The tensor core aligns a block's products to the largest before it
adds them, so when one product dominates its block, the others lose their low bits: the normalised error of a single
32-deep MMA exceeds 8192 on operands whose elements span e4m3's whole range.  32768 * 2^-24 = 2^-9 is also the largest
relative error of a bf16 rounding, so no elementwise bound that the tensor core passes can reject a kernel that rounds
each block's partial sum to bf16.  ``check_exact`` does: on exactly representable operands every partial sum is exact
in fp32, and the output must be the bf16 rounding of the exact result, bit for bit.
"""
import math
from dataclasses import dataclass
from typing import Dict, Optional

import torch

from gemm_reference import C_ACC, U, half_ulp

BLOCK = 32
E4M3_MAX = 448.0
C_MMA = C_ACC[torch.float8_e4m3fn]
TINY = 2.0 ** -149
EPI_NONE, EPI_RELU, EPI_RELU_BWD = 0, 1, 2
# largest normalised errors seen by check(), keyed by the text before the first ':' of its `what`: (|err| - output
# rounding) / rest of the bound (<= 1); and under 'acc', (|err| - every term but the MMA's) / (2^-24 S), which
# C_MMA = C_ACC[e4m3] must cover
OBSERVED: Dict[str, float] = {}


# ------------------------------------------------------------------------------------------------------------------
# quantiser
# ------------------------------------------------------------------------------------------------------------------
def pow2(e: torch.Tensor) -> torch.Tensor:
    """2^e in fp64 for integer-valued e in [-1022, 1023], built from the exponent field (exact on every device; torch's
    ldexp multiplies by pow(2, e), which is not exact for every e on every device)."""
    return ((e.long() + 1023) << 52).view(torch.float64)


def block_exponents(x: torch.Tensor) -> torch.Tensor:
    """Exponents [.., K / 32] (int32) of the 32-element blocks along the last dim of a 16-bit tensor."""
    a = x.double().abs()
    a = torch.where(torch.isnan(a), torch.zeros_like(a), a)
    amax = a.reshape(*x.shape[:-1], x.shape[-1] // BLOCK, BLOCK).amax(-1)
    e = torch.ceil(torch.log2(amax / E4M3_MAX)).clamp(-200, 200)          # +-inf of log2(0) / log2(inf) clamped
    e = torch.where(amax > E4M3_MAX * pow2(e), e + 1, e)                   # log2 is not exact: make e the smallest
    e = torch.where(amax <= E4M3_MAX * pow2(e - 1), e - 1, e)             # integer with amax <= 448 * 2^e
    e = e.clamp(-126, 126)
    return torch.where(amax == 0, torch.full_like(e, -127), e).to(torch.int32)


def e4m3_rn_satfinite(v: torch.Tensor) -> torch.Tensor:
    """fp64 -> e4m3 bytes, round to nearest even, saturating at +-448 (torch's own conversion gives NaN above 464).
    The fp64 -> fp32 step is exact for every |v| >= 2^-126, and smaller values round to +-0 either way."""
    return v.clamp(-E4M3_MAX, E4M3_MAX).float().to(torch.float8_e4m3fn).view(torch.uint8)


def scale_offsets(G: int, R: int, K: int, device=None) -> torch.Tensor:
    """Byte offset [G, R, K / 32] (int64) of each block's scale in the atom layout of csrc/gemm_mx.h."""
    RT, KB = (R + 127) // 128, K // 128
    g = torch.arange(G, device=device).view(G, 1, 1)
    r = torch.arange(R, device=device).view(1, R, 1)
    k = torch.arange(K // BLOCK, device=device).view(1, 1, -1) * BLOCK
    return ((g * KB + k // 128) * RT + r // 128) * 512 + (r % 32) * 16 + ((r % 128) // 32) * 4 + (k % 128) // 32


def pack(e: torch.Tensor) -> torch.Tensor:
    """Exponents [G, R, K / 32] -> flat scale bytes; rows padded to a multiple of 128 carry byte 0."""
    G, R, KB32 = e.shape
    RT = (R + 127) // 128
    sf = torch.zeros(G * (KB32 // 4) * RT * 512, dtype=torch.uint8, device=e.device)
    sf[scale_offsets(G, R, KB32 * BLOCK, e.device).reshape(-1)] = (e + 127).to(torch.uint8).reshape(-1)
    return sf


def scale_bytes(sf: torch.Tensor, G: int, R: int, K: int) -> torch.Tensor:
    """Scale bytes [G, R, K / 32] (int64) of an operand read from the flat atom array."""
    return sf.reshape(-1)[scale_offsets(G, R, K, sf.device)].long()


def quantize(x: torch.Tensor):
    """x [G, R, K] 16 bit -> (q bytes uint8 [G, R, K], sf uint8 flat, nan mask [G, R, K])."""
    G, R, K = x.shape
    assert K % 128 == 0
    e = block_exponents(x)
    inv = pow2(-e).repeat_interleave(BLOCK, -1)
    return e4m3_rn_satfinite(x.double() * inv), pack(e), torch.isnan(x)


def every_positive(dtype: torch.dtype, seed: int = 0) -> torch.Tensor:
    """[1, R, 128] of ``dtype`` in which block i has every positive finite value of the type, in turn, as its largest
    magnitude (at position i % 32, sign alternating), next to 31 random values no larger in magnitude."""
    top = {torch.bfloat16: 0x7F7F, torch.float16: 0x7BFF}[dtype]
    v = torch.arange(1, top + 1, dtype=torch.int32).to(torch.int16).view(dtype).float()
    n = -(-v.numel() // 4) * 4
    v = torch.cat([v, v[: n - v.numel()]])
    gen = torch.Generator().manual_seed(seed)
    x = (v.view(-1, 1) * (torch.rand(n, BLOCK, generator=gen) * 2 - 1)).to(dtype)
    x = torch.where(x.float().abs() > v.view(-1, 1), torch.zeros_like(x), x)
    i = torch.arange(n)
    x[i, i % BLOCK] = torch.where(i % 2 == 0, v, -v).to(dtype)
    return x.view(1, n // 4, 4 * BLOCK)


def special_values(dtype: torch.dtype, G: int = 2, R: int = 130, K: int = 256, seed: int = 0) -> torch.Tensor:
    """[G, R, K] random blocks spread over 2^+-20, with (when the shape has room for them) an all-zero block, -0, a
    block of subnormals holding the largest finite value, +-inf, NaN, an all-NaN block, and block maxima at 448 * 2^n
    and one ulp either side."""
    gen = torch.Generator().manual_seed(seed)
    spread = torch.exp2(torch.randint(-20, 20, (G, R, K // BLOCK, 1), generator=gen).float())
    x = (torch.randn(G, R, K // BLOCK, BLOCK, generator=gen) * spread).view(G, R, K).to(dtype)
    info = torch.finfo(dtype)
    rows = [(0, 0), (0, 1), (0, 2)] + [(G - 1, R - 1 - i) for i in range(5)]
    if R * G < 8:
        rows = [(g, r) for g in range(G) for r in range(R)][:8]
        rows += [rows[-1]] * (8 - len(rows))
    (z, s, n), extremes = rows[:3], rows[3:]
    x[z][:32] = 0
    x[z][32:64] = -0.0
    x[s][:32] = (info.tiny * torch.rand(32, generator=gen)).to(dtype)               # subnormals only
    x[s][40] = info.max
    x[s][64 + 3] = float('inf')
    x[s][96 + 5] = float('-inf')
    x[n][7] = float('nan')
    x[n][32:64] = float('nan')
    x[n][64 + 9] = -float('nan')
    t = torch.tensor([448.0 * 2.0 ** e for e in (-20, -3, 0, 1, 5)], dtype=dtype)
    bits = t.view(torch.int16)
    for (g, r), lo, mid, hi in zip(extremes, (bits - 1).view(dtype), t, (bits + 1).view(dtype)):
        x[g, r, 0], x[g, r, 32], x[g, r, 64], x[g, r, 96] = lo, mid, hi, -mid
    return x


def operands(G: int, M: int, N: int, K: int, spread: int = 30, positive: bool = False, seed: int = 0, device=None):
    """Random finite e4m3 operands a [G, M, K], b [G, N, K] (every finite magnitude, random sign unless ``positive``)
    and their scales, with exponents drawn from [-spread, spread] for every 32-element block."""
    gen = torch.Generator(device=device).manual_seed(seed)

    def one(rows):
        b = torch.randint(0, 0x7F, (G, rows, K), generator=gen, device=device, dtype=torch.int32)
        if not positive:
            b = b | (torch.randint(0, 2, b.shape, generator=gen, device=device, dtype=torch.int32) << 7)
        e = torch.randint(-spread, spread + 1, (G, rows, K // BLOCK), generator=gen, device=device, dtype=torch.int32)
        return b.to(torch.uint8).view(torch.float8_e4m3fn), pack(e)

    aq, sfa = one(M)
    bq, sfb = one(N)
    return aq, sfa, bq, sfb


def bias_aux(acc: torch.Tensor, seed: int = 1):
    """(bias bf16 [G, N] of the columns' typical magnitude, aux bf16 [G, M, N] with rows of +0 and -0 and NaN entries)
    for the epilogues of a GEMM whose plain result is ``acc``."""
    G, M, N = acc.shape
    gen = torch.Generator(device=acc.device).manual_seed(seed)
    scale = acc.abs().median(dim=1).values.float()
    bias = (torch.randn(G, N, generator=gen, device=acc.device) * scale).bfloat16()
    aux = torch.randn(G, M, N, generator=gen, device=acc.device).bfloat16()
    aux[:, ::5] = 0.0
    aux[:, 1::5] = -0.0
    aux[:, 2::7, ::3] = float('nan')
    return bias, aux


def check_quantized(what: str, q: torch.Tensor, sf: torch.Tensor, x: torch.Tensor) -> None:
    """Bit-exact check of a quantiser's output for x [G, R, K].  NaN elements must be NaN (0x7f or 0xff): which sign
    the hardware's satfinite conversion writes for a negative NaN is not part of the contract."""
    wq, wsf, nan = quantize(x)
    got = q.reshape(x.shape).view(torch.uint8)
    assert sf.numel() == wsf.numel(), '%s: %d scale bytes, expected %d' % (what, sf.numel(), wsf.numel())
    bad = sf.reshape(-1) != wsf
    if bool(bad.any()):
        i = int(bad.nonzero()[0])
        raise AssertionError('%s: %d of %d scale bytes differ; first at byte %d: kernel=0x%02x reference=0x%02x' % (
            what, int(bad.sum()), bad.numel(), i, int(sf.reshape(-1)[i]), int(wsf[i])))
    bad = torch.where(nan, (got & 0x7F) != 0x7F, got != wq)
    if bool(bad.any()):
        i = tuple(int(v) for v in bad.nonzero()[0])
        raise AssertionError('%s: %d of %d e4m3 bytes differ; first at %s: x=%r kernel=0x%02x reference=0x%02x' % (
            what, int(bad.sum()), bad.numel(), i, float(x[i]), int(got[i]), int(wq[i])))


# ------------------------------------------------------------------------------------------------------------------
# GEMM
# ------------------------------------------------------------------------------------------------------------------
def dequantize(q: torch.Tensor, sf: torch.Tensor) -> torch.Tensor:
    """fp64 values of an MX operand q [G, R, K] (e4m3 or its bytes); scale byte 0 decodes to 0."""
    G, R, K = q.shape
    b = scale_bytes(sf, G, R, K)
    s = torch.where(b == 0, torch.zeros_like(b, dtype=torch.float64), pow2(b - 127))
    v = q.view(torch.float8_e4m3fn).double()
    return (v.view(G, R, K // BLOCK, BLOCK) * s.unsqueeze(-1)).view(G, R, K)


@dataclass
class Ref:
    val: torch.Tensor                      # fp64 [G, M, N] after the epilogue
    acc: torch.Tensor                      # the bound but for the output rounding
    S: torch.Tensor                        # 2^-24 * sum_k |a_k b_k| 2^(ea + eb)
    other: torch.Tensor                    # every term of acc but the MMA's C_MMA * S
    zero: Optional[torch.Tensor] = None    # RELU_BWD: where the output must be exactly 0


def ref_gemm(aq, sfa, bq, sfb, bias=None, aux=None, epilogue=EPI_NONE) -> Ref:
    """Reference of one ``mx_gemm`` launch: a [G, M, K], b [G, N, K] (e4m3), bias bf16 [G, N], aux bf16 [G, M, N]."""
    A, B = dequantize(aq, sfa), dequantize(bq, sfb)
    K = A.size(2)
    acc = A @ B.transpose(1, 2)
    S = (A.abs() @ B.abs().transpose(1, 2)) * U
    pre = acc if bias is None else acc + bias.double().reshape(acc.size(0), 1, -1)
    other = (K // BLOCK + 2) * S + (U * pre.abs() if bias is not None else 0.0) + (K // BLOCK + 1) * TINY
    r = Ref(pre, C_MMA * S + other, S, other)
    if epilogue == EPI_RELU:
        r.val = pre.clamp_min(0)
    elif epilogue == EPI_RELU_BWD:
        r.zero = ~(aux.double() > 0)
        r.val = torch.where(r.zero, torch.zeros_like(pre), pre)
    return r


def check(what: str, d: torch.Tensor, r: Ref) -> float:
    """Assert ``d`` (bf16) is within the bound everywhere and exactly 0 where the ReLU-backward mask is off.  Returns
    the largest (|err| - output rounding) / rest of the bound, which is <= 1 when it passes."""
    assert d.dtype == torch.bfloat16 and d.shape == r.val.shape, (what, d.dtype, d.shape)
    x = d.double()
    if r.zero is not None:
        bad = r.zero & (x != 0)
        assert not bool(bad.any()), '%s: %d outputs not exactly 0 where aux > 0 is false; first at %s' % (
            what, int(bad.sum()), tuple(int(i) for i in bad.nonzero()[0]))
    err = (x - r.val).abs()
    err = torch.where(torch.isnan(x), torch.full_like(err, math.inf), err)
    rnd = half_ulp(r.val.abs() + r.acc, torch.bfloat16)
    live = torch.ones_like(err, dtype=torch.bool) if r.zero is None else ~r.zero
    norm = torch.where(live, (err - rnd).clamp_min(0) / r.acc, torch.zeros_like(err))
    accn = torch.where(live, (err - rnd - r.other) / r.S.clamp_min(1e-300), torch.full_like(err, -math.inf))
    worst = float(norm.max()) if norm.numel() else 0.0
    if accn.numel():
        key = what.split(':')[0]
        OBSERVED[key] = max(OBSERVED.get(key, -math.inf), worst)
        OBSERVED['acc'] = max(OBSERVED.get('acc', -math.inf), float(accn.max()))
    if not bool((err <= r.acc + rnd)[live].all()):
        i = tuple(int(v) for v in (norm == norm.max()).nonzero()[0])
        raise AssertionError('%s: %d of %d elements outside the bound; worst (err - rounding) / bound %.3g at %s: '
                             'kernel=%r reference=%r bound=%.3g' % (
                                 what, int(((err > r.acc + rnd) & live).sum()), int(live.sum()), worst, i,
                                 float(x[i]), float(r.val[i]), float(r.acc[i] + rnd[i])))
    return worst


def integer_operands(G: int, M: int, N: int, K: int, top: int = 8, spread: int = 2, seed: int = 0, device=None):
    """Operands on which every partial sum is exact in fp32: integers in [-top, top] (exact in e4m3 up to 16) and
    exponents in [-spread, spread]."""
    gen = torch.Generator(device=device).manual_seed(seed)

    def one(rows):
        v = torch.randint(-top, top + 1, (G, rows, K), generator=gen, device=device).float()
        e = torch.randint(-spread, spread + 1, (G, rows, K // BLOCK), generator=gen, device=device, dtype=torch.int32)
        return v.to(torch.float8_e4m3fn), pack(e)

    aq, sfa = one(M)
    bq, sfb = one(N)
    return aq, sfa, bq, sfb


def check_exact(what: str, d: torch.Tensor, aq, sfa, bq, sfb) -> None:
    """On operands from ``integer_operands`` the output must be the bf16 rounding of the exact product, bit for bit."""
    want = (dequantize(aq, sfa) @ dequantize(bq, sfb).transpose(1, 2)).float().bfloat16()
    bad = d.view(torch.int16) != want.view(torch.int16)
    if bool(bad.any()):
        i = tuple(int(v) for v in bad.nonzero()[0])
        raise AssertionError('%s: %d of %d outputs differ from the exact result (exact check); first at %s: kernel=%r '
                             'exact=%r' % (what, int(bad.sum()), bad.numel(), i, float(d[i]), float(want[i])))
