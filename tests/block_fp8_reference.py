"""References with per-element error bounds for the block-scaled fp8 kernels (csrc/gemm_block_fp8.cu).  Plain torch:
runs on the CPU or the GPU.

Quantisers (exact), written from the number format of tutel_b200/ops/block_fp8.py: a block's scale is
``s = max(amax * (1/448), FLT_MIN)`` in fp32 (``1`` when ``amax``, the largest non-NaN magnitude, is 0), and its
elements are ``e4m3_rn_satfinite(x * (1/s))`` with ``1/s`` and the product rounded to fp32.  Index arithmetic gives the
scale layouts: activations ``[G, K/128, roundup(R, 128)]`` (pad rows 0), weights ``[G, N/128, K/128]``, the SwiGLU
forward copy one scale per 64 interleaved rows.

GEMM (bounded).  ``ref_gemm`` computes the result in fp64 from exactly the e4m3 bytes and fp32 scales the kernel read.
The kernel sums each 128-deep K block in the tensor core (four chained ``wgmma k32`` from zero) and promotes it with
``acc = fmaf(part, sa * sb, acc)``:

* each block's MMA error: one calibrated single-block e4m3 term, ``C_BLOCK * 2^-24 * S_kb``, where
  ``S_kb = |sa sb| sum_{k in kb} |a_k b_k|`` (``C_BLOCK = C_ACC[e4m3]`` of tests/gemm_reference.py, calibrated over
  K up to 14336 in the row kernel, which is one long MMA chain);
* ``sa * sb`` rounds once and each promotion rounds once: ``2 * 2^-24 * S_kb`` per block, plus 2 for second-order terms;
* bias: ``2^-24 |acc + bias|``; fp32 subnormals: one subnormal spacing per promotion;
* the bf16 output rounding: half an ulp at ``|ref| + bound``.

So ``|d - ref| <= half_ulp_bf16 + (C_BLOCK + 2 KB + 2) 2^-24 S + 2^-24 |pre| + (KB + 1) 2^-149`` with
``S = sum_kb S_kb``.  The GLU epilogues propagate these bounds through ``act(g) * u`` and ``dh * u * act'(g)`` to first
order (plus the error of the fast ``__expf``); ReLU-backward masks are checked exactly.
"""
import math
from dataclasses import dataclass
from typing import Dict, Optional

import torch

from gemm_reference import C_ACC, FN_REL, LIN_REL, U, half_ulp

TILE = 128
E4M3_MAX = 448.0
C_BLOCK = C_ACC[torch.float8_e4m3fn]
TINY = 2.0 ** -149
EPI_NONE, EPI_RELU, EPI_RELU_BWD, EPI_GLU, EPI_GLU_BWD = 0, 1, 2, 3, 4
ACT = {'relu': 1, 'gelu': 2, 'silu': 3}
# largest normalised errors seen by check(), keyed by the text before the first ':' of its `what`; under 'acc' the
# largest (|err| - every term but the MMA's) / (2^-24 S), which C_BLOCK must cover
OBSERVED: Dict[str, float] = {}


# ------------------------------------------------------------------------------------------------------------------
# quantisers
# ------------------------------------------------------------------------------------------------------------------
def e4m3_rn_satfinite(v: torch.Tensor) -> torch.Tensor:
    """fp32 -> e4m3 bytes, round to nearest even, saturating at +-448 (NaN stays NaN)."""
    return v.clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn).view(torch.uint8)


def scale_of(amax64: torch.Tensor) -> torch.Tensor:
    """fp32 scales of blocks with largest non-NaN magnitude ``amax64`` (exact, any float dtype)."""
    amax = amax64.float()
    s = amax * torch.tensor(1.0 / E4M3_MAX, dtype=torch.float32, device=amax.device)
    s = torch.clamp_min(s, 2.0 ** -126)
    return torch.where(amax > 0, s, torch.ones_like(s))


def _amax(blocks: torch.Tensor, dims) -> torch.Tensor:
    a = blocks.double().abs()
    return torch.where(torch.isnan(a), torch.zeros_like(a), a).amax(dim=dims)


def _q(x: torch.Tensor, s_elem: torch.Tensor) -> torch.Tensor:
    inv = torch.ones_like(s_elem) / s_elem                     # fp32 division, as the kernel's 1.0f / s
    return e4m3_rn_satfinite(x.float() * inv)


def quantize_act(x: torch.Tensor):
    """x [G, R, K] -> (bytes uint8 [G, R, K], s fp32 [G, K/128, roundup(R, 128)])."""
    G, R, K = x.shape
    KT, Rp = K // TILE, -(-R // TILE) * TILE
    s = scale_of(_amax(x.view(G, R, KT, TILE), -1))                                    # [G, R, KT]
    q = _q(x.view(G, R, KT, TILE), s.unsqueeze(-1)).view(G, R, K)
    st = torch.zeros(G, KT, Rp, dtype=torch.float32, device=x.device)
    for g in range(G):
        st[g, :, :R] = s[g].t()
    return q, st


def quantize_weight(w: torch.Tensor):
    """w [G, R, C] -> (bytes [G, R, C], s [G, R/128, C/128])."""
    G, R, C = w.shape
    b = w.view(G, R // TILE, TILE, C // TILE, TILE)
    s = scale_of(_amax(b, (2, 4)))
    return _q(b, s[:, :, None, :, None]).view(G, R, C), s


def glu_rows(n: torch.Tensor, H: int):
    """(gate or up, column) of row n of the interleaved [2H, M] SwiGLU copy."""
    return (n % 128) // 64, (n // 128) * 64 + n % 64


def check_bytes(what: str, got: torch.Tensor, want: torch.Tensor, x: Optional[torch.Tensor] = None) -> None:
    """e4m3 bytes equal; NaN must stay NaN (0x7f / 0xff: the sign the hardware writes for -NaN is not part of the contract)."""
    got = got.reshape(want.shape).view(torch.uint8)
    nan = (want & 0x7F) == 0x7F
    bad = torch.where(nan, (got & 0x7F) != 0x7F, got != want)
    if bool(bad.any()):
        i = tuple(int(v) for v in bad.nonzero()[0])
        raise AssertionError('%s: %d of %d e4m3 bytes differ; first at %s: kernel=0x%02x reference=0x%02x%s' % (
            what, int(bad.sum()), bad.numel(), i, int(got[i]), int(want[i]),
            '' if x is None else ' x=%r' % float(x.reshape(want.shape)[i])))


def check_scales(what: str, got: torch.Tensor, want: torch.Tensor) -> None:
    assert got.shape == want.shape and got.dtype == torch.float32, (what, got.shape, want.shape, got.dtype)
    bad = got.view(torch.int32) != want.view(torch.int32)
    if bool(bad.any()):
        i = tuple(int(v) for v in bad.nonzero()[0])
        raise AssertionError('%s: %d of %d scales differ; first at %s: kernel=%r reference=%r' % (
            what, int(bad.sum()), bad.numel(), i, float(got[i]), float(want[i])))


# ------------------------------------------------------------------------------------------------------------------
# GEMM
# ------------------------------------------------------------------------------------------------------------------
def deq_act(q: torch.Tensor, s: torch.Tensor) -> torch.Tensor:
    G, R, K = q.shape
    v = q.view(torch.float8_e4m3fn).double().view(G, R, K // TILE, TILE)
    return (v * s[:, :, :R].transpose(1, 2).double().unsqueeze(-1)).view(G, R, K)


def deq_weight(q: torch.Tensor, s: torch.Tensor) -> torch.Tensor:
    """[G, N, K] with s [G, N / rows, K / 128] (rows = 128, or 64 for the GLU forward copy)."""
    G, N, K = q.shape
    rows = N // s.size(1)
    v = q.view(torch.float8_e4m3fn).double().view(G, s.size(1), rows, K // TILE, TILE)
    return (v * s.double()[:, :, None, :, None]).view(G, N, K)


def act_fn(g, act):
    if act == 'relu':
        return g.clamp_min(0)
    if act == 'gelu':
        return 0.5 * g * (1 + torch.erf(g / math.sqrt(2)))
    return g * torch.sigmoid(g)


def act_grad(g, act):
    if act == 'relu':
        return (g > 0).to(g.dtype)
    if act == 'gelu':
        return 0.5 * (1 + torch.erf(g / math.sqrt(2))) + g * torch.exp(-0.5 * g * g) / math.sqrt(2 * math.pi)
    s = torch.sigmoid(g)
    return s * (1 + g * (1 - s))


@dataclass
class Ref:
    val: torch.Tensor                      # fp64 after the epilogue
    acc: torch.Tensor                      # the bound but for the output rounding
    S: torch.Tensor                        # 2^-24 * S (the MMA terms' unit), for the report
    other: torch.Tensor                    # every term of acc but C_BLOCK * S
    zero: Optional[torch.Tensor] = None    # where the output must be exactly 0


def _plain(A, B):
    KB = A.size(2) // TILE
    acc = A @ B.transpose(1, 2)
    S = (A.abs() @ B.abs().transpose(1, 2)) * U
    return acc, S, (2 * KB + 2) * S + (KB + 1) * TINY


def ref_gemm(aq, sa, bq, sb, bias=None, aux=None, aux2=None, epilogue=EPI_NONE, act='silu'):
    """Reference of one ``block_fp8_gemm`` launch.  Returns a list of :class:`Ref` in the order of the binding's
    outputs; GLU_BWD returns the two halves (dg, du) of its one buffer."""
    A, B = deq_act(aq, sa), deq_weight(bq, sb)
    acc, S, other = _plain(A, B)
    if epilogue == EPI_GLU:
        G, M, N = acc.shape
        H = N // 2

        def half(t, i):
            return t.view(G, M, H // 64, 2, 64)[:, :, :, i].reshape(G, M, H)
        g, u = half(acc, 0), half(acc, 1)
        Sg, Su = half(S, 0), half(S, 1)
        eg, eu = C_BLOCK * Sg + half(other, 0), C_BLOCK * Su + half(other, 1)
        a, da = act_fn(g, act), act_grad(g, act)
        if act == 'relu':
            da = torch.where(g.abs() <= eg, torch.ones_like(da), da)
        else:
            da = da.abs() + eg            # |act''| <= 1 over the error interval
        h = a * u
        acc_h = da * eg * (u.abs() + eu) + a.abs() * eu + FN_REL * u.abs() * (a.abs() + g.abs()) + LIN_REL * h.abs()
        S_h = da * (u.abs() + eu) * Sg + a.abs() * Su
        return [Ref(h, acc_h, S_h, acc_h - C_BLOCK * S_h), Ref(g, eg, Sg, half(other, 0)), Ref(u, eu, Su, half(other, 1))]
    if epilogue == EPI_GLU_BWD:
        e = C_BLOCK * S + other
        g, u = aux.double(), aux2.double()
        a, da = act_fn(g, act), act_grad(g, act)
        dg = acc * u * da
        du = acc * a
        fdg = FN_REL * (acc * u).abs() * (1 + g.abs()) + LIN_REL * dg.abs()
        fdu = FN_REL * acc.abs() * (a.abs() + g.abs()) + LIN_REL * du.abs()
        return [Ref(dg, (u * da).abs() * e + fdg, (u * da).abs() * S, (u * da).abs() * other + fdg),
                Ref(du, a.abs() * e + fdu, a.abs() * S, a.abs() * other + fdu)]
    pre = acc if bias is None else acc + bias.double().reshape(acc.size(0), 1, -1)
    if bias is not None:
        other = other + U * pre.abs()
    r = Ref(pre, C_BLOCK * S + other, S, other)
    if epilogue == EPI_RELU:
        r.val = pre.clamp_min(0)
    elif epilogue == EPI_RELU_BWD:
        r.zero = ~(aux.double() > 0)
        r.val = torch.where(r.zero, torch.zeros_like(pre), pre)
    return [r]


def check(what: str, d: torch.Tensor, r: Ref) -> float:
    """Assert ``d`` (bf16) is within the bound everywhere and exactly 0 where a ReLU-backward mask is off.  Returns the
    largest (|err| - output rounding) / rest of the bound, <= 1 when it passes."""
    assert d.dtype == torch.bfloat16 and d.shape == r.val.shape, (what, d.dtype, d.shape, r.val.shape)
    x = d.double()
    if r.zero is not None:
        bad = r.zero & (x != 0)
        assert not bool(bad.any()), '%s: %d outputs not exactly 0 where aux > 0 is false' % (what, int(bad.sum()))
    err = (x - r.val).abs()
    err = torch.where(torch.isnan(x), torch.full_like(err, math.inf), err)
    rnd = half_ulp(r.val.abs() + r.acc, torch.bfloat16)
    live = torch.ones_like(err, dtype=torch.bool) if r.zero is None else ~r.zero
    norm = torch.where(live, (err - rnd).clamp_min(0) / r.acc.clamp_min(1e-300), torch.zeros_like(err))
    accn = torch.where(live, (err - rnd - r.other) / r.S.clamp_min(1e-300), torch.full_like(err, -math.inf))
    worst = float(norm.max()) if norm.numel() else 0.0
    if norm.numel():
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


def check_all(what: str, outs, refs) -> float:
    """``check`` every output of a launch (GLU_BWD: the dg and du halves of its one buffer)."""
    if len(outs) == 1 and len(refs) == 2:
        H = refs[0].val.size(-1)
        outs = [outs[0][..., :H], outs[0][..., H:]]
    return max(check('%s[%d]' % (what, i), o, r) for i, (o, r) in enumerate(zip(outs, refs)))


# ------------------------------------------------------------------------------------------------------------------
# operands
# ------------------------------------------------------------------------------------------------------------------
def operands(G: int, M: int, N: int, K: int, spread: int = 30, seed: int = 0, device=None, glu: bool = False):
    """Random finite e4m3 operands a [G, M, K], b [G, N, K] (every finite magnitude, random sign) and fp32 scales whose
    exponents are drawn from [-spread, spread] (random mantissas), in the layouts the kernel reads."""
    gen = torch.Generator(device=device).manual_seed(seed)

    def e4m3(rows):
        b = torch.randint(0, 0x7F, (G, rows, K), generator=gen, device=device, dtype=torch.int32)
        b = b | (torch.randint(0, 2, b.shape, generator=gen, device=device, dtype=torch.int32) << 7)
        return b.to(torch.uint8).view(torch.float8_e4m3fn)

    def scales(*shape):
        e = torch.randint(-spread, spread + 1, shape, generator=gen, device=device).float()
        return (torch.exp2(e) * (1 + torch.rand(shape, generator=gen, device=device))).float()

    aq, bq = e4m3(M), e4m3(N)
    Mp = -(-M // TILE) * TILE
    sa = scales(G, K // TILE, Mp)
    sa[:, :, M:] = 0
    sb = scales(G, N // (64 if glu else 128), K // TILE)
    return aq, sa, bq, sb


def bias_aux(val: torch.Tensor, seed: int = 1):
    """(bias bf16 [G, N] of the columns' typical magnitude, aux bf16 [G, M, N] with +0, -0 and NaN entries)."""
    G, M, N = val.shape
    gen = torch.Generator(device=val.device).manual_seed(seed)
    scale = val.abs().median(dim=1).values.float()
    bias = (torch.randn(G, N, generator=gen, device=val.device) * scale).bfloat16()
    aux = torch.randn(G, M, N, generator=gen, device=val.device).bfloat16()
    aux[:, ::5] = 0.0
    aux[:, 1::5] = -0.0
    aux[:, 2::7, ::3] = float('nan')
    return bias, aux
