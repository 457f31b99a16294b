"""fp64 reference of the grouped GEMM (the contract in csrc/gemm_sm90.h) and a per-element error bound.

``ref_gemm`` computes ``D[g] = epi(A[g] @ B[g // b_group_div])`` in float64 from exactly the operands the kernel read
(the quantised e4m3 / e5m2 values, the 16-bit bias and aux), on the device the operands live on.  Every output element
gets its own tolerance:

    half an output ulp of the reference value                        (final rounding)
  + L * C_ACC[in_dtype] * 2^-24 * S * |sa * sb|                      (accumulation; S = sum_k |a_mk * b_kn|)
  + an evaluation term for the fp32 epilogue math (__expf / erff / one fp32 rounding per operation)

where L bounds the epilogue's slope at that element.  ``check`` compares kernel outputs with the reference under this
bound, checks ReLU masks exactly wherever the reference pre-activation is further from 0 than the accumulation bound,
checks that rows past ``row_counts`` were left untouched, and checks the fused bias gradient (``colsum``).
"""
import math
from dataclasses import dataclass, field
from typing import Dict, Optional

import torch

EPI_NONE, EPI_BIAS, EPI_BIAS_RELU, EPI_BIAS_GELU, EPI_BIAS_SILU, EPI_RELU_BWD = 0, 1, 2, 3, 4, 5
EPI_GLU, EPI_GLU_BWD, EPI_ADD, EPI_ACT_BWD = 6, 7, 8, 9
ACT_RELU, ACT_GELU, ACT_SILU = 1, 2, 3

U = 2.0 ** -24
# Accumulation error constants, in units of 2^-24 * S.  Calibrated on an NVIDIA H100 80GB HBM3 (700 W power limit) as
# about 4x the largest (|out - ref| - 1/2 ulp - evaluation term) / (L * 2^-24 * S) seen over
# tests/test_gpu_gemm_reference.py, whose fp32-output cases run K from 16 to 14336.  The normalised error grows with K
# (bf16 inputs: 0.1 at K = 16, 1.0 at 144, 9.6 at 4096, 15.8 at 14336; fp16 up to 17.6): the wgmma accumulator is not a
# round-to-nearest fp32 sum.  fp8 operands accumulate with far fewer bits: the normalised error is already ~2000 for
# a single 32-deep MMA (K = 16) and ~8000 at K = 4096 (max |err| / max |ref| 4e-3 for e4m3, 7e-3 at K = 14336).
C_ACC = {
    torch.bfloat16: 64.0,          # measured max 15.8
    torch.float16: 64.0,           # measured max 17.6
    torch.float8_e4m3fn: 32768.0,  # measured max 8110
    torch.float8_e5m2: 24576.0,    # measured max 5995
}
# fp32 epilogue arithmetic: one rounding per linear operation, and the approximate __expf / erff of the activations
LIN_REL = 4 * U
FN_REL = 2.0 ** -18
# largest normalised accumulation error seen by check() per input dtype (what C_ACC must cover)
OBSERVED: Dict[torch.dtype, float] = {}

_FMT = {torch.bfloat16: (7, -126), torch.float16: (10, -14), torch.float32: (23, -126)}


def half_ulp(x: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
    """Half the spacing of ``dtype`` values at |x| (subnormal spacing below the normal range)."""
    p, emin = _FMT[dtype]
    _, e = torch.frexp(x)                       # |x| = m * 2^e, 0.5 <= m < 1
    e = torch.where(x == 0, torch.full_like(e, emin + 1), e)
    e = torch.clamp(e - 1, min=emin)
    return torch.ldexp(torch.full_like(x, 0.5), (e - p).to(x.dtype))


def act_fn(x: torch.Tensor, act: int) -> torch.Tensor:
    if act == ACT_RELU:
        return x.clamp_min(0)
    if act == ACT_GELU:
        return 0.5 * x * (1 + torch.erf(x / math.sqrt(2)))
    return x * torch.sigmoid(x)


def act_grad(x: torch.Tensor, act: int) -> torch.Tensor:
    if act == ACT_RELU:
        return (x > 0).to(x.dtype)
    if act == ACT_GELU:
        return 0.5 * (1 + torch.erf(x / math.sqrt(2))) + x * torch.exp(-0.5 * x * x) / math.sqrt(2 * math.pi)
    s = torch.sigmoid(x)
    return s * (1 + x * (1 - s))


@dataclass
class Out:
    val: torch.Tensor     # fp64 reference [G, M, N]
    acc: torch.Tensor     # L * 2^-24 * S (* |sa sb|): multiplied by C_ACC
    fn: torch.Tensor      # evaluation term of the fp32 epilogue


@dataclass
class Ref:
    in_dtype: torch.dtype
    out_dtype: torch.dtype
    valid: torch.Tensor                       # [G, M, 1] rows below min(M, row_counts[g])
    outs: Dict[str, Out] = field(default_factory=dict)
    relu_pre: Optional[torch.Tensor] = None   # BIAS_RELU: the pre-activation and its accumulation bound (/ C_ACC)
    relu_pre_acc: Optional[torch.Tensor] = None
    relu_aux: Optional[torch.Tensor] = None   # RELU_BWD: aux (the mask is exact)
    colsum: Optional[torch.Tensor] = None     # [Gb, N] sum of the fp32 epilogue value over valid rows
    colsum_acc: Optional[torch.Tensor] = None
    colsum_fix: Optional[torch.Tensor] = None


def _operands(a, b, a_mn, b_mn, G, div):
    A = a.double()
    A = A.transpose(1, 2) if a_mn else A                     # [G, M, K]
    B = b.double()
    B = B if b_mn else B.transpose(1, 2)                     # [Gb, K, N]
    return A, B[torch.arange(G, device=B.device) // div]


def ref_gemm(a, b, *, a_mn=False, b_mn=False, epilogue=EPI_NONE, alpha=1.0, bias=None, aux=None, aux2=None, b2=None,
             act=ACT_SILU, scale_a=None, scale_b=None, scale_b2=None, row_counts=None, b_group_div=1,
             out_dtype=torch.bfloat16, want_pre=False) -> Ref:
    """Reference of one launch.  ``a [G, M, K]`` (``[G, K, M]`` when a_mn), ``b [Gb, N, K]`` (``[Gb, K, N]`` when b_mn);
    ``b2`` is the second B of EPI_GLU; ``aux`` / ``aux2`` are g / u of EPI_GLU_BWD."""
    G = a.size(0)
    div = b_group_div
    A, B = _operands(a, b, a_mn, b_mn, G, div)
    M, N = A.size(1), B.size(2)
    gidx = torch.arange(G, device=A.device) // div
    one = torch.ones((), dtype=torch.float64, device=A.device)
    sa = scale_a.double().view(G, M, 1) if scale_a is not None else one
    acc, S = A @ B, A.abs() @ B.abs()
    sb = scale_b.double()[gidx].view(G, 1, N) if scale_b is not None else one
    acc, S = acc * (sa * sb), S * (sa * sb).abs() * U
    if b2 is not None:
        _, B2 = _operands(a, b2, a_mn, b_mn, G, div)
        sb2 = scale_b2.double()[gidx].view(G, 1, N) if scale_b2 is not None else one
        acc2, S2 = (A @ B2) * (sa * sb2), (A.abs() @ B2.abs()) * (sa * sb2).abs() * U
    rows = torch.arange(M, device=A.device).view(1, M, 1)
    count = torch.full((G,), M, device=A.device) if row_counts is None else row_counts.to(A.device).long().clamp(max=M)
    r = Ref(a.dtype, out_dtype, rows < count.view(G, 1, 1))
    lin = lambda v: LIN_REL * v.abs()          # noqa: E731

    if epilogue == EPI_NONE:
        v = acc * alpha
        r.outs['d'] = Out(v, S * abs(alpha), lin(v))
    elif epilogue in (EPI_BIAS, EPI_BIAS_RELU, EPI_BIAS_GELU, EPI_BIAS_SILU):
        pre = acc + (bias.double()[gidx].view(G, 1, N) if bias is not None else 0.0)
        if epilogue == EPI_BIAS:
            r.outs['d'] = Out(pre, S, lin(pre))
        elif epilogue == EPI_BIAS_RELU:
            v = pre.clamp_min(0)
            r.outs['d'] = Out(v, S, lin(pre))
            r.relu_pre, r.relu_pre_acc = pre, S
        else:
            a_ = ACT_GELU if epilogue == EPI_BIAS_GELU else ACT_SILU
            v = act_fn(pre, a_)
            # slope at the element, widened by the largest |act''| (< 1) over the accumulation error
            L = act_grad(pre, a_).abs() + C_ACC[a.dtype] * S
            r.outs['d'] = Out(v, L * S, FN_REL * (v.abs() + pre.abs()) + lin(pre))
            if want_pre:
                r.outs['d2'] = Out(pre, S, lin(pre))
    elif epilogue == EPI_RELU_BWD:
        f = aux.double()
        v = torch.where(f > 0, acc, torch.zeros((), dtype=acc.dtype, device=acc.device))
        r.outs['d'] = Out(v, S, lin(acc))
        r.relu_aux = f
    elif epilogue == EPI_ADD:
        v = acc + aux.double()
        r.outs['d'] = Out(v, S, lin(v) + lin(acc))
    elif epilogue == EPI_ACT_BWD:
        f = aux.double()
        da = act_grad(f, act)
        v = acc * da
        r.outs['d'] = Out(v, S * da.abs(), FN_REL * acc.abs() * (1 + f.abs()) + lin(v))
        if act == ACT_RELU:
            r.relu_aux = f
    elif epilogue == EPI_GLU:
        g, u = acc, acc2
        ag, dg = act_fn(g, act), act_grad(g, act)
        h = ag * u
        # first-order terms act'(g) u dg + act(g) du, widened by |act''| <= 1 over the accumulation error (ReLU: slope
        # 1 wherever the error can reach the kink)
        slack = C_ACC[a.dtype] * (S + S2)
        if act == ACT_RELU:
            dg = torch.where(g.abs() <= C_ACC[a.dtype] * S, torch.ones_like(dg), dg)
        r.outs['d'] = Out(h, (dg.abs() + slack) * (u.abs() + slack) * S + (ag.abs() + slack) * S2,
                          FN_REL * u.abs() * (ag.abs() + g.abs()) + lin(h))
        if want_pre:
            r.outs['d2'] = Out(g, S, lin(g))
            r.outs['d3'] = Out(u, S2, lin(u))
    elif epilogue == EPI_GLU_BWD:
        dh, g, u = acc, aux.double(), aux2.double()
        ag, dg = act_fn(g, act), act_grad(g, act)
        d = dh * u * dg
        d2 = dh * ag
        r.outs['d'] = Out(d, S * (u * dg).abs(), FN_REL * (dh * u).abs() * (1 + g.abs()) + lin(d))
        r.outs['d2'] = Out(d2, S * ag.abs(), FN_REL * dh.abs() * (ag.abs() + g.abs()) + lin(d2))
    else:
        raise ValueError(epilogue)

    o = r.outs['d']
    zero = torch.zeros((), dtype=torch.float64, device=A.device)
    Gb = (G + div - 1) // div
    cs = torch.zeros(Gb, N, dtype=torch.float64, device=A.device)
    cs_acc, cs_fn, cs_abs = torch.zeros_like(cs), torch.zeros_like(cs), torch.zeros_like(cs)
    cs.index_add_(0, gidx, torch.where(r.valid, o.val, zero).sum(1))
    cs_acc.index_add_(0, gidx, torch.where(r.valid, o.acc, zero).sum(1))
    cs_fn.index_add_(0, gidx, torch.where(r.valid, o.fn, zero).sum(1))
    cs_abs.index_add_(0, gidx, torch.where(r.valid, o.val.abs(), zero).sum(1))
    # fp32 additions: the in-register / in-CTA tree over a 128-row tile, then one atomic add per row tile and group
    adds = 16 + div * ((M + 127) // 128)
    r.colsum, r.colsum_acc, r.colsum_fix = cs, cs_acc, cs_fn + adds * U * cs_abs
    return r


def tolerance(r: Ref, name: str, c_acc: Optional[float] = None) -> torch.Tensor:
    o = r.outs[name]
    c = C_ACC[r.in_dtype] if c_acc is None else c_acc
    return half_ulp(o.val, r.out_dtype) + c * o.acc + o.fn


def normalised_error(r: Ref, name: str, out: torch.Tensor) -> float:
    """max over valid elements of (|out - ref| - 1/2 ulp - evaluation term) / (L * 2^-24 * S): what C_ACC must cover."""
    o = r.outs[name]
    excess = (out.double() - o.val).abs() - half_ulp(o.val, r.out_dtype) - o.fn
    ratio = excess / o.acc.clamp_min(1e-300)
    return float(torch.where(r.valid.expand_as(ratio), ratio, torch.full_like(ratio, -math.inf)).max())


def _fail(msg, err, tol, mask, out, val):
    bad = (err > tol) & mask
    idx = tuple(int(i) for i in bad.nonzero()[0])
    return '%s: %d of %d elements outside the bound; worst err/tol %.3g; at %s out=%r ref=%r tol=%.3g' % (
        msg, int(bad.sum()), int(mask.sum()), float(torch.where(mask, err / tol, torch.zeros_like(err)).max()), idx,
        float(out[idx]), float(val[idx]), float(tol[idx]))


def check(r: Ref, d: torch.Tensor, d2: Optional[torch.Tensor] = None, d3: Optional[torch.Tensor] = None,
          colsum: Optional[torch.Tensor] = None, colsum_init: Optional[torch.Tensor] = None, untouched=None,
          c_acc: Optional[float] = None, what: str = '') -> None:
    """Assert that the kernel's outputs satisfy the reference's bound (see the module docstring)."""
    c = C_ACC[r.in_dtype] if c_acc is None else c_acc
    for name, out in (('d', d), ('d2', d2), ('d3', d3)):
        if out is None or name not in r.outs:
            continue
        assert out.dtype == r.out_dtype, (what, name, out.dtype)
        o = r.outs[name]
        x = out.double()
        valid = r.valid.expand_as(x)
        err = (x - o.val).abs()
        err = torch.where(torch.isnan(x), torch.full_like(err, math.inf), err)
        tol = tolerance(r, name, c)
        excess = ((err - half_ulp(o.val, r.out_dtype) - o.fn) / o.acc.clamp_min(1e-300))[valid]
        if excess.numel():
            OBSERVED[r.in_dtype] = max(OBSERVED.get(r.in_dtype, -math.inf), float(excess.max()))
        ok = (err <= tol) | ~valid
        assert bool(ok.all()), _fail('%s %s' % (what, name), err, tol, valid, x, o.val)
        if untouched is not None and not bool(valid.all()):
            kept = x[~valid]
            assert bool((kept == float(untouched)).all()), '%s %s: rows past the count were written' % (what, name)
    x = d.double()
    valid = r.valid.expand_as(x)
    if r.relu_pre is not None:
        bound = c * r.relu_pre_acc
        assert bool((x[valid & (r.relu_pre < -bound)] == 0).all()), '%s: ReLU passed a negative pre-activation' % what
        assert bool((x[valid & (r.relu_pre > bound)] > 0).all()), '%s: ReLU zeroed a positive pre-activation' % what
    if r.relu_aux is not None:
        assert bool((x[valid & (r.relu_aux <= 0)] == 0).all()), '%s: ReLU gradient passed where aux <= 0' % what
    if colsum is not None:
        want = r.colsum + (colsum_init.double() if colsum_init is not None else 0.0)
        got = colsum.double()
        err = (got - want).abs()
        tol = c * r.colsum_acc + r.colsum_fix + half_ulp(want, torch.float32)
        ok = err <= tol
        assert bool(ok.all()), _fail('%s colsum' % what, err, tol, torch.ones_like(ok), got, want)
