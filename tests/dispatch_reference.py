"""References and checkers for the routing and dispatch kernels (csrc/gate_route.cu, csrc/moe_kernels.cu).

Plain torch, no GPU needed.  Every reference takes exactly the tensors the kernel read; where a kernel's contract
depends on an earlier decision it also takes the kernel's own earlier outputs (locations are derived from the
kernel's ``idx``, decode reads the kernel's buffer), so a mismatch points at one kernel.

Two kinds of check:

* exact: integer outputs (ids, locations, slot map, counts) and the outputs that are one fp32 operation and one
  rounding away from their inputs (encode, fp8 encode, dequantisation, transposing quantisation, ``top``) must match
  bit for bit;
* bounded: the fp32 sums (softmax, normalised gates, ``l_aux``, decode, gate gradient, gate backward, column sums) are
  computed in fp64 and each element gets its own bound, derived from the kernel's operation count with u = 2^-24
  (one fp32 rounding), plus half an output ulp where the kernel rounds to a 16-bit type.  A bound is a first-order
  sum of rounding errors; ``SLACK`` covers the second-order terms.

Every failure names the check, the number of bad elements, the worst one, its index, the kernel value, the
reference value and the bound.  ``OBSERVED`` records, per bounded check, the largest normalised error seen:
(|kernel - reference| - output rounding) / accumulation part of the bound, which must stay <= 1.
"""
import math
from typing import Dict, Optional

import torch

from gemm_reference import half_ulp

U = 2.0 ** -24
SLACK = 1.01                      # second-order terms of the first-order bounds below
TINY = 2.0 ** -147                # four fp32 subnormal spacings: expf / products whose result is subnormal
INVALID_LOC = 0x3fffffff          # loc of a choice that routes nowhere
F448 = torch.tensor(1.0 / 448.0, dtype=torch.float32)   # the kernels' fp32 constant 1.0f / 448.0f
FLT_MIN = 2.0 ** -126             # smallest e4m3 row scale: 1 / scale must not overflow
E4M3_MAX = 448.0
OBSERVED: Dict[str, float] = {}


# ------------------------------------------------------------------------------------------------------------------
# reporting
# ------------------------------------------------------------------------------------------------------------------
def _bits(t: torch.Tensor) -> torch.Tensor:
    """Raw bit patterns, so that exact checks also see -0 and NaN payloads."""
    if not t.is_floating_point():
        return t
    return t.view({1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()])


def _value(t: torch.Tensor, i) -> str:
    v = t[i]
    return repr(v.item()) if v.dtype != torch.uint8 else '0x%02x' % int(v)


def assert_equal(what: str, got: torch.Tensor, want: torch.Tensor, mask: Optional[torch.Tensor] = None) -> None:
    """Bit-exact comparison (on ``mask`` only, if given)."""
    assert got.shape == want.shape and got.dtype == want.dtype, (what, got.shape, want.shape, got.dtype, want.dtype)
    bad = _bits(got) != _bits(want)
    if mask is not None:
        bad &= mask
    if bool(bad.any()):
        i = tuple(int(v) for v in bad.nonzero()[0])
        raise AssertionError('%s: %d of %d elements differ (exact check); first at %s: kernel=%s reference=%s' % (
            what, int(bad.sum()), bad.numel() if mask is None else int(mask.sum()), i, _value(got, i), _value(want, i)))


def assert_within(what: str, got: torch.Tensor, want: torch.Tensor, acc: torch.Tensor, rnd=0.0,
                  mask: Optional[torch.Tensor] = None) -> float:
    """|got - want| <= acc + rnd elementwise (on ``mask``), where ``rnd`` is the output rounding (half an ulp of a
    16-bit output) and ``acc`` the rest of the bound.  Records and returns the largest (err - rnd) / acc."""
    x = got.double()
    bound = acc + rnd
    err = (x - want).abs()
    err = torch.where(torch.isnan(x) | torch.isnan(want), torch.full_like(err, math.inf), err)
    ratio = err / bound
    ratio = torch.where(err == 0, torch.zeros_like(ratio), ratio)
    norm = (err - rnd) / acc
    if mask is not None:
        ratio = torch.where(mask, ratio, torch.zeros_like(ratio))
        norm = torch.where(mask, norm, torch.full_like(norm, -math.inf))
    worst = float(ratio.max()) if ratio.numel() else 0.0
    key = what.split(':')[0]
    if norm.numel():
        OBSERVED[key] = max(OBSERVED.get(key, -math.inf), float(norm.max()))
    if worst > 1.0:
        bad = ratio > 1.0
        i = tuple(int(v) for v in (ratio == ratio.max()).nonzero()[0])
        raise AssertionError('%s: %d of %d elements outside the bound; worst err/bound %.3g at %s: kernel=%r '
                             'reference=%r bound=%.3g' % (what, int(bad.sum()), ratio.numel() if mask is None else
                                                          int(mask.sum()), worst, i, float(x[i]), float(want[i]),
                                                          float(bound[i])))
    return worst


def _out_half_ulp(val: torch.Tensor, acc: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
    """Half an output ulp at the largest magnitude the fp32 result can have (its rounding may cross a binade)."""
    return half_ulp(val.abs() + acc, dtype)


# ------------------------------------------------------------------------------------------------------------------
# gate: softmax, top-k, normalised gates
# ------------------------------------------------------------------------------------------------------------------
def ref_softmax(logits: torch.Tensor):
    """fp64 softmax of the logits the kernel read and a per-element bound for gate_route_kernel's fp32 softmax.

    One warp per token, lane l holds experts l, l+32, ...: d = fl(v - max) costs |d| u relative in exp(d); expf is
    within 2 ulp (4u relative); the lane sums of ceil(E/32) terms and 5 shuffle adds give sum(p_e * err_e) +
    (ceil(E/32) - 1 + 5) u on the (positive) sum; the reciprocal and the multiply one rounding each.  Returns
    (p, bound, routable): rows holding a NaN, or with no finite maximum, have NaN scores and route nowhere."""
    v = logits.double()
    mx = v.amax(1, keepdim=True)
    d = v - mx
    routable = ~torch.isnan(d).any(1)
    d = torch.where(routable[:, None], d, torch.zeros_like(d))
    ex = torch.exp(d)
    p = ex / ex.sum(1, keepdim=True)
    rel_e = torch.where(torch.isfinite(d), 4.0 + d.abs(), torch.zeros_like(d)) * U
    lane_terms = -(-v.size(1) // 32)
    rel_sum = (p * rel_e).sum(1, keepdim=True) + (lane_terms - 1 + 5) * U
    bound = p * (rel_e + rel_sum + 2 * U) * SLACK + TINY
    return p, bound, routable


def check_scores(what, logits, scores):
    p, bound, routable = ref_softmax(logits)
    assert_within('scores: ' + what, scores, p, bound, mask=routable[:, None].expand_as(p))
    return p, bound, routable


def check_topk(what, scores, idx, top, p, bound, routable, k):
    """(a) idx is the stable descending sort of the kernel's own fp32 scores (ties -> lower id), exactly;
    (b) in fp64, every chosen expert beats every unchosen one by more than -(bound_chosen + bound_unchosen);
    top is the kernel's score at idx, bit for bit.  Rows that cannot be routed must choose no expert."""
    S, E = scores.shape
    ids = idx.t().long()                                               # [S, k]
    r = routable
    want = torch.sort(scores[r], dim=1, descending=True, stable=True).indices[:, :k]
    assert_equal('top-k ids (stable sort of the kernel scores, ties to the lower id): ' + what, ids[r], want)
    if not bool(r.all()):
        nowhere = (ids[~r] < 0) | (ids[~r] >= E)
        assert bool(nowhere.all()), 'top-k: %s: a row with a NaN score chose an expert' % what
    if not bool(r.any()):
        return
    sel = ids[r]
    assert_equal('top (kernel score at idx): ' + what, top.t()[r].contiguous(), scores[r].gather(1, sel))
    if k < E:
        pr, br = p[r], bound[r]
        chosen = torch.zeros_like(pr, dtype=torch.bool).scatter_(1, sel, True)
        lo = torch.where(chosen, pr + br, torch.full_like(pr, math.inf)).amin(1)
        hi = torch.where(chosen, torch.full_like(pr, -math.inf), pr - br).amax(1)
        bad = lo < hi
        if bool(bad.any()):
            s = int(bad.nonzero()[0])
            raise AssertionError('top-k in fp64: %s: %d rows choose an expert that loses by more than the score bound; '
                                 'first row %d: chosen %s, lowest chosen p+bound %r < highest unchosen p-bound %r' % (
                                     what, int(bad.sum()), s, sel[s].tolist(), float(lo[s]), float(hi[s])))


def ref_gates(top: torch.Tensor, normalize: bool, eps: float):
    """gates = top / max(sum top, eps) (normalize and k > 1) in fp64 from the kernel's top [k, S]: the shuffle sum of
    k positive terms (min(k - 1, 5) roundings) and the division.  Otherwise gates == top exactly (bound None)."""
    k = top.size(0)
    t = top.double()
    if not (normalize and k > 1):
        return t, None
    val = t / t.sum(0, keepdim=True).clamp_min(eps)
    return val, (min(k - 1, 5) + 1) * U * val.abs() * SLACK + TINY


def check_gates(what, top, gates, normalize, eps, routable):
    val, bound = ref_gates(top, normalize, eps)
    mask = routable[None, :].expand_as(gates)
    if bound is None:
        assert_equal('gates (= top): ' + what, gates, top, mask)
    else:
        assert_within('gates: ' + what, gates, val, bound, mask=mask)


# ------------------------------------------------------------------------------------------------------------------
# locations, slot map, counts
# ------------------------------------------------------------------------------------------------------------------
def ref_locations(idx: torch.Tensor, E: int, C: int = 0):
    """Queue positions of the kernel's choices idx [k, S]: choice-major (all first choices in token order, then all
    second choices, ...); an id outside [0, E) routes nowhere (loc = INVALID_LOC).  Returns (loc [k, S] int32,
    counts [E] int32 including dropped tokens, ce [E] fp32 first-choice counts, slot [E*C] int32 or None: token * k +
    choice of the choice queued at (e, l < C), -1 where empty)."""
    k, S = idx.shape
    flat = idx.reshape(-1).long()
    valid = (flat >= 0) & (flat < E)
    key = torch.where(valid, flat, torch.full_like(flat, E))
    order = torch.sort(key, stable=True).indices
    n = torch.bincount(key, minlength=E + 1)
    start = torch.cumsum(n, 0) - n
    rank = torch.empty_like(flat)
    rank[order] = torch.arange(flat.numel(), device=flat.device) - start[key[order]]
    loc = torch.where(valid, rank, torch.full_like(rank, INVALID_LOC))
    counts = n[:E].to(torch.int32)
    ce = torch.bincount(key[:S], minlength=E + 1)[:E].float()
    slot = None
    if C > 0:
        slot = torch.full((E * C,), -1, dtype=torch.int32, device=idx.device)
        src = (torch.arange(S, device=idx.device)[None, :] * k + torch.arange(k, device=idx.device)[:, None]).reshape(-1)
        keep = valid & (loc < C)
        slot[flat[keep] * C + loc[keep]] = src[keep].to(torch.int32)
    return loc.view(k, S).to(torch.int32), counts, ce, slot


def check_locations(what, idx, E, C, loc, counts, ce=None, slot=None):
    rl, rc, rce, rs = ref_locations(idx, E, C)
    assert_equal('loc (choice-major queue order): ' + what, loc, rl)
    assert_equal('counts: ' + what, counts, rc)
    if ce is not None:
        assert_equal('ce (first-choice counts): ' + what, ce, rce)
    if slot is not None:
        assert_equal('slot map: ' + what, slot, rs)


def ref_l_aux(scores: torch.Tensor, ce: torch.Tensor, dtype: torch.dtype):
    """l_aux = E / S^2 * sum_e (sum_s p_se) ce_e in fp64 from the kernel's scores and ce.  fp32 summation in the
    kernels: 8 tokens per lane and tile, 32 warps' shared atomics, the tiles, the product with ce, ceil(E/256) terms
    per thread, 5 shuffle adds, 8 warp partials, S*S / the multiply by E / the division; all terms are >= 0.  Then
    half an ulp of the logits dtype."""
    S, E = scores.shape
    ntiles = -(-S // 256)
    val = (scores.double().sum(0) * ce.double()).sum() * E / (S * S)
    rel = (8 + 32 + ntiles + 1 + (-(-E // 256)) + 5 + 8 + 3) * U
    acc = rel * val.abs() * SLACK
    return val, acc, (_out_half_ulp(val, acc, dtype) if dtype != torch.float32 else 0.0)


def check_l_aux(what, scores, ce, l_aux):
    val, acc, rnd = ref_l_aux(scores, ce, l_aux.dtype)
    assert_within('l_aux: ' + what, l_aux.reshape(1), val.reshape(1), acc.reshape(1), rnd)


def check_gate_route_forward(what, logits, k, C, normalize, eps, outs, check_loss=True):
    """All outputs of gate_route_forward: [scores, idx, top, gates, loc, counts, ce, l_aux(, slot)]."""
    scores, idx, top, gates, loc, counts, ce, l_aux = outs[:8]
    slot = outs[8] if len(outs) > 8 else None
    S, E = logits.shape
    p, bound, routable = check_scores(what, logits, scores)
    check_topk(what, scores, idx, top, p, bound, routable, k)
    check_gates(what, top, gates, normalize, eps, routable)
    check_locations(what, idx, E, C, loc, counts, ce, slot)
    if check_loss:
        check_l_aux(what, scores, ce, l_aux)
    return routable


# ------------------------------------------------------------------------------------------------------------------
# gate backward (closed form of csrc/gate_route.cu, evaluated in fp64 on the kernel's scores / idx / top)
# ------------------------------------------------------------------------------------------------------------------
def ref_gate_backward(scores, idx, top, dgates, ce, dl, normalize, eps, dtype):
    """d logits [S, E] and its bound.

        r_j = top_j, D = sum_j r_j, Dc = max(D, eps)
        dr_j = dg_j / Dc - [D > eps] (sum_i dg_i r_i) / Dc^2          (normalize and k > 1; else dr_j = dg_j)
        dp_e = dl ce_e E / S^2 + sum_j [idx_j == e] dr_j
        dlogit_e = p_e (dp_e - sum_e' dp_e' p_e')

    Rounding errors of gate_route_bwd_kernel: the loss scale dl * E / (S*S) * ce_e (4u); D and dot as 5-step shuffle
    sums; dr as dg/Dc (6u) minus dot/(Dc*Dc) (18u on sum|dg r| / Dc^2) (1u); dp_e one add; the lane sums of
    ceil(E/32) products and 5 shuffle adds for sum dp p; the difference and the product (2u); then the output
    rounding.  Returns (val, acc, rnd, mask): the bound is acc + rnd (rnd: the output rounding); rows whose D is within 8u of eps (either branch may be taken) are masked."""
    S, E = scores.shape
    k = idx.size(0)
    p = scores.double()
    r = top.double().t()
    ids = idx.t().long()
    dg = dgates.double().t() if dgates is not None else torch.zeros_like(r)
    aux = torch.zeros(E, dtype=torch.float64, device=p.device)
    if ce is not None and dl is not None:
        aux = float(dl) * E / (S * S) * ce.double()
    D = r.sum(1, keepdim=True)
    mask = torch.ones(S, dtype=torch.bool, device=p.device)
    if normalize and k > 1:
        Dc = D.clamp_min(eps)
        on = D > eps
        dot = (dg * r).sum(1, keepdim=True)
        sdot = (dg * r).abs().sum(1, keepdim=True)
        dr = dg / Dc - torch.where(on, dot / (Dc * Dc), torch.zeros_like(dot))
        dr_err = 6 * U * (dg / Dc).abs() + torch.where(on, 18 * U * sdot / (Dc * Dc), torch.zeros_like(sdot)) + U * dr.abs()
        mask = ((D - eps).abs() > 8 * U * D).view(S)
    else:
        dr, dr_err = dg, torch.zeros_like(dg)
    valid = (ids >= 0) & (ids < E)
    safe = torch.where(valid, ids, torch.zeros_like(ids))
    zero = torch.zeros_like(dr)
    dp = aux.expand(S, E).clone().scatter_add_(1, safe, torch.where(valid, dr, zero))
    dp_err = (4 * U * aux.abs()).expand(S, E).clone().scatter_add_(1, safe, torch.where(valid, dr_err, zero)) + U * dp.abs()
    acc = (dp * p).sum(1, keepdim=True)
    acc_err = (p * dp_err).sum(1, keepdim=True) + (-(-E // 32) + 6) * U * (dp * p).abs().sum(1, keepdim=True)
    val = p * (dp - acc)
    err = (p * (dp_err + acc_err) + 2 * U * val.abs()) * SLACK + TINY
    return val, err, (_out_half_ulp(val, err, dtype) if dtype != torch.float32 else 0.0), mask


def check_gate_backward(what, dlogits, scores, idx, top, dgates, ce, dl, normalize, eps, routable):
    val, acc, rnd, mask = ref_gate_backward(scores, idx, top, dgates, ce, dl, normalize, eps, dlogits.dtype)
    m = (mask & routable)[:, None].expand_as(val)
    assert_within('gate backward: ' + what, dlogits, val, acc, rnd, m)


# ------------------------------------------------------------------------------------------------------------------
# encode (16-bit / fp32 and e4m3), dequantisation, transposing quantisation: bit-exact
# ------------------------------------------------------------------------------------------------------------------
def _slot_sources(slot, k, gates):
    src = slot.long()
    empty = src < 0
    tok = torch.where(empty, torch.zeros_like(src), src // k)
    j = torch.where(empty, torch.zeros_like(src), src % k)
    g = gates.float()[j, tok] if gates is not None else None
    return empty, tok, g


def ref_encode(x, gates, slot, k, E, C, valid_rows=None):
    """out[e*C + l] = T(fp32(x[tok]) * g) for the choice at slot (e, l) (a plain copy without gates), exactly 0 for an
    empty slot.  Returns (want [E*C, M], keep [E*C]): rows at or past valid_rows[e] must keep what was there."""
    empty, tok, g = _slot_sources(slot, k, gates)
    rows = x[tok]
    if g is not None:
        rows = (rows.float() * g[:, None]).to(x.dtype)
    want = torch.where(empty[:, None], torch.zeros((), dtype=x.dtype, device=x.device), rows)
    keep = torch.zeros(E * C, dtype=torch.bool, device=x.device)
    if valid_rows is not None:
        keep = (torch.arange(C, device=x.device)[None, :] >= valid_rows.long().view(E, 1)[:, :]).reshape(-1)
    return want, keep


def check_encode(what, out, x, gates, slot, k, E, C, valid_rows=None, sentinel=None):
    want, keep = ref_encode(x, gates, slot, k, E, C, valid_rows)
    assert_equal('encode: ' + what, out, want, (~keep)[:, None].expand_as(out))
    if bool(keep.any()):
        s = torch.full_like(out, sentinel)
        assert_equal('encode rows past valid_rows (must keep the sentinel): ' + what, out, s, keep[:, None].expand_as(out))


def to_e4m3(v: torch.Tensor) -> torch.Tensor:
    """fp32 -> e4m3 bytes as the kernels' __nv_fp8x4_e4m3 converts them: round to nearest even, saturating at +-448
    (torch's own conversion returns NaN above 464)."""
    return v.clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn).view(torch.uint8)


def ref_encode_fp8(x, gates, slot, k, E, C):
    """fp8 dispatch rows in fp32, bit for bit: amax = max|x|, amax *= |g|, sc = max(amax * fp32(1/448), FLT_MIN) (1 when amax = 0),
    inv = g / sc, q = e4m3(x * inv).  An empty slot has zero bytes and scale 1.  Returns (q uint8 [E*C, M], sc)."""
    empty, tok, g = _slot_sources(slot, k, gates)
    xf = x.float()[tok]
    if g is None:
        g = torch.ones(xf.size(0), dtype=torch.float32, device=x.device)
    amax = xf.abs().amax(1) * g.abs()
    sc = torch.where(amax > 0, (amax * F448.to(x.device)).clamp_min(FLT_MIN), torch.ones_like(amax))
    inv = g / sc
    q = to_e4m3(xf * inv[:, None])
    q = torch.where(empty[:, None], torch.zeros_like(q), q)
    sc = torch.where(empty, torch.ones_like(sc), sc)
    return q, sc


def check_encode_fp8(what, q, sc, x, gates, slot, k, E, C):
    wq, ws = ref_encode_fp8(x, gates, slot, k, E, C)
    assert_equal('fp8 encode scales: ' + what, sc.reshape(-1), ws)
    assert_equal('fp8 encode bytes: ' + what, q.reshape(wq.shape).view(torch.uint8), wq)


def ref_dequant(q, scale, dtype):
    """y = T(float(q) * scale) per row."""
    return (q.view(torch.float8_e4m3fn).float() * scale.float()[..., None]).to(dtype)


def ref_quantize_transpose(x):
    """x [G, R, K] 16 bit -> (qT uint8 [G, K, R], scale [G, K]): column amax, sc = max(amax * fp32(1/448), FLT_MIN) (1 when 0),
    inv = 1 / sc, e4m3(x * inv) transposed."""
    xf = x.float()
    amax = xf.abs().amax(1)
    sc = torch.where(amax > 0, (amax * F448.to(x.device)).clamp_min(FLT_MIN), torch.ones_like(amax))
    inv = 1.0 / sc
    return to_e4m3(xf * inv[:, None, :]).transpose(1, 2).contiguous(), sc


# ------------------------------------------------------------------------------------------------------------------
# decode, gate gradient, column sums: fp64 with operation-count bounds
# ------------------------------------------------------------------------------------------------------------------
def _gathered(buf, idx, loc, E, C):
    valid = (idx >= 0) & (idx < E) & (loc >= 0) & (loc < C)
    row = torch.where(valid, idx.long() * C + loc.long(), torch.zeros_like(idx, dtype=torch.long))
    return valid, buf.double()[row]                                     # [k, S], [k, S, M]


def ref_decode(buf, gates, idx, loc, E, C):
    """out[s] = sum_j g_j buf[idx_j * C + loc_j] over the valid choices, in fp64.  The kernel's fmaf chain in choice
    order makes nsel roundings: nsel u sum_j |g_j y_j|, then half an output ulp.  Returns (val, acc, rnd, none):
    tokens with no valid choice must be exactly 0."""
    valid, y = _gathered(buf, idx, loc, E, C)
    w = gates.double() if gates is not None else torch.ones(idx.shape, dtype=torch.float64, device=buf.device)
    w = torch.where(valid, w, torch.zeros_like(w))
    terms = w[..., None] * y
    val = terms.sum(0)
    acc = valid.sum(0)[:, None] * U * terms.abs().sum(0) * SLACK + TINY
    return val, acc, _out_half_ulp(val, acc, buf.dtype), ~valid.any(0)


def check_decode(what, out, buf, gates, idx, loc, E, C):
    val, acc, rnd, none = ref_decode(buf, gates, idx, loc, E, C)
    assert_within('decode: ' + what, out, val, acc, rnd, (~none)[:, None].expand_as(val))
    if bool(none.any()):
        assert_equal('decode of a token with no valid choice (exact 0): ' + what, out[none], torch.zeros_like(out[none]))


def ref_gate_grad(a, buf, idx, loc, E, C):
    """dgate[j, s] = a[s] . buf[idx_j * C + loc_j] in fp64, exactly 0 for a dropped or invalid choice.  Kernel: one
    warp per token, each lane an fmaf chain over at most ceil(M/32) + 7 elements (16-byte vectors of up to 8), then 5
    shuffle adds: bound (ceil(M/32) + 7 + 5) u sum|a b|.  Returns (val, bound, valid)."""
    valid, y = _gathered(buf, idx, loc, E, C)
    prod = a.double()[None] * y
    M = a.size(1)
    val = torch.where(valid, prod.sum(-1), torch.zeros(valid.shape, dtype=torch.float64, device=a.device))
    bound = (-(-M // 32) + 7 + 5) * U * prod.abs().sum(-1) * SLACK + TINY
    return val, bound, valid


def check_gate_grad(what, out, a, buf, idx, loc, E, C):
    val, bound, valid = ref_gate_grad(a, buf, idx, loc, E, C)
    assert_within('gate_grad: ' + what, out, val, bound, mask=valid)
    if not bool(valid.all()):
        assert_equal('gate_grad of a dropped choice (exact 0): ' + what, out[~valid], torch.zeros_like(out[~valid]))


def ref_colsum(x):
    """x [G, T, N] -> fp64 column sums and their bound: any fp32 summation tree over T terms (per-thread chains,
    shared-memory sums, fp32 atomics) makes at most T - 1 roundings on a path, so T u sum|x|, then half an ulp.
    Returns (val, acc, rnd)."""
    xd = x.double()
    val = xd.sum(1)
    acc = x.size(1) * U * xd.abs().sum(1) * SLACK + TINY
    return val, acc, (_out_half_ulp(val, acc, x.dtype) if x.dtype != torch.float32 else 0.0)


def check_colsum(what, out, x):
    val, acc, rnd = ref_colsum(x)
    assert_within('colsum: ' + what, out, val, acc, rnd)
