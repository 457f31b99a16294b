"""Reference and checkers for the sigmoid gate kernels (csrc/gate_route.cu, SIGMOID instantiations).

Same conventions as tests/dispatch_reference.py, whose reporting, location reference and constants are reused:

* exact: ids are recomputed from the kernel's own fp32 scores plus the bias (that addition, and the sum of a group's
  two best keys, are single fp32 operations, so the kernel's keys are reproduced bit for bit); ``top`` is the
  kernel's score at each id; locations, slot map and counts come from ``ref_locations``; ce are the all-choice
  counts as fp32;
* bounded: scores, gates, ``l_aux`` and the logits gradient are computed in fp64, each element with a bound derived
  from the kernel's operation count (u = 2^-24, ``SLACK`` for second-order terms).
"""
import math

import torch

from dispatch_reference import SLACK, TINY, U, _out_half_ulp, assert_equal, assert_within, check_locations

FLT_MIN = 2.0 ** -126         # results below the smallest normal fp32 may be flushed or lose all relative precision


def _lanes(E):
    return -(-E // 32)


# ------------------------------------------------------------------------------------------------------------------
# scores
# ------------------------------------------------------------------------------------------------------------------
def ref_sigmoid(logits: torch.Tensor):
    """fp64 sigmoid of the logits the kernel read and the bound of the kernel's 1 / (1 + expf(-z)): expf within
    2 ulp (4u relative, the input is exact), the sum with 1 (1u, and the exponential's error shrinks by e/(1+e) <= 1),
    the division (1u).  Below FLT_MIN the result is subnormal (or 0 once expf overflows): absolute FLT_MIN.
    Returns (p, bound); NaN logits give NaN scores (masked by the callers)."""
    z = logits.double()
    p = torch.sigmoid(z)
    return p, 6 * U * p * SLACK + FLT_MIN


def check_scores(what, logits, scores):
    p, bound = ref_sigmoid(logits)
    assert_within('scores: ' + what, scores, p, bound, mask=~torch.isnan(p))
    return p


# ------------------------------------------------------------------------------------------------------------------
# selection
# ------------------------------------------------------------------------------------------------------------------
def ref_select(scores: torch.Tensor, bias: torch.Tensor, k: int, n_group: int, topk_group: int) -> torch.Tensor:
    """Expected ids [k, S] (int64, E for a choice that routes nowhere) from the kernel's fp32 scores and the bias:
    key = fl(score + bias) (NaN -> -inf); with groups, the group score is fl(sum of its top min(2, E/n_group) keys)
    and the topk_group best groups (stable: ties to the lower group id; NaN / -inf scores never) are kept; then the
    k best keys above -inf, ties to the lower id."""
    S, E = scores.shape
    key = scores.float() + bias.float()
    key = torch.where(torch.isnan(key), torch.full_like(key, -math.inf), key)
    if n_group > 1:
        gsz = E // n_group
        top2 = torch.sort(key.view(S, n_group, gsz), dim=2, descending=True).values[:, :, :min(2, gsz)]
        gs = top2[:, :, 0] + top2[:, :, 1] if gsz > 1 else top2[:, :, 0]
        gs = torch.where(torch.isnan(gs), torch.full_like(gs, -math.inf), gs)
        order = torch.sort(gs, dim=1, descending=True, stable=True).indices[:, :topk_group]
        kept = torch.zeros_like(gs, dtype=torch.bool).scatter_(1, order, True) & (gs > -math.inf)
        key = torch.where(kept.repeat_interleave(gsz, dim=1), key, torch.full_like(key, -math.inf))
    srt = torch.sort(key, dim=1, descending=True, stable=True)
    ids = torch.where(srt.values[:, :k] > -math.inf, srt.indices[:, :k], torch.full_like(srt.indices[:, :k], E))
    return ids.t()


def check_ids(what, scores, bias, idx, top, k, n_group, topk_group):
    S, E = scores.shape
    want = ref_select(scores, bias, k, n_group, topk_group)
    got = idx.long()
    got = torch.where((got < 0) | (got >= E), torch.full_like(got, E), got)
    assert_equal('ids (keys = kernel score + bias, groups, ties to the lower id): ' + what, got, want)
    valid = want < E
    at = scores.t().gather(0, want.clamp(max=E - 1))
    assert_equal('top (unbiased kernel score at idx, 0 where nothing was chosen): ' + what, top,
                 torch.where(valid, at, torch.zeros_like(at)))
    return valid


# ------------------------------------------------------------------------------------------------------------------
# gates, loss
# ------------------------------------------------------------------------------------------------------------------
def ref_gates(top, normalize, eps, scale):
    """gates = scale * (top / max(sum top, eps)) (normalize and k > 1) in fp64 from the kernel's top: the shuffle sum
    of k non-negative terms (min(k - 1, 5) roundings), the division and the product with scale (1u each).
    Otherwise gates = fl(scale * top) exactly (bound None)."""
    k = top.size(0)
    if not (normalize and k > 1):
        return (top.float() * torch.tensor(scale, dtype=torch.float32)), None
    t = top.double()
    val = float(torch.tensor(scale, dtype=torch.float32)) * t / t.sum(0, keepdim=True).clamp_min(eps)
    return val, (min(k - 1, 5) + 2) * U * val.abs() * SLACK + TINY


def check_gates(what, top, gates, normalize, eps, scale, mask):
    val, bound = ref_gates(top, normalize, eps, scale)
    if bound is None:
        assert_equal('gates (= scale * top): ' + what, gates, val, mask)
    else:
        assert_within('gates: ' + what, gates, val, bound, mask=mask)


def ref_l_aux(scores, counts, k, dtype):
    """l_aux = E / (k S^2) sum_e n_e sum_s p_se / T_s in fp64 from the kernel's scores and all-choice counts.
    Kernel: T_s as ceil(E/32) lane terms + 5 shuffle adds, 1 / T_s and the product (fma) with p: ceil(E/32) + 6
    roundings on each (positive) term; then the accumulation of the softmax loss (8 tokens per lane and tile, 32
    warps' shared atomics, the tiles, the product with n_e, ceil(E/256) terms per thread, 5 shuffle adds, 8 warp
    partials) and k * S * S, the multiply by E and the division (4).  Then half an ulp of the logits dtype."""
    S, E = scores.shape
    p = scores.double()
    val = ((p / p.sum(1, keepdim=True)).sum(0) * counts.double()).sum() * E / (k * S * S)
    rel = (_lanes(E) + 6 + 8 + 32 + -(-S // 256) + 1 + -(-E // 256) + 5 + 8 + 4) * U
    acc = rel * val.abs() * SLACK + TINY
    return val, acc, (_out_half_ulp(val, acc, dtype) if dtype != torch.float32 else 0.0)


def check_l_aux(what, scores, counts, k, l_aux):
    val, acc, rnd = ref_l_aux(scores, counts, k, l_aux.dtype)
    assert_within('l_aux: ' + what, l_aux.reshape(1), val.reshape(1), acc.reshape(1), rnd)


def check_forward(what, logits, bias, k, C, normalize, eps, n_group, topk_group, scale, outs, check_loss=True):
    """All outputs of sigmoid_gate_route_forward: [scores, idx, top, gates, loc, counts, ce, l_aux(, slot)].
    Returns the [k, S] mask of choices that route somewhere."""
    scores, idx, top, gates, loc, counts, ce, l_aux = outs[:8]
    slot = outs[8] if len(outs) > 8 else None
    S, E = logits.shape
    check_scores(what, logits, scores)
    valid = check_ids(what, scores, bias, idx, top, k, n_group, topk_group)
    check_gates(what, top, gates, normalize, eps, scale, torch.ones_like(valid))
    check_locations(what, idx, E, C, loc, counts, None, slot)
    assert_equal('ce (all-choice counts as fp32): ' + what, ce, counts.float())
    if check_loss:
        check_l_aux(what, scores, counts, k, l_aux)
    return valid


# ------------------------------------------------------------------------------------------------------------------
# backward (closed form, fp64 on the kernel's scores / idx / top / all-choice counts)
# ------------------------------------------------------------------------------------------------------------------
def ref_backward(scores, idx, top, dgates, ce, dl, normalize, eps, scale, k_loss, dtype):
    """d logits [S, E] and its bound:

        r_j = top_j, D = sum_j r_j, Dc = max(D, eps)
        dr_j = scale (dg_j / Dc - [D > eps] (sum_i dg_i r_i) / Dc^2)     (normalize and k > 1; else scale dg_j)
        T = sum_e p_e, m = sum_e n_e p_e / T, c = dl E / (k S^2 T)
        dp_e = c (n_e - m) + sum_j [idx_j == e] dr_j
        dlogit_e = p_e (1 - p_e) dp_e

    Rounding errors of the kernel: dr as in the softmax backward plus the product with scale (1u); dl E / (k S S)
    (4u), T as ceil(E/32) + 4 adds of positive terms, c = that / T (1u); sum n p as an fma chain of ceil(E/32) terms
    + 5 shuffle adds, m (1u); the difference (1u); the product with c (1u); dp one add; p (1 - p) dp (3u); then the
    output rounding.  Returns (val, acc, rnd, mask): rows whose D is within 8u of eps are masked."""
    S, E = scores.shape
    k = idx.size(0)
    p = scores.double()
    r = top.double().t()
    ids = idx.t().long()
    sc = float(torch.tensor(scale, dtype=torch.float32))
    dg = dgates.double().t() if dgates is not None else torch.zeros_like(r)
    mask = torch.ones(S, dtype=torch.bool, device=p.device)
    if normalize and k > 1:
        D = r.sum(1, keepdim=True)
        Dc = D.clamp_min(eps)
        on = D > eps
        dot = (dg * r).sum(1, keepdim=True)
        sdot = (dg * r).abs().sum(1, keepdim=True)
        dr = dg / Dc - torch.where(on, dot / (Dc * Dc), torch.zeros_like(dot))
        dr_err = 6 * U * (dg / Dc).abs() + torch.where(on, 18 * U * sdot / (Dc * Dc), torch.zeros_like(sdot)) + U * dr.abs()
        mask = ((D - eps).abs() > 8 * U * D).view(S)
    else:
        dr, dr_err = dg, torch.zeros_like(dg)
    dr, dr_err = sc * dr, sc * dr_err + U * (sc * dr).abs()
    a = torch.zeros_like(p)
    a_err = torch.zeros_like(p)
    if ce is not None and dl is not None:
        n = ce.double()[None, :]
        L = _lanes(E)
        T = p.sum(1, keepdim=True)
        c = float(dl) * E / (k_loss * S * S) / T
        c_rel = (4 + L + 4 + 1) * U
        nd = (n * p).sum(1, keepdim=True)
        m = nd / T
        m_err = ((L + 5) + (L + 4) + 1) * U * m.abs()
        diff = n - m
        a = c * diff
        a_err = c.abs() * (m_err + U * diff.abs()) + (c_rel + U) * a.abs()
    valid = (ids >= 0) & (ids < E)
    safe = torch.where(valid, ids, torch.zeros_like(ids))
    zero = torch.zeros_like(dr)
    dp = a.clone().scatter_add_(1, safe, torch.where(valid, dr, zero))
    dp_err = a_err.clone().scatter_add_(1, safe, torch.where(valid, dr_err, zero)) + U * dp.abs()
    w = p * (1 - p)
    val = w * dp
    err = (w * dp_err + 3 * U * val.abs()) * SLACK + TINY
    return val, err, (_out_half_ulp(val, err, dtype) if dtype in (torch.float16, torch.bfloat16) else 0.0), mask


def check_backward(what, dlogits, scores, idx, top, dgates, ce, dl, normalize, eps, scale, row_mask=None):
    k = idx.size(0)
    val, acc, rnd, mask = ref_backward(scores, idx, top, dgates, ce, dl, normalize, eps, scale, k, dlogits.dtype)
    if row_mask is not None:
        mask = mask & row_mask
    m = mask[:, None].expand_as(val)
    assert_within('gate backward: ' + what, dlogits, val, acc, rnd, m)
