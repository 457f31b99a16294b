"""fp64 references of the combine with the shared experts' term and of its backward (csrc/moe_kernels.cu:
decode_rows_kernel and gate_grad_kernel with shared experts), with per-element bounds in the style of
dispatch_reference.py.

Forward, per token s and column m (w_s = 1, or sigmoid of the fp32 shared logit):

    out[s] = T( fmaf chain over the nsel valid routed choices in choice order, then fmaf(w_s, base[s], .) )

Backward of the combine (dy = gradient of out):

    d_buf[slot]        = T(g_j[s] * dy[s])               (the encode of dy, exact: dispatch_reference.ref_encode)
    d_gates[j, s]      = <dy[s], buf[slot_j(s)]>          (fp32, 0 for a dropped choice)
    d_base[s]          = T(w_s * dy[s])                   (dy itself without the shared gate)
    d_shared_logit[s]  = w_s (1 - w_s) <dy[s], base[s]>   (fp32)

Bounds, with u = 2^-24 (one fp32 rounding):

* the kernel's weight ``1 / (1 + expf(-l))`` (IEEE division, no fast-math intrinsics): expf is within 2 ulp (4u
  relative), ``1 + e`` and the division one rounding each, so w_s is within ``SIG_REL = 6u`` of sigmoid(l) relative;
* decode: nsel + 1 fmaf roundings, each at most u times the sum of the magnitudes of all terms, plus w_s's own error on
  the shared term, then half an output ulp;
* d_base: w_s's error and the product's rounding, then half an output ulp;
* d_shared_logit: the dot product as gate_grad's (ceil(M/32) + 7 + 5) u sum|a b|; the weight w (1 - w) is within
  ``SIG_REL sigma^2 + (SIG_REL + 3u) sigma (1 - sigma)`` of sigma (1 - sigma) (the 1 - w subtraction and two products
  add one rounding each).
"""
from typing import Optional

import torch

from dispatch_reference import SLACK, TINY, U, _out_half_ulp, assert_equal, assert_within, ref_encode
from gemm_reference import half_ulp

SIG_REL = 6 * U


def ref_weight(shared_logit: Optional[torch.Tensor]) -> Optional[torch.Tensor]:
    """fp64 sigmoid of the fp32 logits the kernel read, [S, 1]; None (weight 1) without the shared gate."""
    if shared_logit is None:
        return None
    l = shared_logit.float().double().view(-1, 1)
    return 1.0 / (1.0 + torch.exp(-l))


def _rows(idx, loc, E, C, seg_off=None):
    """Buffer row of every choice [k, S] and its validity (padded: e*C + l; packed: seg_off[e] + l, C = R)."""
    valid = (idx >= 0) & (idx < E) & (loc >= 0) & (loc < C)
    e = torch.where(valid, idx.long(), torch.zeros_like(idx, dtype=torch.long))
    l = torch.where(valid, loc.long(), torch.zeros_like(loc, dtype=torch.long))
    row = (seg_off.long()[e] if seg_off is not None else e * C) + l
    return valid, row


def ref_decode_shared(buf, gates, idx, loc, E, C, base, shared_logit=None, seg_off=None):
    """(val, acc, rnd) of the combine with the shared term; ``buf`` is [E*C, M] (padded) or [R, M] (packed, C = R)."""
    valid, row = _rows(idx, loc, E, C, seg_off)
    if buf.size(0) > 0:
        y = buf.double()[row]                                                    # [k, S, M]
    else:                                                                        # C = 0: every choice is dropped
        y = torch.zeros(tuple(idx.shape) + (base.size(1),), dtype=torch.float64, device=buf.device)
    w = gates.double() if gates is not None else torch.ones(idx.shape, dtype=torch.float64, device=buf.device)
    w = torch.where(valid, w, torch.zeros_like(w))
    terms = w[..., None] * y
    ws = ref_weight(shared_logit)
    sh = base.double() if ws is None else ws * base.double()
    val = terms.sum(0) + sh
    mag = terms.abs().sum(0) + sh.abs()
    acc = (valid.sum(0)[:, None] + 1) * U * mag
    if ws is not None:
        acc = acc + SIG_REL * sh.abs()
    acc = acc * SLACK + TINY
    return val, acc, _out_half_ulp(val, acc, buf.dtype)


def check_decode_shared(what, out, buf, gates, idx, loc, E, C, base, shared_logit=None, seg_off=None):
    val, acc, rnd = ref_decode_shared(buf, gates, idx, loc, E, C, base, shared_logit, seg_off)
    return assert_within('decode+shared: ' + what, out, val, acc, rnd)


def ref_gate_grad(a, buf, idx, loc, E, C, seg_off=None):
    """d_gates [k, S] in fp64 and its bound (dispatch_reference.ref_gate_grad, padded or packed)."""
    valid, row = _rows(idx, loc, E, C, seg_off)
    prod = a.double()[None] * buf.double()[row]
    M = a.size(1)
    val = torch.where(valid, prod.sum(-1), torch.zeros(valid.shape, dtype=torch.float64, device=a.device))
    bound = (-(-M // 32) + 7 + 5) * U * prod.abs().sum(-1) * SLACK + TINY
    return val, bound, valid


def check_gate_grad(what, out, a, buf, idx, loc, E, C, seg_off=None):
    val, bound, valid = ref_gate_grad(a, buf, idx, loc, E, C, seg_off)
    assert_within('d_gates: ' + what, out, val, bound, mask=valid)
    if not bool(valid.all()):
        nz = int((out[~valid] != 0).sum())
        assert nz == 0, 'd_gates of a dropped choice: %s: %d values are not 0' % (what, nz)


def ref_d_base(dy, shared_logit):
    """(val, acc, rnd) of d_base = w_s dy[s]; without the shared gate d_base is dy exactly (acc None)."""
    ws = ref_weight(shared_logit)
    if ws is None:
        return dy.double(), None, 0.0
    val = ws * dy.double()
    acc = (SIG_REL + U) * val.abs() * SLACK + TINY
    rnd = half_ulp(val.abs() + acc, dy.dtype) if dy.dtype != torch.float32 else 0.0
    return val, acc, rnd


def check_d_base(what, d_base, dy, shared_logit):
    val, acc, rnd = ref_d_base(dy, shared_logit)
    if acc is None:
        assert_equal('d_base (= dy): ' + what, d_base, dy)
        return 0.0
    return assert_within('d_base: ' + what, d_base, val, acc, rnd)


def ref_d_shared_logit(dy, base, shared_logit):
    """(val, bound) of d_shared_logit = sigma (1 - sigma) <dy[s], base[s]> (fp32 output)."""
    sig = ref_weight(shared_logit).view(-1)
    prod = dy.double() * base.double()
    dot = prod.sum(1)
    M = dy.size(1)
    dot_err = (-(-M // 32) + 7 + 5) * U * prod.abs().sum(1)
    d = sig * (1 - sig)
    val = d * dot
    bound = ((SIG_REL * sig * sig + (SIG_REL + 3 * U) * d) * dot.abs() + d * dot_err) * SLACK + TINY
    return val, bound


def check_d_shared_logit(what, d_logit, dy, base, shared_logit):
    val, bound = ref_d_shared_logit(dy, base, shared_logit)
    return assert_within('d_shared_logit: ' + what, d_logit.view(-1), val, bound)


def check_d_buf(what, d_buf, dy, gates, slot, k, E, C):
    """d_buf is the encode of dy (scaled by the routed gates when they are applied after the experts): exact."""
    want, _ = ref_encode(dy, gates, slot, k, E, C)
    assert_equal('d_buf: ' + what, d_buf.reshape(want.shape), want)
