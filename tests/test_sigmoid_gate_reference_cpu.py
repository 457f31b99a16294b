"""The sigmoid gate reference and checkers (tests/sigmoid_gate_reference.py) on CPU.

An fp32 emulation of the sigmoid kernels passes every check, and each near miss - one plausible kernel bug - is
rejected.  The op-by-op definition (ops/gating.py) passes the same checks, and the closed-form backward of the
reference matches fp64 autograd of that definition.
"""
import math
import re

import pytest
import torch

import dispatch_reference as DR
import sigmoid_gate_reference as R
from tutel_b200.ops.gating import sigmoid_topk_gate

S_, E_, K_, C_ = 600, 48, 4, 40
G_, TG_ = 4, 2
SCALE = 2.5


def _logits(S=S_, E=E_, seed=0, nan=True):
    """Random logits, integer-valued rows (exact ties of keys and group scores), some -inf entries, one NaN."""
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(S, E, generator=gen) * 3
    x[: S // 3] = torch.randint(-2, 3, (S // 3, E), generator=gen).float()
    x[S // 3: S // 3 + 20, ::3] = -math.inf
    if nan:
        x[S // 2, 5] = math.nan
    return x


def _bias(E, kind, seed=1):
    gen = torch.Generator().manual_seed(seed)
    if kind == 'zero':
        return torch.zeros(E)
    if kind == 'random':
        return torch.randn(E, generator=gen) * 0.3
    return -5.0 - torch.rand(E, generator=gen)          # every key negative


# ------------------------------------------------------------------------------------------------------------------
# fp32 emulation of the kernels (``miss`` selects a near miss)
# ------------------------------------------------------------------------------------------------------------------
def _select(key, k, n_group, topk_group, miss):
    S, E = key.shape
    key = torch.where(torch.isnan(key), torch.full_like(key, -math.inf), key)
    excluded = torch.zeros(S, E, dtype=torch.bool)
    if n_group > 1:
        gsz = E // n_group
        srt = torch.sort(key.view(S, n_group, gsz), dim=2, descending=True).values
        gs = srt[:, :, 0] + srt[:, :, 1] if (gsz > 1 and miss != 'group top-1') else srt[:, :, 0]
        gs = torch.where(torch.isnan(gs), torch.full_like(gs, -math.inf), gs)
        kept = torch.zeros(S, n_group, dtype=torch.bool)
        for _ in range(topk_group):
            cand = torch.where(kept, torch.full_like(gs, -math.inf), gs)
            if miss == 'group ties high':
                g = n_group - 1 - torch.argmax(cand.flip(1), dim=1)
            else:
                g = torch.argmax(cand, dim=1)
            ok = cand.gather(1, g[:, None]).squeeze(1) > -math.inf
            kept[ok, g[ok]] = True
        excluded = ~kept.repeat_interleave(gsz, dim=1)
    sentinel = -1.0 if miss == 'sentinel -1' else -math.inf
    ids = torch.full((k, S), E, dtype=torch.int64)
    taken = excluded.clone()
    rows = torch.arange(S)
    for j in range(k):
        cand = torch.where(taken, torch.full_like(key, -math.inf), key)
        e = torch.argmax(cand, dim=1)
        ok = cand[rows, e] > sentinel
        ids[j] = torch.where(ok, e, torch.full_like(e, E))
        taken[rows[ok], e[ok]] = True
    return ids


def emulate_forward(logits, bias, k, C, normalize, eps, n_group, topk_group, scale, miss=None):
    S, E = logits.shape
    z = logits.float()
    scores = 1.0 / (1.0 + torch.exp(-z))
    key = scores if miss == 'no bias in selection' else scores + bias
    ids = _select(key, k, n_group, topk_group, miss)
    valid = ids < E
    src = key if miss == 'gates from key' else scores
    top = torch.where(valid, src.t().gather(0, ids.clamp(max=E - 1)), torch.zeros(()))
    sc = torch.tensor(scale, dtype=torch.float32)
    if normalize and k > 1:
        if miss == 'scale before normalising':
            t = top * sc
            gates = t / t.sum(0, keepdim=True).clamp_min(eps)
        else:
            gates = top / top.sum(0, keepdim=True).clamp_min(eps)
            if miss != 'scale omitted':
                gates = gates * sc
    else:
        gates = top if miss == 'scale omitted' else top * sc
    idx = ids.to(torch.int32)
    loc, counts, _ce, slot = DR.ref_locations(idx, E, C)
    n = counts.float()
    if miss == 'loss on first-choice counts':
        n = torch.bincount(ids[0][valid[0]], minlength=E)[:E].float()
    T = scores.sum(1, keepdim=True)
    me = (scores * (1.0 / T)).sum(0)
    l_aux = (me * n).sum() * E / (k * float(S * S))
    outs = [scores, idx, top, gates, loc, counts, counts.float(), l_aux.reshape(())]
    return outs + ([slot] if C > 0 else [])


def emulate_backward(scores, idx, top, dgates, ce, dl, normalize, eps, scale, miss=None):
    S, E = scores.shape
    k = idx.size(0)
    p, r = scores, top
    dg = dgates if dgates is not None else torch.zeros_like(r)
    dr = dg
    if normalize and k > 1:
        D = r.sum(0, keepdim=True)
        Dc = D.clamp_min(eps)
        dot = (dg * r).sum(0, keepdim=True)
        dr = dg / Dc - torch.where(D > eps, dot / (Dc * Dc), torch.zeros_like(dot))
    dr = dr * torch.tensor(scale, dtype=torch.float32)
    dp = torch.zeros_like(p)
    if ce is not None and dl is not None:
        aux_scale = torch.tensor(float(dl) * E / (k * float(S * S)), dtype=torch.float32)
        T = p.sum(1, keepdim=True)
        m = (ce[None] * p).sum(1, keepdim=True) / T
        dp = (aux_scale / T) * (ce[None] if miss == 'no T coupling' else (ce[None] - m))
    ids = idx.t().long()
    valid = ids < E
    dp = dp.scatter_add(1, ids.clamp(max=E - 1), torch.where(valid, dr.t(), torch.zeros(())))
    return p * (1 - p) * dp


def _check(outs, logits, bias, k, C, normalize, eps, n_group, topk_group, scale, check_loss=True):
    return R.check_forward('cpu', logits, bias, k, C, normalize, eps, n_group, topk_group, scale, outs, check_loss)


# ------------------------------------------------------------------------------------------------------------------
# the emulation passes
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('bias_kind', ['zero', 'random', 'negative'])
@pytest.mark.parametrize('n_group,topk_group', [(1, 1), (G_, TG_), (16, 3)])
@pytest.mark.parametrize('normalize', [True, False])
def test_emulation_passes(bias_kind, n_group, topk_group, normalize):
    logits, bias = _logits(), _bias(E_, bias_kind)
    eps = 1.1920928955078125e-07
    outs = emulate_forward(logits, bias, K_, C_, normalize, eps, n_group, topk_group, SCALE)
    _check(outs, logits, bias, K_, C_, normalize, eps, n_group, topk_group, SCALE, check_loss=False)
    clean = _logits(nan=False)
    outs = emulate_forward(clean, bias, K_, C_, normalize, eps, n_group, topk_group, SCALE)
    _check(outs, clean, bias, K_, C_, normalize, eps, n_group, topk_group, SCALE)
    gen = torch.Generator().manual_seed(3)
    dg = torch.randn(K_, S_, generator=gen)
    dl = torch.tensor(1.75)
    scores, idx, top, ce = outs[0], outs[1], outs[2], outs[6]
    for dgates, loss in [(dg, True), (None, True), (dg, False)]:
        d = emulate_backward(scores, idx, top, dgates, ce if loss else None, dl if loss else None, normalize, eps, SCALE)
        R.check_backward('cpu', d, scores, idx, top, dgates, ce if loss else None, dl if loss else None, normalize,
                         eps, SCALE)


def test_op_by_op_definition_passes():
    """The CPU / op-by-op path (ops/gating.py) against the same reference."""
    for n_group, topk_group, bias_kind in [(1, 1, 'random'), (G_, TG_, 'random'), (G_, 1, 'negative')]:
        logits, bias = _logits(nan=False), _bias(E_, bias_kind)
        idx, gates, l_aux, counts, top1 = sigmoid_topk_gate(logits, bias, K_, True, n_group, topk_group, SCALE)
        scores = torch.sigmoid(logits.float())
        eps = float(torch.finfo(torch.float32).eps)
        top = torch.where(idx < E_, scores.t().gather(0, idx.long().clamp(max=E_ - 1)), torch.zeros(()))
        valid = R.check_ids('op-by-op', scores, bias, idx, top, K_, n_group, topk_group)
        R.check_gates('op-by-op', top, gates.detach(), True, eps, SCALE, torch.ones_like(valid))
        want = torch.bincount(idx.long()[valid], minlength=E_)[:E_].float()
        DR.assert_equal('op-by-op counts', counts, want)
        R.check_l_aux('op-by-op', scores, counts.int(), K_, l_aux.detach())
        DR.assert_equal('op-by-op top1', top1, top[0])


# ------------------------------------------------------------------------------------------------------------------
# near misses
# ------------------------------------------------------------------------------------------------------------------
FWD_MISSES = {
    'gates from key': ('random', G_, TG_, True, 'top (unbiased'),
    'no bias in selection': ('random', 1, 1, True, 'ids'),
    'group top-1': ('random', G_, TG_, True, 'ids'),
    'group ties high': ('zero', G_, TG_, True, 'ids'),
    'sentinel -1': ('negative', 1, 1, True, 'ids'),
    'loss on first-choice counts': ('random', 1, 1, True, 'l_aux'),
    'scale before normalising': ('random', 1, 1, True, 'gates'),
    'scale omitted': ('random', 1, 1, True, 'gates'),
    'scale omitted (no normalisation)': ('random', 1, 1, False, 'gates'),
}


@pytest.mark.parametrize('miss', sorted(FWD_MISSES))
def test_forward_near_miss_rejected(miss):
    bias_kind, n_group, topk_group, normalize, check = FWD_MISSES[miss]
    logits, bias = _logits(nan=False), _bias(E_, bias_kind)
    eps = 1.1920928955078125e-07
    outs = emulate_forward(logits, bias, K_, C_, normalize, eps, n_group, topk_group, SCALE, miss=miss.split(' (')[0])
    with pytest.raises(AssertionError, match='^' + re.escape(check)):
        _check(outs, logits, bias, K_, C_, normalize, eps, n_group, topk_group, SCALE)


def test_backward_without_T_coupling_rejected():
    logits, bias = _logits(nan=False), _bias(E_, 'random')
    eps = 1.1920928955078125e-07
    outs = emulate_forward(logits, bias, K_, C_, True, eps, 1, 1, SCALE)
    scores, idx, top, ce = outs[0], outs[1], outs[2], outs[6]
    dl = torch.tensor(1.75)
    d = emulate_backward(scores, idx, top, None, ce, dl, True, eps, SCALE, miss='no T coupling')
    with pytest.raises(AssertionError, match='^gate backward'):
        R.check_backward('cpu', d, scores, idx, top, None, ce, dl, True, eps, SCALE)


# ------------------------------------------------------------------------------------------------------------------
# the closed form against fp64 autograd of the definition
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('normalize,n_group,topk_group', [(True, 1, 1), (True, G_, TG_), (False, G_, 1)])
def test_closed_form_backward_matches_autograd(normalize, n_group, topk_group):
    logits = _logits(nan=False).double()
    logits[torch.isinf(logits)] = -30.0
    logits.requires_grad_(True)
    bias = _bias(E_, 'random').double()
    idx, gates, l_aux, counts, _ = sigmoid_topk_gate(logits, bias, K_, normalize, n_group, topk_group, SCALE)
    gen = torch.Generator().manual_seed(5)
    dg = torch.randn(K_, S_, generator=gen, dtype=torch.float64)
    dl = 1.75
    ((gates * dg).sum() + dl * l_aux).backward()
    scores = torch.sigmoid(logits.detach())
    ids = idx.long()
    top = torch.where(ids < E_, scores.t().gather(0, ids.clamp(max=E_ - 1)), torch.zeros((), dtype=torch.float64))
    eps = float(torch.finfo(torch.float64).eps)
    val, _, _, _ = R.ref_backward(scores, idx, top, dg, counts, torch.tensor(dl), normalize, eps, SCALE, K_,
                                  torch.float64)
    assert torch.allclose(logits.grad, val, rtol=1e-9, atol=1e-15)
