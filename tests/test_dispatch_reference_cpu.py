"""The routing / dispatch references and checkers (tests/dispatch_reference.py) on CPU.

Faithful fp32 emulations of the kernels pass every check, and each near miss - one plausible kernel bug - is
rejected by the checker that guards it.  The closed form of the gate backward is also checked once against fp64
autograd of softmax -> gather -> normalise -> loss, so the reference does not just restate the kernel's formula.
"""
import re

import pytest
import torch

import dispatch_reference as R

INVALID_ID = 0x7fffffff
S_, E_, K_, C_ = 600, 40, 3, 30


def _logits(S=S_, E=E_, seed=0):
    """Random logits spread by tens, integer-valued rows (ties), rows holding -inf, and one NaN row."""
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(S, E, generator=gen) * 4
    x[: S // 3] = torch.randint(-2, 3, (S // 3, E), generator=gen).float()
    x[S // 3: S // 3 + 20, ::3] = -float('inf')
    x[S // 2, 5] = float('nan')
    return x


# ------------------------------------------------------------------------------------------------------------------
# fp32 emulations of the kernels (``miss`` selects a near miss)
# ------------------------------------------------------------------------------------------------------------------
def _lane_sum(t):
    """gate_route_kernel's reduction of t [S, E]: lane l sums experts l, l+32, ... in order, then 5 xor shuffles."""
    S, E = t.shape
    vpt = -(-E // 32)
    lanes = torch.zeros(S, 32 * vpt, dtype=torch.float32)
    lanes[:, :E] = t
    lanes = lanes.view(S, vpt, 32)
    acc = lanes[:, 0].clone()
    for i in range(1, vpt):
        acc = acc + lanes[:, i]
    lane = torch.arange(32)
    for o in (16, 8, 4, 2, 1):
        acc = acc + acc[:, lane ^ o]
    return acc[:, :1]


def emulate_locations(idx, E, C, token_major=False):
    k, S = idx.shape
    order = idx.t().reshape(-1) if token_major else idx.reshape(-1)
    valid = (order >= 0) & (order < E)
    onehot = torch.nn.functional.one_hot(torch.where(valid, order, 0).long(), E) * valid[:, None]
    pos = (torch.cumsum(onehot, 0) - 1).gather(1, torch.where(valid, order, 0).long()[:, None])[:, 0]
    pos = torch.where(valid, pos, torch.full_like(pos, R.INVALID_LOC)).to(torch.int32)
    loc = pos.view(S, k).t().contiguous() if token_major else pos.view(k, S)
    counts = onehot.sum(0).to(torch.int32)
    ce = torch.bincount(idx[0][(idx[0] >= 0) & (idx[0] < E)].long(), minlength=E).float()
    slot = torch.full((E * C,), -1, dtype=torch.int32)
    for j in range(k):
        for s in range(S):
            e, l = int(idx[j, s]), int(loc[j, s])
            if 0 <= e < E and l < C:
                slot[e * C + l] = s * k + j
    return loc, counts, ce, slot


def emulate_gate_route(logits, k, C, normalize, eps, miss=None):
    v = logits.float()
    S, E = v.shape
    mx = v.nan_to_num(nan=-float('inf')).amax(1, keepdim=True)        # fmaxf ignores NaN
    ex = torch.exp(v - mx)
    p = ex * (1.0 / _lane_sum(ex))
    nan_row = torch.isnan(p).any(1)
    if miss == 'ties_to_higher_id':
        order = E - 1 - torch.sort(p.flip(1), dim=1, descending=True, stable=True).indices
    else:
        order = torch.sort(p, dim=1, descending=True, stable=True).indices
    idx = order[:, :k].t().contiguous().to(torch.int32)
    idx[:, nan_row] = INVALID_ID
    top = p.gather(1, idx.t().long().clamp(max=E - 1)).t().contiguous()
    top[:, nan_row] = -1.0
    gates = top / torch.clamp(_lane_sum(top.t().contiguous()).t(), min=eps) if normalize and k > 1 else top.clone()
    loc, counts, ce, slot = emulate_locations(idx, E, C, token_major=miss == 'token_major_queue')
    me = p.sum(0)
    l_aux = (me * ce).sum() * E / (S if miss == 'l_aux_over_S' else S * S)
    return [p, idx, top, gates, loc, counts, ce, l_aux.to(logits.dtype), slot]


def emulate_encode(x, gates, slot, k, E, C, valid_rows=None, out=None, miss=None):
    empty, tok, g = R._slot_sources(slot, k, gates)
    rows = x[tok]
    if g is not None:
        if miss == 'gate_rounded_first':
            g = g.to(x.dtype).float()
        rows = (rows.float() * g[:, None]).to(x.dtype)
    rows[empty] = 0
    res = out.clone()
    write = torch.ones(E * C, dtype=torch.bool)
    if valid_rows is not None and miss != 'zero_fill_past_valid_rows':
        write = (torch.arange(C)[None, :] < valid_rows.long()[:, None]).reshape(-1)
    res[write] = rows[write]
    if miss == 'zero_fill_past_valid_rows':
        past = (torch.arange(C)[None, :] >= valid_rows.long()[:, None]).reshape(-1)
        res[past] = 0
    return res


def emulate_encode_fp8(x, gates, slot, k, E, C, miss=None):
    empty, tok, g = R._slot_sources(slot, k, gates)
    xf = x.float()[tok]
    amax = xf.abs().amax(1)
    if miss != 'fp8_scale_without_gate':
        amax = amax * g.abs()
    sc = torch.where(amax > 0, (amax * R.F448).clamp_min(R.FLT_MIN), torch.ones_like(amax))
    q = (xf * (g / sc)[:, None]).clamp(-448, 448).to(torch.float8_e4m3fn).view(torch.uint8)
    q[empty] = 0
    sc[empty] = 1.0
    return q, sc


def _fmaf(a, b, c):
    """fp32 fma: the exact product plus c in fp64, one rounding to fp32."""
    return (a.double() * b.double() + c.double()).float()


def emulate_decode(buf, gates, idx, loc, E, C, miss=None):
    k, S = idx.shape
    M = buf.size(1)
    g = gates.clone() if gates is not None else torch.ones(k, S)
    if miss == 'gates_of_choices_swapped':
        g[[0, 1]] = g[[1, 0]]
    acc = torch.zeros(S, M)
    for j in range(k):
        e, l = idx[j].long(), loc[j].long()
        ok = (e >= 0) & (e < E) & (l >= 0) & (l < C)
        y = buf[torch.where(ok, e * C + l, 0)].float()
        nxt = _fmaf(g[j][:, None].expand(S, M), y, acc)
        if miss == 'accumulate_in_16_bit':
            nxt = nxt.to(buf.dtype).float()
        acc = torch.where(ok[:, None], nxt, acc)
    return acc.to(buf.dtype)


def emulate_gate_grad(a, buf, idx, loc, E, C, miss=None):
    k, S = idx.shape
    out = torch.zeros(k, S)
    for j in range(k):
        e, l = idx[j].long(), loc[j].long()
        ok = (e >= 0) & (e < E) & (l >= 0) & (l < C)
        row = torch.where(ok, e * C + l, 0)
        if miss == 'dropped_choice_reads_padded_row':
            dropped = (e >= 0) & (e < E) & (l >= C)
            row = torch.where(dropped, e * C + C - 1, row)
            ok = ok | dropped
        out[j] = torch.where(ok, (a.float() * buf[row].float()).sum(1), torch.zeros(()))
    return out


def emulate_gate_backward(scores, idx, top, dgates, ce, dl, normalize, eps, dtype, miss=None):
    S, E = scores.shape
    k = idx.size(0)
    p = scores.float()
    r = top.t()
    dg = dgates.t() if dgates is not None else torch.zeros(S, k)
    dp = torch.zeros(S, E)
    if ce is not None and miss != 'gate_bwd_without_loss_term':
        dp += (float(dl) * E / (S * S)) * ce[None, :]
    if normalize and k > 1:
        D = r.sum(1, keepdim=True)
        Dc = D.clamp_min(eps)
        corr = (dg * r).sum(1, keepdim=True) / (Dc * Dc)
        if miss != 'gate_bwd_without_eps_indicator':
            corr = torch.where(D > eps, corr, torch.zeros_like(corr))
        dr = dg / Dc - corr
    else:
        dr = dg
    ids = idx.t().long()
    ok = (ids >= 0) & (ids < E)
    dp.scatter_add_(1, torch.where(ok, ids, 0), torch.where(ok, dr, torch.zeros(())))
    acc = _lane_sum(dp * p)
    return (p * (dp - acc)).to(dtype)


# ------------------------------------------------------------------------------------------------------------------
# shared data
# ------------------------------------------------------------------------------------------------------------------
def _routing(S=S_, E=E_, k=K_, C=C_, seed=1):
    gen = torch.Generator().manual_seed(seed)
    idx = torch.topk(torch.rand(S, E, generator=gen), k, dim=1).indices.t().contiguous().to(torch.int32)
    idx[0, 7] = -1
    idx[min(1, k - 1), 11] = E + 3
    loc, _, _, slot = R.ref_locations(idx, E, C)
    gates = torch.rand(k, S, generator=gen) * 2 - 0.5
    return idx, loc, slot, gates


def _rows(S, M, dtype, seed=2):
    gen = torch.Generator().manual_seed(seed)
    return (torch.randn(S, M, generator=gen) * 3).to(dtype)


# ------------------------------------------------------------------------------------------------------------------
# the emulations pass
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize('normalize,eps', [(True, 1e-3), (False, 1e-3), (True, 2.0)])
def test_emulated_gate_route_passes(dtype, normalize, eps):
    x = _logits().to(dtype)
    outs = emulate_gate_route(x, K_, C_, normalize, eps)
    routable = R.check_gate_route_forward('emulated', x, K_, C_, normalize, eps, outs, check_loss=False)
    assert int((~routable).sum()) == 1
    clean = x.clone()
    clean[S_ // 2, 5] = 0.0                                            # l_aux is NaN while a NaN row is routed
    outs = emulate_gate_route(clean, K_, C_, normalize, eps)
    R.check_gate_route_forward('emulated', clean, K_, C_, normalize, eps, outs)


def test_emulated_locations_match_reference():
    idx, _, _, _ = _routing(S=300, E=7, k=4, C=50)
    want = R.ref_locations(idx, 7, 50)
    for got, ref in zip(emulate_locations(idx, 7, 50), want):
        assert torch.equal(got, ref)


@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16, torch.float16])
def test_emulated_gate_backward_passes(dtype):
    x = _logits(seed=3).to(dtype)
    scores, idx, top, _, _, _, ce, _, _ = emulate_gate_route(x, K_, C_, True, 1e-3)
    routable = ~torch.isnan(scores).any(1)
    gen = torch.Generator().manual_seed(4)
    dg = torch.randn(K_, S_, generator=gen)
    dl = torch.tensor(3.0).to(dtype)
    for dgates, c, d, normalize, eps in ((dg, ce, dl, True, 1e-3), (None, ce, dl, True, 1e-3), (dg, None, None, True, 1e-3),
                                         (dg, ce, dl, False, 1e-3), (dg, ce, dl, True, 2.0)):
        out = emulate_gate_backward(scores, idx, top, dgates, c, d, normalize, eps, dtype)
        R.check_gate_backward('emulated', out, scores, idx, top, dgates, c, d, normalize, eps, routable)


@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16, torch.float16])
def test_emulated_encode_decode_gate_grad_pass(dtype):
    idx, loc, slot, gates = _routing()
    x = _rows(S_, 72, dtype)
    vr = torch.tensor([0, 5, C_ + 9] * 13 + [C_], dtype=torch.int32)
    for g in (gates, None):
        for valid_rows in (None, vr):
            sentinel = torch.full((E_ * C_, 72), -7.0).to(dtype)
            out = emulate_encode(x, g, slot, K_, E_, C_, valid_rows, sentinel)
            R.check_encode('emulated', out, x, g, slot, K_, E_, C_, valid_rows, -7.0)
        buf = _rows(E_ * C_, 72, dtype, seed=5)
        R.check_decode('emulated', emulate_decode(buf, g, idx, loc, E_, C_), buf, g, idx, loc, E_, C_)
    R.check_gate_grad('emulated', emulate_gate_grad(x, buf, idx, loc, E_, C_), x, buf, idx, loc, E_, C_)


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16])
def test_emulated_fp8_encode_dequant_passes(dtype):
    idx, loc, slot, gates = _routing()
    x = _rows(S_, 64, dtype)
    x[3] = 0                                                           # amax 0 -> scale 1
    q, sc = emulate_encode_fp8(x, gates, slot, K_, E_, C_)
    R.check_encode_fp8('emulated', q, sc, x, gates, slot, K_, E_, C_)
    R.assert_equal('dequant', R.ref_dequant(q, sc, dtype), (q.view(torch.float8_e4m3fn).float() * sc[:, None]).to(dtype))


def test_e4m3_conversion_saturates_like_the_kernels():
    v = torch.tensor([470.0, -1000.0, 448.0, 447.0, 0.0, -0.0])
    assert R.to_e4m3(v).tolist() == [0x7e, 0xfe, 0x7e, 0x7e, 0x00, 0x80]
    assert torch.isnan(torch.tensor([470.0]).to(torch.float8_e4m3fn).float()).all()   # why the reference clamps


def test_quantize_transpose_reference_matches_row_quantisation_of_the_transpose():
    gen = torch.Generator().manual_seed(6)
    x = (torch.randn(2, 128, 64, generator=gen) * 0.3).bfloat16()
    x[1, :, 5] = 0
    q, sc = R.ref_quantize_transpose(x)
    xt = x.transpose(1, 2).float()
    amax = xt.abs().amax(-1)
    s = torch.where(amax > 0, amax * R.F448, torch.ones_like(amax))
    assert torch.equal(sc, s) and float(sc[1, 5]) == 1.0
    assert torch.equal(q, R.to_e4m3(xt * (1.0 / s)[..., None]))


@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
def test_emulated_colsum_passes(dtype):
    x = _rows(3 * 500, 64, dtype).view(3, 500, 64)
    R.check_colsum('emulated', x.float().sum(1).to(dtype), x)


@pytest.mark.parametrize('normalize,eps', [(True, 1e-3), (True, 2.0), (False, 1e-3)])
def test_gate_backward_closed_form_matches_fp64_autograd(normalize, eps):
    S, E, k = 200, 24, 3
    gen = torch.Generator().manual_seed(7)
    logits = (torch.randn(S, E, generator=gen, dtype=torch.float64) * 2).requires_grad_(True)
    p = torch.softmax(logits, dim=1)
    idx = torch.topk(p.detach(), k, dim=1).indices.t().contiguous().to(torch.int32)
    ce = torch.bincount(idx[0].long(), minlength=E).double()
    dg = torch.randn(k, S, generator=gen, dtype=torch.float64)
    dl = 1.7
    top = p.gather(1, idx.t().long())
    g = top / top.sum(1, keepdim=True).clamp_min(eps) if normalize else top
    loss = (g * dg.t()).sum() + dl * (p.sum(0) * ce).sum() * E / (S * S)
    loss.backward()
    val, _, _, mask = R.ref_gate_backward(p.detach(), idx, top.detach().t(), dg, ce, dl, normalize, eps, torch.float32)
    assert bool(mask.all())
    assert torch.allclose(val, logits.grad, rtol=1e-12, atol=1e-15)


# ------------------------------------------------------------------------------------------------------------------
# each near miss is rejected, by the check that guards it
# ------------------------------------------------------------------------------------------------------------------
def _rejects(miss, match, fn):
    try:
        fn()
    except AssertionError as e:
        assert re.search(match, str(e)), 'near miss %r was rejected by the wrong check: %s' % (miss, e)
        return
    pytest.fail('near miss %r was accepted' % miss)


def _miss_gate_route(miss, dtype=torch.float32):
    x = _logits().to(dtype)
    x[S_ // 2, 5] = 0.0
    R.check_gate_route_forward(str(miss), x, K_, C_, True, 1e-3, emulate_gate_route(x, K_, C_, True, 1e-3, miss=miss))


def _miss_encode(miss, dtype=torch.bfloat16):
    idx, loc, slot, gates = _routing()
    x = _rows(S_, 72, dtype)
    vr = torch.tensor([0, 5, C_ + 9] * 13 + [C_], dtype=torch.int32)
    sentinel = torch.full((E_ * C_, 72), -7.0).to(dtype)
    R.check_encode(str(miss), emulate_encode(x, gates, slot, K_, E_, C_, vr, sentinel, miss=miss), x, gates, slot, K_, E_, C_,
                   vr, -7.0)


def _miss_decode(miss, dtype=torch.bfloat16):
    idx, loc, slot, gates = _routing()
    buf = _rows(E_ * C_, 72, dtype, seed=5)
    R.check_decode(str(miss), emulate_decode(buf, gates, idx, loc, E_, C_, miss=miss), buf, gates, idx, loc, E_, C_)


def _miss_gate_grad(miss, dtype=torch.bfloat16):
    idx, loc, slot, gates = _routing()
    x, buf = _rows(S_, 72, dtype), _rows(E_ * C_, 72, dtype, seed=5)
    R.check_gate_grad(str(miss), emulate_gate_grad(x, buf, idx, loc, E_, C_, miss=miss), x, buf, idx, loc, E_, C_)


def _miss_fp8(miss, dtype=torch.bfloat16):
    idx, loc, slot, gates = _routing()
    x = _rows(S_, 64, dtype)
    q, sc = emulate_encode_fp8(x, gates, slot, K_, E_, C_, miss=miss)
    R.check_encode_fp8(str(miss), q, sc, x, gates, slot, K_, E_, C_)


def _miss_gate_bwd(miss, eps, dtype=torch.float32):
    x = _logits(seed=3).to(dtype)
    x[S_ // 2, 5] = 0.0
    scores, idx, top, _, _, _, ce, _, _ = emulate_gate_route(x, K_, C_, True, eps)
    dg = torch.randn(K_, S_, generator=torch.Generator().manual_seed(4))
    dl = torch.tensor(3.0)
    out = emulate_gate_backward(scores, idx, top, dg, ce, dl, True, eps, dtype, miss=miss)
    R.check_gate_backward(str(miss), out, scores, idx, top, dg, ce, dl, True, eps, torch.ones(S_, dtype=torch.bool))


NEAR_MISSES = {
    'ties_to_higher_id': ('top-k ids', lambda m: _miss_gate_route(m)),
    'token_major_queue': ('loc', lambda m: _miss_gate_route(m)),
    'gate_rounded_first': ('encode:', lambda m: _miss_encode(m)),
    'zero_fill_past_valid_rows': ('past valid_rows', lambda m: _miss_encode(m)),
    'accumulate_in_16_bit': ('decode:', lambda m: _miss_decode(m)),
    'gates_of_choices_swapped': ('decode:', lambda m: _miss_decode(m)),
    'dropped_choice_reads_padded_row': ('dropped choice', lambda m: _miss_gate_grad(m)),
    'fp8_scale_without_gate': ('fp8 encode scales', lambda m: _miss_fp8(m)),
    'gate_bwd_without_eps_indicator': ('gate backward', lambda m: _miss_gate_bwd(m, eps=0.9)),
    'gate_bwd_without_loss_term': ('gate backward', lambda m: _miss_gate_bwd(m, eps=1e-3)),
    'l_aux_over_S': ('l_aux', lambda m: _miss_gate_route(m)),
}


@pytest.mark.parametrize('miss', list(NEAR_MISSES))
def test_near_miss_is_rejected(miss):
    match, fn = NEAR_MISSES[miss]
    fn(None)                                                           # the faithful emulation passes on the same data
    _rejects(miss, match, lambda: fn(miss))


def test_rounding_the_gate_first_is_visible_in_every_16_bit_dtype():
    for dtype in (torch.float16, torch.bfloat16):
        _rejects('gate_rounded_first', 'encode:', lambda: _miss_encode('gate_rounded_first', dtype))
