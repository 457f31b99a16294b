"""The packed-layout reference (tests/packed_reference.py) against the padded routing + dispatch on CPU: the packed
buffer holds the same rows as the padded ``[E, C, M]`` buffer, only in other places, and decodes to the same tokens."""
import pytest
import torch

import packed_reference as P
from tutel_b200.ops import dispatch, routing
from tutel_b200.ops.packed import packed_rows


def _padded(idx, loc, counts, E):
    C = max(int(counts.max()), 1)
    return dispatch.DispatchPlan(E, C, idx, loc), C


# (E, k, S, counts) - empty experts, one-row experts, all tokens on one expert, exact multiples of 128, E up to 256
CASES = [
    (8, 2, 300, [0, 1, 128, 300, 0, 77, 38, 56]),
    (4, 1, 500, [500, 0, 0, 0]),
    (2, 1, 256, [128, 128]),
    (4, 2, 384, [384, 256, 128, 0]),
    (64, 8, 96, None),
    (256, 8, 64, None),
    (256, 1, 1000, None),
]


def _counts(E, k, S, counts, seed):
    if counts is not None:
        return counts
    g = torch.Generator().manual_seed(seed)
    # skewed: a few experts take most of the choices, some take none
    w = torch.rand(E, generator=g) ** 4
    w[torch.randperm(E, generator=g)[: E // 4]] = 0
    raw = torch.distributions.Multinomial(k * S, probs=w / w.sum()).sample().long()
    return [int(c) for c in raw]


@pytest.mark.parametrize('case', range(len(CASES)))
def test_layout_matches_padded(case):
    E, k, S, counts = CASES[case]
    counts = _counts(E, k, S, counts, case)
    idx, loc = P.routing_from_counts(counts, k, S, seed=case)
    R = P.packed_rows(S, k, E)
    assert R == packed_rows(S, k, E)
    seg, bexp, brows, slot = P.layout(idx, loc, torch.tensor(counts), R)
    # alignment, bound and block description
    assert int(seg[0]) == 0 and bool((seg % 128 == 0).all()) and int(seg[-1]) <= R
    assert int(brows.sum()) == sum(counts) and int(brows.max()) <= 128
    assert bool((brows[int(seg[-1]) // 128:] == 0).all())
    # every routed choice sits at seg_off[e] + loc; the padded slot map holds it at e * C + loc
    plan, C = _padded(idx, loc, torch.tensor(counts), E)
    padded_slot = plan.slot_src
    for e in range(E):
        n = counts[e]
        assert torch.equal(slot[int(seg[e]): int(seg[e]) + n], padded_slot[e * C: e * C + n]), e
        assert bool((slot[int(seg[e]) + n: int(seg[e + 1])] == -1).all())
        assert bool((bexp[int(seg[e]) // 128: int(seg[e + 1]) // 128] == e).all())
    assert int((slot >= 0).sum()) == k * S


@pytest.mark.parametrize('gated', [False, True])
@pytest.mark.parametrize('case', [0, 1, 3, 5])
def test_encode_decode_match_padded(case, gated):
    E, k, S, counts = CASES[case]
    counts = _counts(E, k, S, counts, case)
    idx, loc = P.routing_from_counts(counts, k, S, seed=case)
    R = P.packed_rows(S, k, E)
    seg, _, _, slot = P.layout(idx, loc, torch.tensor(counts), R)
    g = torch.Generator().manual_seed(case)
    M = 24
    x = torch.randn(S, M, generator=g, dtype=torch.float64)
    gates = torch.rand(k, S, generator=g, dtype=torch.float64) if gated else None
    plan, C = _padded(idx, loc, torch.tensor(counts), E)
    padded = dispatch.raw_encode(x, gates, plan).view(E, C, M)
    packed = P.encode(x, gates, slot, k)
    for e in range(E):
        n = counts[e]
        assert torch.equal(packed[int(seg[e]): int(seg[e]) + n], padded[e, :n]), e
        assert bool((packed[int(seg[e]) + n: int(seg[e + 1])] == 0).all())
    # decode: the same tokens from the same rows
    y = torch.randn(R, M, generator=g, dtype=torch.float64)
    y_padded = torch.zeros(E, C, M, dtype=torch.float64)
    for e in range(E):
        n = counts[e]
        y_padded[e, :n] = y[int(seg[e]): int(seg[e]) + n]
    want = dispatch.raw_decode(y_padded.view(E * C, M), gates, plan)
    got = P.decode(y, gates, idx, loc, seg)
    assert torch.allclose(got, want, rtol=1e-13, atol=1e-13)
    # gate gradient: the same row dots
    a = torch.randn(S, M, generator=g, dtype=torch.float64)
    want_g = dispatch.raw_gate_grad(a, y_padded.view(E * C, M), plan)
    got_g, _ = P.gate_grad(a, y, idx, loc, seg)
    assert torch.allclose(got_g, want_g, rtol=1e-13, atol=1e-13)


def test_routing_through_extract_critical():
    # the padded dropless routing of real scores: its locations and counts define the same packed layout
    g = torch.Generator().manual_seed(7)
    S, E, k = 400, 16, 4
    logits = torch.randn(S, E, generator=g)
    logits[:, 3] += 4.0          # skewed
    crit, _ = routing.extract_critical(torch.softmax(logits, 1), top_k=k, capacity_factor=0)
    counts = crit[5]
    assert int(crit[4]) == int(counts.max())
    R = P.packed_rows(S, k, E)
    seg, bexp, brows, slot = P.layout(crit.idx_ks, crit.loc_ks, counts, R)
    padded_slot = crit.slot_src
    C = crit[4]
    for e in range(E):
        n = int(counts[e])
        assert torch.equal(slot[int(seg[e]): int(seg[e]) + n], padded_slot[e * C: e * C + n])
    work_padded = E * int(counts.max())
    assert int(seg[-1]) <= work_padded + 127 * E


def test_segment_colsum_reference():
    x = torch.zeros(512, 8, dtype=torch.float64)
    x[:3] = 1.0
    x[256:300] = 2.0
    seg = torch.tensor([0, 128, 256, 384, 384], dtype=torch.int32)
    val, mag = P.segment_colsum(x, seg)
    assert val[:, 0].tolist() == [3.0, 0.0, 88.0, 0.0] and torch.equal(val, mag)
