"""Routing and dispatch kernels (csrc/gate_route.cu, csrc/moe_kernels.cu) against tests/dispatch_reference.py.

Integer outputs and single-rounding outputs are checked bit for bit, fp32 sums element by element under bounds
derived from the kernels' operation counts.  The shapes sit where the kernels branch: the E boundaries of the
gate kernels' per-lane register arrays, the 256-token routing tiles, the 16-row encode units, vector and scalar
paths, dropped and invalid choices, the push-mode pointer / signal tables on one GPU, and the split (atomic)
column sum.
"""
import math

import pytest
import torch

import dispatch_reference as R

pytestmark = pytest.mark.gpu

F32, F16, BF16 = torch.float32, torch.float16, torch.bfloat16
FLOATS = (F32, F16, BF16)
SENTINEL = -7.0


@pytest.fixture(scope='module')
def C():
    from tutel_b200.ops import backend
    return backend.require_ext()


@pytest.fixture(scope='module', autouse=True)
def _report_bounds():
    yield
    print('\nlargest error / bound per bounded check:', {k: round(v, 4) for k, v in sorted(R.OBSERVED.items())})


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _name(dtype):
    return str(dtype)[6:]


# ------------------------------------------------------------------------------------------------------------------
# gate_route_forward / gate_route_backward
# ------------------------------------------------------------------------------------------------------------------
# gate_route_kernel / gate_route_bwd_kernel hold ceil(E/32) <= VPT values per lane, VPT = 1, 2, 4, 8, 16 for
# E <= 32, 64, 128, 256, 512: E sits on both sides of every boundary.  k = 32 at E = 256 and k >= 16 at E = 512 need
# more than the default 48 KB of dynamic shared memory; the last case runs that over 33 routing tiles.
# S = 1, 255, 256, 257, 8195 sit around the 256-token routing tile.
GATE_EKS = [(1, 1, 1), (8, 1, 255), (8, 2, 256), (8, 8, 257), (32, 4, 8195), (32, 32, 1), (33, 2, 255), (33, 8, 256),
            (64, 1, 257), (64, 4, 8195), (65, 2, 1), (65, 8, 255), (128, 2, 256), (129, 4, 257), (256, 8, 8195),
            (256, 32, 1), (257, 2, 255), (257, 8, 256), (512, 1, 257), (512, 8, 257), (512, 16, 1), (512, 32, 255),
            (512, 32, 8195)]
GATE_CASES = [(E, k, S, i) for i, (E, k, S) in enumerate(GATE_EKS)]


def _gate_logits(S, E, dtype, seed, nan_row):
    """Logits spread by tens, integer-valued rows (exact ties), rows holding -inf, and optionally one NaN row."""
    gen = _gen(seed)
    x = torch.randn(S, E, generator=gen) * 3
    x[S // 4: S // 2] *= 8
    x[: S // 4] = torch.randint(-2, 3, (S // 4, E), generator=gen).float()
    if E > 1 and S > 8:
        x[S // 2: S // 2 + 8, ::3] = -math.inf
    if nan_row:
        x[S - 2, E // 2] = math.nan
    return x.to(dtype).cuda()


@pytest.mark.parametrize('dtype', FLOATS, ids=_name)
@pytest.mark.parametrize('E,k,S,case', GATE_CASES, ids=['E%d-k%d-S%d' % c[:3] for c in GATE_CASES])
def test_gate_route_forward_backward(C, dtype, E, k, S, case):
    nan_row = S >= 255 and case % 2 == 1
    logits = _gate_logits(S, E, dtype, 100 + case, nan_row)
    normalize = case % 3 != 2
    eps = float(torch.finfo(dtype).eps)
    cap = 0 if case % 4 == 3 else max(1, S * k // E // 2)         # C = 0: no slot map; else below the load
    what = '%s S=%d E=%d k=%d C=%d' % (_name(dtype), S, E, k, cap)
    outs = C.gate_route_forward(logits, k, cap, normalize, eps)
    assert (len(outs) == 9) == (cap > 0)
    logits_h, outs_h = logits.cpu(), [t.cpu() for t in outs]
    routable = R.check_gate_route_forward(what, logits_h, k, cap, normalize, eps, outs_h, check_loss=not nan_row)
    assert int((~routable).sum()) == int(nan_row)
    if nan_row:
        assert torch.isnan(outs_h[7]).all(), 'l_aux of a batch with a NaN row'

    scores, idx, top, ce = outs[0], outs[1], outs[2], outs[6]
    dg = torch.randn(k, S, generator=_gen(200 + case))
    dl = torch.tensor(1.75, dtype=dtype)
    variants = [('full', dg, True, normalize, eps), ('dgates=None', None, True, normalize, eps),
                ('no loss', dg, False, normalize, eps), ('normalize=False', dg, True, False, eps),
                ('eps above D', dg, True, True, 2.0)]
    for name, dgates, loss, norm, e in variants:
        out = C.gate_route_backward(scores, idx, top, dgates.cuda() if dgates is not None else None,
                                    ce if loss else None, dl.cuda() if loss else None, logits, norm, e)
        assert out.dtype == dtype
        R.check_gate_backward('%s %s' % (what, name), out.cpu(), outs_h[0], outs_h[1], outs_h[2], dgates,
                              outs_h[6] if loss else None, dl if loss else None, norm, e, routable)

    # forward with the clamped normalisation (eps above every D)
    if k > 1:
        outs = [t.cpu() for t in C.gate_route_forward(logits, k, cap, True, 2.0)]
        R.check_gate_route_forward(what + ' eps=2', logits_h, k, cap, True, 2.0, outs, check_loss=not nan_row)


def test_nan_row_changes_no_other_token(C):
    """A NaN row routes nowhere, and every other token's choice, location, slot, count and first-choice count is what
    it is when the row holds zeros instead and then routes nowhere by hand."""
    S, E, k, cap = 1000, 16, 2, 80
    logits = _gate_logits(S, E, F32, 7, nan_row=True)
    s_nan = S - 2
    outs = [t.cpu() for t in C.gate_route_forward(logits, k, cap, True, 1e-6)]
    R.check_gate_route_forward('nan row', logits.cpu(), k, cap, True, 1e-6, outs, check_loss=False)
    clean = logits.clone()
    clean[s_nan] = 0
    ref = [t.cpu() for t in C.gate_route_forward(clean, k, cap, True, 1e-6)]
    others = torch.arange(S) != s_nan
    assert torch.equal(outs[1][:, others], ref[1][:, others])
    assert ((outs[1][:, s_nan] < 0) | (outs[1][:, s_nan] >= E)).all()
    idx = ref[1].clone()
    idx[:, s_nan] = -1
    loc, counts, ce, slot = R.ref_locations(idx, E, cap)
    R.assert_equal('loc', outs[4], loc)
    R.assert_equal('counts', outs[5], counts)
    R.assert_equal('ce', outs[6], ce)
    R.assert_equal('slot', outs[8], slot)


# ------------------------------------------------------------------------------------------------------------------
# route_locations + build_slot_map
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('S,E,k', [(70000, 8, 2), (70000, 3, 1), (4097, 2048, 8), (1, 5, 1), (1025, 130, 3),
                                   (3000, 64, 4), (20000, 2048, 2)])
def test_route_locations_and_slot_map(C, S, E, k):
    gen = _gen(S + E + k)
    idx = torch.randint(0, E, (k, S), generator=gen, dtype=torch.int32)
    bad = torch.rand(k, S, generator=gen) < 0.02
    idx[bad] = torch.where(torch.rand(int(bad.sum()), generator=gen) < 0.5, -1, E + 2).int()
    idx_d = idx.cuda()
    cap = max(1, S * k // E // 2)
    what = 'S=%d E=%d k=%d C=%d' % (S, E, k, cap)
    loc_d, counts, slot = C.route_locations(idx_d, E, cap)
    loc = loc_d.cpu()
    R.check_locations(what, idx, E, cap, loc, counts.cpu(), slot=slot.cpu())
    loc0, counts0 = C.route_locations(idx_d, E, 0)
    assert torch.equal(loc0, loc_d) and torch.equal(counts0, counts)
    for c in (1, cap + 7):
        R.assert_equal('build_slot_map C=%d: %s' % (c, what), C.build_slot_map(idx_d, loc_d, E, c).cpu(),
                       R.ref_locations(idx, E, c)[3])


# ------------------------------------------------------------------------------------------------------------------
# encode_rows / encode_rows_fp8 (local and push mode)
# ------------------------------------------------------------------------------------------------------------------
def _route(S, E, k, cap, seed):
    """Distinct experts per token, some choices routed nowhere; returns CPU idx / loc / slot."""
    gen = _gen(seed)
    idx = torch.topk(torch.rand(S, E, generator=gen), k, dim=1).indices.t().contiguous().to(torch.int32)
    idx[0, 3] = -1
    idx[k - 1, 5] = E + 1
    idx[:, 9] = -1                                                     # a token with no valid choice
    loc, _, _, slot = R.ref_locations(idx, E, cap)
    return idx, loc, slot


def _on_gpu(t, unaligned=False):
    """A CUDA copy of t; with ``unaligned`` it starts one element past a 16-byte boundary (still contiguous)."""
    if not unaligned:
        return t.cuda()
    base = torch.empty(t.numel() + 1, dtype=t.dtype, device='cuda')
    v = base[1:].view(t.shape)
    v.copy_(t)
    assert v.data_ptr() % 16 != 0
    return v


ENC_M = {'vector': {F32: 1028, F16: 2056, BF16: 2056}, 'M%8': {F32: 259, F16: 259, BF16: 259},
         'unaligned x': {F32: 264, F16: 264, BF16: 264}}


@pytest.mark.parametrize('cap', [1, 15, 16, 17, 200])
@pytest.mark.parametrize('mkind', list(ENC_M))
@pytest.mark.parametrize('dtype', FLOATS, ids=_name)
def test_encode_rows(C, dtype, mkind, cap):
    S, E, k = 300, 6, 2
    M = ENC_M[mkind][dtype]
    idx, loc, slot = _route(S, E, k, cap, 11 + cap)
    x = (torch.randn(S, M, generator=_gen(12)) * 3).to(dtype)
    gates = torch.rand(k, S, generator=_gen(13)) * 2 - 0.5
    vr = torch.tensor([0, cap + 5, cap // 2, 1, cap, 3], dtype=torch.int32)
    xd, sd = _on_gpu(x, mkind == 'unaligned x'), slot.cuda()
    for g in (gates, None):
        for valid_rows in (None, vr):
            what = '%s M=%d C=%d gates=%s valid_rows=%s' % (_name(dtype), M, cap, g is not None, valid_rows is not None)
            out = torch.full((E * cap, M), SENTINEL, dtype=dtype, device='cuda')
            C.encode_rows(xd, g.cuda() if g is not None else None, sd, out, k, E, cap, 0, 0, 0, 0, 0, 0,
                          valid_rows.cuda() if valid_rows is not None else None)
            R.check_encode(what, out.cpu(), x, g, slot, k, E, cap, valid_rows, SENTINEL)


@pytest.mark.parametrize('cap', [1, 17, 200])
@pytest.mark.parametrize('dtype', (F16, BF16), ids=_name)
def test_encode_rows_fp8(C, dtype, cap):
    S, E, k, M = 300, 6, 2, 272
    idx, loc, slot = _route(S, E, k, cap, 21 + cap)
    x = (torch.randn(S, M, generator=_gen(22)) * 3).to(dtype)
    x[4] = 0                                                           # amax 0
    x[6, 7] = 900.0                                                    # one large element
    gates = torch.rand(k, S, generator=_gen(23)) * 2 - 0.5
    gates[0, 8] = 0.0
    for g in (gates, None):
        q, sc = C.encode_rows_fp8(x.cuda(), g.cuda() if g is not None else None, slot.cuda(), k, E, cap, 0, 0, 0, 0, 0, 0, 0)
        assert q.dtype == torch.float8_e4m3fn and q.shape == (E * cap, M)
        R.check_encode_fp8('%s C=%d gates=%s' % (_name(dtype), cap, g is not None), q.cpu(), sc.cpu(), x, g, slot, k, E, cap)
        deq = C.dequant_rows(q, sc, dtype)
        R.assert_equal('dequant of the fp8 dispatch rows', deq.cpu(), R.ref_dequant(q.cpu().view(torch.uint8), sc.cpu(), dtype))


@pytest.mark.parametrize('signal_rows,rot', [(48, 0), (24, 3), (0, 3), (200, 0)])
@pytest.mark.parametrize('signal_value', [0, 9])
def test_encode_push_mode_on_one_gpu(C, signal_value, signal_rows, rot):
    """Pointer tables to E separate local buffers, local chunk flags and chunk counters: rows and scales bit-exact,
    every flag at its expected value, every counter re-armed to 0, results independent of the rotation."""
    S, E, k, cap, M = 300, 5, 2, 200, 272
    dtype = BF16
    idx, loc, slot = _route(S, E, k, cap, 31)
    x = (torch.randn(S, M, generator=_gen(32)) * 3).to(dtype)
    gates = torch.rand(k, S, generator=_gen(33)) * 2 - 0.5
    xd, gd, sd = x.cuda(), gates.cuda(), slot.cuda()
    chunk_rows = -(-(signal_rows or 16) // 16) * 16
    chunks = -(-cap // chunk_rows)
    calls = 2 if signal_value == 0 else 1                              # red.add: each launch adds 1
    want_flag = signal_value if signal_value else calls
    what = 'signal_rows=%d rot=%d signal_value=%d' % (signal_rows, rot, signal_value)

    def tables():
        flags = torch.zeros(E, chunks, dtype=torch.int32, device='cuda')
        counters = torch.zeros(E * chunks, dtype=torch.int32, device='cuda')
        s_tab = torch.tensor([flags.data_ptr() + 4 * chunks * e for e in range(E)], dtype=torch.int64, device='cuda')
        return flags, counters, s_tab

    bufs = [torch.full((cap, M), SENTINEL, dtype=dtype, device='cuda') for _ in range(E)]
    d_tab = torch.tensor([b.data_ptr() for b in bufs], dtype=torch.int64, device='cuda')
    flags, counters, s_tab = tables()
    dummy = torch.full((1,), SENTINEL, dtype=dtype, device='cuda')
    for _ in range(calls):
        C.encode_rows(xd, gd, sd, dummy, k, E, cap, d_tab.data_ptr(), s_tab.data_ptr(), signal_rows, rot, signal_value,
                      counters.data_ptr(), None)
    torch.cuda.synchronize()
    assert float(dummy[0]) == SENTINEL
    out = torch.cat(bufs)
    R.check_encode('push ' + what, out.cpu(), x, gates, slot, k, E, cap)
    assert torch.all(flags == want_flag), ('push flags', what, flags.tolist())
    assert torch.all(counters == 0), ('push counters re-armed', what, counters.tolist())
    local = torch.empty(E * cap, M, dtype=dtype, device='cuda')
    C.encode_rows(xd, gd, sd, local, k, E, cap, 0, 0, 0, 0, 0, 0, None)
    assert torch.equal(out, local)

    qbufs = [torch.full((cap, M), 0x55, dtype=torch.uint8, device='cuda') for _ in range(E)]
    sbufs = [torch.full((cap,), SENTINEL, device='cuda') for _ in range(E)]
    q_tab = torch.tensor([b.data_ptr() for b in qbufs], dtype=torch.int64, device='cuda')
    sc_tab = torch.tensor([b.data_ptr() for b in sbufs], dtype=torch.int64, device='cuda')
    flags, counters, s_tab = tables()
    for _ in range(calls):
        assert C.encode_rows_fp8(xd, gd, sd, k, E, cap, q_tab.data_ptr(), sc_tab.data_ptr(), s_tab.data_ptr(), signal_rows,
                                 rot, signal_value, counters.data_ptr()) == []
    torch.cuda.synchronize()
    R.check_encode_fp8('push ' + what, torch.cat(qbufs).cpu(), torch.cat(sbufs).cpu(), x, gates, slot, k, E, cap)
    assert torch.all(flags == want_flag), ('fp8 push flags', what, flags.tolist())
    assert torch.all(counters == 0), ('fp8 push counters re-armed', what, counters.tolist())


# ------------------------------------------------------------------------------------------------------------------
# decode_rows, gate_grad
# ------------------------------------------------------------------------------------------------------------------
DEC_M = {'vector': {F32: 516, F16: 1032, BF16: 1032}, 'M%8': {F32: 131, F16: 131, BF16: 131},
         'unaligned buf': {F32: 136, F16: 136, BF16: 136}}


@pytest.mark.parametrize('mkind', list(DEC_M))
@pytest.mark.parametrize('k', [1, 2, 3, 8, 16])
@pytest.mark.parametrize('dtype', FLOATS, ids=_name)
def test_decode_rows(C, dtype, k, mkind):
    S, E = 333, 20
    M = DEC_M[mkind][dtype]
    cap = max(1, S * k // E // 2)                                      # below the load: dropped choices
    idx, loc, slot = _route(S, E, k, cap, 41 + k)
    buf = (torch.randn(E * cap, M, generator=_gen(42)) * 3).to(dtype)
    gates = torch.rand(k, S, generator=_gen(43)) * 2 - 0.5
    bd, idd, ld = _on_gpu(buf, mkind == 'unaligned buf'), idx.cuda(), loc.cuda()
    outs = {}
    for g in (gates, None):
        out = C.decode_rows(bd, g.cuda() if g is not None else None, idd, ld, E, cap, 0, 0)
        R.check_decode('%s k=%d M=%d C=%d gates=%s' % (_name(dtype), k, M, cap, g is not None), out.cpu(), buf, g, idx, loc,
                       E, cap)
        outs[g is not None] = out
    # flags already at or above the target: no wait, same result
    target = 5
    flags = (target + torch.randint(0, 3, (E,), generator=_gen(44))).to(torch.int32).cuda()
    waited = C.decode_rows(bd, gates.cuda(), idd, ld, E, cap, flags.data_ptr(), target)
    assert torch.equal(waited, outs[True])


def test_decode_rows_rejects_k_above_16(C):
    S, E, k, cap = 40, 20, 17, 8
    idx = torch.arange(k, dtype=torch.int32, device='cuda')[:, None].expand(k, S).contiguous()
    loc = torch.zeros(k, S, dtype=torch.int32, device='cuda')
    buf = torch.zeros(E * cap, 64, dtype=BF16, device='cuda')
    with pytest.raises(RuntimeError, match='invalid argument'):
        C.decode_rows(buf, None, idx, loc, E, cap, 0, 0)


@pytest.mark.parametrize('M', [7, 257, 4096, 14336])
@pytest.mark.parametrize('dtype', FLOATS, ids=_name)
def test_gate_grad(C, dtype, M):
    S, E, k = 96, 6, 2
    cap = S * k // E // 2
    idx, loc, slot = _route(S, E, k, cap, 51)
    a = (torch.randn(S, M, generator=_gen(52)) * 2).to(dtype)
    buf = (torch.randn(E * cap, M, generator=_gen(53)) * 2).to(dtype)
    out = C.gate_grad(a.cuda(), buf.cuda(), idx.cuda(), loc.cuda(), E, cap)
    R.check_gate_grad('%s M=%d' % (_name(dtype), M), out.cpu(), a, buf, idx, loc, E, cap)


# ------------------------------------------------------------------------------------------------------------------
# dequant_rows, quantize_transpose, grouped_colsum
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('R_,K', [(1, 16), (37, 272), (1000, 4096)])
@pytest.mark.parametrize('dtype', (F16, BF16), ids=_name)
def test_dequant_rows(C, dtype, R_, K):
    gen = _gen(R_ + K)
    q = torch.randint(0, 256, (R_, K), generator=gen, dtype=torch.uint8)
    q[(q & 0x7f) == 0x7f] = 0x7e                                       # no NaN codes
    scale = torch.rand(R_, generator=gen) * 2.0 ** torch.randint(-24, -1, (R_,), generator=gen).float()
    y = C.dequant_rows(q.cuda().view(torch.float8_e4m3fn), scale.cuda(), dtype)
    R.assert_equal('dequant_rows %s R=%d K=%d' % (_name(dtype), R_, K), y.cpu(), R.ref_dequant(q, scale, dtype))


@pytest.mark.parametrize('G_,R_,K', [(1, 128, 64), (3, 256, 192), (2, 1024, 1088)])
@pytest.mark.parametrize('dtype', (F16, BF16), ids=_name)
def test_quantize_transpose(C, dtype, G_, R_, K):
    x = torch.randn(G_, R_, K, generator=_gen(G_ * R_ + K)) * 0.3
    x[0, :, 5] = 0                                                     # amax 0 -> scale 1
    x[-1, :, -1] *= 1000
    x = x.to(dtype)
    q, s = C.quantize_transpose(x.cuda())
    rq, rs = R.ref_quantize_transpose(x)
    what = '%s G=%d R=%d K=%d' % (_name(dtype), G_, R_, K)
    R.assert_equal('quantize_transpose scales ' + what, s.cpu(), rs)
    R.assert_equal('quantize_transpose bytes ' + what, q.cpu().view(torch.uint8), rq)


def _colsum_splits(G_, T, N, elem):
    """tb::colsum_row_splits: how many row splits (fp32 atomics into one accumulator) the launcher takes."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    strips = -(-N // (16 * (16 // elem)))
    splits = 1
    while strips * G_ * splits < 2 * sms and T // (splits * 2) >= 64:
        splits *= 2
    return splits


@pytest.mark.parametrize('G_,T,N,split', [(1, 4096, 264, True), (3, 100, 136, False), (2, 20000, 64, True)])
@pytest.mark.parametrize('dtype', FLOATS, ids=_name)
def test_grouped_colsum(C, dtype, G_, T, N, split):
    x = (torch.randn(G_, T, N, generator=_gen(T + N)) * 2).to(dtype).cuda()
    assert (_colsum_splits(G_, T, N, x.element_size()) > 1) == split
    for name, v in (('contiguous', x), ('row view', x[:, 3:]), ('column view', x[:, :, 16:N - 16])):
        R.check_colsum('%s G=%d T=%d N=%d %s' % (_name(dtype), G_, T, N, name), C.grouped_colsum(v).cpu(), v.cpu())
