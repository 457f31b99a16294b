"""The packed-layout kernels against fp64 / exact references: the layout kernel, the block-mapped and ragged-K launch
modes of the grouped GEMM (csrc/gemm_sm90.cu) under the per-element bound of tests/gemm_reference.py, and the packed
encode / decode / gate gradient / segmented column sums (csrc/moe_kernels.cu, csrc/gate_route.cu).

Packed inputs follow the layout's invariant (padding rows zero) and hold NaN in the rows past seg_off[E], which no
kernel may read; outputs are pre-filled with a sentinel, which must survive in the blocks past seg_off[E] and nowhere
else: rows of a computed block past its count must come out exactly zero.
"""
import math

import pytest
import torch

import gemm_reference as R
import packed_reference as P

pytestmark = pytest.mark.gpu

BF16, FP16 = torch.bfloat16, torch.float16
SENTINEL = -7.0
BOTH = (128, 0)
# per-expert row counts: empty experts, one-row experts, exact multiples of 128, a long expert
COUNTS = {
    'mixed': [0, 1, 128, 300, 0, 256, 77, 5],
    'one_expert': [0, 0, 700, 0],
    'aligned': [128, 256, 128],
}


@pytest.fixture(scope='module')
def G():
    from tutel_b200.ops import backend, gemm
    backend.require_ext()
    return gemm


def _gen(seed):
    return torch.Generator(device='cuda').manual_seed(seed)


def _rnd(gen, *shape, scale=0.5, dtype=BF16):
    return (torch.randn(*shape, device='cuda', generator=gen) * scale).to(dtype)


def _layout(counts, k=1):
    from tutel_b200.ops.packed import PackedLayout
    S = sum(counts) // k
    idx, loc = P.routing_from_counts(counts, k, S)
    lay = PackedLayout.build(idx.cuda(), loc.cuda(), torch.tensor(counts, dtype=torch.int32, device='cuda'))
    return lay, idx, loc


def _packed_rows(gen, lay, counts, cols, dtype=BF16, scale=0.5):
    """A packed [R, cols] tensor: random valid rows, zero padding, NaN past seg_off[E]."""
    seg = lay.seg_off.cpu().tolist()
    x = torch.full((lay.R, cols), float('nan'), device='cuda', dtype=dtype)
    for e, c in enumerate(counts):
        x[seg[e]:seg[e + 1]] = 0
        x[seg[e]:seg[e] + c] = _rnd(gen, c, cols, scale=scale, dtype=dtype)
    return x


def _check_padding(d, lay, what):
    """d [R, N]: rows of computed blocks past their count are exactly zero; blocks past seg_off[E] keep the sentinel."""
    used = int(lay.seg_off[-1])
    rows = lay.block_rows.cpu().repeat_interleave(128)
    inner = torch.arange(lay.R) % 128
    pad = (inner >= rows) & (torch.arange(lay.R) < used)
    dc = d.float().cpu()
    assert bool((dc[pad] == 0).all()), '%s: padding rows are not zero' % what
    assert bool((dc[used:] == SENTINEL).all()), '%s: blocks past seg_off[E] were written' % what


# ------------------------------------------------------------------------------------------------------------------
# layout kernel
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('E,k,S', [(8, 2, 300), (64, 6, 512), (256, 8, 256), (4, 1, 640)])
def test_layout_kernel_exact(E, k, S):
    g = torch.Generator().manual_seed(E + k)
    w = torch.rand(E, generator=g) ** 4
    w[: E // 4] = 0
    counts = [int(c) for c in torch.distributions.Multinomial(k * S, probs=w / w.sum()).sample()]
    lay, idx, loc = _layout(counts, k)
    seg, bexp, brows, slot = P.layout(idx, loc, torch.tensor(counts), lay.R)
    assert lay.R == P.packed_rows(S, k, E)
    assert torch.equal(lay.seg_off.cpu(), seg)
    assert torch.equal(lay.block_expert.cpu(), bexp)
    assert torch.equal(lay.block_rows.cpu(), brows)
    assert torch.equal(lay.slot_src.cpu(), slot)


# ------------------------------------------------------------------------------------------------------------------
# block-mapped B
# ------------------------------------------------------------------------------------------------------------------
EPIS = {  # name -> (epilogue, act, needs aux, has pre-activation output, has bias)
    'bias': (R.EPI_BIAS, 0, False, False, True), 'relu': (R.EPI_BIAS_RELU, 0, False, False, True),
    'gelu': (R.EPI_BIAS_GELU, 0, False, True, True), 'silu': (R.EPI_BIAS_SILU, 0, False, True, True),
    'none': (R.EPI_NONE, 0, False, False, False), 'relu_bwd': (R.EPI_RELU_BWD, 0, True, False, False),
    'act_bwd_gelu': (R.EPI_ACT_BWD, R.ACT_GELU, True, False, False),
    'act_bwd_silu': (R.EPI_ACT_BWD, R.ACT_SILU, True, False, False), 'add': (R.EPI_ADD, 0, True, False, False),
}


def _blocks(t, n):
    return t.view(-1, 128, t.size(-1))[:n]


@pytest.mark.parametrize('max_ctas', [0, 3])
@pytest.mark.parametrize('layout', list(COUNTS))
@pytest.mark.parametrize('epi', list(EPIS))
def test_block_mapped(G, epi, layout, max_ctas):
    counts = COUNTS[layout]
    E, K, N = len(counts), 200, 264
    epilogue, act, needs_aux, has_pre, has_bias = EPIS[epi]
    lay, _, _ = _layout(counts)
    gen = _gen(hash((epi, layout)) % 1000)
    x = _packed_rows(gen, lay, counts, K)
    w = _rnd(gen, E, N, K)
    bias = _rnd(gen, E, N, scale=1.0) if has_bias else None
    aux = _packed_rows(gen, lay, counts, N, scale=1.0) if needs_aux else None
    nb = int(lay.seg_off[-1]) // 128
    bexp = lay.block_expert[:nb].long()
    brows = lay.block_rows[:nb]
    r = R.ref_gemm(_blocks(x, nb), w[bexp], epilogue=epilogue, act=act or R.ACT_SILU,
                   bias=bias[bexp] if bias is not None else None, aux=_blocks(aux, nb) if aux is not None else None,
                   row_counts=brows, want_pre=has_pre)
    for bn in BOTH:
        d = torch.full((lay.R, N), SENTINEL, device='cuda', dtype=BF16)
        pre = torch.full_like(d, SENTINEL) if has_pre else None
        cs = torch.zeros(E, N, device='cuda')
        G.raw_gemm(x, w, epilogue=epilogue, act=act, bias=bias, aux=aux, out=d, d2=pre, row_counts=lay.block_rows,
                   b_group_map=lay.block_expert, colsum=cs, block_n=bn, max_ctas=max_ctas)
        what = '%s %s block_n=%d max_ctas=%d' % (epi, layout, bn, max_ctas)
        R.check(r, _blocks(d, nb), d2=_blocks(pre, nb) if pre is not None else None, what=what)
        _check_padding(d, lay, what)
        if pre is not None:
            _check_padding(pre, lay, what + ' pre')
        # colsum: the per-block reference sums, added up per expert
        want, acc, fix = (torch.zeros(E, N, dtype=torch.float64, device='cuda').index_add_(0, bexp, t)
                          for t in (r.colsum, r.colsum_acc, r.colsum_fix))
        err = (cs.double() - want).abs()
        tol = R.C_ACC[BF16] * acc + fix + (nb + 16) * R.U * want.abs() + R.half_ulp(want, torch.float32)
        assert bool((err <= tol).all()), '%s colsum: worst err/tol %.3g' % (what, float((err / tol).max()))


@pytest.mark.parametrize('layout', list(COUNTS))
@pytest.mark.parametrize('act', ['relu', 'gelu', 'silu'])
def test_block_mapped_glu(G, act, layout):
    counts = COUNTS[layout]
    E, K, N = len(counts), 136, 200
    codes = {'relu': R.ACT_RELU, 'gelu': R.ACT_GELU, 'silu': R.ACT_SILU}
    lay, _, _ = _layout(counts)
    gen = _gen(5)
    x = _packed_rows(gen, lay, counts, K)
    w1, w2 = _rnd(gen, E, K, N), _rnd(gen, E, K, N)        # "kn", as llama_ffn stores them
    nb = int(lay.seg_off[-1]) // 128
    bexp = lay.block_expert[:nb].long()
    brows = lay.block_rows[:nb]
    h, g, u = G.glu_gemm(x, w1, w2, b_mn=True, act=act, save_pre=True, row_counts=lay.block_rows,
                         b_group_map=lay.block_expert)
    r = R.ref_gemm(_blocks(x, nb), w1[bexp], b_mn=True, epilogue=R.EPI_GLU, b2=w2[bexp], act=codes[act], row_counts=brows,
                   want_pre=True)
    R.check(r, _blocks(h, nb), d2=_blocks(g, nb), d3=_blocks(u, nb), what='glu %s %s' % (act, layout))
    used = int(lay.seg_off[-1])
    for t in (h, g, u):
        t[used:] = SENTINEL      # (outputs are allocated by glu_gemm: only the padding rows are checked here)
        _check_padding(t, lay, 'glu %s %s' % (act, layout))
    # backward: dh = dy @ W3^T formed in registers, dg / du out
    Mo = 72
    dy = _packed_rows(gen, lay, counts, Mo)
    w3 = _rnd(gen, E, N, Mo)                               # [H, Mout]: "nk" for dh = dy @ W3^T
    dg, du = G.glu_gemm_bwd(dy, w3, g, u, b_mn=False, act=act, row_counts=lay.block_rows, b_group_map=lay.block_expert)
    rb = R.ref_gemm(_blocks(dy, nb), w3[bexp], epilogue=R.EPI_GLU_BWD, aux=_blocks(g, nb), aux2=_blocks(u, nb),
                    act=codes[act], row_counts=brows)
    R.check(rb, _blocks(dg, nb), d2=_blocks(du, nb), what='glu_bwd %s %s' % (act, layout))
    for t in (dg, du):
        t[used:] = SENTINEL
        _check_padding(t, lay, 'glu_bwd %s %s' % (act, layout))


# ------------------------------------------------------------------------------------------------------------------
# ragged K
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('max_ctas', [0, 5])
@pytest.mark.parametrize('layout', list(COUNTS))
@pytest.mark.parametrize('dtype', [BF16, FP16], ids=['bf16', 'fp16'])
def test_ragged_k(G, dtype, layout, max_ctas):
    counts = COUNTS[layout]
    E, M, N = len(counts), 264, 200
    lay, _, _ = _layout(counts)
    gen = _gen(7)
    a = _packed_rows(gen, lay, counts, M, dtype=dtype)
    b = _packed_rows(gen, lay, counts, N, dtype=dtype)
    seg = lay.seg_off.cpu().tolist()
    kmax = max(max(seg[e + 1] - seg[e] for e in range(E)), 64)
    a_pad = torch.zeros(E, kmax, M, device='cuda', dtype=dtype)
    b_pad = torch.zeros(E, kmax, N, device='cuda', dtype=dtype)
    for e in range(E):
        a_pad[e, :seg[e + 1] - seg[e]] = a[seg[e]:seg[e + 1]]
        b_pad[e, :seg[e + 1] - seg[e]] = b[seg[e]:seg[e + 1]]
    r = R.ref_gemm(a_pad, b_pad, a_mn=True, b_mn=True, out_dtype=dtype)
    for bn in BOTH:
        d = torch.full((E, M, N), SENTINEL, device='cuda', dtype=dtype)
        G.raw_gemm(a, b, a_mn=True, b_mn=True, out=d, k_offsets=lay.seg_off, block_n=bn, max_ctas=max_ctas)
        R.check(r, d, what='ragged K %s block_n=%d' % (layout, bn))
        for e in range(E):
            if counts[e] == 0:
                assert bool((d[e] == 0).all()), 'empty expert %d: the tile is not zero' % e


def test_refusals(G):
    lay, _, _ = _layout(COUNTS['mixed'])
    x = torch.zeros(lay.R, 64, device='cuda', dtype=BF16)
    w = torch.zeros(8, 64, 64, device='cuda', dtype=BF16)
    with pytest.raises(RuntimeError):      # fp8 operands have no ragged-K mode
        G.raw_gemm(x.to(torch.float8_e4m3fn).unsqueeze(0), x.to(torch.float8_e4m3fn).unsqueeze(0), k_offsets=lay.seg_off)
    with pytest.raises(RuntimeError):      # both modes at once
        G.raw_gemm(x, w, b_group_map=lay.block_expert, k_offsets=lay.seg_off)


# ------------------------------------------------------------------------------------------------------------------
# packed encode / decode / gate gradient / segmented column sums
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('dtype', [BF16, FP16], ids=['bf16', 'fp16'])
@pytest.mark.parametrize('k,E', [(1, 8), (2, 8), (8, 64)])
def test_dispatch_kernels(k, E, dtype):
    from tutel_b200.ops import packed
    S, M = 384, 200
    g = torch.Generator().manual_seed(k * E)
    w = torch.rand(E, generator=g) ** 3
    w[0] = 0
    counts = [int(c) for c in torch.distributions.Multinomial(k * S, probs=w / w.sum()).sample()]
    lay, idx, loc = _layout(counts, k)
    idx_d, loc_d = idx.cuda(), loc.cuda()
    x = (torch.randn(S, M, generator=g)).to(dtype).cuda()
    gates = torch.rand(k, S, generator=g).cuda()
    seg = lay.seg_off.cpu()
    # encode: exact (the gate product is one fp32 multiply, rounded once)
    enc = packed.encode(x, None, lay)
    want = P.encode(x, None, lay.slot_src, k)
    used = int(seg[-1])
    assert torch.equal(enc[:used].double().cpu(), want[:used])
    enc_g = packed.encode(x, gates, lay)
    tok = lay.slot_src.long().clamp_min(0) // k
    j = lay.slot_src.long().clamp_min(0) % k
    want_g = torch.where((lay.slot_src >= 0).unsqueeze(1), (x.float()[tok] * gates[j, tok].unsqueeze(1)).to(dtype),
                         torch.zeros((), dtype=dtype, device='cuda'))
    assert torch.equal(enc_g[:used], want_g[:used])
    # decode: fp32 accumulation of k products, one rounding
    buf = _packed_rows(_gen(3), lay, counts, M, dtype=dtype)
    out = packed.decode(buf, gates, idx_d, loc_d, lay)
    ref = P.decode(buf, gates, idx, loc, seg)
    mag = P.decode(buf.abs(), gates.abs(), idx, loc, seg)
    tol = R.half_ulp(ref, dtype) + 2 * k * R.U * mag
    assert bool(((out.double().cpu() - ref).abs() <= tol).all())
    # gate gradient: fp32 dot products of M terms
    dg = packed.gate_grad(x, buf, idx_d, loc_d, lay)
    ref, mag = P.gate_grad(x, buf, idx, loc, seg)
    assert bool(((dg.double().cpu() - ref).abs() <= (M + 2) * R.U * mag + 1e-30).all())
    # segmented column sums (the fc2 bias gradient)
    cs = packed.segment_colsum(buf[:used].contiguous() if used == lay.R else torch.cat(
        [buf[:used], torch.zeros(lay.R - used, M, device='cuda', dtype=dtype)]), lay)
    ref, mag = P.segment_colsum(torch.nan_to_num(buf[:used].float()).double(), seg)
    rows = max(max(int(seg[e + 1] - seg[e]) for e in range(E)), 1)
    tol = R.half_ulp(ref, dtype) + (rows + 2) * R.U * mag
    assert bool(((cs.double().cpu() - ref).abs() <= tol).all())
