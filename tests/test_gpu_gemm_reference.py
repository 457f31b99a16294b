"""The grouped GEMM (csrc/gemm_sm90.cu) against the fp64 reference of tests/gemm_reference.py, element by element.

Every case runs the 128 x 128 configuration (block_n=128) and the launcher's own choice (block_n=0), and both are
checked against the reference under its per-element bound: epilogues x dtypes, shape edges, fp8 with row / column
scales, grouping (row counts, grouped B, max_ctas), GLU, operand views and argument checks, and the fused engine's
launch arguments on one GPU.
"""
import math

import pytest
import torch

import gemm_reference as R

pytestmark = pytest.mark.gpu

BF16, FP16, FP32 = torch.bfloat16, torch.float16, torch.float32
E4M3, E5M2 = torch.float8_e4m3fn, torch.float8_e5m2
BOTH = (128, 0)
SENTINEL = -7.0


@pytest.fixture(scope='module')
def G():
    from tutel_b200.ops import backend, gemm
    backend.require_ext()
    return gemm


@pytest.fixture(scope='module', autouse=True)
def _report_accumulation_error():
    yield
    print('\nlargest normalised accumulation error per input dtype (C_ACC covers it):',
          {str(k)[6:]: round(v, 3) for k, v in R.OBSERVED.items()})


def _gen(seed):
    return torch.Generator(device='cuda').manual_seed(seed)


def _rnd(gen, *shape, scale=0.5, dtype=BF16):
    return (torch.randn(*shape, device='cuda', generator=gen) * scale).to(dtype)


def _quant(x, dtype):
    """Row-scaled fp8 copy of x [.., K] and its scales: e4m3 by the native quantiser, e5m2 like it in torch."""
    from tutel_b200.ops import gemm
    if dtype == E4M3:
        return gemm.quantize_rows(x)
    amax = x.float().abs().amax(-1)
    s = torch.where(amax > 0, amax * (1.0 / 57344.0), torch.ones_like(amax))
    return (x.float() * (1.0 / s)[..., None]).clamp(-57344.0, 57344.0).to(E5M2), s


ACT = {'relu': R.ACT_RELU, 'gelu': R.ACT_GELU, 'silu': R.ACT_SILU}
EPIS = {  # name -> (epilogue, act, needs aux, has pre-activation output)
    'none': (R.EPI_NONE, 0, False, False), 'bias': (R.EPI_BIAS, 0, False, False),
    'bias_relu': (R.EPI_BIAS_RELU, 0, False, False), 'gelu': (R.EPI_BIAS_GELU, 0, False, True),
    'silu': (R.EPI_BIAS_SILU, 0, False, True), 'relu_bwd': (R.EPI_RELU_BWD, 0, True, False),
    'add': (R.EPI_ADD, 0, True, False), 'act_bwd_gelu': (R.EPI_ACT_BWD, R.ACT_GELU, True, False),
    'act_bwd_silu': (R.EPI_ACT_BWD, R.ACT_SILU, True, False), 'act_bwd_relu': (R.EPI_ACT_BWD, R.ACT_RELU, True, False),
}


def run_case(G, a, b, *, epi='none', a_mn=False, b_mn=False, out_dtype=None, bias=None, aux=None, scale_a=None, scale_b=None,
             row_counts=None, b_group_div=1, colsum=False, sentinel=None, block_ns=BOTH, what='', **extra):
    """Launch with each block_n, check every output against the reference, return {block_n: (d, pre, colsum)}."""
    epilogue, act, _, has_pre = EPIS[epi]
    alpha = 0.375 if epi == 'none' and a.element_size() == 2 else 1.0
    Gn = a.size(0)
    M = a.size(2) if a_mn else a.size(1)
    N = b.size(2) if b_mn else b.size(1)
    out_dtype = out_dtype or (a.dtype if a.element_size() == 2 else BF16)
    r = R.ref_gemm(a, b, a_mn=a_mn, b_mn=b_mn, epilogue=epilogue, alpha=alpha, bias=bias, aux=aux, act=act or R.ACT_SILU,
                   scale_a=scale_a, scale_b=scale_b, row_counts=row_counts, b_group_div=b_group_div, out_dtype=out_dtype,
                   want_pre=has_pre)
    res = {}
    for bn in block_ns:
        fill = (lambda: torch.full((Gn, M, N), sentinel, device='cuda', dtype=out_dtype)) if sentinel is not None else \
            (lambda: torch.empty((Gn, M, N), device='cuda', dtype=out_dtype))
        d = fill()
        pre = fill() if has_pre else None
        cs = torch.zeros((Gn + b_group_div - 1) // b_group_div, N, device='cuda') if colsum else None
        G.raw_gemm(a, b, a_mn=a_mn, b_mn=b_mn, epilogue=epilogue, alpha=alpha, bias=bias, aux=aux, act=act, out=d, d2=pre,
                   scale_a=scale_a, scale_b=scale_b, row_counts=row_counts, b_group_div=b_group_div, colsum=cs, block_n=bn,
                   **extra)
        R.check(r, d, d2=pre, colsum=cs, untouched=sentinel, what='%s %s block_n=%d' % (what, epi, bn))
        res[bn] = (d, pre, cs)
    return res


def _epi_inputs(gen, epi, Gn, M, N, dtype, div=1):
    _, _, needs_aux, _ = EPIS[epi]
    bias = _rnd(gen, (Gn + div - 1) // div, N, scale=1.0, dtype=dtype) if epi in ('bias', 'bias_relu', 'gelu', 'silu') else None
    aux = _rnd(gen, Gn, M, N, scale=1.0, dtype=dtype) if needs_aux else None
    return dict(bias=bias, aux=aux)


# ------------------------------------------------------------------------------------------------------------------
# epilogues x dtypes
# ------------------------------------------------------------------------------------------------------------------
# fp32 outputs: every epilogue without an aux operand (aux operands are 16-bit, of the output dtype)
EPI_OUT = [(e, False) for e in EPIS] + [(e, True) for e in ('none', 'bias', 'bias_relu', 'gelu', 'silu')]


@pytest.mark.parametrize('dtype', [BF16, FP16], ids=['bf16', 'fp16'])
@pytest.mark.parametrize('epi,out32', EPI_OUT, ids=['%s-%s' % (e, 'out32' if o else 'out16') for e, o in EPI_OUT])
def test_epilogue_dtype(G, epi, out32, dtype):
    # a partial row block, a partial 256-wide tile and a partial 64-deep K block
    Gn, M, N, K = 3, 328, 264, 200
    gen = _gen(1)
    a, b = _rnd(gen, Gn, M, K, dtype=dtype), _rnd(gen, Gn, N, K, dtype=dtype)
    run_case(G, a, b, epi=epi, out_dtype=FP32 if out32 else dtype, colsum=True, **_epi_inputs(gen, epi, Gn, M, N, dtype))


@pytest.mark.parametrize('epi', list(EPIS))
def test_epilogue_many_tiles(G, epi):
    # 8 x 8 x 8 tiles of 128 x 256: every CTA runs several tiles
    Gn, M, N, K = 8, 1024, 2048, 256
    gen = _gen(2)
    a, b = _rnd(gen, Gn, M, K), _rnd(gen, Gn, N, K)
    run_case(G, a, b, epi=epi, colsum=epi in ('relu_bwd', 'act_bwd_gelu'), **_epi_inputs(gen, epi, Gn, M, N, BF16))


# ------------------------------------------------------------------------------------------------------------------
# shape edges, all four operand layouts
# ------------------------------------------------------------------------------------------------------------------
EDGES = [('K', 8), ('K', 16), ('K', 56), ('K', 64), ('K', 72), ('K', 4104), ('M', 1), ('M', 8), ('M', 127), ('M', 129),
         ('N', 8), ('N', 120), ('N', 136), ('N', 248), ('N', 256), ('N', 264), ('G', 160)]


@pytest.mark.parametrize('a_mn,b_mn', [(False, False), (False, True), (True, False), (True, True)],
                         ids=['kk', 'kn', 'mk', 'mn'])
@pytest.mark.parametrize('epi', ['none', 'bias_relu'])
@pytest.mark.parametrize('dim,val', EDGES, ids=['%s%d' % e for e in EDGES])
def test_shape_edges(G, dim, val, epi, a_mn, b_mn):
    shape = dict(G=3, M=136, N=264, K=200)
    if dim == 'G':
        shape.update(G=160, M=64, N=128, K=64)    # more tiles than SMs, all of them small
    shape[dim] = val
    Gn, M, N, K = shape['G'], shape['M'], shape['N'], shape['K']
    gen = _gen(3)
    a, b = _rnd(gen, Gn, M, K), _rnd(gen, Gn, N, K)
    a_op = a.transpose(1, 2).contiguous() if a_mn else a
    b_op = b.transpose(1, 2).contiguous() if b_mn else b
    kw = _epi_inputs(gen, epi, Gn, M, N, BF16)
    if a_mn and M % 8:
        # an MN-major A has rows of M elements: M % 8 != 0 breaks the 16-byte stride rule of the tensor maps (M = 1: the
        # [G, K, 1] view keeps a non-unit innermost stride, which the binding refuses first)
        with pytest.raises(RuntimeError, match='16-byte|innermost dim must be contiguous'):
            G.raw_gemm(a_op, b_op, a_mn=True, b_mn=b_mn, epilogue=EPIS[epi][0], **kw)
        return
    run_case(G, a_op, b_op, epi=epi, a_mn=a_mn, b_mn=b_mn, **kw)


# ------------------------------------------------------------------------------------------------------------------
# fp8
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('dtype', [BF16, FP16])
def test_quantize_rows_bit_exact(G, dtype):
    # moe_kernels.h: q = e4m3(x * (1 / s)), s = max|x| / 448 (1 for an all-zero row); rounding to nearest, saturating
    gen = _gen(4)
    x = _rnd(gen, 3, 200, 264, scale=3.0, dtype=dtype)
    x[1, 7] = 0
    x[2, 9, 5] = 1000.0
    q, s = G.quantize_rows(x)
    amax = x.float().abs().amax(-1)
    s_ref = torch.where(amax > 0, amax * (1.0 / 448.0), torch.ones_like(amax))
    q_ref = (x.float() * (1.0 / s_ref)[..., None]).clamp(-448.0, 448.0).to(E4M3)
    assert torch.equal(s, s_ref)
    assert torch.equal(q.view(torch.uint8), q_ref.view(torch.uint8))


@pytest.mark.parametrize('out_dtype', [BF16, FP16], ids=['bf16', 'fp16'])
@pytest.mark.parametrize('dtype', [E4M3, E5M2], ids=['e4m3', 'e5m2'])
@pytest.mark.parametrize('epi', ['none', 'bias', 'bias_relu'])
def test_fp8_epilogues(G, epi, dtype, out_dtype):
    Gn, M, N, K = 3, 328, 264, 208
    gen = _gen(5)
    (aq, sa), (bq, sb) = _quant(_rnd(gen, Gn, M, K), dtype), _quant(_rnd(gen, Gn, N, K), dtype)
    run_case(G, aq, bq, epi=epi, out_dtype=out_dtype, scale_a=sa, scale_b=sb, **_epi_inputs(gen, epi, Gn, M, N, out_dtype))


@pytest.mark.parametrize('dtype', [E4M3, E5M2], ids=['e4m3', 'e5m2'])
@pytest.mark.parametrize('epi', ['relu_bwd', 'add'])
def test_fp8_backward_shapes(G, epi, dtype):
    # dh of the fp8 ReLU FFN (RELU_BWD + bias gradient + row counts) and dx of the fp8 GLU FFN (ADD), on 128 x 256 tiles
    Gn, M, N, K = 4, 640, 1032, 512
    gen = _gen(6)
    (aq, sa), (bq, sb) = _quant(_rnd(gen, Gn, M, K), dtype), _quant(_rnd(gen, Gn, N, K), dtype)
    rc = torch.tensor([640, 300, 0, 129], device='cuda', dtype=torch.int32) if epi == 'relu_bwd' else None
    run_case(G, aq, bq, epi=epi, scale_a=sa, scale_b=sb, row_counts=rc, colsum=epi == 'relu_bwd', sentinel=SENTINEL,
             **_epi_inputs(gen, epi, Gn, M, N, BF16))


@pytest.mark.parametrize('dtype', [BF16, FP16, E4M3, E5M2], ids=['bf16', 'fp16', 'e4m3', 'e5m2'])
@pytest.mark.parametrize('K', [16, 48, 144, 4096, 14336])
def test_accumulation_vs_k(G, K, dtype):
    # fp32 output, so that the accumulation error is not hidden by a 16-bit rounding; prints the normalised error
    # max (|out - ref| - 1/2 ulp) / (2^-24 S) that C_ACC covers
    Gn, M, N = 2, 256, 512
    gen = _gen(7)
    sa = sb = None
    if dtype in (E4M3, E5M2):
        (a, sa), (b, sb) = _quant(_rnd(gen, Gn, M, K), dtype), _quant(_rnd(gen, Gn, N, K), dtype)
    else:
        a, b = _rnd(gen, Gn, M, K, dtype=dtype), _rnd(gen, Gn, N, K, dtype=dtype)
    r = R.ref_gemm(a, b, scale_a=sa, scale_b=sb, out_dtype=FP32)
    outs = {bn: G.raw_gemm(a, b, scale_a=sa, scale_b=sb, out_dtype=FP32, block_n=bn) for bn in BOTH}
    v = r.outs['d'].val
    rel = max(float(((d.double() - v).abs() / v.abs().amax()).max()) for d in outs.values())
    print('\n%s K=%d normalised accumulation error %.3g, max|err| / max|ref| %.2e' % (
        str(dtype)[6:], K, max(R.normalised_error(r, 'd', d) for d in outs.values()), rel))
    for bn, d in outs.items():
        R.check(r, d, what='K=%d block_n=%d' % (K, bn))


# ------------------------------------------------------------------------------------------------------------------
# grouping
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('epi', ['relu_bwd', 'gelu', 'add', 'bias_relu'])
def test_row_counts(G, epi):
    # counts of 0, 1, a block minus one, one block, one block plus one and more than M; NaN in A's and aux's rows past
    # the count must reach neither the valid rows nor the bias gradient
    Gn, M, N, K = 6, 384, 520, 192
    counts = [0, 1, 127, 128, 129, 1000]
    gen = _gen(9)
    a = _rnd(gen, Gn, M, K)
    kw = _epi_inputs(gen, epi, Gn, M, N, BF16)
    for g, c in enumerate(counts):
        a[g, c:] = float('nan')
        if kw['aux'] is not None:
            kw['aux'][g, c:] = float('nan')
    rc = torch.tensor(counts, device='cuda', dtype=torch.int32)
    run_case(G, a, _rnd(gen, Gn, N, K), epi=epi, row_counts=rc, colsum=True, sentinel=SENTINEL, **kw)


@pytest.mark.parametrize('div', [2, 4])
@pytest.mark.parametrize('epi', ['bias', 'relu_bwd'])
def test_b_group_div(G, epi, div):
    # several groups share one B, one bias row and one bias-gradient row
    Gn, M, N, K = 8, 200, 264, 136
    gen = _gen(10)
    a, b = _rnd(gen, Gn, M, K), _rnd(gen, Gn // div, N, K)
    run_case(G, a, b, epi=epi, b_group_div=div, colsum=True, **_epi_inputs(gen, epi, Gn, M, N, BF16, div=div))


@pytest.mark.parametrize('max_ctas', [1, 7])
def test_max_ctas(G, max_ctas):
    Gn, M, N, K = 5, 520, 776, 128
    gen = _gen(11)
    a, b = _rnd(gen, Gn, M, K), _rnd(gen, Gn, N, K)
    run_case(G, a, b, epi='relu_bwd', colsum=True, max_ctas=max_ctas, **_epi_inputs(gen, 'relu_bwd', Gn, M, N, BF16))


# ------------------------------------------------------------------------------------------------------------------
# GLU
# ------------------------------------------------------------------------------------------------------------------
def _glu(G, a, b, b2, *, b_mn, act, scale_a=None, scale_b=None, scale_b2=None, row_counts=None, div=1):
    C = G.backend.require_ext()
    Gn, M = a.size(0), a.size(1)
    N = b.size(2) if b_mn else b.size(1)
    h, g, u = (torch.full((Gn, M, N), SENTINEL, device='cuda', dtype=BF16) for _ in range(3))
    C.gemm_glu(a, b, b2, h, g, u, None, None, b_mn, ACT[act], scale_a, scale_b, scale_b2, row_counts, div, 0, 0, 0, 0, 0, 0, 1)
    r = R.ref_gemm(a, b, b_mn=b_mn, epilogue=R.EPI_GLU, b2=b2, act=ACT[act], scale_a=scale_a, scale_b=scale_b,
                   scale_b2=scale_b2, row_counts=row_counts, b_group_div=div, want_pre=True)
    R.check(r, h, d2=g, d3=u, untouched=SENTINEL, what='glu %s' % act)
    dy = _rnd(_gen(13), Gn, M, 200)
    w = _rnd(_gen(14), (Gn + div - 1) // div, N, 200)       # dh = dy @ w^T ("nk")
    dg, du = (torch.full((Gn, M, N), SENTINEL, device='cuda', dtype=BF16) for _ in range(2))
    gg, uu = g.clone(), u.clone()
    if row_counts is not None:
        for i, c in enumerate(row_counts.tolist()):
            gg[i, c:] = float('nan')
            uu[i, c:] = float('nan')
    C.gemm_glu(dy, w, None, dg, du, None, gg, uu, False, ACT[act], None, None, None, row_counts, div, 0, 0, 0, 0, 0, 0, 1)
    rb = R.ref_gemm(dy, w, epilogue=R.EPI_GLU_BWD, aux=gg, aux2=uu, act=ACT[act], row_counts=row_counts, b_group_div=div)
    R.check(rb, dg, d2=du, untouched=SENTINEL, what='glu_bwd %s' % act)


@pytest.mark.parametrize('variant', ['plain', 'row_counts', 'div2', 'e4m3'])
@pytest.mark.parametrize('act', ['relu', 'gelu', 'silu'])
def test_glu(G, act, variant):
    Gn, M, N, K = 4, 328, 264, 208
    gen = _gen(12)
    div = 2 if variant == 'div2' else 1
    a = _rnd(gen, Gn, M, K)
    rc = torch.tensor([328, 0, 129, 5], device='cuda', dtype=torch.int32) if variant == 'row_counts' else None
    if variant == 'e4m3':
        (aq, sa), (bq, sb), (b2q, sb2) = _quant(a, E4M3), _quant(_rnd(gen, Gn, N, K), E4M3), _quant(_rnd(gen, Gn, N, K), E4M3)
        _glu(G, aq, bq, b2q, b_mn=False, act=act, scale_a=sa, scale_b=sb, scale_b2=sb2)
        return
    b, b2 = _rnd(gen, Gn // div, K, N), _rnd(gen, Gn // div, K, N)
    _glu(G, a, b, b2, b_mn=True, act=act, row_counts=rc, div=div)


# ------------------------------------------------------------------------------------------------------------------
# memory layout and argument checks
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('pad', ['ld', 'group'])
@pytest.mark.parametrize('epi', ['add', 'gelu', 'bias_relu'])
def test_strided_views(G, epi, pad):
    # A, B, aux and out are slices of wider tensors: a padded leading dimension or a padded group stride
    Gn, M, N, K = 3, 328, 264, 200
    gen = _gen(15)
    wide = lambda *s: _rnd(gen, *s)                                                   # noqa: E731
    if pad == 'ld':
        a, b = wide(Gn, M, K + 24)[..., :K], wide(Gn, N, K + 8)[..., :K]
        base = torch.full((Gn, M, N + 16), SENTINEL, device='cuda', dtype=BF16)
        out = base[..., :N]
        aux = wide(Gn, M, N + 8)[..., :N] if EPIS[epi][2] else None
    else:
        a, b = wide(Gn, M + 8, K)[:, :M], wide(Gn, N + 16, K)[:, :N]
        base = torch.full((Gn, M + 40, N), SENTINEL, device='cuda', dtype=BF16)
        out = base[:, :M]
        aux = wide(Gn, M + 8, N)[:, :M] if EPIS[epi][2] else None
    epilogue, _, _, has_pre = EPIS[epi]
    bias = _rnd(gen, Gn, N, scale=1.0) if aux is None else None
    r = R.ref_gemm(a, b, epilogue=epilogue, bias=bias, aux=aux)
    for bn in BOTH:
        base.fill_(SENTINEL)
        d = G.raw_gemm(a, b, epilogue=epilogue, bias=bias, aux=aux, out=out, block_n=bn)
        assert d.data_ptr() == out.data_ptr()
        R.check(r, out, what='%s %s bn=%d' % (epi, pad, bn))
        rest = base.clone()
        rest[:, :M, :N] = SENTINEL
        assert torch.all(rest == SENTINEL), 'the padding around the output view was written'


def test_inplace_add(G):
    Gn, M, N, K = 3, 328, 264, 200
    gen = _gen(16)
    a, b, aux = _rnd(gen, Gn, M, K), _rnd(gen, Gn, N, K), _rnd(gen, Gn, M, N, scale=1.0)
    r = R.ref_gemm(a, b, epilogue=R.EPI_ADD, aux=aux)
    for bn in BOTH:
        buf = aux.clone()
        G.raw_gemm(a, b, epilogue=R.EPI_ADD, aux=buf, out=buf, block_n=bn)
        R.check(r, buf, what='in-place add bn=%d' % bn)


def test_colsum_unaligned_view(G):
    # a bias-gradient row at a 4-byte but not 16-byte offset takes the scalar-atomic path
    Gn, M, N, K = 3, 328, 264, 200
    gen = _gen(17)
    a, b, aux = _rnd(gen, Gn, M, K), _rnd(gen, Gn, N, K), _rnd(gen, Gn, M, N, scale=1.0)
    r = R.ref_gemm(a, b, epilogue=R.EPI_RELU_BWD, aux=aux)
    for bn in BOTH:
        flat = torch.zeros(Gn * N + 4, device='cuda')
        cs = flat[1:1 + Gn * N].view(Gn, N)
        assert cs.data_ptr() % 16 == 4
        d = G.raw_gemm(a, b, epilogue=R.EPI_RELU_BWD, aux=aux, colsum=cs, block_n=bn)
        R.check(r, d, colsum=cs, what='bn=%d' % bn)
        assert flat[0].item() == 0 and torch.all(flat[1 + Gn * N:] == 0)


@pytest.mark.parametrize('which', ['a', 'b', 'aux'])
def test_expanded_operands(G, which):
    # a stride-0 group dimension (one matrix broadcast to every group) is materialised, and both configurations agree
    Gn, M, N, K = 4, 256, 264, 64
    gen = _gen(18)
    a, b, aux = _rnd(gen, Gn, M, K), _rnd(gen, Gn, N, K), _rnd(gen, Gn, M, N, scale=1.0)
    if which == 'a':
        a = _rnd(gen, 1, M, K).expand(Gn, M, K)
    elif which == 'b':
        b = _rnd(gen, 1, N, K).expand(Gn, N, K)
    else:
        aux = _rnd(gen, 1, M, N, scale=1.0).expand(Gn, M, N)
    res = run_case(G, a, b, epi='add', aux=aux)
    assert torch.equal(res[128][0], res[0][0])


def test_expanded_operand_rejected_by_the_launcher(G):
    C = G.backend.require_ext()
    a = _rnd(_gen(19), 1, 256, 64).expand(4, 256, 64)
    b = _rnd(_gen(20), 4, 128, 64)
    d = torch.empty(4, 256, 128, device='cuda', dtype=BF16)
    with pytest.raises(RuntimeError, match='group strides'):
        C.gemm_ex(a, b, d, False, False, 0, None, None, None, 1.0, 1, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1, None, None, None, None, 0)


def test_misaligned_side_inputs(G):
    # bias and scale_b views at odd element offsets: raw_gemm copies them, the binding refuses them
    Gn, M, N, K = 3, 328, 264, 208
    gen = _gen(21)
    a, b = _rnd(gen, Gn, M, K), _rnd(gen, Gn, N, K)
    bias = _rnd(gen, Gn * N + 1, scale=1.0)[1:].view(Gn, N)
    assert bias.data_ptr() % 16 == 2
    run_case(G, a, b, epi='bias_relu', bias=bias)
    (aq, sa), (bq, sb) = _quant(a, E4M3), _quant(b, E4M3)
    flat = torch.empty(Gn * N + 1, device='cuda')
    flat[1:] = sb.flatten()
    sb_odd = flat[1:].view(Gn, N)
    assert sb_odd.data_ptr() % 8 == 4
    run_case(G, aq, bq, epi='bias', bias=_rnd(gen, Gn, N, scale=1.0), scale_a=sa, scale_b=sb_odd)
    C = G.backend.require_ext()
    d = torch.empty(Gn, M, N, device='cuda', dtype=BF16)
    with pytest.raises(RuntimeError, match='bias rows'):
        C.gemm_ex(a, b, d, False, False, R.EPI_BIAS, bias, None, None, 1.0, 1, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1, None, None, None, None, 0)
    with pytest.raises(RuntimeError, match='scale_b rows'):
        C.gemm_ex(aq, bq, d, False, False, 0, None, None, None, 1.0, 1, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1, sa, sb_odd, None, None, 0)
    with pytest.raises(RuntimeError, match='bias must be'):      # a bias with fewer rows than B groups
        C.gemm_ex(a, b, d, False, False, R.EPI_BIAS, bias[:2].contiguous(), None, None, 1.0, 1, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1,
                  None, None, None, None, 0)


def test_argument_checks(G):
    gen = _gen(22)
    a, b = _rnd(gen, 6, 128, 64), _rnd(gen, 6, 128, 64)
    with pytest.raises(RuntimeError, match='group_mod'):
        G.raw_gemm(a, b, group_rot=1, group_mod=4)                        # 6 groups in blocks of 4
    with pytest.raises(RuntimeError, match='group_mod'):
        G.raw_gemm(a, b, group_rot=0, group_mod=-4)
    with pytest.raises(RuntimeError, match='alpha'):
        G.raw_gemm(a, b, epilogue=R.EPI_BIAS, bias=_rnd(gen, 6, 128), alpha=0.5)


# ------------------------------------------------------------------------------------------------------------------
# the fused engine's launch arguments on one GPU (no peers)
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('rot,mod', [(1, 4), (2, -4)])
def test_fused_engine_arguments(G, rot, mod):
    Gn, W, M, N, K = 8, 2, 300, 264, 192
    gen = _gen(23)
    a, b = _rnd(gen, Gn, M, K), _rnd(gen, Gn // W, N, K)
    bias = _rnd(gen, Gn // W, N, scale=1.0)
    rows_per_flag, target = 64, 5
    flags_per_group = -(-M // rows_per_flag)
    # every flag index the producer can compute is inside the group's flags, and all of them are already at the target,
    # so no wait can spin
    for m0 in range(0, M, 128):
        assert m0 // rows_per_flag < flags_per_group and (min(m0 + 128, M) - 1) // rows_per_flag < flags_per_group
    flags = torch.full((Gn * flags_per_group,), target, device='cuda', dtype=torch.int32)
    outs = [torch.full((M, N), SENTINEL, device='cuda', dtype=BF16) for _ in range(Gn)]
    d_tab = torch.tensor([t.data_ptr() for t in outs], device='cuda', dtype=torch.int64)
    counters = torch.zeros(Gn, device='cuda', dtype=torch.int32)
    s_tab = torch.tensor([counters.data_ptr() + 4 * g for g in range(Gn)], device='cuda', dtype=torch.int64)
    dummy = torch.full((Gn, M, N), SENTINEL, device='cuda', dtype=BF16)
    G.raw_gemm(a, b, epilogue=R.EPI_BIAS_RELU, bias=bias, b_group_div=W, block_n=128, out=dummy, d_ptr_table=d_tab.data_ptr(),
               signal_ptr_table=s_tab.data_ptr(), wait_flags=flags.data_ptr(), wait_rows_per_flag=rows_per_flag,
               wait_flags_per_group=flags_per_group, wait_target=target, group_rot=rot, group_mod=mod)
    torch.cuda.synchronize()
    assert torch.all(dummy == SENTINEL), 'with a pointer table the output tensor itself is not written'
    assert counters.tolist() == [math.ceil(M / 128) * math.ceil(N / 128)] * Gn
    d = torch.stack(outs)
    r = R.ref_gemm(a, b, epilogue=R.EPI_BIAS_RELU, bias=bias, b_group_div=W)
    R.check(r, d, what='fused rot=%d mod=%d' % (rot, mod))
    plain = G.raw_gemm(a, b, epilogue=R.EPI_BIAS_RELU, bias=bias, b_group_div=W, block_n=128)
    assert torch.equal(d, plain)
