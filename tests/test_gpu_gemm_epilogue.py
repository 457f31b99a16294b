"""The 128 x 256 configuration's register epilogue (TMA-stored output, TMA-loaded aux operand, CTA-reduced bias
gradient) against the 128 x 128 configuration (block_n=128): both apply the same per-element formulas to the same
accumulators, so every output must agree bit for bit."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def G():
    from tutel_b200.ops import backend, gemm
    backend.require_ext()
    return gemm


def _rand(gen, *shape, scale=1.0, dtype=torch.bfloat16):
    return (torch.randn(*shape, device='cuda', generator=gen) * scale).to(dtype)


def _both(fn):
    """fn(block_n) -> tuple of tensors; returns (narrow, wide)."""
    return fn(128), fn(0)


def _epi_kwargs(G, epi, gen, Gn, M, N, dtype):
    bias = _rand(gen, Gn, N, dtype=dtype)
    aux = _rand(gen, Gn, M, N, dtype=dtype)
    if epi == 'none':
        return dict(alpha=0.5), False
    if epi == 'bias':
        return dict(epilogue=G.EPI_BIAS, bias=bias), False
    if epi == 'bias_relu':
        return dict(epilogue=G.EPI_BIAS_RELU, bias=bias), False
    if epi in ('gelu', 'silu'):
        return dict(epilogue=G.FWD_EPILOGUE[epi], bias=bias), True
    if epi == 'relu_bwd':
        return dict(epilogue=G.EPI_RELU_BWD, aux=aux), False
    if epi in ('act_bwd_gelu', 'act_bwd_silu'):
        return dict(epilogue=G.EPI_ACT_BWD, aux=aux, act=G.ACT_CODES[epi[8:]]), False
    assert epi == 'add'
    return dict(epilogue=G.EPI_ADD, aux=aux), False


EPILOGUES = ['none', 'bias', 'bias_relu', 'gelu', 'silu', 'relu_bwd', 'act_bwd_gelu', 'act_bwd_silu', 'add']


def _run(G, a, b, kw, with_pre, shape, dtype, **extra):
    def fn(bn):
        pre = torch.full(shape, 3.0, device='cuda', dtype=dtype) if with_pre else None
        d = G.raw_gemm(a, b, block_n=bn, d2=pre, **kw, **extra)
        return (d,) if pre is None else (d, pre)
    return _both(fn)


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16])
@pytest.mark.parametrize('epi', EPILOGUES)
def test_epilogue_bit_identical_many_tiles(G, epi, dtype):
    # 8 x 8 x 8 = 512 tiles of 128 x 256: every CTA runs several tiles back to back, so the output tile is reused and
    # the aux operand is prefetched while the previous tile's store drains
    Gn, M, N, K = 8, 1024, 2048, 256
    gen = torch.Generator(device='cuda').manual_seed(11)
    a, b = _rand(gen, Gn, M, K, scale=0.5, dtype=dtype), _rand(gen, Gn, N, K, scale=0.5, dtype=dtype)
    kw, with_pre = _epi_kwargs(G, epi, gen, Gn, M, N, dtype)
    narrow, wide = _run(G, a, b, kw, with_pre, (Gn, M, N), dtype)
    for x, y in zip(narrow, wide):
        assert torch.equal(x, y)


@pytest.mark.parametrize('epi', ['none', 'bias_relu', 'gelu', 'relu_bwd', 'add'])
@pytest.mark.parametrize('a_mn,b_mn', [(False, True), (True, False), (True, True)])
def test_epilogue_bit_identical_mn_major_tails(G, epi, a_mn, b_mn):
    # M = 328 and N = 264: partial row block and a 256-wide tile with a single valid 64-column box (TMA-clipped)
    Gn, M, N, K = 3, 328, 264, 200
    gen = torch.Generator(device='cuda').manual_seed(12)
    a, b = _rand(gen, Gn, M, K, scale=0.5), _rand(gen, Gn, N, K, scale=0.5)
    a_op = a.transpose(1, 2).contiguous() if a_mn else a
    b_op = b.transpose(1, 2).contiguous() if b_mn else b
    kw, with_pre = _epi_kwargs(G, epi, gen, Gn, M, N, torch.bfloat16)
    narrow, wide = _run(G, a_op, b_op, kw, with_pre, (Gn, M, N), torch.bfloat16, a_mn=a_mn, b_mn=b_mn)
    for x, y in zip(narrow, wide):
        assert torch.equal(x, y)


@pytest.mark.parametrize('epi', ['none', 'bias', 'bias_relu'])
def test_epilogue_bit_identical_e4m3_scales(G, epi):
    Gn, M, N, K = 2, 392, 776, 512
    gen = torch.Generator(device='cuda').manual_seed(13)
    a, b = _rand(gen, Gn, M, K, scale=0.5), _rand(gen, Gn, N, K, scale=0.5)
    aq, sa = G.quantize_rows(a)
    bq, sb = G.quantize_rows(b)
    kw, _ = _epi_kwargs(G, epi, gen, Gn, M, N, torch.bfloat16)
    narrow, wide = _run(G, aq, bq, kw, False, None, torch.bfloat16, scale_a=sa, scale_b=sb, out_dtype=torch.bfloat16)
    assert torch.equal(narrow[0], wide[0])
    ref = torch.matmul(a.float(), b.float().transpose(1, 2))
    if epi == 'none':
        assert ((wide[0].float() - 0.5 * ref).norm() / (0.5 * ref).norm()).item() < 0.06


@pytest.mark.parametrize('epi', ['relu_bwd', 'bias_relu', 'gelu'])
def test_epilogue_row_counts_straddle(G, epi):
    # counts end inside a row block (the row-guarded copy), on a block boundary, at zero and past M
    Gn, M, N, K = 5, 512, 520, 192
    counts = [300, 0, 128, 1, 512]
    gen = torch.Generator(device='cuda').manual_seed(14)
    a, b = _rand(gen, Gn, M, K, scale=0.5), _rand(gen, Gn, N, K, scale=0.5)
    rc = torch.tensor(counts, device='cuda', dtype=torch.int32)
    kw, with_pre = _epi_kwargs(G, epi, gen, Gn, M, N, torch.bfloat16)

    def fn(bn):
        d = torch.full((Gn, M, N), 7.0, device='cuda', dtype=torch.bfloat16)
        pre = torch.full((Gn, M, N), 3.0, device='cuda', dtype=torch.bfloat16) if with_pre else None
        G.raw_gemm(a, b, block_n=bn, row_counts=rc, out=d, d2=pre, **kw)
        return (d,) if pre is None else (d, pre)

    narrow, wide = _both(fn)
    for x, y in zip(narrow, wide):
        assert torch.equal(x, y)
    for g, c in enumerate(counts):
        assert torch.all(wide[0][g, c:] == 7.0)      # rows past the count are never written
        if with_pre:
            assert torch.all(wide[1][g, c:] == 3.0)


@pytest.mark.parametrize('counts', [None, [1024, 700, 0, 129, 1024, 5, 1000, 1023]])
def test_epilogue_colsum(G, counts):
    # the bias gradient summed in the CTA (one global add per column and tile) against an fp32 sum of the output
    Gn, M, N, K = 8, 1024, 2048, 256
    gen = torch.Generator(device='cuda').manual_seed(15)
    a, b = _rand(gen, Gn, M, K, scale=0.5), _rand(gen, Gn, N, K, scale=0.5)
    aux = _rand(gen, Gn, M, N)
    rc = torch.tensor(counts, device='cuda', dtype=torch.int32) if counts is not None else None
    outs = {}
    for bn in (128, 0):
        cs = torch.zeros(Gn, N, device='cuda')
        d = torch.zeros(Gn, M, N, device='cuda', dtype=torch.bfloat16)
        G.raw_gemm(a, b, epilogue=G.EPI_RELU_BWD, aux=aux, colsum=cs, row_counts=rc, out=d, block_n=bn)
        outs[bn] = (d, cs)
    assert torch.equal(outs[128][0], outs[0][0])
    ref = torch.where(aux.float() > 0, torch.matmul(a.float(), b.float().transpose(1, 2)), torch.zeros((), device='cuda'))
    if counts is not None:
        for g, c in enumerate(counts):
            ref[g, c:] = 0
    want = ref.sum(1)
    scale = want.abs().max().item()
    for bn in (128, 0):
        assert (outs[bn][1] - want).abs().max().item() <= 2e-3 * scale
    # the two configurations differ only in the order of the fp32 additions
    assert (outs[0][1] - outs[128][1]).abs().max().item() <= 5e-4 * scale


def test_epilogue_consecutive_calls_reuse(G):
    # back-to-back wide launches with different epilogues on the same stream: nothing leaks between calls
    Gn, M, N, K = 4, 512, 1024, 128
    gen = torch.Generator(device='cuda').manual_seed(16)
    a, b = _rand(gen, Gn, M, K, scale=0.5), _rand(gen, Gn, N, K, scale=0.5)
    aux = _rand(gen, Gn, M, N)
    ref = torch.matmul(a.float(), b.float().transpose(1, 2))
    d1 = G.raw_gemm(a, b, epilogue=G.EPI_ADD, aux=aux)
    d2 = G.raw_gemm(a, b)
    d3 = G.raw_gemm(a, b, epilogue=G.EPI_RELU_BWD, aux=aux)
    assert torch.allclose(d1.float(), ref + aux.float(), atol=0.1, rtol=2e-2)
    assert torch.allclose(d2.float(), ref, atol=0.08, rtol=2e-2)
    assert torch.allclose(d3.float(), torch.where(aux.float() > 0, ref, torch.zeros((), device='cuda')), atol=0.08, rtol=2e-2)
