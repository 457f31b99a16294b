"""Protocol edges of the 128 x 256 grouped GEMM's store warp: the warp that stores each output tile, loads the next
tile's aux operand into it, copies bias / column scales into shared memory and reduces the bias gradient.

Every output is compared bit for bit with the 128 x 128 configuration (block_n=128), which has no store warp and
computes each element with the same formula and K order; the bias gradient, whose fp32 summation order differs between
the two, is checked against the fp64 reference of tests/gemm_reference.py.
"""
import pytest
import torch

import gemm_reference as R

pytestmark = pytest.mark.gpu

SENTINEL = -7.0


@pytest.fixture(scope='module')
def G():
    from tutel_b200.ops import backend, gemm
    backend.require_ext()
    return gemm


def _rand(gen, *shape, scale=1.0, dtype=torch.bfloat16):
    return (torch.randn(*shape, device='cuda', generator=gen) * scale).to(dtype)


def _both(G, a, b, **kw):
    """Run the same launch in both configurations into sentinel-filled outputs; returns (wide, narrow)."""
    outs = []
    for bn in (0, 128):
        d = torch.full((a.size(0), a.size(1), b.size(1)), SENTINEL, device='cuda', dtype=torch.bfloat16)
        G.raw_gemm(a, b, out=d, block_n=bn, **kw)
        outs.append(d)
    torch.cuda.synchronize()
    return outs


def _epi_kwargs(G, epi, gen, Gn, M, N):
    if epi == 'relu_bwd':
        return dict(epilogue=G.EPI_RELU_BWD, aux=_rand(gen, Gn, M, N))
    if epi == 'add':
        return dict(epilogue=G.EPI_ADD, aux=_rand(gen, Gn, M, N))
    if epi == 'act_bwd':
        return dict(epilogue=G.EPI_ACT_BWD, aux=_rand(gen, Gn, M, N), act=G.ACT_CODES['gelu'])
    if epi == 'bias_relu':
        return dict(epilogue=G.EPI_BIAS_RELU, bias=_rand(gen, Gn, N, scale=0.5))
    if epi == 'bias':
        return dict(epilogue=G.EPI_BIAS, bias=_rand(gen, Gn, N, scale=0.5))
    return {}


@pytest.mark.parametrize('K', [64, 128])
@pytest.mark.parametrize('epi', ['relu_bwd', 'add', 'act_bwd'])
def test_short_k_aux(G, K, epi):
    # one or two K blocks per tile: the aux load for tile i + 1 and the store of tile i overlap almost nothing
    gen = torch.Generator(device='cuda').manual_seed(10 + K)
    Gn, M, N = 3, 384, 776
    a, b = _rand(gen, Gn, M, K), _rand(gen, Gn, N, K, scale=K ** -0.5)
    wide, narrow = _both(G, a, b, **_epi_kwargs(G, epi, gen, Gn, M, N))
    assert torch.equal(wide, narrow)


@pytest.mark.parametrize('max_ctas', [1, 3])
@pytest.mark.parametrize('epi', ['relu_bwd', 'bias_relu', 'none', 'gelu'])
def test_few_ctas_many_tiles(G, max_ctas, epi):
    # 4 x 8 x 8 = 256 tiles on one or three CTAs: every barrier phase wraps many times
    gen = torch.Generator(device='cuda').manual_seed(20 + max_ctas)
    Gn, M, N, K = 4, 1024, 2048, 128
    a, b = _rand(gen, Gn, M, K), _rand(gen, Gn, N, K, scale=K ** -0.5)
    if epi == 'gelu':
        bias = _rand(gen, Gn, N, scale=0.5)
        pres = [torch.full((Gn, M, N), SENTINEL, device='cuda', dtype=torch.bfloat16) for _ in range(2)]
        outs = [torch.empty(Gn, M, N, device='cuda', dtype=torch.bfloat16) for _ in range(2)]
        for bn, d, pre in zip((0, 128), outs, pres):
            G.raw_gemm(a, b, out=d, epilogue=G.EPI_BIAS_GELU, bias=bias, d2=pre, block_n=bn,
                       max_ctas=max_ctas if bn == 0 else 0)
        assert torch.equal(outs[0], outs[1])
        assert torch.equal(pres[0], pres[1])
        return
    kw = _epi_kwargs(G, epi, gen, Gn, M, N)
    wide = torch.empty(Gn, M, N, device='cuda', dtype=torch.bfloat16)
    G.raw_gemm(a, b, out=wide, max_ctas=max_ctas, **kw)
    narrow = G.raw_gemm(a, b, block_n=128, **kw)
    assert torch.equal(wide, narrow)


@pytest.mark.parametrize('epi', ['relu_bwd', 'bias_relu', 'add'])
@pytest.mark.parametrize('max_ctas', [0, 2])
def test_row_counts_interleaved(G, epi, max_ctas):
    # empty groups between groups with straddling row blocks; rows past each count must keep the sentinel
    gen = torch.Generator(device='cuda').manual_seed(30)
    counts = [300, 0, 128, 0, 515, 1, 0, 640]
    Gn, M, N, K = len(counts), 640, 520, 192
    a, b = _rand(gen, Gn, M, K), _rand(gen, Gn, N, K, scale=K ** -0.5)
    rc = torch.tensor(counts, device='cuda', dtype=torch.int32)
    kw = _epi_kwargs(G, epi, gen, Gn, M, N)
    outs = []
    for bn in (0, 128):
        d = torch.full((Gn, M, N), SENTINEL, device='cuda', dtype=torch.bfloat16)
        G.raw_gemm(a, b, out=d, row_counts=rc, block_n=bn, max_ctas=max_ctas if bn == 0 else 0, **kw)
        outs.append(d)
    assert torch.equal(outs[0], outs[1])
    for g, c in enumerate(counts):
        assert bool((outs[0][g, c:] == SENTINEL).all()), 'group %d: rows past the count were written' % g


@pytest.mark.parametrize('N', [136, 520])
@pytest.mark.parametrize('epi', ['bias', 'bias_relu'])
def test_bias_n_tail(G, N, epi):
    gen = torch.Generator(device='cuda').manual_seed(40 + N)
    Gn, M, K = 3, 256, 256
    a, b = _rand(gen, Gn, M, K), _rand(gen, Gn, N, K, scale=K ** -0.5)
    wide, narrow = _both(G, a, b, max_ctas=2, **_epi_kwargs(G, epi, gen, Gn, M, N))
    assert torch.equal(wide, narrow)


@pytest.mark.parametrize('N', [136, 520])
@pytest.mark.parametrize('aligned', [True, False])
def test_fp8_scale_b_n_tail(G, N, aligned):
    # scale_b rows need only 8-byte alignment; rows that are not all 16-byte aligned cannot be bulk-copied and take the
    # 128 x 128 configuration
    from tutel_b200.ops import backend
    gen = torch.Generator(device='cuda').manual_seed(50 + N)
    Gn, M, K = 2, 256, 256
    aq, sa = G.quantize_rows(_rand(gen, Gn, M, K))
    bq, sb = G.quantize_rows(_rand(gen, Gn, N, K))
    sb = sb.reshape(Gn, N).float()
    if not aligned:
        # rows of N + 2 floats starting 8 bytes into a 16-byte aligned buffer
        buf = torch.zeros(Gn, N + 2, device='cuda')
        buf[:, 2:] = sb
        sb = buf[:, 2:]
        assert sb.data_ptr() % 16 == 8
    bias = _rand(gen, Gn, N, scale=0.5)
    C = backend.require_ext()
    outs = []
    for bn in (0, 128):
        d = torch.full((Gn, M, N), SENTINEL, device='cuda', dtype=torch.bfloat16)
        C.gemm_ex(aq, bq, d, False, False, G.EPI_BIAS, bias, None, None, 1.0, 1, 0, bn, 0, 0, 0, 0, 0, 0,
                  1 if bn == 0 else 0, 0, 1, sa, sb, None, None, 0)
        outs.append(d)
    torch.cuda.synchronize()
    assert torch.equal(outs[0], outs[1])


@pytest.mark.parametrize('max_ctas', [1, 0])
def test_colsum_against_reference(G, max_ctas):
    # bias gradient of the ReLU backward GEMM, with straddling and empty groups, against the fp64 reference
    gen = torch.Generator(device='cuda').manual_seed(60)
    counts = [640, 0, 200, 513]
    Gn, M, N, K = len(counts), 640, 776, 128
    a, b = _rand(gen, Gn, M, K), _rand(gen, Gn, N, K, scale=K ** -0.5)
    aux = _rand(gen, Gn, M, N)
    rc = torch.tensor(counts, device='cuda', dtype=torch.int32)
    init = torch.randn(Gn, N, device='cuda', generator=gen)
    colsum = init.clone()
    d = torch.full((Gn, M, N), SENTINEL, device='cuda', dtype=torch.bfloat16)
    G.raw_gemm(a, b, out=d, epilogue=G.EPI_RELU_BWD, aux=aux, row_counts=rc, colsum=colsum, max_ctas=max_ctas)
    ref = R.ref_gemm(a, b, epilogue=R.EPI_RELU_BWD, aux=aux, row_counts=rc)
    R.check(ref, d, colsum=colsum, colsum_init=init, untouched=SENTINEL, what='relu_bwd colsum max_ctas=%d' % max_ctas)
    narrow = torch.full_like(d, SENTINEL)
    G.raw_gemm(a, b, out=narrow, epilogue=G.EPI_RELU_BWD, aux=aux, row_counts=rc, block_n=128)
    assert torch.equal(d, narrow)


def test_back_to_back_same_output(G):
    # consecutive launches into one output, the second reading the first's result as its aux operand and the third
    # adding to it: each launch's last stores must have landed before the next launch reads them
    gen = torch.Generator(device='cuda').manual_seed(70)
    Gn, M, N, K = 2, 512, 1024, 256
    a, b = _rand(gen, Gn, M, K), _rand(gen, Gn, N, K, scale=K ** -0.5)
    bias = _rand(gen, Gn, N, scale=0.5)
    res = []
    for bn in (0, 128):
        h = torch.empty(Gn, M, N, device='cuda', dtype=torch.bfloat16)
        g2 = torch.empty_like(h)
        G.raw_gemm(a, b, out=h, epilogue=G.EPI_BIAS_RELU, bias=bias, block_n=bn)
        G.raw_gemm(a, b, out=g2, epilogue=G.EPI_RELU_BWD, aux=h, block_n=bn)
        G.raw_gemm(a, b, out=g2, epilogue=G.EPI_ADD, aux=g2, block_n=bn)
        for _ in range(3):
            G.raw_gemm(a, b, out=h, epilogue=G.EPI_BIAS_RELU, bias=bias, block_n=bn)
        res.append((h, g2))
    torch.cuda.synchronize()
    assert torch.equal(res[0][0], res[1][0])
    assert torch.equal(res[0][1], res[1][1])
