"""The 128 x 256 tile configuration of the grouped GEMM (block_n=0, the launcher's choice) against fp32 PyTorch
references, and against the 128 x 128 configuration (block_n=128) that the fused multi-GPU engine runs."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def G():
    from tutel_b200.ops import backend, gemm
    backend.require_ext()
    return gemm


def _operands(G_, M, N, K, dtype, seed, gb=None):
    g = torch.Generator(device='cuda').manual_seed(seed)
    a = (torch.randn(G_, M, K, device='cuda', generator=g) * 0.5).to(dtype)
    b = (torch.randn(gb or G_, N, K, device='cuda', generator=g) * 0.5).to(dtype)
    return a, b


def _mm(a, b, div=1):
    bb = b.float().repeat_interleave(div, dim=0)[: a.size(0)]
    return torch.matmul(a.float(), bb.transpose(1, 2))


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16])
@pytest.mark.parametrize('a_mn,b_mn', [(False, False), (False, True), (True, False), (True, True)])
def test_wide_all_layouts(G, dtype, a_mn, b_mn):
    # M = 328 (a partial last row block) and N = 264 (a partial 256-wide tile)
    a, b = _operands(3, 328, 264, 200, dtype, 0)
    a_op = a.transpose(1, 2).contiguous() if a_mn else a
    b_op = b.transpose(1, 2).contiguous() if b_mn else b
    d = G.raw_gemm(a_op, b_op, a_mn=a_mn, b_mn=b_mn)
    assert torch.allclose(d.float(), _mm(a, b), atol=0.08, rtol=2e-2)


@pytest.mark.parametrize('epi', ['none', 'bias', 'bias_relu', 'gelu', 'silu', 'relu_bwd', 'act_bwd', 'add'])
def test_wide_epilogues(G, epi):
    M, N, K = 640, 520, 1096
    a, b = _operands(2, M, N, K, torch.bfloat16, 1)
    a, b = a * 0.5, b * 0.5
    gen = torch.Generator(device='cuda').manual_seed(2)
    bias = torch.randn(2, N, device='cuda', generator=gen).bfloat16()
    aux = torch.randn(2, M, N, device='cuda', generator=gen).bfloat16()
    ref = _mm(a, b)
    kw, pre = {}, None
    if epi == 'none':
        kw, want = dict(alpha=0.5), ref * 0.5
    elif epi == 'bias':
        kw, want = dict(epilogue=G.EPI_BIAS, bias=bias), ref + bias.float().unsqueeze(1)
    elif epi == 'bias_relu':
        kw, want = dict(epilogue=G.EPI_BIAS_RELU, bias=bias), torch.relu(ref + bias.float().unsqueeze(1))
    elif epi in ('gelu', 'silu'):
        pre = torch.empty(2, M, N, device='cuda', dtype=torch.bfloat16)
        x = ref + bias.float().unsqueeze(1)
        kw = dict(epilogue=G.FWD_EPILOGUE[epi], bias=bias, d2=pre)
        want = torch.nn.functional.gelu(x) if epi == 'gelu' else torch.nn.functional.silu(x)
    elif epi == 'relu_bwd':
        kw, want = dict(epilogue=G.EPI_RELU_BWD, aux=aux), torch.where(aux.float() > 0, ref, torch.zeros((), device='cuda'))
    elif epi == 'act_bwd':
        f = aux.float()
        sg = torch.sigmoid(f)
        kw, want = dict(epilogue=G.EPI_ACT_BWD, aux=aux, act=G.ACT_CODES['silu']), ref * sg * (1 + f * (1 - sg))
    else:
        kw, want = dict(epilogue=G.EPI_ADD, aux=aux), ref + aux.float()
    d = G.raw_gemm(a, b, **kw)
    assert torch.allclose(d.float(), want, atol=0.1, rtol=2e-2)
    if pre is not None:
        assert torch.allclose(pre.float(), ref + bias.float().unsqueeze(1), atol=0.1, rtol=2e-2)


def test_wide_colsum_row_counts(G):
    # counts leave row blocks whole, partial and skipped; group 1 is empty
    M, N, K = 512, 264, 320
    counts = [512, 0, 130, 257, 385]
    a, b = _operands(len(counts), M, N, K, torch.bfloat16, 3)
    rc = torch.tensor(counts, device='cuda', dtype=torch.int32)
    gen = torch.Generator(device='cuda').manual_seed(4)
    aux = torch.randn(len(counts), M, N, device='cuda', generator=gen).bfloat16()
    colsum = torch.zeros(len(counts), N, device='cuda')
    d = torch.full((len(counts), M, N), 7.0, device='cuda', dtype=torch.bfloat16)
    G.raw_gemm(a, b, epilogue=G.EPI_RELU_BWD, aux=aux, row_counts=rc, colsum=colsum, out=d)
    ref = torch.where(aux.float() > 0, _mm(a, b), torch.zeros((), device='cuda'))
    for g, c in enumerate(counts):
        assert torch.allclose(d[g, :c].float(), ref[g, :c], atol=0.3, rtol=2e-2)
        assert torch.all(d[g, c:] == 7.0)            # rows past the count are never written
        want = d[g, :c].float().sum(0)
        assert torch.allclose(colsum[g], want, atol=0.5, rtol=1e-2)


def test_wide_grouped_b_div(G):
    a, b = _operands(4, 384, 520, 264, torch.bfloat16, 5, gb=2)
    d = G.raw_gemm(a, b, b_group_div=2)
    assert torch.allclose(d.float(), _mm(a, b, div=2), atol=0.08, rtol=2e-2)


def test_wide_fp8_scales(G):
    a, b = _operands(2, 384, 520, 512, torch.bfloat16, 6)
    aq, sa = G.quantize_rows(a)
    bq, sb = G.quantize_rows(b)
    d = G.raw_gemm(aq, bq, scale_a=sa, scale_b=sb, out_dtype=torch.bfloat16)
    ref = _mm(a, b)
    assert ((d.float() - ref).norm() / ref.norm()).item() < 0.06


@pytest.mark.parametrize('epi', ['bias_relu', 'relu_bwd_colsum'])
def test_wide_matches_narrow(G, epi):
    # same inputs through block_n=128 and the automatic choice: every element sums the same products in
    # the same K order, so the results agree to the last bit (the atomically accumulated colsum to rounding)
    a, b = _operands(3, 520, 1032, 776, torch.bfloat16, 7)
    gen = torch.Generator(device='cuda').manual_seed(8)
    bias = torch.randn(3, 1032, device='cuda', generator=gen).bfloat16()
    aux = torch.randn(3, 520, 1032, device='cuda', generator=gen).bfloat16()
    outs = []
    for bn in (128, 0):
        if epi == 'bias_relu':
            outs.append((G.raw_gemm(a, b, epilogue=G.EPI_BIAS_RELU, bias=bias, block_n=bn), None))
        else:
            cs = torch.zeros(3, 1032, device='cuda')
            outs.append((G.raw_gemm(a, b, epilogue=G.EPI_RELU_BWD, aux=aux, colsum=cs, block_n=bn), cs))
    assert torch.equal(outs[0][0], outs[1][0])
    if outs[0][1] is not None:
        assert torch.allclose(outs[0][1], outs[1][1], atol=1e-3, rtol=1e-5)
