"""Dropless ("Megablocks") inference for SwiGLU (`llama_ffn`) experts: the one-launch skinny GLU kernel against a float64
reference, and the layer's choice between it, the dual-B wgmma kernel with row counts and the padded path."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

ACTS = {'relu': 1, 'gelu': 2, 'silu': 3}
# Largest |act'(v)|: 1 for ReLU, 1.0998 for SiLU, 1.1289 for erf-GELU.  Bounds the layer-1 error's effect on act(g).
ACT_LIPSCHITZ = 1.13
U32 = 2.0 ** -24
# C_GLU = 2: with fp32 accumulation, the gate / up sums over M and the output sums over H each carry at most
# n * 2^-24 * sum|terms| of rounding error to first order, i.e. c = 1 for the bound below.  The factor 2 covers the
# second-order terms and the few ulps of erff / __expf and of the act(g) * u product, which (M + H) * |h| dominates.
C_GLU = 2.0


@pytest.fixture(scope='module')
def C():
    from tutel_b200.ops import backend
    return backend.require_ext()


def _ref_and_bound(x, w1, w2, w3, act):
    """float64 y = (act(x @ W1) * (x @ W2)) @ W3 from the operands as the kernel read them, and a per-element bound:
    output rounding + C_GLU * (M + H) * 2^-24 * sum_j |W3[j, n]| * (L * Sg_j * |u_j| + |act(g_j)| * Su_j + |h_j|), where
    Sg / Su are sum_k |x_k W1[k, j]| / sum_k |x_k W2[k, j]| and L = ACT_LIPSCHITZ."""
    xd, w1d, w2d, w3d = (t.double() for t in (x, w1, w2, w3))
    g, u = xd @ w1d, xd @ w2d
    fn = {'relu': torch.relu, 'gelu': F.gelu, 'silu': F.silu}[act]
    a = fn(g)
    h = a * u
    y = h @ w3d
    sg, su = xd.abs() @ w1d.abs(), xd.abs() @ w2d.abs()
    terms = (ACT_LIPSCHITZ * sg * u.abs() + a.abs() * su + h.abs()) @ w3d.abs()
    M, H = w1.size(1), w1.size(2)
    return y, U32 * y.abs() + C_GLU * (M + H) * U32 * terms


@pytest.mark.parametrize('M,H,N', [(200, 264, 136), (1048, 40, 72)])
@pytest.mark.parametrize('act', ['relu', 'gelu', 'silu'])
@pytest.mark.parametrize('dtype', [torch.float32, torch.float16, torch.bfloat16])
def test_skinny_glu_ffn_matches_fp64_reference(C, dtype, act, M, H, N):
    """Counts of 0, the 1- and 2-row specialisations, 3 (a padded 4-row pass), several passes, the cap and above it;
    M, H and N are not multiples of the 64-unit slice (the second shape has one partial slice only)."""
    torch.manual_seed(21)
    R = 12
    counts = torch.tensor([0, 1, 2, 3, 5, 9, R, R + 7], device='cuda', dtype=torch.int32)
    G = counts.numel()
    x = torch.randn(G, R, M, device='cuda').to(dtype)
    w1 = (torch.randn(G, M, H, device='cuda') * M ** -0.5).to(dtype)
    w2 = (torch.randn(G, M, H, device='cuda') * M ** -0.5).to(dtype)
    w3 = (torch.randn(G, H, N, device='cuda') * H ** -0.5).to(dtype)
    y = C.skinny_glu_ffn(x, w1, w2, w3, counts, ACTS[act])
    assert y.dtype == torch.float32 and y.shape == (G, R, N)
    ref, bound = _ref_and_bound(x, w1, w2, w3, act)
    for g, c in enumerate(counts.clamp(max=R).tolist()):
        err = (y[g, :c].double() - ref[g, :c]).abs()
        assert bool((err <= bound[g, :c]).all()), (g, float((err / bound[g, :c]).max()))
        assert torch.count_nonzero(y[g, c:]) == 0           # rows at or past the count (all rows of an idle expert)


def test_skinny_glu_ffn_rejects_what_it_cannot_stage(C):
    """x rows beyond the shared-memory staging limit: the launcher refuses and the Python side never selects it."""
    from tutel_b200.ops import gemm as G
    M, H = 12288, 64
    x = torch.randn(1, 1, M, device='cuda', dtype=torch.bfloat16)
    w1 = torch.zeros(1, M, H, device='cuda', dtype=torch.bfloat16)
    w3 = torch.zeros(1, H, 64, device='cuda', dtype=torch.bfloat16)
    with torch.no_grad():
        assert not G.can_use_skinny_glu_ffn(x, w1, w1, w3, 'silu')
        assert G.can_use_skinny_glu_ffn(x[..., :4096], w1[:, :4096], w1[:, :4096], w3, 'silu')
    with pytest.raises(RuntimeError, match='invalid argument'):
        C.skinny_glu_ffn(x, w1, w1, w3, None, 3)
    with pytest.raises(RuntimeError, match='act'):
        C.skinny_glu_ffn(x[..., :4096].contiguous(), w1[:, :4096].contiguous(), w1[:, :4096].contiguous(), w3, None, 0)


def _llama_layer(E, dim, hidden, dtype, fp8=False, k=1):
    from tutel_b200 import moe
    torch.manual_seed(3)
    layer = moe.moe_layer(gate_type={'type': 'top', 'k': k, 'capacity_factor': 0.0}, model_dim=dim,
                          experts={'type': 'llama_ffn', 'num_experts_per_device': E, 'hidden_size_per_expert': hidden,
                                   'fp8': fp8}, seeds=(1, 1, 1)).cuda().to(dtype).eval()
    with torch.no_grad():                   # weights large enough that outputs are O(1), not O(1e-4)
        for p in layer.experts.parameters():
            p.normal_(0, dim ** -0.5)
    return layer


def _rel(a, b):
    return float((a.float() - b.float()).norm() / b.float().norm())


@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
@pytest.mark.parametrize('E', [16, 64])
def test_llama_dropless_skinny_matches_padded(monkeypatch, E, dtype):
    from tutel_b200.ops import gemm as G
    layer = _llama_layer(E, 256, 512, dtype)
    x = torch.randn(1, 32, 256, device='cuda', dtype=dtype)
    calls = []
    real = G.skinny_glu_ffn
    monkeypatch.setattr(G, 'skinny_glu_ffn', lambda *a, **kw: calls.append(1) or real(*a, **kw))
    with torch.no_grad():
        padded = layer(x)
        assert not calls
        fast = layer(x, megablocks_size=1)
    assert len(calls) == 1
    # the padded path rounds the hidden activations to bf16 (the skinny kernel keeps them in fp32)
    assert _rel(fast, padded) < (1e-5 if dtype == torch.float32 else 1e-2)


@pytest.mark.parametrize('tokens', [512, 32])
@pytest.mark.parametrize('fp8', [False, True])
def test_llama_dropless_wgmma_row_counts_match_padded(monkeypatch, fp8, tokens):
    """Above 64 rows (512 tokens), or with more than one skinny pass for the average expert (32 tokens x top-2 over 8
    experts), the dual-B GLU kernel and the down projection get the device row counts."""
    from tutel_b200.ops import gemm as G
    layer = _llama_layer(8, 256, 512, torch.bfloat16, fp8=fp8, k=2)
    x = torch.randn(1, tokens, 256, device='cuda', dtype=torch.bfloat16)
    seen = {'glu': [], 'raw': []}
    real_glu, real_raw = G.glu_gemm, G.raw_gemm

    def glu(*a, **kw):
        seen['glu'].append(kw.get('row_counts'))
        return real_glu(*a, **kw)

    def raw(*a, **kw):
        seen['raw'].append(kw.get('row_counts'))
        return real_raw(*a, **kw)
    monkeypatch.setattr(G, 'glu_gemm', glu)
    monkeypatch.setattr(G, 'raw_gemm', raw)
    with torch.no_grad():
        padded = layer(x)
        assert seen['glu'] == [None] and seen['raw'] == [None]
        fast = layer(x, megablocks_size=1)
    counts = layer.dispatch_count.int()
    assert len(seen['glu']) == 2 and len(seen['raw']) == 2
    assert torch.equal(seen['glu'][1], counts) and torch.equal(seen['raw'][1], counts)
    assert _rel(fast, padded) < 1e-2


class _Probe(torch.nn.Module):
    """A custom expert that records the dispatch buffer it is given."""

    def __init__(self, model_dim, num_experts_per_device, sharded_count):
        super().__init__()
        self.w = torch.nn.Parameter(torch.ones(1))
        self.seen = []

    def forward(self, x, ctx):
        self.seen.append(x.clone())
        return x * self.w


class _RowwiseProbe(_Probe):
    rows_independent = True


def _plan_valid_rows(layer, x):
    from tutel_b200.ops.dispatch import DispatchPlan
    crits = []
    route = layer._route
    layer._route = lambda *a, **kw: crits.append(route(*a, **kw)) or crits[-1]
    with torch.no_grad():
        layer(x, megablocks_size=1)
    del layer._route
    return DispatchPlan.from_critical(crits[0][1]).valid_rows


def test_dropless_padding_follows_rows_independent():
    from tutel_b200 import moe
    x = torch.randn(1, 32, 128, device='cuda')
    layer = _llama_layer(8, 128, 256, torch.float32)
    assert _plan_valid_rows(layer, x) is not None             # llama_ffn: rows past the counts are not zero-filled
    for probe, skips in ((_Probe, False), (_RowwiseProbe, True)):
        torch.manual_seed(3)
        layer = moe.moe_layer(gate_type={'type': 'top', 'k': 1, 'capacity_factor': 0.0}, model_dim=128,
                              experts={'type': 'custom', 'module': probe, 'num_experts_per_device': 8}).cuda().eval()
        assert (_plan_valid_rows(layer, x) is not None) == skips
        if not skips:
            buf, counts = layer.experts.seen[-1], layer.dispatch_count
            rows = torch.arange(buf.size(1), device='cuda').view(1, -1, 1)
            assert torch.count_nonzero(torch.where(rows >= counts.view(-1, 1, 1), buf, torch.zeros_like(buf))) == 0


def test_graphed_llama_dropless_forward_matches_eager():
    from tutel_b200.utils.graph import GraphedForward
    layer = _llama_layer(32, 128, 256, torch.float32, k=2)
    xs = [torch.randn(1, 16, 128, device='cuda') for _ in range(3)]
    fast = GraphedForward(lambda t: layer(t, megablocks_size=1), xs[0])
    for x in xs[1:] + xs[:1]:
        with torch.no_grad():
            want = layer(x, megablocks_size=1)
        got = fast(x).clone()
        assert torch.allclose(got, want, atol=1e-5, rtol=1e-5)


def test_fused_glu_ffn_with_row_counts_has_no_backward():
    from tutel_b200.ops import gemm as G
    torch.manual_seed(4)
    x = torch.randn(2, 128, 128, device='cuda', dtype=torch.bfloat16, requires_grad=True)
    w1, w2 = (torch.randn(2, 128, 256, device='cuda', dtype=torch.bfloat16) * 0.1 for _ in range(2))
    w3 = torch.randn(2, 256, 128, device='cuda', dtype=torch.bfloat16) * 0.1
    counts = torch.tensor([100, 128], device='cuda', dtype=torch.int32)
    y = G.fused_glu_ffn(x, w1, w2, w3, 'silu', False, counts)
    with pytest.raises(RuntimeError, match='row_counts'):
        y.float().sum().backward()
