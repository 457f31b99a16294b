"""Dropless fp8 decoding: the weight-only e4m3 skinny FFN and SwiGLU kernels against the float64 reference of the
quantised weights they read (tests/skinny_fp8_reference.py), their refusals, and the expert layers' choice of them."""
import pytest
import torch
import torch.nn.functional as F

import skinny_fp8_reference as R

pytestmark = pytest.mark.gpu

ROWS = 12
COUNTS = [0, 1, 2, 3, 5, 9, ROWS, ROWS + 7]      # idle, the 1- / 2-row passes, a padded 4-row pass, several, the cap, above
U16 = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}
# K (M), H, N: multiples of 16 but not of the 128-unit hidden slice; the second has one partial slice only
SHAPES = [(208, 272, 144), (1040, 48, 80)]


@pytest.fixture(scope='module')
def C():
    from tutel_b200.ops import backend
    return backend.require_ext()


def _weights(G, rows, cols, gen):
    return R.quantize((torch.randn(G, rows, cols, device='cuda', generator=gen) * cols ** -0.5))


@pytest.mark.parametrize('bias', ['none', 'b1', 'b2', 'both'])
@pytest.mark.parametrize('K,H,N', SHAPES)
@pytest.mark.parametrize('act', ['relu', 'gelu', 'silu'])
@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16])
def test_skinny_ffn_fp8_matches_fp64_reference(C, dtype, act, K, H, N, bias):
    gen = torch.Generator(device='cuda').manual_seed(31)
    counts = torch.tensor(COUNTS, device='cuda', dtype=torch.int32)
    G = counts.numel()
    x = torch.randn(G, ROWS, K, device='cuda', generator=gen).to(dtype)
    (q1, s1), (q2, s2) = _weights(G, H, K, gen), _weights(G, N, H, gen)
    b1 = torch.randn(G, H, device='cuda', generator=gen).to(dtype) if bias in ('b1', 'both') else None
    b2 = torch.randn(G, N, device='cuda', generator=gen).to(dtype) if bias in ('b2', 'both') else None
    y = C.skinny_ffn_fp8(x, q1, s1, b1, q2, s2, b2, counts, R.ACTS[act])
    assert y.dtype == torch.float32 and y.shape == (G, ROWS, N)
    ref, bound = R.ffn_reference(x, q1, s1, b1, q2, s2, b2, act)
    assert R.check(y, ref, bound, counts) <= 1.0


@pytest.mark.parametrize('M,H,N', SHAPES)
@pytest.mark.parametrize('act', ['relu', 'gelu', 'silu'])
@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16])
def test_skinny_glu_ffn_fp8_matches_fp64_reference(C, dtype, act, M, H, N):
    gen = torch.Generator(device='cuda').manual_seed(32)
    counts = torch.tensor(COUNTS, device='cuda', dtype=torch.int32)
    G = counts.numel()
    x = torch.randn(G, ROWS, M, device='cuda', generator=gen).to(dtype)
    (q1, s1), (q2, s2), (q3, s3) = _weights(G, H, M, gen), _weights(G, H, M, gen), _weights(G, N, H, gen)
    y = C.skinny_glu_ffn_fp8(x, q1, s1, q2, s2, q3, s3, counts, R.ACTS[act])
    assert y.dtype == torch.float32 and y.shape == (G, ROWS, N)
    ref, bound = R.glu_reference(x, q1, s1, q2, s2, q3, s3, act)
    assert R.check(y, ref, bound, counts) <= 1.0


def test_fp8_skinny_refusals(C):
    """A dimension that is not a multiple of 16, a wrong dtype and x rows beyond the staging limit: the launchers refuse
    and ``can_use_*`` never selects them."""
    from tutel_b200.ops import gemm as G
    bf = torch.bfloat16

    def glu_ops(M, H, N, dtype=bf):
        x = torch.randn(1, 1, M, device='cuda', dtype=dtype)
        w1, w3 = torch.zeros(1, M, H, device='cuda', dtype=dtype), torch.zeros(1, H, N, device='cuda', dtype=dtype)
        (q1, s1), (q3, s3) = R.quantize(w1.transpose(1, 2)), R.quantize(w3.transpose(1, 2))
        return x, w1, w3, (q1, s1, q1, s1, q3, s3)

    def ffn_ops(K, H, N, dtype=bf):
        x = torch.randn(1, 1, K, device='cuda', dtype=dtype)
        w1, w2 = torch.zeros(1, H, K, device='cuda', dtype=dtype), torch.zeros(1, H, N, device='cuda', dtype=dtype)
        (q1, s1), (q2, s2) = R.quantize(w1), R.quantize(w2.transpose(1, 2))
        return x, w1, w2, (q1, s1, None, q2, s2, None)

    with torch.no_grad():
        x, w1, w3, _ = glu_ops(256, 128, 128)
        assert G.can_use_skinny_glu_ffn_fp8(x, w1, w1, w3, 'silu')
        x, w1, w2, _ = ffn_ops(256, 128, 128)
        assert G.can_use_skinny_ffn_fp8(x, w1, w2, 'relu')
        for dims in [(200, 128, 128), (256, 136, 128), (256, 128, 136), (12800, 128, 128)]:
            x, w1, w3, ops = glu_ops(*dims)
            assert not G.can_use_skinny_glu_ffn_fp8(x, w1, w1, w3, 'silu'), dims
            with pytest.raises(RuntimeError, match='invalid argument'):
                C.skinny_glu_ffn_fp8(x, *ops, None, 3)
            x, w1, w2, ops = ffn_ops(*dims)
            assert not G.can_use_skinny_ffn_fp8(x, w1, w2, 'relu'), dims
            with pytest.raises(RuntimeError, match='invalid argument'):
                C.skinny_ffn_fp8(x, *ops, None, 1)
        # fp32 activations: the 16-bit rules still hold, the fp8 kernels do not take them
        x, w1, w3, ops = glu_ops(256, 128, 128, torch.float32)
        assert G.can_use_skinny_glu_ffn(x, w1, w1, w3, 'silu') and not G.can_use_skinny_glu_ffn_fp8(x, w1, w1, w3, 'silu')
        with pytest.raises(RuntimeError, match='float16 or bfloat16'):
            C.skinny_glu_ffn_fp8(x, *ops, None, 3)
        x, w1, w2, ops = ffn_ops(256, 128, 128, torch.float32)
        assert G.can_use_skinny_ffn(x, w1, w2, 'relu') and not G.can_use_skinny_ffn_fp8(x, w1, w2, 'relu')
        with pytest.raises(RuntimeError, match='float16 or bfloat16'):
            C.skinny_ffn_fp8(x, *ops, None, 1)
        # 16-bit weights where e4m3 ones belong, act in 1..3
        x, w1, w3, (q1, s1, q2, s2, q3, s3) = glu_ops(256, 128, 128)
        with pytest.raises(RuntimeError, match='float8_e4m3fn'):
            C.skinny_glu_ffn_fp8(x, w1.transpose(1, 2).contiguous(), s1, q2, s2, q3, s3, None, 3)
        with pytest.raises(RuntimeError, match='act'):
            C.skinny_glu_ffn_fp8(x, q1, s1, q2, s2, q3, s3, None, 0)
        x, w1, w2, (q1, s1, _, q2, s2, _) = ffn_ops(256, 128, 128)
        with pytest.raises(RuntimeError, match='biases'):
            C.skinny_ffn_fp8(x, q1, s1, torch.zeros(1, 128, device='cuda'), q2, s2, None, None, 1)


# ------------------------------------------------------------------------------------------------------------------
# layers
# ------------------------------------------------------------------------------------------------------------------
def _layer(kind, fp8, E=8, dim=256, hidden=512, k=2, seed=3, dtype=torch.bfloat16):
    from tutel_b200 import moe
    torch.manual_seed(seed)
    experts = {'type': kind, 'num_experts_per_device': E, 'hidden_size_per_expert': hidden, 'fp8': fp8}
    if kind == 'ffn':
        experts['activation_fn'] = lambda t: F.relu(t)
    layer = moe.moe_layer(gate_type={'type': 'top', 'k': k, 'capacity_factor': 0.0}, model_dim=dim, experts=experts,
                          seeds=(1, 1, 1)).cuda().to(dtype).eval()
    torch.manual_seed(seed)                 # moe_layer re-seeds its own initialisation (seeds=...)
    with torch.no_grad():                   # weights large enough that outputs are O(1)
        for p in layer.experts.parameters():
            p.normal_(0, dim ** -0.5)
    return layer


def _rel(a, b):
    return float((a.float() - b.float()).norm() / b.float().norm())


class _Spy:
    """Counts the calls of the ops the layer may take and records what fp8_weight hands out."""

    def __init__(self, monkeypatch):
        from tutel_b200.ops import gemm as G
        self.calls = {n: 0 for n in ('skinny_ffn_fp8', 'skinny_glu_ffn_fp8', 'skinny_ffn', 'skinny_glu_ffn')}
        self.weights = []
        for name in self.calls:
            real = getattr(G, name)
            monkeypatch.setattr(G, name, self._counted(name, real))
        real_w = G.fp8_weight

        def fp8_weight(w, layout):
            out = real_w(w, layout)
            self.weights.append(out)
            return out
        monkeypatch.setattr(G, 'fp8_weight', fp8_weight)

    def _counted(self, name, real):
        def f(*a, **kw):
            self.calls[name] += 1
            return real(*a, **kw)
        return f


def _expert_io(layer, x):
    """(dispatch buffer, expert output, counts) of one dropless call."""
    seen = {}
    h1 = layer.experts.register_forward_pre_hook(lambda m, a: seen.__setitem__('x', a[0]))
    h2 = layer.experts.register_forward_hook(lambda m, a, y: seen.__setitem__('y', y))
    try:
        out = layer(x, megablocks_size=1)
    finally:
        h1.remove()
        h2.remove()
    return out, seen['x'], seen['y'], layer.dispatch_count.int()


@pytest.mark.parametrize('kind', ['ffn', 'llama_ffn'])
def test_fp8_layer_decode_takes_fp8_skinny_kernel(monkeypatch, kind):
    """Decode (4 tokens, top-2, 8 experts): the fp8 layer takes the fp8 skinny kernel once and matches the fp64 reference
    of its quantised weights; its error against the 16-bit padded path stays within the fp8 layer budget; the e4m3
    tensors it reads are the cached copies the wgmma fp8 forward of the same layer gets."""
    fp8_layer, bf_layer = _layer(kind, True), _layer(kind, False)
    x = torch.randn(1, 4, 256, device='cuda', dtype=torch.bfloat16)
    spy = _Spy(monkeypatch)
    fp8_name = 'skinny_ffn_fp8' if kind == 'ffn' else 'skinny_glu_ffn_fp8'
    with torch.no_grad():
        padded = bf_layer(x)
        bf_layer(x, megablocks_size=1)
        assert spy.calls[fp8_name] == 0 and spy.calls[fp8_name[:-4]] == 1       # a 16-bit layer never takes it
        spy.weights.clear()
        fast, buf, y, counts = _expert_io(fp8_layer, x)
        decode_weights = list(spy.weights)
        assert spy.calls[fp8_name] == 1 and spy.calls[fp8_name[:-4]] == 1
        spy.weights.clear()
        fp8_layer(x)                                                              # padded: the wgmma fp8 forward
        wgmma_weights = list(spy.weights)
    assert len(decode_weights) == (2 if kind == 'ffn' else 3)
    ids = {id(t) for pair in wgmma_weights for t in pair}
    assert all(id(q) in ids and id(s) in ids for q, s in decode_weights)          # one e4m3 copy per weight
    e = fp8_layer.experts
    if kind == 'ffn':
        (q1, s1), (q2, s2) = decode_weights
        ref, bound = R.ffn_reference(buf, q1, s1, e.batched_fc1_bias, q2, s2, e.batched_fc2_bias, 'relu')
    else:
        (q1, s1), (q2, s2), (q3, s3) = decode_weights
        ref, bound = R.glu_reference(buf, q1, s1, q2, s2, q3, s3, 'silu')
    # the layer hands back x's dtype: one more bf16 rounding of the output
    assert R.check(y, ref, bound + U16[torch.bfloat16] * ref.abs(), counts) <= 1.0
    assert _rel(fast, padded) < 0.08


@pytest.mark.parametrize('kind', ['ffn', 'llama_ffn'])
def test_fp8_layer_decode_not_taken_where_it_cannot_run(monkeypatch, kind):
    """A model dimension that is a multiple of 8 but not of 16 keeps the 16-bit skinny kernel."""
    layer = _layer(kind, True, dim=200, hidden=256)
    spy = _Spy(monkeypatch)
    with torch.no_grad():
        layer(torch.randn(1, 4, 200, device='cuda', dtype=torch.bfloat16), megablocks_size=1)
    fp8_name = 'skinny_ffn_fp8' if kind == 'ffn' else 'skinny_glu_ffn_fp8'
    assert spy.calls[fp8_name] == 0 and spy.calls[fp8_name[:-4]] == 1


@pytest.mark.parametrize('kind', ['ffn', 'llama_ffn'])
def test_fp8_decode_follows_loaded_weights(kind):
    """load_state_dict with other weights: the next decode uses them (the e4m3 cache is not stale)."""
    a, b = _layer(kind, True, seed=3), _layer(kind, True, seed=4)
    x = torch.randn(1, 4, 256, device='cuda', dtype=torch.bfloat16)
    with torch.no_grad():
        before = a(x, megablocks_size=1).clone()
        want = b(x, megablocks_size=1).clone()
        a.load_state_dict(b.state_dict())
        after = a(x, megablocks_size=1)
    assert _rel(before, want) > 0.1
    assert _rel(after, want) < 1e-2              # same weights; only the fp32 atomics' order may differ


@pytest.mark.parametrize('kind', ['ffn', 'llama_ffn'])
def test_graphed_fp8_dropless_decode_matches_eager(kind):
    from tutel_b200.utils.graph import GraphedForward
    layer = _layer(kind, True, E=16)
    xs = [torch.randn(1, 4, 256, device='cuda', dtype=torch.bfloat16) for _ in range(3)]
    with torch.no_grad():
        layer(xs[0], megablocks_size=1)          # quantise the weights outside the capture
    fast = GraphedForward(lambda t: layer(t, megablocks_size=1), xs[0])
    for x in xs[1:] + xs[:1]:
        with torch.no_grad():
            want = layer(x, megablocks_size=1)
        got = fast(x).clone()
        assert _rel(got, want) < 1e-2
