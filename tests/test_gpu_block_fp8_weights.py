"""Stored block-fp8 SwiGLU experts on the H100: the one-launch skinny decode kernel against an fp64 reference of the bytes
it reads, the block GEMM's device row counts, bitwise equality with a bf16 ``fp8='block'`` layer on the padded path,
decode and dropless prefill paths, host synchronisation, graph replay and memory."""
import pytest
import torch
import torch.nn.functional as F

from tutel_b200 import moe
from tutel_b200.ops import backend
from tutel_b200.ops import block_fp8 as BF8
from tutel_b200.utils.graph import GraphedForward

import skinny_block_fp8_reference as SR

pytestmark = pytest.mark.gpu
ACTS = {'silu': F.silu, 'gelu': F.gelu, 'relu': F.relu}


def _stored_weights(G, M, H, seed=0, dev='cuda'):
    """Random stored operands: e4m3 bytes over the whole range and block scales spread over 2^-12 .. 2^-4."""
    g = torch.Generator(device=dev).manual_seed(seed)
    def q(*shape):
        return (torch.randn(*shape, device=dev, generator=g) * 100).clamp(-448, 448).to(torch.float8_e4m3fn)
    def s(*shape):
        return 2.0 ** (torch.rand(*shape, device=dev, generator=g) * 8 - 12)
    return q(G, 2 * H, M), s(G, 2 * H // 64, M // 128), q(G, M, H), s(G, M // 128, H // 128)


KERNEL_CASES = [
    (128, 128, [0, 1, 4, 5, 64, 0, 2, 3] * 8),        # G = 64
    (2048, 1408, [5, 0, 1, 4, 64]),
    (7168, 2048, [1, 0, 4, 5]),
    (7168, 2048, [64, 0]),
]


@pytest.mark.parametrize('act', ['silu', 'gelu', 'relu'])
@pytest.mark.parametrize('M,H,counts', KERNEL_CASES)
def test_skinny_kernel_against_fp64_reference(M, H, counts, act):
    G, R = len(counts), 64
    qglu, sglu, q3t, s3t = _stored_weights(G, M, H, seed=M + H)
    x = torch.randn(G, R, M, device='cuda').bfloat16()
    rows = torch.tensor(counts, dtype=torch.int32, device='cuda')
    y = backend.require_ext().skinny_glu_ffn_block_fp8(x, qglu, sglu, q3t, s3t, rows, BF8.ACT_CODES[act])
    assert y.dtype == torch.float32 and y.shape == (G, R, M)
    live = [g for g, c in enumerate(counts) if c > 0]
    ref, bound = SR.glu_reference(x, qglu, sglu, q3t, s3t, act, groups=live)
    worst = SR.check(y, ref, bound, rows.cpu())
    print('M=%d H=%d %s: worst error / bound %.3f' % (M, H, act, worst))


def test_skinny_kernel_refuses_bad_operands():
    qglu, sglu, q3t, s3t = _stored_weights(2, 256, 128)
    x = torch.randn(2, 4, 256, device='cuda').bfloat16()
    ext = backend.require_ext()
    with pytest.raises(RuntimeError, match='bf16'):
        ext.skinny_glu_ffn_block_fp8(x.half(), qglu, sglu, q3t, s3t, None, 3)
    with pytest.raises(RuntimeError, match='sglu'):
        ext.skinny_glu_ffn_block_fp8(x, qglu, sglu[:, :2], q3t, s3t, None, 3)
    with pytest.raises(RuntimeError, match='q3t'):
        ext.skinny_glu_ffn_block_fp8(x, qglu, sglu, q3t.view(torch.uint8), s3t, None, 3)


@pytest.mark.parametrize('epi', [BF8.EPI_NONE, BF8.EPI_RELU, BF8.EPI_GLU])
def test_gemm_row_counts(epi):
    G, M, K, N = 6, 300, 512, 384 if epi != BF8.EPI_GLU else 512
    counts = torch.tensor([0, 1, 127, 128, 129, 300], dtype=torch.int32, device='cuda')
    x = torch.randn(G, M, K, device='cuda').bfloat16()
    poisoned = BF8.zero_rows_past(x, counts) + torch.where(
        torch.arange(M, device='cuda').view(1, -1, 1) >= counts.view(-1, 1, 1).long(), float('nan'), 0.0).bfloat16()
    if epi == BF8.EPI_GLU:                                    # gate / up [G, K, N / 2] -> the interleaved [G, N, K]
        w1, w2 = ((torch.randn(G, K, N // 2, device='cuda') * 0.05).bfloat16() for _ in range(2))
        _, _, q, s = BF8.quantize_glu_weight(w1, w2)
    else:
        q, s, _, _ = BF8.quantize_weight((torch.randn(G, N, K, device='cuda') * 0.05).bfloat16())
    bias = torch.randn(G, N, device='cuda').bfloat16() if epi == BF8.EPI_RELU else None
    a, sa = BF8.quantize_act(poisoned)
    plain = BF8.block_fp8_gemm(a, sa, q, s, bias=bias, epilogue=epi)
    counted = BF8.block_fp8_gemm(a, sa, q, s, bias=bias, epilogue=epi, row_counts=counts)
    assert len(plain) == len(counted)
    for p, c in zip(plain, counted):
        for g, n in enumerate(counts.tolist()):
            assert torch.equal(c[g, :n], p[g, :n]), (g, n)
            assert torch.count_nonzero(c[g, n:]) == 0, 'rows past the count %d of group %d are not zero' % (n, g)
        assert not torch.isnan(c.float()).any()


def _bf16_and_stored(E=8, M=512, H=256, k=2, shared=None, gate=None, act=F.silu):
    spec = {'type': 'top', 'k': k}
    if gate == 'sigmoid':
        spec.update(scoring_func='sigmoid', n_group=4, topk_group=2)
    def build(**extra):
        return moe.moe_layer(gate_type=dict(spec), model_dim=M, seeds=(1, 2, 3), shared_experts=shared,
                             experts=dict({'type': 'llama_ffn', 'num_experts_per_device': E, 'hidden_size_per_expert': H,
                                           'activation_fn': act}, **extra)).cuda().bfloat16()
    ref = build(fp8='block')
    with torch.no_grad():
        for p in ref.parameters():
            if p.dim() == 1 and p.numel() % 128 == 0 and p.numel() >= 128 * 128:
                p.normal_(0, 0.05)                        # expert weights of a useful magnitude
    layer = build(weight_format='fp8_block')
    layer.load_state_dict({k_: v for k_, v in ref.state_dict().items()
                           if not k_.startswith(('experts.', 'shared_experts.'))}, strict=False)
    layer.experts.load_fp8_block_weights(*ref.experts.export_fp8_block_weights())
    if shared is not None:
        layer.shared_experts.load_fp8_block_weights(*ref.shared_experts.export_fp8_block_weights())
    return ref, layer


@pytest.mark.parametrize('cf', [1.0, 0.0])
@pytest.mark.parametrize('shared,gate', [(None, None), ({'num_experts': 1}, None), ({'num_experts': 2, 'gate': True}, None),
                                         ({'num_experts': 1, 'gate': True}, 'sigmoid'), (None, 'sigmoid')])
def test_layer_bitwise_equal_to_the_bf16_block_layer(cf, shared, gate):
    ref, layer = _bf16_and_stored(k=4 if gate == 'sigmoid' else 2, shared=shared, gate=gate)
    x = torch.randn(128, 512, device='cuda').bfloat16()       # > 64 tokens: the shared experts take the GEMMs too
    with torch.no_grad():
        y0 = ref(x, capacity_factor=cf)
        y1 = layer(x, capacity_factor=cf)
    assert torch.isfinite(y0.float()).all()
    assert torch.equal(y0, y1), (y0.float() - y1.float()).abs().max()


class _Spy:
    def __init__(self, monkeypatch):
        self.skinny, self.gemm = [], []
        real_skinny, real_gemm = BF8.skinny_glu_ffn_block_fp8, BF8.block_fp8_gemm
        def skinny(x, qglu, sglu, q3t, s3t, rows, act='silu'):
            y = real_skinny(x, qglu, sglu, q3t, s3t, rows, act)
            self.skinny.append((x, qglu, sglu, q3t, s3t, rows.clone(), act, y))
            return y
        def gemm(*a, **kw):
            self.gemm.append(kw.get('row_counts'))
            return real_gemm(*a, **kw)
        monkeypatch.setattr(BF8, 'skinny_glu_ffn_block_fp8', skinny)
        monkeypatch.setattr(BF8, 'block_fp8_gemm', gemm)


@pytest.mark.parametrize('k', [2, 8])
@pytest.mark.parametrize('tokens', [1, 4, 64])
def test_decode_against_fp64_and_the_path_taken(monkeypatch, tokens, k):
    E = 16
    _, layer = _bf16_and_stored(E=E, k=k, shared={'num_experts': 1})
    spy = _Spy(monkeypatch)
    x = torch.randn(tokens, 512, device='cuda').bfloat16()
    with torch.no_grad():
        y = layer(x, megablocks_size=1)
    assert torch.isfinite(y.float()).all()
    if tokens == 1:                                          # routed and shared experts: one launch each, no GEMM
        assert len(spy.skinny) == 2 and not spy.gemm
    assert spy.skinny or spy.gemm
    assert all(rc is not None for rc in spy.gemm)            # dropless: the GEMMs get the device row counts
    for xx, qglu, sglu, q3t, s3t, rows, act, yy in spy.skinny:
        y32 = backend.require_ext().skinny_glu_ffn_block_fp8(xx.contiguous(), qglu, sglu, q3t, s3t, rows, BF8.ACT_CODES[act])
        assert torch.equal(y32.bfloat16(), yy)
        live = [g for g, c in enumerate(rows.tolist()) if c > 0]
        ref, bound = SR.glu_reference(xx, qglu, sglu, q3t, s3t, act, groups=live)
        SR.check(y32, ref, bound, rows.cpu())


def test_dropless_prefill_runs_the_gemm_with_row_counts(monkeypatch):
    ref, layer = _bf16_and_stored(E=8, k=2)
    with torch.no_grad():
        layer.gates[0].wg.weight[0] += 0.5                    # skewed routing: expert 0 gets most tokens
    x = torch.randn(512, 512, device='cuda').bfloat16()
    with torch.no_grad():
        y_pad = layer(x, capacity_factor=0.0)
        spy = _Spy(monkeypatch)
        y = layer(x, megablocks_size=1)
    assert not spy.skinny and len(spy.gemm) == 2 and all(rc is not None for rc in spy.gemm)
    assert torch.equal(y, y_pad), (y.float() - y_pad.float()).abs().max()


def test_no_host_sync_and_graph_replay():
    _, layer = _bf16_and_stored(E=8, k=2, shared={'num_experts': 1, 'gate': True})
    xs = [torch.randn(n, 512, device='cuda').bfloat16() for n in (4, 4, 512)]
    with torch.no_grad():
        for x in xs:
            layer(x, megablocks_size=1)                       # warm-up: attributes and lazy initialisation
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode('error')
        try:
            for x in xs:
                layer(x, megablocks_size=1)
        finally:
            torch.cuda.set_sync_debug_mode('default')
        eager = [layer(x, megablocks_size=1) for x in xs[:2]]
    fast = GraphedForward(lambda t: layer(t, megablocks_size=1), xs[0])
    for x, e in zip(xs[:2], eager):
        assert torch.equal(fast(x), e)


def test_memory():
    E, M, H = 8, 2048, 1408
    layer = moe.moe_layer(gate_type={'type': 'top', 'k': 2}, model_dim=M, seeds=(1, 1, 1),
                          experts={'type': 'llama_ffn', 'num_experts_per_device': E, 'hidden_size_per_expert': H,
                                   'weight_format': 'fp8_block'}).cuda().bfloat16()
    ex = layer.experts
    nbytes = sum(b.numel() * b.element_size() for b in ex.buffers())
    assert nbytes == E * 3 * M * H + 4 * E * (2 * H // 64 * M // 128 + M // 128 * H // 128)
    x = torch.randn(1, M, device='cuda').bfloat16()
    with torch.no_grad():
        layer(x, megablocks_size=1)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        layer(x, megablocks_size=1)
        torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    assert peak < 3 * M * H * 2, 'a decode step allocated %d bytes' % peak
