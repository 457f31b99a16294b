"""Group-32 int4 SwiGLU experts on the H100: the one-launch decode kernel and the mixed-input wgmma GEMM of the prefill
path (``w4a16_gemm_kernel``: nibbles expanded on chip to bf16_rn(q * s)) element by element against the fp64 references
and bounds of tests/int4_reference.py, the launchers' refusals, the paths the layer takes, the layer against a bf16 layer
holding bf16_rn(q * s), host synchronisation, graph replay and memory."""
import pytest
import torch
import torch.nn.functional as F

from tutel_b200 import moe
from tutel_b200.ops import backend
from tutel_b200.ops import int4 as I4
from tutel_b200.utils.graph import GraphedForward

import int4_reference as R

pytestmark = pytest.mark.gpu
ACTS = {'silu': F.silu, 'gelu': F.gelu, 'relu': F.relu}


def _stored_weights(E, M, H, seed=0, dev='cuda'):
    """Random stored operands: every nibble value, scales spread over 2^-10 .. 2^-4."""
    g = torch.Generator(device=dev).manual_seed(seed)
    def q(*shape):
        return torch.randint(0, 256, shape, device=dev, generator=g, dtype=torch.int32).to(torch.uint8)
    def s(*shape):
        return (2.0 ** (torch.rand(*shape, device=dev, generator=g) * 6 - 10)).bfloat16()
    return q(E, 2 * H, M // 2), s(E, 2 * H, M // 32), q(E, M, H // 2), s(E, M, H // 32)


def _poisoned(G_, R_, M, counts, seed=1):
    g = torch.Generator(device='cuda').manual_seed(seed)
    x = torch.randn(G_, R_, M, device='cuda', generator=g).bfloat16()
    dead = torch.arange(R_, device='cuda').view(1, -1, 1) >= torch.tensor(counts, device='cuda').view(-1, 1, 1)
    return torch.where(dead, torch.full((), float('nan'), device='cuda', dtype=torch.bfloat16), x)


DECODE_CASES = [
    (128, 128, [0, 1, 2, 3, 4, 5, 64, 0] * 8),       # G = 64
    (2048, 1408, [5, 0, 1, 4, 64]),
    (7168, 2048, [1, 0, 4, 5]),
    (7168, 2048, [64, 0]),
]


@pytest.mark.parametrize('act', ['silu', 'gelu', 'relu'])
@pytest.mark.parametrize('M,H,counts', DECODE_CASES)
def test_decode_kernel_against_fp64(M, H, counts, act):
    E, Rw = len(counts), 64
    qglu, sglu, q3t, s3t = _stored_weights(E, M, H, seed=M + H)
    x = _poisoned(E, Rw, M, counts)
    rows = torch.tensor(counts, dtype=torch.int32, device='cuda')
    y = backend.require_ext().skinny_glu_ffn_int4(x, qglu, sglu, q3t, s3t, rows, I4.ACT_CODES[act])
    assert y.dtype == torch.float32 and y.shape == (E, Rw, M)
    live = [g for g, c in enumerate(counts) if c > 0]
    ref, bound = R.stored_reference(torch.nan_to_num(x), qglu, sglu, q3t, s3t, act, 'decode', groups=live)
    worst = R.check(y, ref, bound, counts)
    print('decode M=%d H=%d %s: worst error / bound %.3f' % (M, H, act, worst))


GEMM_CASES = [
    (1, 128, 128, [1]),
    (5, 300, 256, [0, 127, 128, 129, 300]),              # M at tile edges, NaN rows past the counts
    (70, 129, 128, [129, 1] * 35),                         # more tiles than SMs
    (2, 200, 14336, [200, 77]),                            # K = 14336: the 8-stage ring wraps many times per tile
    (3, 64, 4096, None),                                   # no row counts
]


@pytest.mark.parametrize('G_,M,K,counts', GEMM_CASES)
def test_gemm_against_fp64(G_, M, K, counts):
    N = 256
    g = torch.Generator(device='cuda').manual_seed(K + M)
    q = torch.randint(0, 256, (G_, N, K // 2), device='cuda', generator=g, dtype=torch.int32).to(torch.uint8)
    s = (2.0 ** (torch.rand(G_, N, K // 32, device='cuda', generator=g) * 6 - 10)).bfloat16()
    x = _poisoned(G_, M, K, counts if counts is not None else [M] * G_)
    rows = None if counts is None else torch.tensor(counts, dtype=torch.int32, device='cuda')
    y = I4.w4a16_gemm(x, q, s, None, rows)
    assert y.dtype == torch.bfloat16 and y.shape == (G_, M, N)
    w = R.stored_values(q, s)
    xd = torch.nan_to_num(x).double()
    ref = xd @ w.transpose(1, 2)
    bound = R.U16 * ref.abs() + (R.U16 + R.C_ACC * K * R.U32) * (xd.abs() @ w.abs().transpose(1, 2))
    worst = R.check(y, ref, bound, counts)
    print('gemm G=%d M=%d K=%d: worst error / bound %.3f' % (G_, M, K, worst))


PREFILL_CASES = [
    (128, 128, [0, 1, 2, 3, 4, 5, 64, 127, 128, 129] * 7),       # G = 70: more tiles than SMs
    (7168, 2048, [129, 0, 1, 128]),
    (4096, 14336, [127, 3]),                                       # K = 14336 in the down GEMM
    (1024, 512, [200, 77, 0]),                                     # 200 rows: two row tiles, the ring wraps mid-expert
]


@pytest.mark.parametrize('act', ['silu', 'gelu', 'relu'])
@pytest.mark.parametrize('M,H,counts', PREFILL_CASES)
def test_prefill_against_fp64(M, H, counts, act):
    E = len(counts)
    Rw = max(max(counts), 1)
    qglu, sglu, q3t, s3t = _stored_weights(E, M, H, seed=M + 2 * H)
    x = _poisoned(E, Rw, M, counts)
    rows = torch.tensor(counts, dtype=torch.int32, device='cuda')
    y = I4.glu_ffn_int4(x, qglu, sglu, q3t, s3t, act, rows)
    assert y.dtype == torch.bfloat16 and y.shape == (E, Rw, M)
    live = [g for g, c in enumerate(counts) if c > 0]
    ref, bound = R.stored_reference(torch.nan_to_num(x), qglu, sglu, q3t, s3t, act, 'prefill', groups=live)
    worst = R.check(y, ref, bound, counts)
    print('prefill M=%d H=%d %s: worst error / bound %.3f' % (M, H, act, worst))


def test_launchers_refuse_bad_operands():
    qglu, sglu, q3t, s3t = _stored_weights(2, 256, 128)
    x = torch.randn(2, 4, 256, device='cuda').bfloat16()
    ext = backend.require_ext()
    with pytest.raises(RuntimeError, match='bf16'):
        ext.skinny_glu_ffn_int4(x.half(), qglu, sglu, q3t, s3t, None, 3)
    with pytest.raises(RuntimeError, match='sglu'):
        ext.skinny_glu_ffn_int4(x, qglu, sglu[:, :, :2].contiguous(), q3t, s3t, None, 3)
    with pytest.raises(RuntimeError, match='q3t'):
        ext.skinny_glu_ffn_int4(x, qglu, sglu, q3t.view(torch.int8), s3t, None, 3)
    with pytest.raises(RuntimeError, match='s3t'):
        ext.skinny_glu_ffn_int4(x, qglu, sglu, q3t, s3t.float(), None, 3)
    with pytest.raises(RuntimeError, match='act'):
        ext.skinny_glu_ffn_int4(x, qglu, sglu, q3t, s3t, None, 0)
    with pytest.raises(RuntimeError, match='multiples of 128'):
        ext.skinny_glu_ffn_int4(x[:, :, :192].contiguous(), qglu, sglu, q3t, s3t, None, 3)
    h = torch.randn(2, 4, 128, device='cuda').bfloat16()
    with pytest.raises(RuntimeError, match='bf16'):
        ext.w4a16_gemm(h.half(), q3t, s3t, None, 0, 0)
    with pytest.raises(RuntimeError, match='sb must be'):
        ext.w4a16_gemm(h, q3t, s3t.float(), None, 0, 0)
    with pytest.raises(RuntimeError, match='b must be'):
        ext.w4a16_gemm(h, q3t.view(torch.int8), s3t, None, 0, 0)
    with pytest.raises(RuntimeError, match='N of 128'):
        ext.w4a16_gemm(h, q3t[:, :64].contiguous(), s3t[:, :64].contiguous(), None, 0, 0)
    with pytest.raises(RuntimeError, match='epilogue'):
        ext.w4a16_gemm(h, q3t, s3t, None, 2, 0)
    with pytest.raises(RuntimeError, match='act'):
        ext.w4a16_gemm(x, qglu, sglu, None, 1, 0)
    with pytest.raises(RuntimeError, match='row_counts'):
        ext.w4a16_gemm(h, q3t, s3t, torch.ones(2, dtype=torch.int64, device='cuda'), 0, 0)


def _bf16_and_int4(E=8, M=512, H=256, k=2, shared=None, gate=None, act=F.silu, int4_shared=True):
    """A bf16 layer whose expert weights are bf16_rn(q * s) of an int4 export, and the int4 layer of that export."""
    spec = {'type': 'top', 'k': k}
    if gate == 'sigmoid':
        spec.update(scoring_func='sigmoid', n_group=4, topk_group=2)
    def build(fmt, shared_spec):
        return moe.moe_layer(gate_type=dict(spec), model_dim=M, seeds=(1, 2, 3), shared_experts=shared_spec,
                             experts={'type': 'llama_ffn', 'num_experts_per_device': E, 'hidden_size_per_expert': H,
                                      'activation_fn': act, 'weight_format': fmt}).cuda().bfloat16()
    ref = build(None, shared)
    with torch.no_grad():
        for p in ref.parameters():
            if p.dim() == 1 and p.numel() >= 128 * 128:
                p.normal_(0, 0.05)
    lshared = None if shared is None else dict(shared, **({} if int4_shared else {'weight_format': None}))
    layer = build('int4', lshared)
    layer.load_state_dict({k_: v for k_, v in ref.state_dict().items()
                           if not k_.startswith(('experts.', 'shared_experts.'))}, strict=False)
    mods = [('experts', True)] + ([('shared_experts', int4_shared)] if shared is not None else [])
    with torch.no_grad():
        for name, quantised in mods:
            src, dst = getattr(ref, name), getattr(layer, name)
            if not quantised:
                dst.load_state_dict(src.state_dict())
                continue
            gate_, gs, up, us, down, ds = src.export_int4_weights()
            dst.load_int4_weights(gate_, gs, up, us, down, ds)
            for n, (q, s) in (('W_fc1', (gate_, gs)), ('W_fc2', (up, us)), ('W_fc3', (down, ds))):
                w = R.values(q, s).bfloat16().transpose(1, 2).contiguous()     # [E, M, H] / [E, H, M]
                getattr(src, n).copy_(w.reshape(-1))
    return ref, layer


def _close(y, y0):
    """Both layers see identical bf16 weights; only the GEMM layouts (and so the fp32 summation order) differ."""
    err = (y.float() - y0.float()).abs()
    tol = 4 * R.U16 * y0.float().abs() + 2.0 ** -6 * y0.float().pow(2).mean().sqrt()
    assert bool((err <= tol).all()), float((err / tol).max())


@pytest.mark.parametrize('cf', [1.0, 0.0])
@pytest.mark.parametrize('shared,gate,int4_shared', [
    (None, None, True), ({'num_experts': 1}, None, True), ({'num_experts': 2, 'gate': True}, None, False),
    ({'num_experts': 1, 'gate': True}, 'sigmoid', True), (None, 'sigmoid', True)])
def test_layer_against_the_bf16_layer(cf, shared, gate, int4_shared):
    ref, layer = _bf16_and_int4(k=4 if gate == 'sigmoid' else 2, shared=shared, gate=gate, int4_shared=int4_shared)
    x = torch.randn(128, 512, device='cuda').bfloat16()
    with torch.no_grad():
        y0 = ref(x, capacity_factor=cf)
        y1 = layer(x, capacity_factor=cf)
    assert torch.isfinite(y0.float()).all()
    _close(y1, y0)


class _Spy:
    def __init__(self, monkeypatch):
        self.skinny, self.gemm = [], []
        real_skinny, real_gemm = I4.skinny_glu_ffn_int4, I4.glu_ffn_int4
        def skinny(x, qglu, sglu, q3t, s3t, rows, act='silu'):
            y = real_skinny(x, qglu, sglu, q3t, s3t, rows, act)
            self.skinny.append((x, qglu, sglu, q3t, s3t, rows.clone(), act, y))
            return y
        def gemm(x, qglu, sglu, q3t, s3t, act='silu', row_counts=None):
            self.gemm.append(row_counts)
            return real_gemm(x, qglu, sglu, q3t, s3t, act, row_counts)
        monkeypatch.setattr(I4, 'skinny_glu_ffn_int4', skinny)
        monkeypatch.setattr(I4, 'glu_ffn_int4', gemm)


@pytest.mark.parametrize('k', [2, 8])
@pytest.mark.parametrize('tokens', [1, 4, 64])
def test_decode_path_and_fp64(monkeypatch, tokens, k):
    _, layer = _bf16_and_int4(E=16, k=k, shared={'num_experts': 1})
    spy = _Spy(monkeypatch)
    x = torch.randn(tokens, 512, device='cuda').bfloat16()
    with torch.no_grad():
        y = layer(x, megablocks_size=1)
    assert torch.isfinite(y.float()).all()
    if tokens == 1:                                          # routed and shared experts: one launch each, no GEMM
        assert len(spy.skinny) == 2 and not spy.gemm
    assert spy.skinny or spy.gemm
    assert all(rc is not None for rc in spy.gemm)
    for xx, qglu, sglu, q3t, s3t, rows, act, yy in spy.skinny:
        y32 = backend.require_ext().skinny_glu_ffn_int4(xx.contiguous(), qglu, sglu, q3t, s3t, rows, I4.ACT_CODES[act])
        assert torch.equal(y32.bfloat16(), yy)
        live = [g for g, c in enumerate(rows.tolist()) if c > 0]
        ref, bound = R.stored_reference(torch.nan_to_num(xx), qglu, sglu, q3t, s3t, act, 'decode', groups=live)
        R.check(y32, ref, bound, rows.tolist())


def test_dropless_prefill_takes_the_gemms_with_row_counts(monkeypatch):
    _, layer = _bf16_and_int4(E=8, k=2)
    with torch.no_grad():
        layer.gates[0].wg.weight[0] += 0.5                    # skewed routing: expert 0 gets most tokens
    x = torch.randn(512, 512, device='cuda').bfloat16()
    with torch.no_grad():
        y_pad = layer(x, capacity_factor=0.0)
        spy = _Spy(monkeypatch)
        y = layer(x, megablocks_size=1)
    assert not spy.skinny and len(spy.gemm) == 1 and spy.gemm[0] is not None
    assert torch.equal(y, y_pad), (y.float() - y_pad.float()).abs().max()


def test_no_host_sync_and_graph_replay():
    _, layer = _bf16_and_int4(E=8, k=2, shared={'num_experts': 1, 'gate': True})
    xs = [torch.randn(n, 512, device='cuda').bfloat16() for n in (4, 4, 512)]
    with torch.no_grad():
        for x in xs:
            layer(x, megablocks_size=1)
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
                                   'weight_format': 'int4'}).cuda().bfloat16()
    nbytes = sum(b.numel() * b.element_size() for b in layer.experts.buffers())
    assert nbytes == E * 3 * M * H // 2 + 2 * E * 3 * M * H // 32           # 0.5625 bytes per weight
    x = torch.randn(1, M, device='cuda').bfloat16()
    with torch.no_grad():
        layer(x, megablocks_size=1)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        layer(x, megablocks_size=1)
        torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    assert peak < M * H, 'a decode step allocated %d bytes' % peak
    # prefill: the weights are expanded on chip, so a forward allocates activations only, never a bf16 weight copy
    x = torch.randn(256, M, device='cuda').bfloat16()
    with torch.no_grad():
        layer(x, megablocks_size=1)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        layer(x, megablocks_size=1)
        torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    assert peak < E * M * H * 2, 'a prefill step allocated %d bytes (a bf16 copy of the experts is %d)' % (
        peak, 3 * E * M * H * 2)
