"""Stored block-fp8 SwiGLU experts (``llama_ffn`` with ``weight_format='fp8_block'``) on CPU, through the pure-torch
references of ops/block_fp8.py: the checkpoint exporter and loader, the module's buffers, refusals and state dict, and a
two-rank Gloo run."""
import types

import pytest
import torch
import torch.nn.functional as F

from tutel_b200 import moe
from tutel_b200.models.experts.llama_ffn import LlamaFFNNetwork
from tutel_b200.ops import block_fp8 as BF8

from helpers import run_workers

E, M, H = 3, 256, 256


def _bf16_weights(seed=0, E=E, M=M, H=H):
    """w1, w2 [E, M, H], w3 [E, H, M] bf16 whose 128 x 128 block (i, j) has magnitude 4^(i - j), so that a scale applied
    to the transposed block is 16 times off or more."""
    g = torch.Generator().manual_seed(seed)
    def one(r, c):
        w = torch.randn(E, r, c, generator=g)
        i, j = torch.arange(r // 128).view(-1, 1), torch.arange(c // 128).view(1, -1)
        mag = (4.0 ** (i - j)).float().expand(E, -1, -1)
        return (w * mag.repeat_interleave(128, 1).repeat_interleave(128, 2) * 0.05).bfloat16()
    return one(M, H), one(M, H), one(H, M)


def _stored(ckpt, E=E, M=M, H=H, act=F.silu):
    ex = LlamaFFNNetwork(M, H, E, 1, activation_fn=act, weight_format='fp8_block')
    ex.load_fp8_block_weights(*ckpt)
    return ex


def _ctx(rows=None, top_k=1):
    return types.SimpleNamespace(group=None, adaptive_degree=1, top_k=top_k, megablocks_size=0 if rows is None else 1,
                                 dispatch_count=rows)


def _fp64_reference(x, ckpt, act='silu'):
    """The layer composed in fp64 from the dequantised checkpoint tensors (HF orientation: y = down(act(gate x) * up x))."""
    gate, gs, up, us, down, ds = ckpt
    wg, wu, wd = (BF8.dequantize_weight(q, s).double() for q, s in ((gate, gs), (up, us), (down, ds)))
    xd = x.double()
    g, u = xd @ wg.transpose(1, 2), xd @ wu.transpose(1, 2)
    return (BF8._act(g, act)[0] * u) @ wd.transpose(1, 2)


def _rel(y, ref):
    return float((y.double() - ref).norm() / ref.norm())


def test_export_then_load_is_the_forward_copy_bit_for_bit():
    w1, w2, w3 = _bf16_weights()
    ckpt = BF8.export_glu_weights(w1, w2, w3)
    gate, gs, up, us, down, ds = ckpt
    assert gate.shape == (E, H, M) and gs.shape == (E, H // 128, M // 128) and down.shape == (E, M, H)
    assert all(t.dtype == torch.float8_e4m3fn for t in (gate, up, down))
    qglu, sglu, q3t, s3t = BF8.load_glu_weights(*ckpt)
    _, _, qglu0, sglu0 = BF8.glu_weight(w1, w2)
    _, _, q3t0, s3t0 = BF8.weight(w3)
    assert torch.equal(qglu.view(torch.uint8), qglu0.view(torch.uint8))
    assert torch.equal(sglu, sglu0) and torch.equal(s3t, s3t0)
    assert torch.equal(q3t.view(torch.uint8), q3t0.view(torch.uint8))
    ex = _stored(ckpt)
    for name, t in zip(LlamaFFNNetwork.FP8_BLOCK_BUFFERS, (qglu0, sglu0, q3t0, s3t0)):
        assert torch.equal(getattr(ex, name).view(torch.uint8), t.view(torch.uint8)), name


def test_module_export_matches_the_function():
    ex16 = LlamaFFNNetwork(M, H, E, 1, fp8='block').bfloat16()
    w = [getattr(ex16, n).view(ex16.full_shapes[n]) for n in ('W_fc1', 'W_fc2', 'W_fc3')]
    for a, b in zip(ex16.export_fp8_block_weights(), BF8.export_glu_weights(*w)):
        assert torch.equal(a.view(torch.uint8), b.view(torch.uint8))


@pytest.mark.parametrize('decode', [False, True])
@pytest.mark.parametrize('act', ['silu', 'gelu', 'relu'])
def test_layer_output_against_fp64_composition_and_near_misses(decode, act):
    fn = {'silu': F.silu, 'gelu': F.gelu, 'relu': F.relu}[act]
    ckpt = BF8.export_glu_weights(*_bf16_weights(1))
    x = torch.randn(E, 6, M, generator=torch.Generator().manual_seed(2)).bfloat16()
    rows = torch.tensor([6, 1, 0], dtype=torch.int32) if decode else None
    ref = _fp64_reference(x, ckpt, act)
    if decode:
        ref = BF8.zero_rows_past(ref, rows)
    # decode: fp32 on the stored weights, x unquantised (relative error 0.002 here); prefill: x and h in 1 x 128 e4m3
    # tiles as on the GPU (0.044).  Each near miss is off by 0.8 or more.
    tol = 0.01 if decode else 0.06

    def err(c):
        with torch.no_grad():
            return _rel(_stored(c, act=fn)(x, _ctx(rows)), ref)

    gate, gs, up, us, down, ds = ckpt
    misses = {
        'gate and up swapped': (up, us, gate, gs, down, ds),
        'gate scales transposed': (gate, gs.transpose(1, 2).contiguous(), up, us, down, ds),
        'down scales transposed': (gate, gs, up, us, down, ds.transpose(1, 2).contiguous()),
    }
    assert err(ckpt) < tol
    for name, c in misses.items():
        assert err(c) > 5 * tol, name


def test_decode_kernel_reference_zeroes_rows_past_the_counts():
    ckpt = BF8.export_glu_weights(*_bf16_weights(3))
    ex = _stored(ckpt)
    x = torch.full((E, 5, M), float('nan')).bfloat16()
    x[0, :2] = torch.randn(2, M).bfloat16()
    rows = torch.tensor([2, 0, 0], dtype=torch.int32)
    with torch.no_grad():
        y = ex(x, _ctx(rows))
    assert torch.isfinite(y[0, :2].float()).all() and torch.count_nonzero(y[0, 2:]) == 0 and torch.count_nonzero(y[1:]) == 0
    # the prefill GEMMs with row counts (the layer's path above SKINNY_PASS_ROWS rows per expert) too
    q, s = BF8.quantize_act(x)
    out = BF8.block_fp8_gemm(q, s, ex.W_gate_up, ex.W_gate_up_scale, epilogue=BF8.EPI_GLU, row_counts=rows)
    for t in out:
        assert torch.isfinite(t[0, :2].float()).all() and torch.count_nonzero(t[0, 2:]) == 0 and torch.count_nonzero(t[1:]) == 0


def test_construction_refusals():
    with pytest.raises(ValueError, match='multiples of 128'):
        LlamaFFNNetwork(192, 256, 2, 1, weight_format='fp8_block')
    with pytest.raises(ValueError, match='multiples of 128'):
        LlamaFFNNetwork(256, 200, 2, 1, weight_format='fp8_block')
    with pytest.raises(ValueError, match='sharded_count'):
        LlamaFFNNetwork(256, 256, 1, 2, weight_format='fp8_block')
    for fp8 in (True, False, 'row', 'mx'):
        with pytest.raises(ValueError, match='fp8 must be unset'):
            LlamaFFNNetwork(256, 256, 2, 1, fp8=fp8, weight_format='fp8_block')
    with pytest.raises(ValueError, match='weight_format'):
        LlamaFFNNetwork(256, 256, 2, 1, weight_format='fp8')
    LlamaFFNNetwork(256, 256, 2, 1, fp8='block', weight_format='fp8_block')
    with pytest.raises(ValueError, match='ffn experts'):
        moe.moe_layer(gate_type={'type': 'top', 'k': 2}, model_dim=256,
                      experts={'type': 'ffn', 'num_experts_per_device': 2, 'hidden_size_per_expert': 256,
                               'weight_format': 'fp8_block'})


def test_no_parameters_and_the_default_is_unchanged():
    ex = LlamaFFNNetwork(M, H, E, 1, weight_format='fp8_block')
    assert list(ex.parameters()) == []
    assert set(ex.state_dict()) == set(LlamaFFNNetwork.FP8_BLOCK_BUFFERS)
    torch.manual_seed(5)
    a = LlamaFFNNetwork(M, H, E, 1)
    torch.manual_seed(5)
    b = LlamaFFNNetwork(M, H, E, 1, weight_format=None)
    assert set(a.state_dict()) == {'W_fc1', 'W_fc2', 'W_fc3'}
    assert all(torch.equal(a.state_dict()[k], b.state_dict()[k]) for k in a.state_dict())
    torch.manual_seed(5)
    LlamaFFNNetwork(M, H, E, 1, weight_format='fp8_block')      # draws no random numbers
    after = torch.randn(4)
    torch.manual_seed(5)
    assert torch.equal(after, torch.randn(4))


def test_buffer_dtypes_survive_dtype_casts():
    ex = _stored(BF8.export_glu_weights(*_bf16_weights(4)))
    raw = {n: getattr(ex, n).clone() for n in LlamaFFNNetwork.FP8_BLOCK_BUFFERS}
    for cast in (lambda m: m.bfloat16(), lambda m: m.half(), lambda m: m.float(), lambda m: m.double(),
                 lambda m: m.to(torch.float16), lambda m: m.to('cpu', torch.bfloat16), lambda m: m.cpu()):
        cast(ex)
        for n, t in raw.items():
            b = getattr(ex, n)
            assert b.dtype == t.dtype, (n, b.dtype)
            assert torch.equal(b.view(torch.uint8), t.view(torch.uint8)), n


def _layer(seed=1, shared=None, E_local=4, M=256, H=128, k=2):
    return moe.moe_layer(gate_type={'type': 'top', 'k': k}, model_dim=M, seeds=(seed, seed, seed), shared_experts=shared,
                         experts={'type': 'llama_ffn', 'num_experts_per_device': E_local, 'hidden_size_per_expert': H,
                                  'weight_format': 'fp8_block'}).bfloat16()


@pytest.mark.parametrize('shared', [None, {'num_experts': 1, 'gate': True}])
def test_state_dict_round_trip_and_grad_refusal(shared):
    layer = _layer(shared=shared)
    assert list(layer.experts.parameters()) == []
    ckpt = BF8.export_glu_weights(*_bf16_weights(6, E=4, M=256, H=128))
    layer.experts.load_fp8_block_weights(*ckpt)
    if shared is not None:
        assert layer.shared_experts.weight_format == 'fp8_block'
        layer.shared_experts.load_fp8_block_weights(*BF8.export_glu_weights(*_bf16_weights(7, E=1, M=256, H=128)))
    x = torch.randn(32, 256).bfloat16()
    with torch.no_grad():
        y = layer(x)
    fresh = _layer(seed=9, shared=shared)
    fresh.load_state_dict(layer.state_dict())
    with torch.no_grad():
        assert torch.equal(fresh(x), y)
    with pytest.raises(RuntimeError, match='inference-only'):
        layer(x.clone().requires_grad_(True))
    with pytest.raises(ValueError, match='bf16'), torch.no_grad():
        layer.float()(x.float())


def test_loader_refuses_bad_shapes_and_dtypes():
    gate, gs, up, us, down, ds = BF8.export_glu_weights(*_bf16_weights(8, M=256, H=128))
    ex = LlamaFFNNetwork(256, 128, E, 1, weight_format='fp8_block')
    with pytest.raises(ValueError, match='gate_scale'):
        ex.load_fp8_block_weights(gate, gs.transpose(1, 2), up, us, down, ds)
    with pytest.raises(ValueError, match='down'):
        ex.load_fp8_block_weights(gate, gs, up, us, down.float(), ds)
    with pytest.raises(ValueError, match='up'):
        ex.load_fp8_block_weights(gate, gs, up[:, :, :128], us, down, ds)
    with pytest.raises(ValueError, match='W_gate_up'):
        LlamaFFNNetwork(256, 128, E + 1, 1, weight_format='fp8_block').load_fp8_block_weights(gate, gs, up, us, down, ds)


GLOO = r'''
sys.path.insert(0, os.getcwd())
from tutel_b200 import moe, system
from tutel_b200.ops import block_fp8 as BF8
env = system.init_data_model_parallel(backend='gloo')
W, r = env.global_size, env.global_rank
path = os.environ['CKPT_DIR']
torch.manual_seed(0)
x = torch.randn(24, 256).bfloat16()
g = torch.Generator().manual_seed(3)
w1, w2 = (torch.randn(4, 256, 128, generator=g) * 0.05).bfloat16(), (torch.randn(4, 256, 128, generator=g) * 0.05).bfloat16()
w3 = (torch.randn(4, 128, 256, generator=g) * 0.05).bfloat16()
ckpt = BF8.export_glu_weights(w1, w2, w3)
nle = 4 // W
layer = moe.moe_layer(gate_type={'type': 'top', 'k': 2}, model_dim=256, seeds=(1, 1, 1),
                      experts={'type': 'llama_ffn', 'num_experts_per_device': nle, 'hidden_size_per_expert': 128,
                               'weight_format': 'fp8_block'}).bfloat16()
layer.experts.load_fp8_block_weights(*(t[r * nle:(r + 1) * nle] for t in ckpt))
with torch.no_grad():
    y = layer(x)
if W == 1:
    torch.save(y, path + '/out.pt')
else:
    try:
        layer(x, adaptive_r=0)
        raise SystemExit('adaptive_r=0 was not refused')
    except ValueError:
        pass
    y0 = torch.load(path + '/out.pt')
    assert torch.equal(y, y0), (y.float() - y0.float()).abs().max()
    if r == 0:
        print('BLOCK_FP8_WEIGHTS_OK')
'''


def test_two_gloo_ranks_equal_one_rank(tmp_path):
    env = {'CKPT_DIR': str(tmp_path)}
    run_workers(GLOO, nproc=1, env=env)
    out = run_workers(GLOO, nproc=2, env=env)
    assert 'BLOCK_FP8_WEIGHTS_OK' in out
