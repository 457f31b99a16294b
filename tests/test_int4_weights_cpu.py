"""Group-32 int4 SwiGLU experts (``llama_ffn`` with ``weight_format='int4'``) on CPU: the format's packing, unpacking and
quantiser against the element-by-element definitions of tests/int4_reference.py, the loader, the module's buffers,
refusals and state dict, the shared-expert override, the layer against the fp64 composition, near misses that the
kernels' bounds reject, and a two-rank Gloo run."""
import types

import pytest
import torch
import torch.nn.functional as F

from tutel_b200 import moe
from tutel_b200.models.experts.llama_ffn import LlamaFFNNetwork
from tutel_b200.ops import int4 as I4

import int4_reference as R
from helpers import run_workers

E, M, H = 3, 256, 128


def _bf16_weights(seed=0, E=E, M=M, H=H, scale=0.05):
    g = torch.Generator().manual_seed(seed)
    w1, w2 = ((torch.randn(E, M, H, generator=g) * scale).bfloat16() for _ in range(2))
    return w1, w2, (torch.randn(E, H, M, generator=g) * scale).bfloat16()


def _stored(ckpt, E=E, M=M, H=H, act=F.silu):
    ex = LlamaFFNNetwork(M, H, E, 1, activation_fn=act, weight_format='int4')
    ex.load_int4_weights(*ckpt)
    return ex


def _ctx(rows=None, top_k=1):
    return types.SimpleNamespace(group=None, adaptive_degree=1, top_k=top_k, megablocks_size=0 if rows is None else 1,
                                 dispatch_count=rows)


def test_pack_unpack_and_int32_against_the_definitions():
    q = torch.randint(-8, 8, (2, 3, 64), generator=torch.Generator().manual_seed(1), dtype=torch.int8)
    packed = I4.pack_reference(q)
    assert packed.dtype == torch.uint8 and torch.equal(packed, R.pack(q))
    assert torch.equal(I4.unpack_reference(packed), q) and torch.equal(R.unpack(packed), q)
    words = R.pack_int32(q)
    assert torch.equal(I4.unpack_int32(words, 64), q)
    # one hand-written word: elements 0..7 = -8, -7, 0, 7, 1, -1, 3, -4 -> nibbles 0, 1, 8, 15, 9, 7, 11, 4
    w = torch.tensor([[0x4B79F810]], dtype=torch.int32)
    assert I4.unpack_int32(w, 8).tolist() == [[-8, -7, 0, 7, 1, -1, 3, -4]]
    assert R.pack(torch.tensor([[-8, -7]], dtype=torch.int8)).tolist() == [[0x10]]
    with pytest.raises(ValueError, match='int32'):
        I4.unpack_int32(words.to(torch.int64), 64)


def test_quantiser_against_the_definition():
    g = torch.Generator().manual_seed(2)
    w = (torch.randn(2, 4, 128, generator=g) * torch.logspace(-6, 2, 4).view(1, 4, 1)).bfloat16()
    w[0, 0, :32] = 0                                   # all-zero group: s = 1
    w[0, 1, 32:64] = 1e-40                             # subnormal amax: s clamps to the smallest normal
    w[1, 2, 5] = float('nan')                          # NaN: not in amax, q = 0
    w[1, 3, 64:96] = torch.tensor([3.5, -3.5] * 16).bfloat16()   # w / s = +-7 exactly
    q, s = I4.quantize_reference(w)
    q0, s0 = R.quantize(w)
    assert torch.equal(q, q0) and torch.equal(s.view(torch.int16), s0.view(torch.int16))
    assert float(s[0, 0, 0]) == 1.0 and float(s[0, 1, 1]) == 2.0 ** -126 and int(q[1, 2, 5]) == 0
    assert int(q.min()) >= -8 and int(q.max()) <= 7


def test_export_then_load_bit_for_bit():
    w1, w2, w3 = _bf16_weights()
    ckpt = I4.export_glu_weights(w1, w2, w3)
    gate, gs, up, us, down, ds = ckpt
    assert gate.shape == (E, H, M) and gs.shape == (E, H, M // 32) and down.shape == (E, M, H) and ds.shape == (E, M, H // 32)
    assert gate.dtype == torch.int8 and gs.dtype == torch.bfloat16
    for (q, s), w in (((gate, gs), w1.transpose(1, 2)), ((up, us), w2.transpose(1, 2)), ((down, ds), w3.transpose(1, 2))):
        q0, s0 = R.quantize(w.contiguous())
        assert torch.equal(q, q0) and torch.equal(s, s0)
    ex = _stored(ckpt)
    wg, wu = R.split_glu(R.stored_values(ex.W_gate_up, ex.W_gate_up_scale))
    assert torch.equal(wg, R.values(gate, gs)) and torch.equal(wu, R.values(up, us))
    assert torch.equal(R.stored_values(ex.W_down, ex.W_down_scale), R.values(down, ds))
    assert torch.equal(ex.W_down, R.pack(down))
    # the module exporter is the function
    ex16 = LlamaFFNNetwork(M, H, E, 1).bfloat16()
    w = [getattr(ex16, n).view(ex16.full_shapes[n]) for n in ('W_fc1', 'W_fc2', 'W_fc3')]
    for a, b in zip(ex16.export_int4_weights(), I4.export_glu_weights(*w)):
        assert torch.equal(a, b)


def test_loader_refusals():
    gate, gs, up, us, down, ds = I4.export_glu_weights(*_bf16_weights(3))
    ex = LlamaFFNNetwork(M, H, E, 1, weight_format='int4')
    with pytest.raises(ValueError, match='up'):
        ex.load_int4_weights(gate, gs, up[:, :, :128], us, down, ds)
    with pytest.raises(ValueError, match='down'):
        ex.load_int4_weights(gate, gs, up, us, down.to(torch.int16), ds)
    with pytest.raises(ValueError, match='gate_scale'):
        ex.load_int4_weights(gate, gs.float(), up, us, down, ds)
    with pytest.raises(ValueError, match='down_scale'):
        ex.load_int4_weights(gate, gs, up, us, down, ds[:, :, :2])
    bad = gate.clone()
    bad[1, 2, 3] = 8
    with pytest.raises(ValueError, match='outside the int4 range'):
        ex.load_int4_weights(bad, gs, up, us, down, ds)
    bad = down.clone()
    bad[0, 0, 0] = -9
    with pytest.raises(ValueError, match='outside the int4 range'):
        ex.load_int4_weights(gate, gs, up, us, bad, ds)
    with pytest.raises(ValueError, match='W_gate_up'):
        LlamaFFNNetwork(M, H, E + 1, 1, weight_format='int4').load_int4_weights(gate, gs, up, us, down, ds)
    with pytest.raises(ValueError, match="weight_format='int4'"):
        LlamaFFNNetwork(M, H, E, 1, weight_format='fp8_block').load_int4_weights(gate, gs, up, us, down, ds)


def test_construction_refusals():
    with pytest.raises(ValueError, match='multiples of 128'):
        LlamaFFNNetwork(192, 256, 2, 1, weight_format='int4')
    with pytest.raises(ValueError, match='multiples of 128'):
        LlamaFFNNetwork(256, 200, 2, 1, weight_format='int4')
    with pytest.raises(ValueError, match='sharded_count'):
        LlamaFFNNetwork(256, 256, 1, 2, weight_format='int4')
    for fp8 in (True, False, 'row', 'block', 'mx'):
        with pytest.raises(ValueError, match='fp8 must be unset'):
            LlamaFFNNetwork(256, 256, 2, 1, fp8=fp8, weight_format='int4')
    with pytest.raises(ValueError, match='fp8_wgrad'):
        LlamaFFNNetwork(256, 256, 2, 1, weight_format='int4', fp8_wgrad=True)
    with pytest.raises(ValueError, match='fp8_packed'):
        LlamaFFNNetwork(256, 256, 2, 1, weight_format='int4', fp8_packed=True)
    with pytest.raises(ValueError, match='weight_format'):
        LlamaFFNNetwork(256, 256, 2, 1, weight_format='int8')
    with pytest.raises(ValueError, match='ffn experts'):
        moe.moe_layer(gate_type={'type': 'top', 'k': 2}, model_dim=256,
                      experts={'type': 'ffn', 'num_experts_per_device': 2, 'hidden_size_per_expert': 256,
                               'weight_format': 'int4'})


def test_no_parameters_rng_untouched_and_buffer_dtypes_survive_casts():
    ex = LlamaFFNNetwork(M, H, E, 1, weight_format='int4')
    assert list(ex.parameters()) == []
    assert set(ex.state_dict()) == set(LlamaFFNNetwork.INT4_BUFFERS)
    assert 'int4' in repr(ex)
    torch.manual_seed(5)
    LlamaFFNNetwork(M, H, E, 1, weight_format='int4')          # draws no random numbers
    after = torch.randn(4)
    torch.manual_seed(5)
    assert torch.equal(after, torch.randn(4))
    ex.load_int4_weights(*I4.export_glu_weights(*_bf16_weights(4)))
    raw = {n: getattr(ex, n).clone() for n in LlamaFFNNetwork.INT4_BUFFERS}
    for cast in (lambda m: m.bfloat16(), lambda m: m.half(), lambda m: m.float(), lambda m: m.double(),
                 lambda m: m.to(torch.float16), lambda m: m.to('cpu', torch.bfloat16), lambda m: m.cpu()):
        cast(ex)
        for n, t in raw.items():
            b = getattr(ex, n)
            assert b.dtype == t.dtype and torch.equal(b, t), (n, b.dtype)


def _layer(seed=1, shared=None, E_local=4, M=256, H=128, k=2, fmt='int4'):
    return moe.moe_layer(gate_type={'type': 'top', 'k': k}, model_dim=M, seeds=(seed, seed, seed), shared_experts=shared,
                         experts={'type': 'llama_ffn', 'num_experts_per_device': E_local, 'hidden_size_per_expert': H,
                                  'weight_format': fmt}).bfloat16()


@pytest.mark.parametrize('shared', [None, {'num_experts': 1, 'gate': True}])
def test_state_dict_round_trip_and_forward_refusals(shared):
    layer = _layer(shared=shared)
    layer.experts.load_int4_weights(*I4.export_glu_weights(*_bf16_weights(6, E=4)))
    if shared is not None:
        assert layer.shared_experts.weight_format == 'int4'
        layer.shared_experts.load_int4_weights(*I4.export_glu_weights(*_bf16_weights(7, E=1)))
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


def test_shared_expert_weight_format_override():
    layer = _layer(shared={'num_experts': 2, 'weight_format': None})
    assert layer.experts.weight_format == 'int4' and layer.shared_experts.weight_format is None
    assert {n for n, _ in layer.shared_experts.named_parameters()} == {'W_fc1', 'W_fc2', 'W_fc3'}
    assert layer.shared_experts.full_shapes['W_fc1'] == (1, 256, 256)
    layer = _layer(shared={'num_experts': 1, 'weight_format': 'fp8_block'})
    assert layer.shared_experts.weight_format == 'fp8_block'
    layer = _layer(shared={'num_experts': 1, 'weight_format': 'int4'}, fmt=None)
    assert layer.experts.weight_format is None and layer.shared_experts.weight_format == 'int4'
    assert _layer(shared={'num_experts': 1}).shared_experts.weight_format == 'int4'      # no key: inherited
    with pytest.raises(ValueError, match='weight_format'):
        _layer(shared={'num_experts': 1, 'weight_format': 'int8'})
    with pytest.raises(ValueError, match='Unrecognized shared_experts'):
        _layer(shared={'num_experts': 1, 'format': 'int4'})
    # a 16-bit shared expert beside int4 routed ones runs and equals the same layer built in bf16 for the shared part
    layer = _layer(shared={'num_experts': 1, 'weight_format': None, 'gate': True})
    layer.experts.load_int4_weights(*I4.export_glu_weights(*_bf16_weights(8, E=4)))
    with torch.no_grad():
        y = layer(torch.randn(16, 256).bfloat16())
    assert torch.isfinite(y.float()).all()


def _fake(x, qglu, sglu, q3t, s3t, act, kernel, counts=None, miss=None):
    """A CPU stand-in for one of the two kernels on the stored operands, with one deliberate mistake ``miss``."""
    def vals(packed, s):
        lo, hi = (packed & 15).to(torch.int16), (packed >> 4).to(torch.int16)
        if miss == 'nibble order':
            lo, hi = hi, lo
        q = torch.stack([lo, hi], dim=-1).reshape(*packed.shape[:-1], -1)
        q = torch.where(q >= 8, q - 16, q) if miss == "two's complement" else q - 8
        if miss == 'neighbour scale':
            s = s.roll(1, dims=-1)
        v = R.values(q, s)
        if miss == 'dropped last group':
            v[..., -32:] = 0
        return v
    wg, wu = R.split_glu(vals(qglu, sglu))
    w3 = vals(q3t, s3t)
    if miss == 'gate and up swapped':
        wg, wu = wu, wg
    if kernel == 'prefill':                                 # bf16 weights, bf16 h, as on the GPU
        wg, wu, w3 = (w.to(torch.bfloat16).double() for w in (wg, wu, w3))
    xd = x.double()
    h = R._FN['none' if miss == 'missing activation' else act](xd @ wg.transpose(1, 2)) * (xd @ wu.transpose(1, 2))
    if kernel == 'prefill':
        h = h.to(torch.bfloat16).double()
    y = (h @ w3.transpose(1, 2)).float()
    if counts is not None:
        y = torch.where(torch.arange(y.size(1)).view(1, -1, 1) < counts.view(-1, 1, 1), y, torch.zeros(()))
    return y.bfloat16() if kernel == 'prefill' else y


MISSES = ['nibble order', "two's complement", 'neighbour scale', 'gate and up swapped', 'dropped last group',
          'missing activation']


@pytest.mark.parametrize('kernel', ['decode', 'prefill'])
@pytest.mark.parametrize('act', ['silu', 'gelu', 'relu'])
def test_layer_against_fp64_and_near_misses_the_bounds_reject(kernel, act):
    fn = {'silu': F.silu, 'gelu': F.gelu, 'relu': F.relu}[act]
    w1, w2, w3 = _bf16_weights(1, scale=0.2)
    ckpt = I4.export_glu_weights(w1, w2, w3)
    ex = _stored(ckpt, act=fn)
    x = torch.randn(E, 6, M, generator=torch.Generator().manual_seed(2)).bfloat16()
    rows = torch.tensor([6, 1, 0], dtype=torch.int32)
    ref, bound = R.stored_reference(x, ex.W_gate_up, ex.W_gate_up_scale, ex.W_down, ex.W_down_scale, act, kernel)
    # the module's CPU path (the kernels' references), decode with row counts and prefill without
    with torch.no_grad():
        y = ex(x, _ctx(rows if kernel == 'decode' else None))
    # the op returns x's dtype: the decode kernel's fp32 output rounds once more to bf16
    R.check(y, ref, bound + (R.U16 * ref.abs() if kernel == 'decode' else 0), rows if kernel == 'decode' else None)
    ops = (x, ex.W_gate_up, ex.W_gate_up_scale, ex.W_down, ex.W_down_scale, act, kernel)
    R.check(_fake(*ops, counts=rows), ref, bound, rows)
    for miss in MISSES:
        if miss == 'missing activation' and act == 'relu':
            continue                      # relu(g) * u and g * u differ only where g < 0: still checked below for silu / gelu
        with pytest.raises(AssertionError):
            R.check(_fake(*ops, counts=rows, miss=miss), ref, bound, rows)


def test_decode_reference_zeroes_rows_past_the_counts():
    ex = _stored(I4.export_glu_weights(*_bf16_weights(3)))
    x = torch.full((E, 5, M), float('nan')).bfloat16()
    x[0, :2] = torch.randn(2, M).bfloat16()
    rows = torch.tensor([2, 0, 0], dtype=torch.int32)
    with torch.no_grad():
        y = ex(x, _ctx(rows))
        y2 = I4.glu_ffn_int4(x, ex.W_gate_up, ex.W_gate_up_scale, ex.W_down, ex.W_down_scale, 'silu', rows)
    for t in (y, y2):
        assert torch.isfinite(t[0, :2].float()).all() and torch.count_nonzero(t[0, 2:]) == 0 and torch.count_nonzero(t[1:]) == 0


GLOO = r'''
sys.path.insert(0, os.getcwd())
from tutel_b200 import moe, system
from tutel_b200.ops import int4 as I4
env = system.init_data_model_parallel(backend='gloo')
W, r = env.global_size, env.global_rank
path = os.environ['CKPT_DIR']
torch.manual_seed(0)
x = torch.randn(24, 256).bfloat16()
g = torch.Generator().manual_seed(3)
w1, w2 = (torch.randn(4, 256, 128, generator=g) * 0.05).bfloat16(), (torch.randn(4, 256, 128, generator=g) * 0.05).bfloat16()
w3 = (torch.randn(4, 128, 256, generator=g) * 0.05).bfloat16()
ckpt = I4.export_glu_weights(w1, w2, w3)
nle = 4 // W
layer = moe.moe_layer(gate_type={'type': 'top', 'k': 2}, model_dim=256, seeds=(1, 1, 1),
                      experts={'type': 'llama_ffn', 'num_experts_per_device': nle, 'hidden_size_per_expert': 128,
                               'weight_format': 'int4'}).bfloat16()
layer.experts.load_int4_weights(*(t[r * nle:(r + 1) * nle] for t in ckpt))
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
        print('INT4_WEIGHTS_OK')
'''


def test_two_gloo_ranks_equal_one_rank(tmp_path):
    env = {'CKPT_DIR': str(tmp_path)}
    run_workers(GLOO, nproc=1, env=env)
    out = run_workers(GLOO, nproc=2, env=env)
    assert 'INT4_WEIGHTS_OK' in out
