"""Shared experts on the CPU: the combine bounds of tests/shared_expert_reference.py against fp32 emulations of the
kernels (the faithful one passes, likely bugs fail), the torch combine paths, the autograd function, the layer's API
(parameters, RNG, refusals, checkpoints) and a two-rank Gloo run."""
import pytest
import torch
import torch.nn.functional as F

import shared_expert_reference as R
from helpers import run_workers


# ------------------------------------------------------------------------------------------------------------------
# fp32 emulations of decode_rows_kernel / gate_grad_kernel with the shared term
# ------------------------------------------------------------------------------------------------------------------
def _fma(a, b, c):
    """fmaf on fp32 tensors: the fp64 product of two fp32 values is exact, the sum is rounded once to fp32."""
    return (a.double() * b.double() + c.double()).float()


def _sigmoid32(logit):
    one = torch.ones((), dtype=torch.float32)
    return one / (one + torch.exp(-logit.float()))


def emu_decode(buf, gates, idx, loc, E, C, base, logit, bug=None):
    valid, row = R._rows(idx, loc, E, C)
    S, M = idx.size(1), buf.size(1)
    acc = torch.zeros(S, M, dtype=torch.float32)
    for j in range(idx.size(0)):
        w = (gates[j].float() if gates is not None else torch.ones(S))[:, None].expand(S, M)
        acc = torch.where(valid[j][:, None], _fma(w, buf[row[j]].float(), acc), acc)
    if bug == 'round_routed_first':
        acc = acc.to(buf.dtype).float()
    ws = torch.ones(S, 1) if logit is None else _sigmoid32(logit).view(-1, 1)
    if bug == 'logit_not_sigmoid':
        ws = logit.float().view(-1, 1)
    out = _fma(ws.expand(S, M), base.float(), acc)
    if bug == 'skip_dropped':
        out = torch.where(valid.any(0)[:, None], out, acc)
    return out.to(buf.dtype)


def emu_shared_grad(dy, base, logit, bug=None):
    ws = _sigmoid32(logit).view(-1, 1)
    d_base = dy if bug == 'd_base_unscaled' else (dy.float() * ws).to(dy.dtype)
    dot = (dy.double() * base.double()).sum(1).float()
    d_logit = dot if bug == 'no_sigmoid_derivative' else ws.view(-1) * (1 - ws.view(-1)) * dot
    return d_base, d_logit


def _case(dtype=torch.bfloat16, S=256, M=64, k=4, E=8, C=96, seed=0, base_scale=0.25):
    g = torch.Generator().manual_seed(seed)
    idx = torch.randint(0, E, (k, S), generator=g, dtype=torch.int32)
    from dispatch_reference import INVALID_LOC, ref_locations
    loc = ref_locations(idx, E)[0]                               # some choices past C: dropped
    loc[:, :5] = INVALID_LOC                                     # fully dropped tokens
    buf = torch.randn(E * C, M, generator=g).to(dtype)
    gates = torch.rand(k, S, generator=g)
    base = (torch.randn(S, M, generator=g) * base_scale).to(dtype)
    logit = torch.randn(S, generator=g) * 2
    dy = torch.randn(S, M, generator=g).to(dtype)
    assert bool((loc >= C).any()), 'the case must drop choices'
    return buf, gates, idx, loc, E, C, base, logit, dy


@pytest.mark.parametrize('gated', [False, True])
@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16, torch.float32])
def test_faithful_emulation_passes(dtype, gated):
    buf, gates, idx, loc, E, C, base, logit, dy = _case(dtype)
    logit = logit if gated else None
    R.check_decode_shared('emulation', emu_decode(buf, gates, idx, loc, E, C, base, logit), buf, gates, idx, loc, E, C,
                          base, logit)
    R.check_decode_shared('emulation, pre-scored', emu_decode(buf, None, idx, loc, E, C, base, logit), buf, None, idx, loc,
                          E, C, base, logit)
    if gated:
        d_base, d_logit = emu_shared_grad(dy, base, logit)
        R.check_d_base('emulation', d_base, dy, logit)
        R.check_d_shared_logit('emulation', d_logit, dy, base, logit)
    else:
        R.check_d_base('ungated', dy, dy, None)


@pytest.mark.parametrize('bug', ['round_routed_first', 'logit_not_sigmoid', 'skip_dropped'])
def test_decode_bound_rejects_likely_bugs(bug):
    buf, gates, idx, loc, E, C, base, logit, dy = _case()
    bad = emu_decode(buf, gates, idx, loc, E, C, base, logit, bug=bug)
    with pytest.raises(AssertionError):
        R.check_decode_shared(bug, bad, buf, gates, idx, loc, E, C, base, logit)


@pytest.mark.parametrize('bug', ['d_base_unscaled', 'no_sigmoid_derivative'])
def test_backward_bound_rejects_likely_bugs(bug):
    buf, gates, idx, loc, E, C, base, logit, dy = _case()
    d_base, d_logit = emu_shared_grad(dy, base, logit, bug=bug)
    with pytest.raises(AssertionError):
        if bug == 'd_base_unscaled':
            R.check_d_base(bug, d_base, dy, logit)
        else:
            R.check_d_shared_logit(bug, d_logit, dy, base, logit)


# ------------------------------------------------------------------------------------------------------------------
# the torch combine paths (CPU) and the autograd function
# ------------------------------------------------------------------------------------------------------------------
def _plan(idx, loc, E, C):
    from tutel_b200.ops.dispatch import DispatchPlan
    return DispatchPlan(E, C, idx, loc)


@pytest.mark.parametrize('gated', [False, True])
@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16, torch.float32])
def test_cpu_combine_paths_within_bound(dtype, gated):
    from tutel_b200.ops.dispatch import raw_decode, raw_shared_grad
    buf, gates, idx, loc, E, C, base, logit, dy = _case(dtype)
    logit = logit if gated else None
    plan = _plan(idx, loc, E, C)
    out = raw_decode(buf, gates, plan, base, logit)
    assert out.dtype == dtype
    R.check_decode_shared('cpu %s' % dtype, out, buf, gates, idx, loc, E, C, base, logit)
    if gated:
        dg, d_base, d_logit = raw_shared_grad(dy, buf, plan, base, logit)
        R.check_gate_grad('cpu', dg.float(), dy, buf, idx, loc, E, C)
        R.check_d_base('cpu', d_base, dy, logit)
        R.check_d_shared_logit('cpu', d_logit.float(), dy, base, logit)
        none, d_base2, d_logit2 = raw_shared_grad(dy, None, plan, base, logit, routed=False)
        assert none is None and torch.equal(d_base2, d_base) and torch.equal(d_logit2, d_logit)


@pytest.mark.parametrize('postscore', [True, False])
@pytest.mark.parametrize('gated', [False, True])
def test_gating_decoder_gradcheck(gated, postscore):
    from tutel_b200.ops.dispatch import GatingDecoder
    buf, gates, idx, loc, E, C, base, logit, dy = _case(torch.float32, S=12, M=8, k=2, E=4, C=5)
    plan = _plan(idx, loc, E, C)
    buf = buf.double().requires_grad_(True)
    g = gates.double().requires_grad_(True) if postscore else None
    b = base.double().requires_grad_(True)
    l = logit.double().requires_grad_(True) if gated else None
    inputs = [t for t in (buf, g, b, l) if t is not None]

    def fn(*ts):
        it = iter(ts)
        bb = next(it)
        gg = next(it) if postscore else None
        bs = next(it)
        ll = next(it) if gated else None
        return GatingDecoder.apply(plan, bb, gg, bs, ll)
    assert torch.autograd.gradcheck(fn, inputs)


def test_gating_decoder_without_shared_terms_is_unchanged():
    from tutel_b200.ops.dispatch import GatingDecoder
    buf, gates, idx, loc, E, C, base, logit, dy = _case(torch.float32, S=12, M=8, k=2, E=4, C=5)
    plan = _plan(idx, loc, E, C)
    a = buf.clone().requires_grad_(True)
    ga = gates.clone().requires_grad_(True)
    y = GatingDecoder.apply(plan, a, ga)
    y.backward(dy)
    b = buf.clone().requires_grad_(True)
    gb = gates.clone().requires_grad_(True)
    z = GatingDecoder.apply(plan, b, gb, torch.zeros_like(base), None)
    z.backward(dy)
    assert torch.equal(y, z) and torch.equal(a.grad, b.grad) and torch.equal(ga.grad, gb.grad)


# ------------------------------------------------------------------------------------------------------------------
# the layer
# ------------------------------------------------------------------------------------------------------------------
def _layer(expert='ffn', shared=None, seeds=(1, 2, 3), E=4, k=2, M=16, H=24, **kw):
    from tutel_b200 import moe
    if expert == 'llama_ffn':
        experts = {'type': 'llama_ffn', 'num_experts_per_device': E, 'hidden_size_per_expert': H}
    else:
        experts = {'type': 'ffn', 'num_experts_per_device': E, 'hidden_size_per_expert': H, 'activation_fn': F.relu}
    args = dict(gate_type={'type': 'top', 'k': k}, model_dim=M, experts=experts, seeds=seeds, **kw)
    if shared is not None:
        args['shared_experts'] = shared
    return moe.moe_layer(**args)


@pytest.mark.parametrize('expert', ['ffn', 'llama_ffn'])
@pytest.mark.parametrize('gated', [False, True])
def test_parameter_names_and_shapes(expert, gated):
    M, H, n = 16, 24, 2
    layer = _layer(expert, {'num_experts': n, 'gate': gated}, M=M, H=H)
    plain = _layer(expert, None, M=M, H=H)
    sd, sd0 = layer.state_dict(), plain.state_dict()
    extra = {k: tuple(v.shape) for k, v in sd.items() if k not in sd0}
    if expert == 'ffn':
        want = {'shared_experts.batched_fc1_w': (1, n * H, M), 'shared_experts.batched_fc2_w': (1, n * H, M),
                'shared_experts.batched_fc1_bias': (1, n * H), 'shared_experts.batched_fc2_bias': (1, M)}
    else:
        want = {'shared_experts.W_fc1': (M * n * H,), 'shared_experts.W_fc2': (M * n * H,),
                'shared_experts.W_fc3': (n * H * M,)}
    if gated:
        want['shared_expert_gate.weight'] = (1, M)
    assert extra == want
    assert list(sd.keys())[:len(sd0)] == list(sd0.keys())
    for name, p in layer.named_parameters():
        assert hasattr(p, '_tutel_expert') == name.startswith('experts.'), name
    assert type(layer.shared_experts) is type(layer.experts)
    from tutel_b200.parallel.optimizer import TutelDistributedOptimizer
    opt = TutelDistributedOptimizer(layer.parameters())
    shared_ids = {id(p) for n_, p in layer.named_parameters() if n_.startswith('shared_')}
    assert shared_ids <= {id(p) for p in opt.params}


def test_shared_experts_keep_the_routed_options():
    from tutel_b200 import moe
    layer = moe.moe_layer(gate_type={'type': 'top', 'k': 2}, model_dim=16, shared_experts={'num_experts': 3},
                          experts={'type': 'ffn', 'num_experts_per_device': 4, 'hidden_size_per_expert': 8,
                                   'activation_fn': F.gelu, 'has_fc2_bias': False, 'fp8': True})
    se = layer.shared_experts
    assert se.fp8 and se.activation_fn is F.gelu and se.batched_fc2_bias is None and se.hidden_size == 24
    assert se.local_experts == 1 and se.sharded_count == 1


def test_none_leaves_state_dict_and_rng_unchanged():
    for seeds in (None, (1, 2, 3)):
        torch.manual_seed(7)
        a = _layer(shared=None, seeds=seeds)
        ra = torch.rand(4)
        torch.manual_seed(7)
        from tutel_b200 import moe
        b = moe.moe_layer(gate_type={'type': 'top', 'k': 2}, model_dim=16, seeds=seeds, shared_experts=None,
                          experts={'type': 'ffn', 'num_experts_per_device': 4, 'hidden_size_per_expert': 24,
                                   'activation_fn': F.relu})
        rb = torch.rand(4)
        assert torch.equal(ra, rb)
        sa, sb = a.state_dict(), b.state_dict()
        assert list(sa) == list(sb) and all(torch.equal(sa[k], sb[k]) for k in sa)
        assert a.shared_experts is None and a.shared_expert_gate is None
    # with shared experts the routed experts and gates draw exactly what they drew before, and with `seeds` so does
    # everything after the layer
    plain, shared = _layer(shared=None), _layer(shared={'num_experts': 2, 'gate': True})
    r0 = torch.rand(4)
    r1 = (_layer(shared=None), torch.rand(4))[1]
    assert torch.equal(r0, r1)
    sp, ss = plain.state_dict(), shared.state_dict()
    assert all(torch.equal(sp[k], ss[k]) for k in sp)


def test_refusals():
    from tutel_b200 import moe

    class Custom(torch.nn.Module):
        def __init__(self, model_dim, num_experts_per_device, sharded_count):
            super().__init__()
            self.w = torch.nn.Parameter(torch.zeros(num_experts_per_device, model_dim, model_dim))

        def forward(self, x, ctx):
            return torch.matmul(x, self.w)
    with pytest.raises(ValueError, match='custom'):
        moe.moe_layer(gate_type={'type': 'top', 'k': 1}, model_dim=8, shared_experts={'num_experts': 1},
                      experts={'type': 'custom', 'module': Custom, 'num_experts_per_device': 2})
    for bad in ({'num_experts': 0}, {'num_experts': 1.5}, {'num_experts': 1, 'scale': 2}, {}, 2):
        with pytest.raises(ValueError):
            _layer(shared=bad)
    layer = _layer(shared={'num_experts': 1}, M=16)
    with pytest.raises(ValueError, match='reserve_dims'):
        layer(torch.randn(4, 8, 2, 8), reserve_dims=2)
    _layer(shared=None, M=16)(torch.randn(4, 8, 2, 8), reserve_dims=2)      # unchanged without shared experts


@pytest.mark.parametrize('expert', ['ffn', 'llama_ffn'])
@pytest.mark.parametrize('gated', [False, True])
@pytest.mark.parametrize('postscore', [True, False])
def test_layer_equals_routed_layer_plus_shared_module(expert, gated, postscore):
    """fp64 on the CPU: y = routed layer + w * shared(x), and every gradient equals the torch composition's."""
    torch.manual_seed(0)
    layer = _layer(expert, {'num_experts': 2, 'gate': gated}, is_postscore=postscore).double()
    plain = _layer(expert, None, is_postscore=postscore).double()
    plain.load_state_dict({k: v for k, v in layer.state_dict().items() if not k.startswith('shared_')})
    x = torch.randn(2, 20, 16, dtype=torch.float64)
    xa = x.clone().requires_grad_(True)
    y = layer(xa)
    (y.pow(2).sum() + y.l_aux).backward()

    from tutel_b200.models.moe_layer import _SharedExpertContext
    xb = x.clone().requires_grad_(True)
    xs = xb.view(-1, 16)
    shared = layer.shared_experts(xs.view(1, 40, 16), _SharedExpertContext(layer, None)).view(40, 16)
    if gated:
        shared = torch.sigmoid(F.linear(xs, layer.shared_expert_gate.weight)) * shared
    grads = {n: p.grad.clone() for n, p in layer.named_parameters()}
    for p in layer.parameters():
        p.grad = None
    zp = plain(xb)
    z = zp + shared.view(2, 20, 16)
    (z.pow(2).sum() + zp.l_aux).backward()
    assert torch.allclose(y, z, rtol=1e-12, atol=1e-12)
    assert torch.allclose(xa.grad, xb.grad, rtol=1e-10, atol=1e-12)
    ref = dict(plain.named_parameters())
    for n, g in grads.items():
        want = ref[n].grad if n in ref else dict(layer.named_parameters())[n].grad
        assert want is not None and torch.allclose(g, want, rtol=1e-10, atol=1e-12), n


@pytest.mark.parametrize('gated', [False, True])
def test_checkpoint_gather_scatter_treat_shared_experts_as_replicated(gated):
    from tutel_b200.checkpoint.gather import gather_states
    from tutel_b200.checkpoint.scatter import scatter_state
    model = torch.nn.ModuleDict({'moe': _layer('ffn', {'num_experts': 2, 'gate': gated}, E=4)})
    state = model.state_dict()
    shared_keys = [k for k in state if '.shared_' in k]
    assert shared_keys
    shards = scatter_state(state, 2)
    for shard in shards:
        assert shard['moe.experts.batched_fc1_w'].size(0) == 2
        for k in shared_keys:
            assert torch.equal(shard[k], state[k]), k
    merged = gather_states(shards)
    assert set(merged) == set(state) and all(torch.equal(merged[k], state[k]) for k in state)


GLOO = r'''
sys.path.insert(0, os.getcwd())
import torch.nn.functional as F
from tutel_b200 import moe, system
env = system.init_data_model_parallel(backend='gloo')
W, r = env.global_size, env.global_rank
path = os.environ['CKPT_DIR']
gated = os.environ['GATED'] == '1'
torch.manual_seed(0)
x = torch.randn(16, 8, dtype=torch.float64)
def build(nle):
    return moe.moe_layer(gate_type={'type': 'top', 'k': 2}, model_dim=8, seeds=(1, 1, 1),
                         shared_experts={'num_experts': 2, 'gate': gated},
                         experts={'type': 'ffn', 'num_experts_per_device': nle, 'hidden_size_per_expert': 12,
                                  'activation_fn': lambda t: F.relu(t)}).double()
def run(layer):
    xx = x.clone().requires_grad_(True)
    y = layer(xx)
    y.pow(2).sum().backward()
    g = {n: p.grad for n, p in layer.named_parameters() if n.startswith('shared_')}
    return y.detach(), xx.grad, g
if W == 1:
    layer = build(2)
    torch.save(layer.state_dict(), path + '/full.ckpt')
    torch.save(run(layer), path + '/out.pt')
else:
    layer = build(1)
    layer.load_state_dict(torch.load(path + '/%d-of-2.ckpt' % r))
    y, dx, g = run(layer)
    y0, dx0, g0 = torch.load(path + '/out.pt')
    assert torch.allclose(y, y0, rtol=1e-12, atol=1e-12), (y - y0).abs().max()
    assert torch.allclose(dx, dx0, rtol=1e-12, atol=1e-12), (dx - dx0).abs().max()
    assert g.keys() == g0.keys() and len(g) == (5 if gated else 4)
    for n in g:
        assert torch.allclose(g[n], g0[n], rtol=1e-12, atol=1e-12), n
    if r == 0:
        print('SHARED_OK')
'''


@pytest.mark.parametrize('gated', [False, True])
def test_two_gloo_ranks_equal_one_rank(tmp_path, gated):
    env = {'CKPT_DIR': str(tmp_path), 'GATED': '1' if gated else '0'}
    run_workers(GLOO, nproc=1, env=env)
    from tutel_b200.checkpoint import scatter
    scatter.main(['--input', str(tmp_path / 'full.ckpt'), '--output_size', '2', '--outputs',
                  str(tmp_path / '{rank}-of-{size}.ckpt')])
    out = run_workers(GLOO, nproc=2, env=env)
    assert 'SHARED_OK' in out
