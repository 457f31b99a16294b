"""Shared experts on the GPU: the combine kernels with the shared term against tests/shared_expert_reference.py, the
layer's combine against the fp64 composition of what its experts produced, packed dropless training against the padded
path (bitwise), no host synchronisation, CUDA-graph replay, the skinny decoding path and launch counts."""
import pytest
import torch
import torch.nn.functional as F

import shared_expert_reference as R
from dispatch_reference import INVALID_LOC, ref_locations

pytestmark = pytest.mark.gpu

DTYPES = {'bf16': torch.bfloat16, 'fp16': torch.float16, 'fp32': torch.float32}


def _ext():
    from tutel_b200.ops import backend
    return backend.require_ext()


# ------------------------------------------------------------------------------------------------------------------
# kernels
# ------------------------------------------------------------------------------------------------------------------
def _routing(S, k, E, C, seed, packed):
    """idx / loc [k, S] with dropped choices (padded: past C) and fully dropped tokens; packed: seg_off and R."""
    g = torch.Generator().manual_seed(seed)
    idx = torch.randint(0, E, (k, S), generator=g, dtype=torch.int32)
    loc, counts = ref_locations(idx, E)[:2]
    drop = torch.rand(k, S, generator=g) < 0.1
    loc = torch.where(drop, torch.full_like(loc, INVALID_LOC), loc)
    loc[:, : min(3, S)] = INVALID_LOC                               # tokens whose choices were all dropped
    seg_off = None
    if packed:
        rounded = (counts + 127) // 128 * 128
        seg = torch.zeros(E + 1, dtype=torch.int32)
        seg[1:] = torch.cumsum(rounded, 0)
        seg_off = seg.cuda()
        C = (k * S + 127) // 128 * 128 + 128 * E                   # packed rows R
    return idx.cuda(), loc.cuda(), C, seg_off


KERNEL_CASES = [(dt, M, packed, gated, k) for dt in DTYPES for M in (256, 203) for packed in (False, True)
                for gated in (False, True) for k in (1, 4, 16)]


@pytest.mark.parametrize('dt,M,packed,gated,k', KERNEL_CASES,
                         ids=['%s-M%d-%s-%s-k%d' % (c[0], c[1], 'packed' if c[2] else 'padded', 'gated' if c[3] else 'w1',
                                                    c[4]) for c in KERNEL_CASES])
def test_kernels_against_reference(dt, M, packed, gated, k):
    dtype = DTYPES[dt]
    S, E = 300, 8
    C = max(1, k * S // E * 3 // 4)                                # capacity binds: choices past C are dropped
    idx, loc, C, seg_off = _routing(S, k, E, C, 1000 + k, packed)
    g = torch.Generator(device='cuda').manual_seed(k)
    rows = C if packed else E * C
    buf = torch.randn(rows, M, device='cuda', generator=g).to(dtype)
    gates = torch.rand(k, S, device='cuda', generator=g)
    base = (torch.randn(S, M, device='cuda', generator=g) * 0.5).to(dtype)
    logit = (torch.randn(S, device='cuda', generator=g) * 3) if gated else None
    dy = torch.randn(S, M, device='cuda', generator=g).to(dtype)
    ext = _ext()
    for gv in (gates, None):                                       # routed gates after (post-score) / before the experts
        out = ext.decode_rows(buf, gv, idx, loc, E, C, 0, 0, seg_off, base, logit)
        R.check_decode_shared('%s M=%d k=%d' % (dt, M, k), out.cpu(), buf.cpu(), None if gv is None else gv.cpu(),
                              idx.cpu(), loc.cpu(), E, C, base.cpu(), None if logit is None else logit.cpu(),
                              None if seg_off is None else seg_off.cpu())
    if not gated:
        return
    dg, d_base, d_logit = ext.gate_grad(dy, buf, idx, loc, E, C, seg_off, base, logit)
    R.check_gate_grad(dt, dg.cpu(), dy.cpu(), buf.cpu(), idx.cpu(), loc.cpu(), E, C,
                      None if seg_off is None else seg_off.cpu())
    R.check_d_base(dt, d_base.cpu(), dy.cpu(), logit.cpu())
    R.check_d_shared_logit(dt, d_logit.cpu(), dy.cpu(), base.cpu(), logit.cpu())
    assert torch.equal(dg, ext.gate_grad(dy, buf, idx, loc, E, C, seg_off)), 'routed dots changed by the shared term'
    none, d_base0, d_logit0 = ext.gate_grad(dy, None, idx[:0], loc[:0], E, C, None, base, logit)
    assert none.shape == (0, S) and torch.equal(d_base0, d_base) and torch.equal(d_logit0, d_logit)


@pytest.mark.parametrize('gated', [False, True])
def test_decode_with_empty_buffer(gated):
    """C = 0: every choice is dropped and each token gets the shared term alone."""
    S, M, E, k = 40, 64, 4, 2
    idx = torch.randint(0, E, (k, S), dtype=torch.int32, device='cuda')
    loc = torch.zeros(k, S, dtype=torch.int32, device='cuda')
    buf = torch.empty(0, M, dtype=torch.bfloat16, device='cuda')
    base = torch.randn(S, M, device='cuda').to(torch.bfloat16)
    logit = torch.randn(S, device='cuda') if gated else None
    out = _ext().decode_rows(buf, torch.rand(k, S, device='cuda'), idx, loc, E, 0, 0, 0, None, base, logit)
    R.check_decode_shared('C=0', out.cpu(), buf.cpu(), None, idx.cpu(), loc.cpu(), E, 0, base.cpu(),
                          None if logit is None else logit.cpu())
    if not gated:
        assert torch.equal(out, base)


# ------------------------------------------------------------------------------------------------------------------
# the layer
# ------------------------------------------------------------------------------------------------------------------
ACTS = {'relu': F.relu, 'gelu': F.gelu, 'silu': F.silu}


def _layer(expert, E=8, k=2, gate='softmax', dtype=torch.bfloat16, M=256, H=512, shared=2, gated=False, fp8=False,
           postscore=True, cf=None, seeds=(1, 2, 3)):
    from tutel_b200 import moe
    if expert == 'llama':
        experts = {'type': 'llama_ffn', 'num_experts_per_device': E, 'hidden_size_per_expert': H}
    else:
        experts = {'type': 'ffn', 'num_experts_per_device': E, 'hidden_size_per_expert': H, 'activation_fn': ACTS[expert]}
    if fp8:
        experts['fp8'] = True
    spec = {'type': 'top', 'k': k}
    if cf is not None:
        spec['capacity_factor'] = cf
    if gate == 'sigmoid':
        spec.update(scoring_func='sigmoid', bias_update_speed=0.001)
    se = None if shared is None else {'num_experts': shared, 'gate': gated}
    layer = moe.moe_layer(gate_type=spec, model_dim=M, experts=experts, seeds=seeds, shared_experts=se,
                          is_postscore=postscore).cuda().to(dtype)
    with torch.no_grad():
        w = layer.gates[0].wg.weight
        w.mul_(4.0)
        w[: max(E // 8, 1)] += 0.5
        if layer.shared_expert_gate is not None:
            layer.shared_expert_gate.weight.mul_(8.0)               # logits of a few units: weights away from 1/2
    return layer


LAYER_CASES = [('relu', 'softmax', True, False, False), ('gelu', 'sigmoid', True, True, False),
               ('silu', 'softmax', False, True, False), ('llama', 'sigmoid', True, False, False),
               ('llama', 'softmax', False, True, False), ('relu', 'sigmoid', True, True, True),
               ('llama', 'softmax', True, True, True), ('silu', 'sigmoid', False, False, False)]


@pytest.mark.parametrize('expert,gate,postscore,gated,fp8', LAYER_CASES,
                         ids=['%s-%s-%s-%s%s' % (c[0], c[1], 'post' if c[2] else 'pre', 'gated' if c[3] else 'w1',
                                                  '-fp8' if c[4] else '') for c in LAYER_CASES])
@pytest.mark.parametrize('cf', [1.0, 0])
def test_layer_combine_against_fp64_composition(expert, gate, postscore, gated, fp8, cf):
    from tutel_b200.ops import dispatch as D
    torch.manual_seed(0)
    layer = _layer(expert, gate=gate, postscore=postscore, gated=gated, fp8=fp8, cf=cf)
    S, M = 512, 256
    x = torch.randn(S, M, device='cuda', dtype=torch.bfloat16, requires_grad=True)
    hooked = {}
    h1 = layer.shared_experts.register_forward_hook(lambda m, i, o: hooked.__setitem__('shared', o))
    h2 = layer.experts.register_forward_hook(lambda m, i, o: hooked.__setitem__('routed', o))
    rec = {}
    orig = D.raw_decode

    def spy(buf, gates, plan, base=None, shared_logit=None):
        out = orig(buf, gates, plan, base, shared_logit)
        if base is not None:
            rec.update(buf=buf, gates=gates, plan=plan, base=base, logit=shared_logit, out=out)
        return out
    D.raw_decode = spy
    try:
        y = layer(x)
    finally:
        D.raw_decode = orig
        h1.remove()
        h2.remove()
    plan = rec['plan']
    assert torch.equal(rec['base'], hooked['shared'].reshape(S, -1))
    if 'routed' in hooked:
        assert torch.equal(rec['buf'].reshape(-1), hooked['routed'].reshape(-1))
    else:
        assert plan.layout is not None                              # the packed path calls forward_packed
    if gated:
        assert torch.equal(rec['logit'], F.linear(x.detach(), layer.shared_expert_gate.weight).view(-1))
    else:
        assert rec['logit'] is None
    assert (postscore and rec['gates'] is not None) or (not postscore and rec['gates'] is None)
    packed = plan.layout is not None
    E, C = (plan.E, plan.layout.R) if packed else (plan.E, plan.C)
    buf = rec['buf'].reshape(C if packed else E * C, -1)
    R.check_decode_shared('layer %s %s' % (expert, gate), rec['out'].cpu(), buf.cpu(),
                          None if rec['gates'] is None else rec['gates'].float().cpu(), plan.idx_ks.cpu(),
                          plan.loc_ks.cpu(), E, C, rec['base'].cpu(), None if rec['logit'] is None else rec['logit'].cpu(),
                          plan.layout.seg_off.cpu() if packed else None)
    assert torch.equal(y.detach().view(S, -1), rec['out'])
    (y.float().pow(2).mean() + 0.01 * y.l_aux.float()).backward()
    for n, p in layer.named_parameters():
        if n.startswith('shared_'):
            assert p.grad is not None and torch.isfinite(p.grad.float()).all() and bool((p.grad != 0).any()), n


def _step(layer, x, cf):
    for p in layer.parameters():
        p.grad = None
    xx = x.detach().clone().requires_grad_(True)
    y = layer(xx, capacity_factor=cf)
    loss = y.float().pow(2).mean() + 0.01 * y.l_aux.float()
    loss.backward()
    grads = {n: p.grad.clone() for n, p in layer.named_parameters() if p.grad is not None}
    return y.detach(), y.l_aux.detach(), xx.grad.clone(), grads, layer.dispatch_count.clone()


def _bias_bound(ref, dtype, rows):
    ulp = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}[dtype]
    return ulp * ref.abs().float() + (rows + 16) * 2.0 ** -24 * ref.abs().float().max() + 1e-7


PACKED_CASES = [(ex, gate, gated, post, dt) for ex, gate in (('relu', 'softmax'), ('gelu', 'sigmoid'), ('silu', 'softmax'),
                                                             ('llama', 'sigmoid'))
                for gated, post in ((False, True), (True, True), (True, False)) for dt in ('bf16',)]
PACKED_CASES += [('llama', 'softmax', True, True, 'fp16'), ('relu', 'sigmoid', True, True, 'fp16')]


@pytest.mark.parametrize('expert,gate,gated,postscore,dt', PACKED_CASES,
                         ids=['%s-%s-%s-%s-%s' % (c[0], c[1], 'gated' if c[2] else 'w1', 'post' if c[3] else 'pre', c[4])
                              for c in PACKED_CASES])
def test_packed_training_matches_padded(expert, gate, gated, postscore, dt):
    dtype = DTYPES[dt]
    E, k, S = 8, 2, 512
    torch.manual_seed(0)
    layer = _layer(expert, E=E, k=k, gate=gate, dtype=dtype, gated=gated, postscore=postscore, cf=0)
    x = torch.randn(S, 256, device='cuda', dtype=dtype)
    from tutel_b200.ops import routing
    calls = []
    orig = routing._packed_critical
    routing._packed_critical = lambda *a: calls.append(1) or orig(*a)
    try:
        y, l_aux, dx, grads, counts = _step(layer, x, None)
    finally:
        routing._packed_critical = orig
    assert calls, 'capacity_factor=0 did not take the packed path'
    y_r, l_r, dx_r, grads_r, counts_r = _step(layer, x, -E)
    assert torch.equal(counts, counts_r)
    assert torch.equal(y, y_r)
    assert torch.equal(l_aux, l_r)
    assert torch.equal(dx, dx_r)
    assert grads.keys() == grads_r.keys()
    assert any(n.startswith('shared_experts.') for n in grads) and (not gated or 'shared_expert_gate.weight' in grads)
    for n in grads:
        if 'bias' in n and 'e_score' not in n:
            bound = _bias_bound(grads_r[n], dtype, S if n.startswith('shared_') else int(counts.max()))
            assert bool(((grads[n].float() - grads_r[n].float()).abs() <= bound).all()), n
        else:
            assert torch.equal(grads[n], grads_r[n]), n


def test_no_host_sync():
    """Packed dropless training and bound-based dropless decoding of one token, with gated shared experts."""
    layer = _layer('silu', gate='sigmoid', gated=True, cf=0)
    x = torch.randn(512, 256, device='cuda', dtype=torch.bfloat16, requires_grad=True)
    _step(layer, x, None)
    with torch.no_grad():
        layer(x[:1], megablocks_size=1)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        y = layer(x)
        (y.float().pow(2).mean() + y.l_aux.float()).backward()
        with torch.no_grad():
            layer(x[:1], megablocks_size=1)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()


@pytest.mark.parametrize('expert', ['relu', 'llama'])
def test_graphed_train_step(expert):
    from tutel_b200.utils.graph import GraphedTrainStep
    torch.manual_seed(0)
    S = 512
    xs = [torch.randn(S, 256, device='cuda', dtype=torch.bfloat16) for _ in range(4)]

    def make():
        layer = _layer(expert, gate='sigmoid', gated=True, cf=0)
        opt = torch.optim.SGD(layer.parameters(), lr=0.05)

        def step(x):
            opt.zero_grad(set_to_none=True)
            y = layer(x)
            loss = y.float().pow(2).mean() + 0.01 * y.l_aux.float()
            loss.backward()
            opt.step()
            return loss.detach()
        return layer, step

    eager_layer, eager_step = make()
    eager = [eager_step(x).clone() for x in [xs[0]] * 3 + xs]
    graph_layer, graph_step = make()
    fast = GraphedTrainStep(graph_step, xs[0], warmup=3)
    graphed = [fast(x).clone() for x in xs]
    for a, b in zip(eager[3:], graphed):
        assert torch.equal(a, b)
    sd0, sd1 = eager_layer.state_dict(), graph_layer.state_dict()
    assert 'shared_expert_gate.weight' in sd1
    for n in sd0:
        assert torch.equal(sd0[n], sd1[n]), n
    g = eager_layer.shared_expert_gate.weight.grad
    assert g is not None and bool((g != 0).any()), 'the shared gate received no gradient'


@pytest.mark.parametrize('expert,fp8', [('relu', False), ('relu', True), ('llama', False), ('llama', True),
                                        ('gelu', False)])
def test_one_token_decode_takes_the_skinny_kernel(expert, fp8):
    from tutel_b200.ops import gemm as G
    layer = _layer(expert, fp8=fp8, gated=True)
    names = ['skinny_ffn', 'skinny_ffn_fp8', 'skinny_glu_ffn', 'skinny_glu_ffn_fp8']
    calls, saved = [], {n: getattr(G, n) for n in names}

    def wrap(n):
        return lambda x, *a: calls.append((n, tuple(x.shape))) or saved[n](x, *a)
    for n in names:
        setattr(G, n, wrap(n))
    x = torch.randn(1, 256, device='cuda', dtype=torch.bfloat16)
    try:
        with torch.no_grad():
            y = layer(x)
    finally:
        for n in names:
            setattr(G, n, saved[n])
    want = {('relu', True): 'skinny_ffn_fp8', ('llama', False): 'skinny_glu_ffn', ('llama', True): 'skinny_glu_ffn_fp8'}
    assert calls[0] == (want.get((expert, fp8), 'skinny_ffn'), (1, 1, 256)), calls
    assert torch.isfinite(y.float()).all()


def _ctx(layer, rows):
    from tutel_b200.models.moe_layer import _SharedExpertContext
    return _SharedExpertContext(layer, rows)


@pytest.mark.parametrize('postscore,gated,cf', [(True, False, 1.0), (True, True, 1.0), (True, True, 0), (False, True, 1.0),
                                                (False, False, 0)])
def test_launch_counts(postscore, gated, cf):
    """Shared experts add their FFN's own launches (and the torch GEMV of the shared gate, which is not one of the
    project's launches); the combine stays one launch forward and one backward - with pre-scored routing and the
    shared gate the backward runs the gate-gradient kernel with zero routed choices."""
    from tutel_b200.ops import backend
    layer = _layer('relu', gated=gated, postscore=postscore, cf=cf)
    x = torch.randn(512, 256, device='cuda', dtype=torch.bfloat16)

    def count(fn):
        fn()
        torch.cuda.synchronize()
        n0 = backend.launch_count()
        fn()
        return backend.launch_count() - n0

    def step():
        xx = x.clone().requires_grad_(True)
        y = layer(xx)
        (y.float().pow(2).mean() + 0.01 * y.l_aux.float()).backward()
    with_shared = count(step)
    se, sg = layer.shared_experts, layer.shared_expert_gate
    layer.shared_experts, layer.shared_expert_gate = None, None
    try:
        without = count(step)
    finally:
        layer.shared_experts, layer.shared_expert_gate = se, sg

    def shared_alone():
        xx = x.clone().requires_grad_(True)
        se(xx.view(1, 512, 256), _ctx(layer, None)).float().sum().backward()
    own = count(shared_alone)
    extra = 1 if (gated and not postscore) else 0
    assert with_shared == without + own + extra, (with_shared, without, own)
