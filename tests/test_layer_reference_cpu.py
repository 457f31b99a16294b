"""The layer reference of tests/layer_reference.py on CPU: a faithful emulation of the GPU step passes every check,
and near misses of the layer's wiring each fail the check that guards them.

The emulation is fp32 autograd of the layer's documented step with the GPU path's 16-bit stores: ``Store`` rounds a
tensor to bf16 in forward and the gradient reaching it in backward (logits / dlogits, hidden activations / dh, expert
output / encoded gradient rows, the shared-gate logit / its gradient), then ``y``, ``dx`` and every parameter gradient
are rounded.  Its expert buffer is ``[E, C, M]`` with C from the capacity rule, read back at ``e * C + loc``.
"""
import pytest
import torch
import torch.nn.functional as F

import layer_reference as LR

DT = torch.bfloat16


class Store(torch.autograd.Function):
    @staticmethod
    def forward(ctx, t):
        return t.to(DT).float()

    @staticmethod
    def backward(ctx, g):
        return g.to(DT).float()


class SoftmaxNoJacobian(torch.autograd.Function):
    """softmax whose backward forgets the Jacobian (near miss 7)."""
    @staticmethod
    def forward(ctx, z):
        return torch.softmax(z, 1)

    @staticmethod
    def backward(ctx, g):
        return g


class SigmoidNoSlope(torch.autograd.Function):
    """sigmoid whose backward forgets w (1 - w) (near miss 8)."""
    @staticmethod
    def forward(ctx, z):
        return torch.sigmoid(z)

    @staticmethod
    def backward(ctx, g):
        return g


def make_params(E=4, M=32, H=48, shared=True, seed=0):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s, sc=1.0: (torch.randn(*s, generator=g) * sc).to(DT)     # noqa: E731
    P = {'gates.0.wg.weight': r(E, M, sc=0.3),
         'experts.batched_fc1_w': r(E, H, M, sc=M ** -0.5), 'experts.batched_fc1_bias': r(E, H, sc=0.1),
         'experts.batched_fc2_w': r(E, H, M, sc=H ** -0.5), 'experts.batched_fc2_bias': r(E, M, sc=0.1)}
    if shared:
        P.update({'shared_experts.batched_fc1_w': r(1, 2 * H, M, sc=M ** -0.5),
                  'shared_experts.batched_fc1_bias': r(1, 2 * H, sc=0.1),
                  'shared_experts.batched_fc2_w': r(1, 2 * H, M, sc=(2 * H) ** -0.5),
                  'shared_experts.batched_fc2_bias': r(1, M, sc=0.1),
                  'shared_expert_gate.weight': r(1, M, sc=0.3)})
    return P


def config(**kw):
    c = dict(E=4, k=2, dtype=DT, logit_dtype=DT, cf=0.6, alignment=1, shared=True, shared_gated=True)
    c.update(kw)
    return LR.Config(**c)


def emulate(cfg, x, P, dy, dl, miss=None, stale=None):
    """One step of the GPU path in fp32 with bf16 stores; ``miss`` selects a near miss; ``stale``: parameters the
    step really ran on (the Step still reports ``P``)."""
    Q = {n: t.float().requires_grad_(True) for n, t in (stale or P).items()}
    xx = x.float().requires_grad_(True)
    S, M = x.shape
    E, k = cfg.E, cfg.k
    z = Store.apply((xx.detach() if miss == 'no gate term in dx' else xx) @ Q['gates.0.wg.weight'].t())
    z.retain_grad()
    p = SoftmaxNoJacobian.apply(z) if miss == 'wg grad before softmax jacobian' else torch.softmax(z, 1)
    ids = torch.sort(p.detach(), dim=1, descending=True, stable=True).indices[:, :k].t().contiguous()          # [k, S]
    r = p.t().gather(0, ids)
    g = r / r.sum(0, keepdim=True).clamp_min(torch.finfo(DT).eps) if cfg.normalize and k > 1 else r
    ce = torch.bincount(ids[0], minlength=E).float()
    l_aux = (p.sum(0) * ce).sum() * E / (S * S)
    if miss == 'l_aux grad x k':
        l_aux = l_aux + (k - 1) * (l_aux - l_aux.detach())
    if miss == 'l_aux grad missing':
        l_aux = l_aux.detach()
    onehot = F.one_hot(ids.reshape(-1), E)
    loc = ((onehot.cumsum(0) - 1) * onehot).sum(1).view(k, S)
    counts = onehot.sum(0)
    C = LR.capacity_rule(S, E, k, cfg.cf, counts, cfg.alignment)
    kept = loc < C
    buf = torch.zeros(E, C, M)
    jj, ss = kept.nonzero(as_tuple=True)
    rows = xx[ss] if cfg.postscore else Store.apply(xx[ss] * g[jj, ss][:, None])
    buf = buf.index_put((ids[jj, ss], loc[jj, ss]), rows)
    h = Store.apply(torch.relu(buf @ Q['experts.batched_fc1_w'].transpose(1, 2) + Q['experts.batched_fc1_bias'][:, None]))
    o = Store.apply(h @ Q['experts.batched_fc2_w'] + Q['experts.batched_fc2_bias'][:, None]).reshape(E * C, M)
    stride = C - 1 if miss == 'neighbour slots' else C
    y = torch.zeros(S, M)
    for j in range(k):
        m = kept[j] if miss != 'dropped choice in y' else torch.ones_like(kept[j])
        row = (ids[j] * stride + loc[j].clamp(max=C - 1)).clamp(max=E * C - 1)
        oj = o[row]
        if miss == 'dropped choice in y':        # the dropped choice's expert output, as if it had a slot
            xj = xx
            hj = Store.apply(torch.relu(torch.einsum('sm,shm->sh', xj, Q['experts.batched_fc1_w'][ids[j]]) +
                                        Q['experts.batched_fc1_bias'][ids[j]]))
            oj = torch.where(kept[j][:, None], oj, Store.apply(torch.einsum('sh,shm->sm', hj, Q['experts.batched_fc2_w'][ids[j]]) +
                                                               Q['experts.batched_fc2_bias'][ids[j]]))
        if cfg.postscore:
            gj = r[j] if miss == 'unnormalised gates' else g[j]
            y = y + (gj[:, None] * oj) * m[:, None]
        else:
            y = y + oj * m[:, None] * (g[j][:, None] if miss == 'prescore gate twice' else 1.0)
        if miss == 'dropped choice in gate grad':
            oe = Store.apply(torch.relu(torch.einsum('sm,shm->sh', xx, Q['experts.batched_fc1_w'][ids[j]]) +
                                        Q['experts.batched_fc1_bias'][ids[j]]))
            oe = torch.einsum('sh,shm->sm', oe, Q['experts.batched_fc2_w'][ids[j]]) + Q['experts.batched_fc2_bias'][ids[j]]
            y = y + ((g[j] - g[j].detach())[:, None] * oe.detach()) * (~kept[j])[:, None]
    if cfg.shared:
        hs = Store.apply(torch.relu(xx @ Q['shared_experts.batched_fc1_w'][0].t() + Q['shared_experts.batched_fc1_bias'][0]))
        base = Store.apply(hs @ Q['shared_experts.batched_fc2_w'][0] + Q['shared_experts.batched_fc2_bias'][0])
        if cfg.shared_gated:
            sl = Store.apply(xx @ Q['shared_expert_gate.weight'].t())
            w = SigmoidNoSlope.apply(sl) if miss == 'shared gate without w(1-w)' else torch.sigmoid(sl)
            base = base * w
        y = y + base
    y = Store.apply(y)
    l_out = l_aux.to(DT)
    loss = (y * dy.float()).sum() + dl * l_aux
    loss.backward()
    grads = {n: Q[n].grad.to(DT) if Q[n].grad is not None else None for n in Q}
    return LR.Step(x=x, params=P, logits=z.detach().to(DT), idx=ids.int(), loc=loc.int(), counts=counts.int(),
                   capacity=C, y=y.detach().to(DT), l_aux=l_out.detach(), dy=dy, dl=dl,
                   dlogits=z.grad.to(DT), dx=xx.grad.to(DT), grads=grads)


def _case(S=96, seed=0, dl=0.7, only_aux=False, **kw):
    cfg = config(**kw)
    P = make_params(shared=cfg.shared, seed=seed)
    g = torch.Generator().manual_seed(seed + 1)
    x = torch.randn(S, 32, generator=g).to(DT)
    dy = (torch.randn(S, 32, generator=g) * 0.1).to(DT)
    if only_aux:
        dy = torch.zeros_like(dy)
    return cfg, P, x, dy, dl


@pytest.mark.parametrize('kw', [dict(), dict(postscore=False), dict(k=1), dict(normalize=False), dict(cf=0.3),
                                dict(cf=0.6, alignment=3), dict(shared_gated=False), dict(shared=False, shared_gated=False)],
                         ids=['default', 'prescore', 'k1', 'unnormalised', 'cf0.3', 'aligned', 'shared', 'no shared'])
def test_emulation_passes(kw):
    cfg, P, x, dy, dl = _case(**kw)
    st = emulate(cfg, x, P, dy, dl)
    ref = LR.reference(cfg, st)
    LR.autograd_check(cfg, st, ref)
    worst = LR.check_step(cfg, st, ref)
    assert worst['y'] > 1e-3            # the bound is not vacuous
    st = emulate(cfg, x, P, torch.zeros_like(dy), 2.0)
    LR.check_step(cfg, st)


NEAR_MISSES = [
    ('unnormalised gates', {}, 'y'),
    ('dropped choice in y', dict(cf=0.3), 'y'),
    ('dropped choice in gate grad', dict(cf=0.3), 'dlogits'),
    ('no gate term in dx', dict(only_aux=True, dl=3.0), 'dx'),
    ('l_aux grad x k', dict(only_aux=True, dl=3.0), 'dlogits'),
    ('l_aux grad missing', dict(only_aux=True, dl=3.0), 'dlogits'),
    ('prescore gate twice', dict(postscore=False), 'y'),
    ('neighbour slots', dict(alignment=3), 'y'),
    ('wg grad before softmax jacobian', {}, 'gates.0.wg.weight'),
    ('shared gate without w(1-w)', {}, 'shared_expert_gate.weight'),
]


@pytest.mark.parametrize('miss,kw,guard', NEAR_MISSES, ids=[m[0] for m in NEAR_MISSES])
def test_near_miss_fails(miss, kw, guard):
    cfg, P, x, dy, dl = _case(**kw)
    LR.check_step(cfg, emulate(cfg, x, P, dy, dl))
    with pytest.raises(AssertionError) as ex:
        LR.check_step(cfg, emulate(cfg, x, P, dy, dl, miss=miss))
    assert any(line.startswith(guard + ':') for line in str(ex.value).splitlines()), str(ex.value)[:2000]


def test_near_miss_stale_second_step():
    """Step 2 computed with the expert weights from before the SGD update (stale copies of them; the gate weight is
    current, so the decision check passes and the outputs must catch it)."""
    cfg, P, x, dy, dl = _case()
    st1 = emulate(cfg, x, P, dy, dl)
    P2 = {n: (P[n].float() - 0.05 * st1.grads[n].float()).to(DT) for n in P}
    LR.check_step(cfg, emulate(cfg, x, P2, dy, dl))
    stale = {n: (P[n] if n.startswith(('experts.', 'shared_experts.')) else P2[n]) for n in P}
    with pytest.raises(AssertionError) as ex:
        LR.check_step(cfg, emulate(cfg, x, P2, dy, dl, stale=stale))
    assert any(line.startswith('y:') for line in str(ex.value).splitlines()), str(ex.value)[:2000]


# ------------------------------------------------------------------------------------------------------------------
# the real layer on CPU, through the capture path
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('dtype,variant', [(torch.float32, 'ffn shared gated'), (torch.bfloat16, 'ffn shared gated'),
                                           (torch.float32, 'llama_ffn prescore'), (torch.bfloat16, 'llama_ffn prescore'),
                                           (torch.float32, 'sigmoid'), (torch.float32, 'sigmoid batch prioritised')])
def test_cpu_layer_through_capture(dtype, variant):
    """The capture, decision check and reference on the layer's CPU path.  The CPU experts run torch.matmul and round
    before adding the bias, which the reference (modelling the GPU kernels) does not charge: bf16 with the sigmoid gate
    exceeds the fc2 weight-gradient bound there, so that pair runs in fp32 only."""
    from tutel_b200 import moe
    torch.manual_seed(0)
    spec = {'type': 'top', 'k': 2, 'capacity_factor': 0.5}
    kw = {}
    if variant == 'sigmoid batch prioritised':
        kw['batch_prioritized_routing'] = True
    if variant.startswith('sigmoid'):
        spec.update(scoring_func='sigmoid', n_group=2, topk_group=1, routed_scaling_factor=2.0, k=3)
        spec['capacity_factor'] = 0.8
    experts = {'type': 'ffn', 'num_experts_per_device': 4, 'hidden_size_per_expert': 96,
               'activation_fn': lambda t: F.relu(t)}
    if variant == 'llama_ffn prescore':
        experts = {'type': 'llama_ffn', 'num_experts_per_device': 4, 'hidden_size_per_expert': 96}
        kw['is_postscore'] = False
    if variant == 'ffn shared gated':
        kw['shared_experts'] = {'num_experts': 2, 'gate': True}
    E = 8 if variant.startswith('sigmoid') else 4
    experts['num_experts_per_device'] = E
    layer = moe.moe_layer(gate_type=spec, model_dim=64, experts=experts, seeds=(1, 2, 3), **kw).to(dtype)
    if variant == 'llama_ffn prescore':
        with torch.no_grad():
            for n, p in layer.named_parameters():
                if 'W_fc' in n:
                    p.normal_(0, 0.125)
    if variant.startswith('sigmoid'):
        with torch.no_grad():
            layer.gates[0].e_score_correction_bias.copy_(torch.linspace(-0.05, 0.05, E))
    x = torch.randn(40, 64).to(dtype).requires_grad_(True)
    params = LR.snapshot(layer)
    with LR.recording(layer) as recs:
        y = layer(x)
        (-F.log_softmax(y.float().sum(1), 0)[0] + 0.3 * y.l_aux.float()).backward()
    st = LR.make_step(layer, recs[-1], x, params, x.grad)
    cfg = LR.config_of(layer, x)
    ref = LR.reference(cfg, st)
    LR.autograd_check(cfg, st, ref)
    LR.check_step(cfg, st, ref)


def test_every_gradient_needs_a_reference():
    """A parameter gradient the reference does not model, or a missing gate gradient, fails instead of being skipped."""
    cfg, P, x, dy, dl = _case()
    st = emulate(cfg, x, P, dy, dl)
    extra = LR.Step(**{**st.__dict__, 'grads': {**st.grads, 'experts.new_w': torch.zeros(3, dtype=DT)}})
    with pytest.raises(AssertionError, match='experts.new_w: a gradient the reference does not model'):
        LR.check_step(cfg, extra)
    with pytest.raises(AssertionError, match='dlogits: no gradient'):
        LR.check_step(cfg, LR.Step(**{**st.__dict__, 'dlogits': None}))
