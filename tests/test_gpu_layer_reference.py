"""Whole training steps of ``MOELayer`` on one GPU against the fp64 reference of tests/layer_reference.py.

Each case runs real steps (forward, loss, backward, SGD) of a layer, eagerly or replayed from a ``GraphedTrainStep``,
records what the layer routed with and returned, and checks the routing decision, ``y``, ``l_aux``, ``dlogits``,
``dx`` and every parameter gradient against the reference under its per-element bound.  A second step after the SGD
update is checked at the updated parameters (stale fp8 / MX weight copies, stale cached state).  Steps whose loss is
``l_aux`` alone check the gate path on its own.  The cases cover the configuration ``bench.py`` times, the gates, the
capacity rules, the expert kinds, shared experts, dtypes and ``a2a_ffn_overlap_degree=2``; see the module docstring of
tests/layer_reference.py for what is out of scope.
"""
import copy
import json
import os

import pytest
import torch
import torch.nn.functional as F

import layer_reference as LR

pytestmark = pytest.mark.gpu

ACTS = {'relu': lambda t: F.relu(t), 'gelu': F.gelu, 'silu': F.silu}
WORST = {}


@pytest.fixture(scope='module', autouse=True)
def report():
    yield
    out = os.environ.get('LAYER_REFERENCE_REPORT')
    text = json.dumps(WORST, indent=1, sort_keys=True)
    print('\nlargest err / bound per case and output:\n' + text)
    if out:
        with open(out, 'w') as f:
            f.write(text)


def make_layer(expert='ffn', act='relu', E=8, k=2, cf=1.0, dtype=torch.bfloat16, M=256, H=512, fp32_gate=False,
               gate='softmax', normalize=True, postscore=True, shared=None, fp8=None, biases=True, bpr=False, overlap=1,
               seed=1):
    from tutel_b200 import moe
    spec = {'type': 'top', 'k': k, 'fp32_gate': fp32_gate, 'capacity_factor': cf}
    if gate == 'sigmoid':
        spec.update(scoring_func='sigmoid', n_group=4, topk_group=2, routed_scaling_factor=2.5)
    if expert == 'llama_ffn':
        experts = {'type': 'llama_ffn', 'num_experts_per_device': E, 'hidden_size_per_expert': H}
    else:
        experts = {'type': 'ffn', 'num_experts_per_device': E, 'hidden_size_per_expert': H, 'activation_fn': ACTS[act]}
        if not biases:
            experts.update(has_fc1_bias=False, has_fc2_bias=False)
    if fp8:
        experts['fp8'] = fp8
    layer = moe.moe_layer(gate_type=spec, model_dim=M, experts=experts, seeds=(seed, seed + 1, seed + 2),
                          is_postscore=postscore, normalize_gate=normalize, batch_prioritized_routing=bpr,
                          a2a_ffn_overlap_degree=overlap, shared_experts=shared).cuda().to(dtype)
    if gate == 'sigmoid':
        with torch.no_grad():
            layer.gates[0].e_score_correction_bias.copy_(torch.linspace(-0.05, 0.05, E))
    if expert == 'llama_ffn':
        with torch.no_grad():          # unit-scale hidden activations (the default init gives ~1e-4)
            for n, p in layer.named_parameters():
                if 'W_fc' in n:
                    p.normal_(0, M ** -0.5 if 'fc3' not in n else H ** -0.5)
    return layer


def bench_loss(y, t):
    return F.nll_loss(F.log_softmax(torch.sum(y, dim=2), dim=1), t)


def mixed_loss(y, t):
    w = torch.linspace(-1, 1, y.size(-1), device=y.device, dtype=torch.float32)
    return (y.float() * w).sum() / y.size(0) + 0.5 * y.l_aux.float()


def aux_loss(y, t):
    return 3.0 * y.l_aux.float()


def run_steps(layer, x, t, loss_fn, steps=1, graphed=False, lr=0.0, **fwd):
    """Steps of zero_grad + forward + loss + backward + SGD; returns one layer_reference.Step per step."""
    from tutel_b200.utils.graph import GraphedTrainStep
    opt = torch.optim.SGD(layer.parameters(), lr=lr)

    def step_fn(xx, tt):
        opt.zero_grad(set_to_none=True)
        xx.grad = None
        loss = loss_fn(layer(xx, **fwd), tt)
        loss.backward()
        opt.step()
        return loss

    out = []
    with LR.recording(layer) as recs:
        if graphed:
            g = GraphedTrainStep(step_fn, x, t, warmup=2)
            gx = g.static_inputs[0]
            for _ in range(steps):
                params = LR.snapshot(layer)
                g(x, t)
                torch.cuda.synchronize()
                out.append(LR.make_step(layer, recs[-1], gx, params, gx.grad))
        else:
            for _ in range(steps):
                params = LR.snapshot(layer)
                xx = x.detach().clone().requires_grad_(True)
                step_fn(xx, t)
                torch.cuda.synchronize()
                out.append(LR.make_step(layer, recs[-1], xx, params, xx.grad))
    return out


def check(name, layer, x, steps, capacity_factor=None, top_k=None, overlap=None, autograd=True):
    worst = {}
    for i, st in enumerate(steps):
        cfg = LR.config_of(layer, x, capacity_factor, top_k, overlap)
        ref = LR.reference(cfg, st)
        if autograd and i == 0:
            LR.autograd_check(cfg, st, ref)
        for key, v in LR.check_step(cfg, st, ref).items():
            worst[key] = max(worst.get(key, 0.0), v)
        check_gate_kernel(cfg, st)
    WORST[name] = worst
    return worst


def check_gate_kernel(cfg, st):
    """The gate kernels' own checkers on the logits the layer routed with: their ids and counts must be the layer's, bit
    for bit, and so must their locations unless the layer queued by confidence (batch-prioritised routing, which the
    sigmoid gate then runs in torch: same selection rule, fp32 as well)."""
    if cfg.gate_path != 'fused':
        return
    from tutel_b200.ops import backend
    import dispatch_reference as DR
    import sigmoid_gate_reference as SR
    ext = backend.require_ext()
    lg = st.logits.contiguous()
    C = st.capacity or 0
    eps = float(torch.finfo(lg.dtype).eps)
    if cfg.scoring == 'softmax':
        outs = ext.gate_route_forward(lg, cfg.k, C, cfg.normalize, eps)
        DR.check_gate_route_forward('layer logits', lg, cfg.k, C, cfg.normalize, eps, outs)
    else:
        outs = ext.sigmoid_gate_route_forward(lg, st.bias, cfg.k, C, cfg.normalize, eps, cfg.n_group, cfg.topk_group,
                                              cfg.scale, None)
        SR.check_forward('layer logits', lg, st.bias, cfg.k, C, cfg.normalize, eps, cfg.n_group, cfg.topk_group,
                         cfg.scale, outs)
    assert torch.equal(outs[1], st.idx) and torch.equal(outs[5], st.counts)
    assert cfg.bpr or torch.equal(outs[4], st.loc)


def _data(S, M, dtype, batch=2, seed=0):
    g = torch.Generator(device='cuda').manual_seed(seed)
    x = torch.randn(batch, S // batch, M, device='cuda', generator=g).to(dtype)
    t = torch.zeros(batch, dtype=torch.long, device='cuda')
    return x.requires_grad_(True), t


# ---------------------------------------------------------------------------------------------------------- bench
@pytest.mark.parametrize('graphed', [False, True], ids=['eager', 'graphed'])
def test_bench_configuration(graphed):
    """bench.py's layer: ffn with a lambda ReLU, top-2 of 8, capacity factor 1 (drops), bf16 logits, its loss; two steps
    with an SGD update in between."""
    torch.manual_seed(0)
    layer = make_layer()
    x, t = _data(512, 256, torch.bfloat16)
    steps = run_steps(layer, x, t, bench_loss, steps=2, graphed=graphed, lr=0.5)
    assert any((s.loc >= s.capacity).any() for s in steps), 'no choice was dropped'
    check('bench ' + ('graphed' if graphed else 'eager'), layer, x, steps)


def test_bench_configuration_full_size():
    """The bench layer at model_dim 4096 / hidden 14336 on fewer tokens; the reference runs one expert at a time."""
    torch.manual_seed(0)
    layer = make_layer(M=4096, H=14336)
    x, t = _data(512, 4096, torch.bfloat16)
    steps = run_steps(layer, x, t, bench_loss)
    check('bench full size', layer, x, steps, autograd=False)


# ---------------------------------------------------------------------------------------------------------- gates
GATE_CASES = {
    'fused k1': dict(k=1),
    'fused k8': dict(k=8, cf=0.75),
    'fused unnormalised': dict(normalize=False),
    'fused prescore': dict(postscore=False),
    'fused fp32_gate': dict(fp32_gate=True),
    'batch prioritised': dict(bpr=True, cf=0.5),
    'sigmoid groups': dict(gate='sigmoid', E=16, k=3),
    'sigmoid prescore unnormalised': dict(gate='sigmoid', E=16, k=3, postscore=False, normalize=False),
    'sigmoid batch prioritised (torch gate)': dict(gate='sigmoid', E=16, k=3, bpr=True, cf=0.5),
}


@pytest.mark.parametrize('case', list(GATE_CASES))
def test_gates(case):
    torch.manual_seed(0)
    layer = make_layer(**GATE_CASES[case])
    x, t = _data(384, 256, torch.bfloat16)
    check('gate: ' + case, layer, x, run_steps(layer, x, t, mixed_loss))
    # the gate path alone: dlogits, wg.grad and dx of an l_aux-only loss
    check('gate: %s, l_aux only' % case, layer, x, run_steps(layer, x, t, aux_loss))


@pytest.mark.parametrize('case', ['op-by-op softmax', 'op-by-op softmax, batch prioritised'])
def test_op_by_op_gate(case, monkeypatch):
    monkeypatch.setenv('TUTEL_B200_FUSED_GATE', '0' if 'prioritised' not in case else '1')
    torch.manual_seed(0)
    layer = make_layer(bpr='prioritised' in case, cf=0.5)
    x, t = _data(384, 256, torch.bfloat16)
    check(case, layer, x, run_steps(layer, x, t, mixed_loss))
    check(case + ', l_aux only', layer, x, run_steps(layer, x, t, aux_loss))


# ---------------------------------------------------------------------------------------------------------- capacity
CAP_CASES = {
    'cf 0.5': dict(cf=0.5),
    'dropless packed ffn': dict(cf=0),
    'dropless packed llama_ffn': dict(cf=0, expert='llama_ffn'),
    'dropless fp32 (padded, host read)': dict(cf=0, dtype=torch.float32),
    'cf -0.5': dict(cf=-0.5),
    'S 300': dict(S=300),
    'S 1': dict(S=1, batch=1),
}


@pytest.mark.parametrize('case', list(CAP_CASES))
def test_capacity(case):
    opts = dict(CAP_CASES[case])
    S, batch = opts.pop('S', 384), opts.pop('batch', 2)
    dtype = opts.get('dtype', torch.bfloat16)
    torch.manual_seed(0)
    layer = make_layer(**opts)
    x, t = _data(S, 256, dtype, batch=batch)
    steps = run_steps(layer, x, t, mixed_loss)
    if opts.get('cf') == 0 and dtype != torch.float32:
        assert steps[0].layout is not None, 'the dropless step did not take the packed layout'
    check('capacity: ' + case, layer, x, steps)


# ---------------------------------------------------------------------------------------------------------- experts
EXPERT_CASES = {
    'ffn gelu': dict(act='gelu'),
    'ffn silu': dict(act='silu'),
    'ffn no biases': dict(biases=False),
    'llama_ffn': dict(expert='llama_ffn'),
    'ffn fp8 row': dict(fp8='row'),
    'llama_ffn fp8 row': dict(expert='llama_ffn', fp8='row'),
    'ffn fp8 mx': dict(fp8='mx'),
    'ffn fp16': dict(dtype=torch.float16),
    'ffn fp32': dict(dtype=torch.float32),
    'shared': dict(shared={'num_experts': 2}),
    'shared gated': dict(shared={'num_experts': 2, 'gate': True}),
    'shared gated llama_ffn prescore': dict(shared={'num_experts': 1, 'gate': True}, expert='llama_ffn',
                                            postscore=False),
}


@pytest.mark.parametrize('case', list(EXPERT_CASES))
def test_experts(case):
    opts = dict(EXPERT_CASES[case])
    dtype = opts.get('dtype', torch.bfloat16)
    torch.manual_seed(0)
    layer = make_layer(**opts)
    x, t = _data(384, 256, dtype)
    check('experts: ' + case, layer, x, run_steps(layer, x, t, mixed_loss))
    if 'shared gated' in case:
        check('experts: %s, l_aux only' % case, layer, x, run_steps(layer, x, t, aux_loss))


# ---------------------------------------------------------------------------------------------------------- two steps
TWO_STEP_CASES = {
    'fp8 row': dict(fp8='row'),
    'fp8 mx': dict(fp8='mx'),
    'llama_ffn fp8 row': dict(expert='llama_ffn', fp8='row'),
    'dropless packed': dict(cf=0),
    'shared gated': dict(shared={'num_experts': 2, 'gate': True}),
}


EXPERT_WEIGHTS = ('experts.', 'shared_experts.')


@pytest.mark.parametrize('graphed', [False, True], ids=['eager', 'graphed'])
@pytest.mark.parametrize('case', list(TWO_STEP_CASES))
def test_two_steps(case, graphed):
    """Step 2 runs at the parameters the SGD update of step 1 produced.  It is checked against the reference at those
    parameters, and bit for bit against a fresh layer loaded with them and run the same way (eager or graphed): a
    step 2 that used expert weight copies (e4m3, MX) made before the update differs from the fresh layer's.  The e4m3
    bound is wider than the update, so the reference alone cannot see stale fp8 copies; for 16-bit experts it can, and
    step 2 against the reference with only the expert weights left at their step-1 values must fail."""
    opts = TWO_STEP_CASES[case]
    torch.manual_seed(0)
    layer = make_layer(**opts)
    x, t = _data(384, 256, torch.bfloat16)
    steps = run_steps(layer, x, t, mixed_loss, steps=2, graphed=graphed, lr=1e-3)
    check('two steps: %s %s' % (case, 'graphed' if graphed else 'eager'), layer, x, steps)
    fresh = make_layer(**opts)
    with torch.no_grad():
        for n, p in fresh.named_parameters():
            p.copy_(steps[1].params[n])
    again = run_steps(fresh, x, t, mixed_loss, graphed=graphed)[0]
    for what in ('logits', 'y', 'l_aux', 'dlogits', 'dx'):
        assert torch.equal(getattr(steps[1], what), getattr(again, what)), what
    for n, g in steps[1].grads.items():
        if 'bias' not in n:           # (bias gradients are fp32 atomic sums: checked against the reference above)
            assert torch.equal(g, again.grads[n]), n
    if not opts.get('fp8'):
        params = {n: (steps[0].params[n] if n.startswith(EXPERT_WEIGHTS) else p) for n, p in steps[1].params.items()}
        with pytest.raises(AssertionError) as ex:
            LR.check_step(LR.config_of(layer, x), LR.Step(**{**steps[1].__dict__, 'params': params}))
        assert any(line.startswith('y:') for line in str(ex.value).splitlines()), str(ex.value)[:2000]


def test_fp8_row_quantisation_of_tiny_rows():
    """Rows whose largest magnitude is below 448 * 2^-126 (a near-zero gate times dy, in the fp8 dgrad) get the
    smallest normal scale: 1 / scale overflowed before, and the row's zeros came out as 0 * inf = NaN."""
    from tutel_b200.ops import gemm as G
    import expert_ffn_reference as ER
    x = torch.zeros(4, 64, device='cuda', dtype=torch.bfloat16)
    x[0, :8] = torch.linspace(-1, 1, 8) * 1e-38
    x[1, 3] = 2e-40
    x[2] = torch.randn(64)
    q, sc = G.quantize_rows(x)
    assert not bool(torch.isnan(q.view(torch.float8_e4m3fn).float()).any())
    wq, ws = ER.quantize_rows_reference(x)
    assert torch.equal(sc.reshape(-1), ws.reshape(-1)) and torch.equal(q.view(torch.uint8), wq.view(torch.uint8))


# ---------------------------------------------------------------------------------------------------------- overlap
@pytest.mark.parametrize('cf', [1.0, 0.7], ids=['same capacity', 'aligned capacity'])
def test_overlap_degree_2(cf):
    """a2a_ffn_overlap_degree=2 on one GPU: the capacity is aligned to 2; where it equals the degree-1 capacity the
    step is also bitwise equal to degree 1 (parallel/overlap.py)."""
    torch.manual_seed(0)
    layer = make_layer(cf=cf, E=8)
    twin = copy.deepcopy(layer)
    # cf 1, top-2: capacity 2 * 46 = 92 at both degrees;  cf 0.7, top-1: int(0.7 * 25) = 17, aligned to 18 at degree 2
    S, k = (8 * 46, 2) if cf == 1.0 else (8 * 25, 1)
    x, t = _data(S, 256, torch.bfloat16, batch=1)
    s2 = run_steps(layer, x, t, mixed_loss, a2a_ffn_overlap_degree=2, top_k=k)
    s1 = run_steps(twin, x, t, mixed_loss, a2a_ffn_overlap_degree=1, top_k=k)
    check('overlap 2: cf %s' % cf, layer, x, s2, top_k=k, overlap=2)
    if s1[0].capacity == s2[0].capacity:
        assert cf == 1.0
        assert torch.equal(s1[0].y, s2[0].y) and torch.equal(s1[0].dx, s2[0].dx)
        for n, g in s1[0].grads.items():
            assert torch.equal(g, s2[0].grads[n]), n
    else:
        assert cf == 0.7 and s2[0].capacity == s1[0].capacity + 1
