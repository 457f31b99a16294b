"""Dropless training on the expert-packed layout (a gate with capacity_factor=0, one GPU) against the padded path.

The reference is the same layer run through the padded dispatch with a non-binding negative capacity factor:
``capacity_factor=-E`` caps at ``k * E * ceil(S / E) >= max(count)``, so no token is dropped and every expert GEMM
computes the same rows with the same kernel, K order and per-row math.  The forward output and the auxiliary loss are
therefore compared bitwise, and so are the input, weight and gate gradients (padded K blocks only add zero products);
bias gradients are column sums that both paths add up with fp32 atomics in a different order, and are compared under the
bound of that summation.
"""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

ACTS = {'relu': F.relu, 'gelu': F.gelu, 'silu': F.silu}


def _layer(expert, E, k, gate, dtype, M=256, H=512):
    from tutel_b200 import moe
    if expert == 'llama':
        experts = {'type': 'llama_ffn', 'num_experts_per_device': E, 'hidden_size_per_expert': H}
    else:
        experts = {'type': 'ffn', 'num_experts_per_device': E, 'hidden_size_per_expert': H, 'activation_fn': ACTS[expert]}
    spec = {'type': 'top', 'k': k, 'capacity_factor': 0}      # dropless (a per-call factor of 0 means "the gate's")
    if gate == 'sigmoid':
        spec.update(scoring_func='sigmoid', bias_update_speed=0.001)
    layer = moe.moe_layer(gate_type=spec, model_dim=M, experts=experts, seeds=(1, 2, 3)).cuda().to(dtype)
    with torch.no_grad():
        # skewed routing: a few experts get most tokens, and the gate weight decides it
        w = layer.gates[0].wg.weight
        w.mul_(4.0)
        w[: max(E // 8, 1)] += 0.5
    return layer


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


CASES = [(ex, gate, k, E, torch.bfloat16) for ex in ('relu', 'gelu', 'silu', 'llama') for gate in ('softmax', 'sigmoid')
         for k, E in ((1, 8), (2, 8), (8, 64))]
CASES += [(ex, gate, 2, 8, torch.float16) for ex in ('relu', 'silu', 'llama') for gate in ('softmax', 'sigmoid')]


@pytest.mark.parametrize('expert,gate,k,E,dtype', CASES,
                         ids=['%s-%s-k%d-E%d-%s' % (c[0], c[1], c[2], c[3], str(c[4])[6:]) for c in CASES])
def test_training_step_matches_padded(expert, gate, k, E, dtype):
    torch.manual_seed(0)
    layer = _layer(expert, E, k, gate, dtype)
    S = 512
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
    assert 4 * int(counts.max()) > 5 * k * S // E, 'routing is not skewed'
    assert torch.equal(y, y_r)
    assert torch.equal(l_aux, l_r)
    assert torch.equal(dx, dx_r)
    assert grads.keys() == grads_r.keys()
    for n in grads:
        if 'bias' in n and 'e_score' not in n:
            bound = _bias_bound(grads_r[n], dtype, int(counts.max()))
            assert bool(((grads[n].float() - grads_r[n].float()).abs() <= bound).all()), n
        else:
            assert torch.equal(grads[n], grads_r[n]), n


def test_no_host_sync():
    layer = _layer('silu', 8, 2, 'sigmoid', torch.bfloat16)
    x = torch.randn(512, 256, device='cuda', dtype=torch.bfloat16, requires_grad=True)
    _step(layer, x, None)                  # warm-up (lazy initialisation)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        y = layer(x)
        (y.float().pow(2).mean() + y.l_aux.float()).backward()
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
        layer = _layer(expert, 8, 2, 'sigmoid', torch.bfloat16)
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
    eager = [eager_step(x).clone() for x in [xs[0]] * 3 + xs]      # the same warm-up the graph runs
    graph_layer, graph_step = make()
    fast = GraphedTrainStep(graph_step, xs[0], warmup=3)
    graphed = [fast(x).clone() for x in xs]
    for a, b in zip(eager[3:], graphed):
        assert torch.equal(a, b)
    for (n, p), (_, q) in zip(eager_layer.state_dict().items(), graph_layer.state_dict().items()):
        assert torch.equal(p, q), n
    bias = graph_layer.gates[0].e_score_correction_bias
    assert bool((bias != 0).any()), 'the sigmoid gate bias was not updated'


@pytest.mark.parametrize('variant', ['fp8', 'mx', 'custom', 'megablocks', 'reserve_dims'])
def test_ineligible_configurations_take_the_padded_path(variant):
    from tutel_b200 import moe
    from tutel_b200.ops import routing
    torch.manual_seed(0)
    E, M = 8, 256
    experts = {'type': 'ffn', 'num_experts_per_device': E, 'hidden_size_per_expert': 512}
    if variant == 'fp8':
        experts['fp8'] = True
    if variant == 'mx':
        experts['fp8'] = 'mx'
    if variant == 'custom':
        class Custom(torch.nn.Module):
            def __init__(self, model_dim, num_experts_per_device, sharded_count):
                super().__init__()
                self.w = torch.nn.Parameter(torch.randn(num_experts_per_device, model_dim, model_dim) * 0.02)

            def forward(self, x, ctx):
                return torch.matmul(x, self.w)
        experts = {'type': 'custom', 'module': Custom, 'num_experts_per_device': E}
    layer = moe.moe_layer(gate_type={'type': 'top', 'k': 2, 'capacity_factor': 0}, model_dim=M, experts=experts, seeds=(1, 2, 3)).cuda().bfloat16()
    x = torch.randn(4, 128, M, device='cuda', dtype=torch.bfloat16)
    calls = []
    orig = routing._packed_critical
    routing._packed_critical = lambda *a: calls.append(1) or orig(*a)
    try:
        if variant == 'megablocks':          # (bound-based dropless decoding: inference only)
            with torch.no_grad():
                y = layer(x.view(-1, M), megablocks_size=1)
        elif variant == 'reserve_dims':
            y = layer(x.view(4, 128, 2, M // 2), reserve_dims=2)
        else:
            y = layer(x)
    finally:
        routing._packed_critical = orig
    assert not calls, 'an ineligible configuration took the packed path'
    assert torch.isfinite(y.detach().float()).all()
