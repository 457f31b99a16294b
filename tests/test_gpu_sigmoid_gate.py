"""Sigmoid gate kernels (csrc/gate_route.cu, SIGMOID instantiations) against tests/sigmoid_gate_reference.py, and
the layer's sigmoid routing on the GPU: fused against op-by-op in every capacity mode, dropless decoding, CUDA-graph
replay of the bias update, and the load accumulator's training-only rule."""
import math

import pytest
import torch
import torch.nn.functional as F

import dispatch_reference as DR
import sigmoid_gate_reference as R

pytestmark = pytest.mark.gpu

F32, F16, BF16 = torch.float32, torch.float16, torch.bfloat16
FLOATS = (F32, F16, BF16)


@pytest.fixture(scope='module')
def C():
    from tutel_b200.ops import backend
    return backend.require_ext()


@pytest.fixture(scope='module', autouse=True)
def _report_bounds():
    yield
    print('\nlargest error / bound per bounded check:', {k: round(v, 4) for k, v in sorted(DR.OBSERVED.items())})


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _name(dtype):
    return str(dtype)[6:]


# E on both sides of every per-lane boundary (VPT = 1, 2, 4, 8, 16 for E <= 32, 64, 128, 256, 512), k up to 32,
# n_group in {1, 2, 8, 32} (also one expert per group), S around the 256-token routing tile.
CASES = [(8, 2, 255, 2, 1), (32, 4, 256, 8, 2), (32, 32, 1, 1, 1), (33, 8, 257, 1, 1), (64, 6, 8195, 1, 1),
         (64, 8, 255, 32, 4), (65, 2, 256, 1, 1), (128, 8, 257, 8, 4), (129, 4, 255, 1, 1), (256, 8, 8195, 8, 4),
         (256, 32, 256, 2, 1), (257, 8, 255, 1, 1), (384, 8, 1000, 32, 8), (512, 16, 257, 32, 2),
         (512, 32, 8195, 8, 4), (32, 4, 257, 32, 8)]
CASES = [c + (i,) for i, c in enumerate(CASES)]
BIASES = ('zero', 'random', 'negative')


def _logits(S, E, dtype, seed, nan):
    """Logits spread by tens, integer-valued rows (exact ties of keys and group scores), -inf entries, one NaN."""
    gen = _gen(seed)
    x = torch.randn(S, E, generator=gen) * 3
    x[: S // 4] = torch.randint(-2, 3, (S // 4, E), generator=gen).float()
    if S > 8 and E > 1:
        x[S // 2: S // 2 + 8, ::3] = -math.inf
    if nan:
        x[S - 2, E // 2] = math.nan
    return x.to(dtype)


def _bias(E, kind, seed):
    gen = _gen(seed)
    if kind == 'zero':
        return torch.zeros(E)
    if kind == 'random':
        return torch.randn(E, generator=gen) * 0.3
    return -50.0 - torch.rand(E, generator=gen)          # every key negative


@pytest.mark.parametrize('dtype', FLOATS, ids=_name)
@pytest.mark.parametrize('E,k,S,G,TG,case', CASES, ids=['E%d-k%d-S%d-g%d-%d' % c[:5] for c in CASES])
def test_sigmoid_gate_forward_backward(C, dtype, E, k, S, G, TG, case):
    nan = S >= 255 and case % 2 == 1
    kind = BIASES[case % 3]
    logits = _logits(S, E, dtype, 300 + case, nan)
    bias = _bias(E, kind, 400 + case)
    normalize = case % 4 != 2
    eps = float(torch.finfo(dtype).eps)
    scale = 2.5 if case % 2 == 0 else 1.0
    cap = 0 if case % 4 == 3 else max(1, S * k // E // 2)
    what = '%s S=%d E=%d k=%d groups=%d/%d bias=%s C=%d' % (_name(dtype), S, E, k, G, TG, kind, cap)
    load = torch.full((E,), 3.0, device='cuda')
    outs = C.sigmoid_gate_route_forward(logits.cuda(), bias.cuda(), k, cap, normalize, eps, G, TG, scale, load)
    assert (len(outs) == 9) == (cap > 0)
    outs_h = [t.cpu() for t in outs]
    R.check_forward(what, logits, bias, k, cap, normalize, eps, G, TG, scale, outs_h, check_loss=not nan)
    DR.assert_equal('expert_load += counts: ' + what, load.cpu(), outs_h[5].float() + 3.0)

    rows = torch.ones(S, dtype=torch.bool)
    if nan:
        rows[S - 2] = False
        assert torch.isnan(outs_h[7]).all(), 'l_aux of a batch with a NaN logit'
    scores, idx, top, ce = outs[0], outs[1], outs[2], outs[6]
    dg = torch.randn(k, S, generator=_gen(500 + case))
    dl = torch.tensor(1.75, dtype=dtype)
    variants = [('full', dg, True, normalize, eps), ('dgates=None', None, True, normalize, eps),
                ('no loss', dg, False, normalize, eps), ('normalize=False', dg, True, False, eps),
                ('eps above D', dg, True, True, 2.0)]
    for name, dgates, loss, norm, e in variants:
        out = C.sigmoid_gate_route_backward(scores, idx, top, dgates.cuda() if dgates is not None else None,
                                            ce if loss else None, dl.cuda() if loss else None, logits.cuda(), norm, e,
                                            scale)
        assert out.dtype == dtype
        R.check_backward('%s %s' % (what, name), out.cpu(), outs_h[0], outs_h[1], outs_h[2], dgates,
                         outs_h[6] if loss else None, dl if loss else None, norm, e, scale, rows)


def test_refusals(C):
    x = torch.randn(16, 24, device='cuda')
    b = torch.zeros(24, device='cuda')
    for G, TG, k in [(5, 1, 2), (4, 0, 2), (4, 5, 2), (4, 1, 7), (48, 1, 1)]:
        with pytest.raises(RuntimeError):
            C.sigmoid_gate_route_forward(x, b, k, 0, True, 1e-6, G, TG, 1.0, None)
    with pytest.raises(RuntimeError):
        C.sigmoid_gate_route_forward(x, b.half(), 2, 0, True, 1e-6, 1, 1, 1.0, None)


# ------------------------------------------------------------------------------------------------------------------
# the layer
# ------------------------------------------------------------------------------------------------------------------
def _layer(E=64, k=6, M=128, H=256, experts='ffn', dtype=torch.float32, speed=1e-3, groups=(8, 4)):
    from tutel_b200 import moe
    ex = {'type': experts, 'num_experts_per_device': E, 'hidden_size_per_expert': H}
    if experts == 'ffn':
        ex['activation_fn'] = F.relu
    layer = moe.moe_layer(gate_type={'type': 'top', 'k': k, 'scoring_func': 'sigmoid', 'n_group': groups[0],
                                     'topk_group': groups[1], 'routed_scaling_factor': 2.5,
                                     'bias_update_speed': speed},
                          model_dim=M, experts=ex, seeds=(1, 1, 1)).cuda().to(dtype)
    with torch.no_grad():
        layer.gates[0].e_score_correction_bias.copy_(torch.randn(E, generator=_gen(9)) * 0.2)
    return layer


def _run(layer, x, **kw):
    x = x.clone().requires_grad_(True)
    layer.zero_grad(set_to_none=True)
    y = layer(x, **kw)
    (y.float().pow(2).mean() + 0.1 * y.l_aux.float()).backward()
    return y.detach(), y.l_aux.detach(), x.grad, layer.gates[0].wg.weight.grad


@pytest.mark.parametrize('cf', [1.0, 0.0, -0.5])
def test_layer_fused_matches_op_by_op(monkeypatch, cf):
    layer = _layer()
    x = torch.randn(512, 128, device='cuda', generator=torch.Generator('cuda').manual_seed(1))
    fused = _run(layer, x, capacity_factor=cf)
    load_fused = layer.gates[0].expert_load.clone()
    layer.gates[0].expert_load.zero_()
    monkeypatch.setenv('TUTEL_B200_FUSED_GATE', '0')
    ref = _run(layer, x, capacity_factor=cf)
    assert torch.equal(load_fused, layer.gates[0].expert_load)
    assert float(load_fused.sum()) == 512 * 6
    for name, a, b in zip(('y', 'l_aux', 'dx', 'dwg'), fused, ref):
        assert torch.allclose(a, b, rtol=1e-4, atol=1e-6), (name, (a - b).abs().max())


def test_dropless_bound_and_decoding_match_op_by_op(monkeypatch):
    """Inference with megablocks_size=1 and capacity_factor=0: the sync-free row bound (and for llama_ffn experts the
    skinny one-launch kernels at decode sizes) with a non-zero bias, against op-by-op routing."""
    for experts, dtype, S in [('ffn', torch.float32, 512), ('llama_ffn', torch.bfloat16, 4),
                              ('llama_ffn', torch.bfloat16, 64)]:
        layer = _layer(E=16, k=4, M=256, H=512, experts=experts, dtype=dtype, groups=(4, 2)).eval()
        x = torch.randn(S, 256, device='cuda', generator=torch.Generator('cuda').manual_seed(2)).to(dtype)
        monkeypatch.delenv('TUTEL_B200_FUSED_GATE', raising=False)
        with torch.no_grad():
            y = layer(x, capacity_factor=0.0, megablocks_size=1)
        monkeypatch.setenv('TUTEL_B200_FUSED_GATE', '0')
        with torch.no_grad():
            want = layer(x, capacity_factor=0.0)
        tol = 1e-4 if dtype == torch.float32 else 3e-2
        assert torch.allclose(y.float(), want.float(), rtol=tol, atol=tol), (experts, S, (y.float() - want.float()).abs().max())
        assert torch.equal(layer.gates[0].expert_load, torch.zeros(16, device='cuda'))


def test_expert_load_untouched_in_eval_and_no_grad():
    layer = _layer()
    x = torch.randn(256, 128, device='cuda')
    layer.eval()
    layer(x)
    layer.train()
    with torch.no_grad():
        layer(x)
    assert torch.equal(layer.gates[0].expert_load, torch.zeros(64, device='cuda'))
    layer(x)
    assert float(layer.gates[0].expert_load.sum()) == 256 * 6


def test_graphed_train_step_replays_bias_update():
    """lr = 0: the bias after warm-up plus n replays equals the bias after as many eager steps, bit for bit."""
    from tutel_b200.utils.graph import GraphedTrainStep
    n, warmup = 5, 3
    x = torch.randn(1024, 128, device='cuda', generator=torch.Generator('cuda').manual_seed(3))

    def make():
        layer = _layer(speed=1e-3)
        opt = torch.optim.SGD(layer.parameters(), lr=0.0)

        def step(inp):
            opt.zero_grad(set_to_none=True)
            y = layer(inp)
            loss = y.float().pow(2).mean() + 0.01 * y.l_aux.float()
            loss.backward()
            opt.step()
            return loss.detach()
        return layer, step

    eager, step = make()
    for _ in range(warmup + n):
        step(x)
    torch.cuda.synchronize()
    graphed, gstep = make()
    fast = GraphedTrainStep(gstep, x, warmup=warmup)
    after_warmup = graphed.gates[0].e_score_correction_bias.clone()
    for _ in range(n):
        fast(x)
    torch.cuda.synchronize()
    b_eager = eager.gates[0].e_score_correction_bias
    b_graph = graphed.gates[0].e_score_correction_bias
    assert not torch.equal(after_warmup, b_graph), 'the replays did not update the bias'
    assert torch.equal(b_eager, b_graph)
    assert torch.equal(graphed.gates[0].expert_load, torch.zeros(64, device='cuda'))
