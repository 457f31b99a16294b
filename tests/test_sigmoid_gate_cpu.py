"""Sigmoid gate options, buffers and auxiliary-loss-free bias balancing on CPU (models/gates/top.py)."""
import pytest
import torch
import torch.nn.functional as F

from helpers import run_workers
from tutel_b200 import moe
from tutel_b200.models.gates.top import LinearTopKGate
from tutel_b200.ops.gating import expert_bias_update


def _layer(gate, E=16, M=32, **kw):
    return moe.moe_layer(gate_type=dict({'type': 'top'}, **gate), model_dim=M,
                         experts={'type': 'ffn', 'num_experts_per_device': E, 'hidden_size_per_expert': 64,
                                  'activation_fn': F.relu}, seeds=(1, 1, 1), **kw)


@pytest.mark.parametrize('opts,msg', [
    ({'n_group': 3}, 'n_group'),
    ({'n_group': 4, 'topk_group': 0}, 'topk_group'),
    ({'n_group': 4, 'topk_group': 5}, 'topk_group'),
    ({'k': 9, 'n_group': 4, 'topk_group': 2}, 'top_k'),
    ({'bias_update_speed': -1e-3}, 'bias_update_speed'),
    ({'scoring_func': 'tanh'}, 'scoring_func'),
])
def test_option_validation(opts, msg):
    with pytest.raises(ValueError, match=msg):
        LinearTopKGate(8, 16, **dict({'k': 2, 'scoring_func': 'sigmoid'}, **opts))


def test_softmax_rejects_sigmoid_options_and_sigmoid_rejects_load_importance_loss():
    with pytest.raises(ValueError, match='sigmoid'):
        LinearTopKGate(8, 16, k=2, n_group=4)
    with pytest.raises(ValueError, match='is_gshard_loss'):
        _layer({'k': 2, 'scoring_func': 'sigmoid'}, is_gshard_loss=False)


def test_top_k_override_is_validated():
    layer = _layer({'k': 2, 'scoring_func': 'sigmoid', 'n_group': 4, 'topk_group': 1})
    layer(torch.randn(8, 32), top_k=4)
    with pytest.raises(ValueError, match='top_k'):
        layer(torch.randn(8, 32), top_k=5)


def test_state_dict_and_fp32_buffers():
    soft = _layer({'k': 2})
    keys = list(soft.state_dict())
    assert 'gates.0.e_score_correction_bias' not in keys and not hasattr(soft.gates[0], 'expert_load')
    sig = _layer({'k': 2, 'scoring_func': 'sigmoid', 'bias_update_speed': 1e-3})
    assert sorted(sig.state_dict()) == sorted(keys + ['gates.0.e_score_correction_bias'])
    gate = sig.gates[0]
    gate.e_score_correction_bias.fill_(1e-3 * 3)
    want = gate.e_score_correction_bias.clone()
    for cast in (torch.nn.Module.bfloat16, torch.nn.Module.half, torch.nn.Module.double):
        cast(sig)
        assert gate.e_score_correction_bias.dtype == torch.float32 and gate.expert_load.dtype == torch.float32
        assert torch.equal(gate.e_score_correction_bias, want)
    assert gate.wg.weight.dtype == torch.float64
    assert 'gates.0.expert_load' not in sig.state_dict()


def test_bias_arithmetic_is_exact():
    """n updates with the same counts move each bias by exactly +-n * gamma (fp32 gamma), or leave it at 0."""
    E, gamma, n = 8, 2.0 ** -10, 7                  # gamma and its multiples are exact in fp32
    bias = torch.zeros(E)
    load = torch.zeros(E)
    counts = torch.tensor([5., 1., 3., 3., 9., 0., 3., 0.])       # mean 3: below, above and equal
    for _ in range(n):
        load += counts
        expert_bias_update(bias, load, gamma)
        assert torch.equal(load, torch.zeros(E))
    assert torch.equal(bias, torch.sign(3.0 - counts) * (n * gamma))


def test_training_forward_accumulates_and_step_updates():
    layer = _layer({'k': 2, 'scoring_func': 'sigmoid', 'bias_update_speed': 1e-3})
    gate = layer.gates[0]
    opt = torch.optim.SGD(layer.parameters(), lr=0.0)
    x = torch.randn(64, 32)
    layer.eval()
    layer(x)
    assert torch.equal(gate.expert_load, torch.zeros(16))
    layer.train()
    with torch.no_grad():
        layer(x)
    assert torch.equal(gate.expert_load, torch.zeros(16))
    y = layer(x)
    assert float(gate.expert_load.sum()) == 2 * 64
    load = gate.expert_load.clone()
    y.sum().backward()
    opt.step()
    assert torch.equal(gate.expert_load, torch.zeros(16))
    assert torch.equal(gate.e_score_correction_bias, torch.sign(load.mean() - load) * torch.tensor(1e-3))
    layer(x).sum().backward()
    layer.update_expert_bias()                      # loops without torch.optim
    assert torch.equal(gate.expert_load, torch.zeros(16))


def test_balancing_reduces_skew():
    """A frozen gate (lr = 0) skewed towards experts 0-3 of 32: the first step sends every token there (max/mean load
    8), and after 130 bias updates at gamma = 3e-3 the max/mean load of each of the next 20 steps is below 1.5.
    Seeded and deterministic."""
    E, k, M, S = 32, 4, 32, 512
    layer = _layer({'k': k, 'scoring_func': 'sigmoid', 'n_group': 8, 'topk_group': 4, 'bias_update_speed': 3e-3},
                   E=E, M=M)
    gate = layer.gates[0]
    with torch.no_grad():
        gate.wg.weight.mul_(0.2)
        gate.wg.weight[:4] += 0.06
    x = torch.randn(S, M, generator=torch.Generator().manual_seed(0)).abs()
    opt = torch.optim.SGD(layer.parameters(), lr=0.0)
    skew = []
    for _ in range(150):
        opt.zero_grad()
        y = layer(x)
        load = gate.expert_load.clone()
        (y.sum() + y.l_aux).backward()
        opt.step()
        skew.append(float(load.max() / load.mean()))
    print('max/mean load: first step %.3f, worst of steps 131-150 %.3f' % (skew[0], max(skew[130:])))
    assert skew[0] == 8.0 and max(skew[130:]) < 1.5


def test_frozen_bias_accumulates_nothing():
    layer = _layer({'k': 2, 'scoring_func': 'sigmoid'})
    gate = layer.gates[0]
    opt = torch.optim.SGD(layer.parameters(), lr=0.0)
    layer(torch.randn(64, 32)).sum().backward()
    assert torch.equal(gate.expert_load, torch.zeros(16))
    opt.step()
    layer.update_expert_bias()
    assert torch.equal(gate.e_score_correction_bias, torch.zeros(16))


GLOO_WORKER = r'''
sys.path.insert(0, os.getcwd())
dist.init_process_group('gloo')
from tutel_b200.models.gates.top import LinearTopKGate, apply_pending_bias_updates
from tutel_b200.ops.gating import expert_bias_update
r = dist.get_rank()
# three gates, two of the same size; rank 1 allocates between them, so the gates' addresses (and the order of any
# address-keyed set) differ between the ranks
junk = []
gates = []
for i, E in enumerate((8, 8, 12)):
    if r == 1:
        junk += [object() for _ in range(1000 * (3 - i))]
    g = LinearTopKGate(16, E, k=2, scoring_func='sigmoid', bias_update_speed=1e-3 * (i + 1))
    g.balance_group = dist.group.WORLD
    gates.append(g)
def counts(i, rank, step):
    gen = torch.Generator().manual_seed(100 * i + 10 * rank + step)
    return torch.randint(0, 20, (gates[i].expert_load.numel(),), generator=gen).float()
for step in range(4):
    order = range(3) if r == 0 else reversed(range(3))      # the forwards mark the gates pending in different orders
    for i in order:
        gates[i].expert_load.add_(counts(i, r, step))
        gates[i].note_training_forward()
    apply_pending_bias_updates()
for i, g in enumerate(gates):
    want_b = torch.zeros_like(g.e_score_correction_bias)
    for step in range(4):
        load = counts(i, 0, step) + counts(i, 1, step)
        expert_bias_update(want_b, load, g.bias_update_speed)
    assert torch.equal(g.e_score_correction_bias, want_b), (r, i, g.e_score_correction_bias, want_b)
    assert bool((want_b != 0).any())
    both = [torch.zeros_like(want_b) for _ in range(2)]
    dist.all_gather(both, g.e_score_correction_bias)
    assert torch.equal(both[0], both[1])
print('BIAS_SYNC_OK')
dist.destroy_process_group()
'''


def test_two_rank_gloo_bias_sync():
    """Different tokens per rank: every gate of a several-gate model ends with the same bias on both ranks, equal to
    the single-rank updates from its own summed counts, whatever the gates' addresses and pending order."""
    assert 'BIAS_SYNC_OK' in run_workers(GLOO_WORKER, nproc=2, timeout=300)
