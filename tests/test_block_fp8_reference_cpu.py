"""The block-fp8 references (tests/block_fp8_reference.py) on the CPU: the module's own CPU definitions
(tutel_b200/ops/block_fp8.py) and an fp32 emulation of the kernel pass; each likely kernel bug fails the check that
guards it; the expert option is parsed as documented and a CPU layer stays on its 16-bit path."""
import pytest
import torch
import torch.nn.functional as F

import block_fp8_reference as R
from tutel_b200.ops import block_fp8 as BF


def _special(G, rows, K, seed=0):
    gen = torch.Generator().manual_seed(seed)
    spread = torch.exp2(torch.randint(-20, 20, (G, rows, K // 128, 1), generator=gen).float())
    x = (torch.randn(G, rows, K // 128, 128, generator=gen) * spread).view(G, rows, K)
    x[0, 0, :128] = 0
    x[0, 0, 128:256] = torch.randn(128, generator=gen) * 1e-37           # below 448 * FLT_MIN
    x[G - 1, rows - 1, 7] = float('nan')
    x[G - 1, rows // 2, 3] = float('inf')
    x[G - 1, rows // 2, K - 1] = float('-inf')
    return x.bfloat16()


def test_cpu_quantisers_match_the_reference():
    x = _special(2, 130, 384, seed=1)
    q, s = BF.quantize_act_reference(x)
    wq, ws = R.quantize_act(x)
    R.check_scales('act scales', s, ws)
    R.check_bytes('act', q, wq, x)
    assert bool((s[:, :, 130:] == 0).all())
    assert float(ws[0, 1, 0]) == 2.0 ** -126, 'a tiny tile gets the FLT_MIN scale'
    assert float(ws[0, 0, 0]) == 1.0, 'a zero tile gets scale 1'
    w = _special(2, 256, 384, seed=2)
    q, s, qT, sT = BF.quantize_weight_reference(w)
    wq, ws = R.quantize_weight(w)
    R.check_scales('weight scales', s, ws)
    R.check_bytes('weight', q, wq, w)
    assert torch.equal(qT.view(torch.uint8), wq.transpose(1, 2))
    assert torch.equal(sT, ws.transpose(1, 2))


# ------------------------------------------------------------------------------------------------------------------
# an fp32 emulation of the kernel, and its near misses
# ------------------------------------------------------------------------------------------------------------------
def emulate(a, sa, b, sb, bias=None, aux=None, aux2=None, epilogue=R.EPI_NONE, act='silu', miss=None):
    G, M, K = a.shape
    N = b.size(1)
    KB = K // 128
    rows_b = N // sb.size(1)
    acc = torch.zeros(G, M, N)
    for kb in range(KB):
        if miss == 'dropped K step' and kb == KB - 1:
            continue
        k = slice(kb * 128, (kb + 1) * 128)
        part = a.float()[:, :, k] @ b.float()[:, :, k].transpose(1, 2)
        ka = (kb + 1) % KB if miss == 'scale of the wrong K block' else kb
        s_a = sa[:, ka, :M]
        if miss == 'per-128-row A scale':
            s_a = s_a[:, ::128].repeat_interleave(128, dim=1)[:, :M]
        s_b = sb[:, :, kb].repeat_interleave(rows_b, dim=1)
        if miss == 'B scale of the wrong N block':
            s_b = s_b.roll(128, dims=1)
        acc = (part.double() * (s_a.unsqueeze(-1) * s_b.unsqueeze(1)).double() + acc.double()).float()
    if epilogue == R.EPI_GLU:
        H = N // 2
        t = acc.view(G, M, H // 64, 2, 64)
        g, u = t[:, :, :, 0].reshape(G, M, H), t[:, :, :, 1].reshape(G, M, H)
        if miss == 'swapped gate/up halves':
            g, u = u, g
        return [(BF._act(g, act)[0] * u).bfloat16(), g.bfloat16(), u.bfloat16()]
    if epilogue == R.EPI_RELU and miss == 'bias after ReLU':
        return [(acc.clamp_min(0) + bias.float().view(G, 1, N)).bfloat16()]
    if bias is not None:
        acc = acc + bias.float().view(G, 1, N)
    if epilogue == R.EPI_RELU:
        acc = acc.clamp_min(0)
    elif epilogue == R.EPI_RELU_BWD:
        keep = aux.float() >= 0 if miss == '>= ReLU-backward mask' else aux.float() > 0
        acc = torch.where(keep, acc, torch.zeros_like(acc))
    return [acc.bfloat16()]


def _plain_case(K=512, seed=0):
    return R.operands(2, 300, 384, K, spread=10, seed=seed)


def test_emulation_passes_every_epilogue():
    aq, sa, bq, sb = _plain_case()
    r = R.ref_gemm(aq, sa, bq, sb)
    bias, aux = R.bias_aux(r[0].val)
    for epi, kw in ((R.EPI_NONE, {}), (R.EPI_NONE, dict(bias=bias)), (R.EPI_RELU, dict(bias=bias)),
                    (R.EPI_RELU_BWD, dict(aux=aux))):
        R.check_all('emulation %d' % epi, emulate(aq, sa, bq, sb, epilogue=epi, **kw), R.ref_gemm(aq, sa, bq, sb, epilogue=epi, **kw))
        R.check_all('module %d' % epi, BF.block_fp8_gemm_reference(aq, sa, bq, sb, epilogue=epi, **kw),
                    R.ref_gemm(aq, sa, bq, sb, epilogue=epi, **kw))
    for act in ('silu', 'gelu', 'relu'):
        ops = R.operands(2, 130, 256, 384, spread=3, seed=5, glu=True)
        R.check_all('glu ' + act, emulate(*ops, epilogue=R.EPI_GLU, act=act), R.ref_gemm(*ops, epilogue=R.EPI_GLU, act=act))


@pytest.mark.parametrize('miss', ['scale of the wrong K block', 'B scale of the wrong N block', 'per-128-row A scale',
                                  'dropped K step'])
def test_accumulation_near_misses_fail(miss):
    aq, sa, bq, sb = _plain_case(seed=1)
    with pytest.raises(AssertionError):
        R.check(miss, emulate(aq, sa, bq, sb, miss=miss)[0], R.ref_gemm(aq, sa, bq, sb)[0])


def test_epilogue_near_misses_fail():
    aq, sa, bq, sb = _plain_case(seed=2)
    r = R.ref_gemm(aq, sa, bq, sb)
    bias, aux = R.bias_aux(r[0].val)
    with pytest.raises(AssertionError):
        R.check('bias after relu', emulate(aq, sa, bq, sb, bias=bias, epilogue=R.EPI_RELU, miss='bias after ReLU')[0],
                R.ref_gemm(aq, sa, bq, sb, bias=bias, epilogue=R.EPI_RELU)[0])
    with pytest.raises(AssertionError, match='exactly 0'):
        R.check('>= mask', emulate(aq, sa, bq, sb, aux=aux, epilogue=R.EPI_RELU_BWD, miss='>= ReLU-backward mask')[0],
                R.ref_gemm(aq, sa, bq, sb, aux=aux, epilogue=R.EPI_RELU_BWD)[0])
    ops = R.operands(2, 130, 256, 384, spread=3, seed=6, glu=True)
    with pytest.raises(AssertionError):
        R.check_all('swapped', emulate(*ops, epilogue=R.EPI_GLU, miss='swapped gate/up halves'),
                    R.ref_gemm(*ops, epilogue=R.EPI_GLU))


def test_transposed_weight_scale_indexing_fails():
    """The dgrad copy W^T must carry the transposed scales; the forward scales read in the transposed copy's index
    order (a reshape instead of a transpose) is caught."""
    gen = torch.Generator().manual_seed(3)
    w = (torch.randn(1, 256, 384, generator=gen) * torch.exp2(torch.randint(-8, 8, (1, 256, 384), generator=gen).float())).bfloat16()
    x = torch.randn(1, 200, 256, generator=gen).bfloat16()
    _, s, qT, sT = BF.quantize_weight_reference(w)
    xq, xs = R.quantize_act(x)
    xq = xq.view(torch.float8_e4m3fn)
    ref = R.ref_gemm(xq, xs, qT, sT)[0]
    R.check('transposed copy', emulate(xq, xs, qT, sT)[0], ref)
    wrong = s.reshape(sT.shape)
    assert not torch.equal(wrong, sT)
    with pytest.raises(AssertionError):
        R.check('reshaped scales', emulate(xq, xs, qT, wrong)[0], ref)


def test_glu_backward_emulation_passes():
    ops = R.operands(2, 130, 256, 384, spread=3, seed=7)
    gen = torch.Generator().manual_seed(8)
    g = (torch.randn(2, 130, 256, generator=gen) * 2).bfloat16()
    u = torch.randn(2, 130, 256, generator=gen).bfloat16()
    for act in ('silu', 'gelu', 'relu'):
        got = BF.block_fp8_gemm_reference(*ops, aux=g, aux2=u, epilogue=R.EPI_GLU_BWD, act=act)
        R.check_all('glu_bwd ' + act, got, R.ref_gemm(*ops, aux=g, aux2=u, epilogue=R.EPI_GLU_BWD, act=act))
        swapped = [torch.cat([got[0][..., 256:], got[0][..., :256]], dim=2)]
        with pytest.raises(AssertionError):
            R.check_all('glu_bwd swapped ' + act, swapped, R.ref_gemm(*ops, aux=g, aux2=u, epilogue=R.EPI_GLU_BWD, act=act))


# ------------------------------------------------------------------------------------------------------------------
# options
# ------------------------------------------------------------------------------------------------------------------
def test_block_option_is_accepted_and_typos_are_refused(monkeypatch):
    from tutel_b200.models.experts.ffn import FusedExpertsNetwork
    from tutel_b200.models.experts.llama_ffn import LlamaFFNNetwork
    ffn = FusedExpertsNetwork(128, 128, 2, 1, fp8='block')
    assert ffn.block and not ffn.fp8 and not ffn.mx
    llama = LlamaFFNNetwork(128, 128, 2, 1, fp8='BLOCK')
    assert llama.block and not llama.fp8
    monkeypatch.setenv('TUTEL_B200_FP8', 'block')
    assert FusedExpertsNetwork(128, 128, 2, 1).block and LlamaFFNNetwork(128, 128, 2, 1).block
    for bad in ('blokc', 'blocks'):
        with pytest.raises(AssertionError, match='block'):
            FusedExpertsNetwork(128, 128, 2, 1, fp8=bad)
        with pytest.raises(AssertionError, match='block'):
            LlamaFFNNetwork(128, 128, 2, 1, fp8=bad)
    # no new parameters: the state dict is that of the 16-bit experts
    assert ffn.state_dict().keys() == FusedExpertsNetwork(128, 128, 2, 1, fp8=False).state_dict().keys()


@pytest.mark.parametrize('kind', ['ffn', 'llama_ffn'])
def test_cpu_layer_takes_the_16_bit_path(monkeypatch, kind):
    from tutel_b200 import moe
    calls = []
    for name in ('fused_relu_ffn_block_fp8', 'fused_glu_ffn_block_fp8'):
        monkeypatch.setattr(BF, name, lambda *a, **k: calls.append(a))
    experts = {'type': kind, 'num_experts_per_device': 2, 'hidden_size_per_expert': 128, 'fp8': 'block'}
    if kind == 'ffn':
        experts['activation_fn'] = lambda t: F.relu(t)
    torch.manual_seed(0)
    layer = moe.moe_layer(gate_type={'type': 'top', 'k': 1}, model_dim=128, experts=experts, seeds=(1, 1, 1))
    x = torch.randn(2, 16, 128, requires_grad=True)
    y = layer(x)
    y.float().sum().backward()
    assert not calls and torch.isfinite(y).all()
    assert not layer.experts.supports_packed(x)
