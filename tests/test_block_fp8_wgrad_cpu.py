"""Block-fp8 weight gradients (``fp8_wgrad``) on the CPU: the dual quantiser's CPU definition matches the exact
reference of tests/block_fp8_wgrad_reference.py, an fp32 emulation of the weight-gradient GEMM passes the fp64 bound, each
likely kernel bug fails the check that guards it, the option is refused where it cannot apply, and a CPU layer with it
stays on its 16-bit path."""
import pytest
import torch
import torch.nn.functional as F

import block_fp8_reference as R
import block_fp8_wgrad_reference as W
from tutel_b200.ops import block_fp8 as BF


def _special(G, rows, K, seed=0):
    """Random values spread over 2^+-20 per 128 x 128 tile, with a zero column block, a column of values below
    448 * FLT_MIN, NaN and +-inf."""
    gen = torch.Generator().manual_seed(seed)
    spread = torch.exp2(torch.randint(-20, 20, (G, 1, K // 128, 1), generator=gen).float())
    x = (torch.randn(G, rows, K // 128, 128, generator=gen) * spread).view(G, rows, K)
    x[0, :, :128] = 0
    x[0, :, 130] = torch.randn(rows, generator=gen) * 1e-37
    x[G - 1, rows - 1, 7] = float('nan')
    x[G - 1, rows // 2, 3] = float('inf')
    x[G - 1, rows // 2, K - 1] = float('-inf')
    return x.bfloat16()


def _check_dual(what, got, want):
    q, s, qT, sT = got
    wq, ws, wqT, wsT = want
    R.check_scales(what + ' row scales', s, ws)
    R.check_bytes(what + ' rows', q, wq)
    R.check_scales(what + ' column scales', sT, wsT)
    R.check_bytes(what + ' columns', qT, wqT)


@pytest.mark.parametrize('rows', [1, 127, 129, 300])
def test_cpu_dual_quantiser_matches_the_reference(rows):
    x = _special(2, rows, 384, seed=rows)
    got = BF.quantize_act_dual_reference(x)
    _check_dual('dual R=%d' % rows, got, W.quantize_act_dual(x))
    q, s = BF.quantize_act_reference(x)
    assert torch.equal(got[0].view(torch.uint8), q.view(torch.uint8)) and torch.equal(got[1], s)
    Rp = -(-rows // 128) * 128
    assert got[2].shape == (2, 384, Rp) and got[3].shape == (2, Rp // 128, 384)
    assert bool((got[2].view(torch.uint8)[:, :, rows:] == 0).all()), 'pad rows of x^T are zero bytes'
    assert float(got[3][0, 0, 0]) == 1.0, 'an all-zero column block gets scale 1'
    assert float(got[3][0, 0, 130]) == 2.0 ** -126, 'a tiny column block gets the FLT_MIN scale'
    col_only = BF.quantize_act_dual_reference(x, rowwise=False)
    assert col_only[0] is None and col_only[1] is None
    assert torch.equal(col_only[2].view(torch.uint8), got[2].view(torch.uint8)) and torch.equal(col_only[3], got[3])


def test_dual_quantiser_near_misses_fail():
    x = _special(2, 200, 256, seed=3)
    want = W.quantize_act_dual(x)
    q, s, qT, sT = BF.quantize_act_dual_reference(x)
    # pad rows given a non-zero scale (row-wise and column-wise halves)
    bad_s = s.clone()
    bad_s[:, :, 200:] = 1.0
    with pytest.raises(AssertionError):
        _check_dual('pad row scale', (q, bad_s, qT, sT), want)
    # the amax of the partial last block taken over pad rows that hold NaN (as if rows past R were read)
    Rp = 256
    xp = torch.full((2, Rp, 256), float('nan'))
    xp[:, :200] = x.float()
    amax = xp.abs().view(2, 2, 128, 256).amax(2)
    bad_sT = R.scale_of(amax)
    with pytest.raises(AssertionError):
        _check_dual('NaN pad rows', (q, s, qT, bad_sT), want)
    # one scale per 128 x 128 block instead of per column
    blk = R.scale_of(R._amax(torch.cat([x.float(), torch.zeros(2, 56, 256)], 1).view(2, 2, 128, 2, 128), (2, 4)))
    with pytest.raises(AssertionError):
        _check_dual('block scales', (q, s, qT, blk.repeat_interleave(128, dim=2)), want)


# ------------------------------------------------------------------------------------------------------------------
# the weight-gradient GEMM
# ------------------------------------------------------------------------------------------------------------------
def _operands(G, M, N, K, seed=0):
    """Column-wise operands: aT [G, M, K] + saT [G, K/128, M], bT [G, N, K] + sbT [G, K/128, N], random e4m3 bytes and
    scale exponents over +-30; K steps past the real tokens hold zero bytes and pad scales."""
    aq, sa, _, _ = R.operands(G, M, 128, K, seed=seed)
    bq, sb, _, _ = R.operands(G, N, 128, K, seed=seed + 1)
    return aq, sa, bq, sb


@pytest.mark.parametrize('G,M,N,K,split', [(1, 128, 128, 128, None), (2, 256, 384, 384, None), (3, 128, 512, 256, 256),
                                           (1, 384, 256, 640, 128)])
def test_wgrad_emulation_passes_the_bound(G, M, N, K, split):
    aq, sa, bq, sb = _operands(G, M, N, K, seed=M + N + K)
    out = BF.wgrad_gemm_reference(aq, sa, bq, sb, split)
    ref = W.ref_wgrad(aq, sa, bq, sb)
    d = out[0] if split is None else torch.cat(out, dim=2)
    if split is not None:
        assert len(out) == 2 and all(t.shape == (G, M, split) and t.is_contiguous() for t in out)
    R.check('wgrad emulation G=%d M=%d N=%d K=%d' % (G, M, N, K), d, ref)


def test_wgrad_near_misses_fail():
    G, M, N, K = 2, 256, 256, 512
    aq, sa, bq, sb = _operands(G, M, N, K, seed=7)
    ref = W.ref_wgrad(aq, sa, bq, sb)
    R.check('wgrad', BF.wgrad_gemm_reference(aq, sa, bq, sb)[0], ref)
    near = {
        # one B scale per 128-column block (the forward's weight-block layout) instead of per column
        'per-block B scales': (aq, sa, bq, sb[:, :, ::128].repeat_interleave(128, dim=2)),
        # sT read transposed: [G, N, K/128] memory taken for [G, K/128, N]
        'transposed sT': (aq, sa, bq, sb.transpose(1, 2).contiguous().view(G, K // 128, N)),
        # each K step promoted with the next step's scales
        'K step off by one': (aq, sa.roll(-1, dims=1), bq, sb.roll(-1, dims=1)),
    }
    for what, ops in near.items():
        with pytest.raises(AssertionError):
            R.check('wgrad ' + what, BF.wgrad_gemm_reference(*ops)[0], ref)


def test_wgrad_of_quantised_activations_matches_fp64():
    """``dW = dh^T x`` through the dual quantiser and the emulated GEMM is the fp64 product of the dequantised operands
    within the bound, with a partial last token block."""
    gen = torch.Generator().manual_seed(5)
    x = torch.randn(2, 200, 256, generator=gen).bfloat16()
    dh = torch.randn(2, 200, 384, generator=gen).bfloat16()
    _, _, xqT, xsT = BF.quantize_act_dual_reference(x, rowwise=False)
    _, _, hqT, hsT = BF.quantize_act_dual_reference(dh, rowwise=False)
    d = BF.wgrad_gemm_reference(hqT, hsT, xqT, xsT)[0]
    R.check('dW1 C=200', d, W.ref_wgrad(hqT, hsT, xqT, xsT))
    exact = dh.double().transpose(1, 2) @ x.double()
    assert float((d.double() - exact).abs().max() / exact.abs().max()) < 0.1


# ------------------------------------------------------------------------------------------------------------------
# the option
# ------------------------------------------------------------------------------------------------------------------
def test_option_is_refused_where_it_cannot_apply(monkeypatch):
    from tutel_b200.models.experts.ffn import FusedExpertsNetwork
    from tutel_b200.models.experts.llama_ffn import LlamaFFNNetwork
    monkeypatch.delenv('TUTEL_B200_FP8', raising=False)
    for fp8 in (None, False, True, 'row', 'mx'):
        with pytest.raises(ValueError, match='fp8_wgrad'):
            FusedExpertsNetwork(128, 128, 2, 1, fp8=fp8, fp8_wgrad=True)
    for fp8 in (None, False, True, 'row'):
        with pytest.raises(ValueError, match='fp8_wgrad'):
            LlamaFFNNetwork(128, 128, 2, 1, fp8=fp8, fp8_wgrad=True)
    with pytest.raises(ValueError, match='fp8_wgrad'):
        LlamaFFNNetwork(128, 128, 2, 1, weight_format='fp8_block', fp8_wgrad=True)
    ffn = FusedExpertsNetwork(128, 128, 2, 1, fp8='block', fp8_wgrad=True)
    llama = LlamaFFNNetwork(128, 128, 2, 1, fp8='block', fp8_wgrad=True)
    assert ffn.fp8_wgrad and llama.fp8_wgrad
    assert 'fp8_wgrad=True' in repr(ffn) and 'fp8_wgrad=True' in repr(llama)
    assert 'fp8_wgrad' not in repr(FusedExpertsNetwork(128, 128, 2, 1, fp8='block'))
    # the state dict is that of the 16-bit experts
    assert ffn.state_dict().keys() == FusedExpertsNetwork(128, 128, 2, 1).state_dict().keys()
    assert llama.state_dict().keys() == LlamaFFNNetwork(128, 128, 2, 1).state_dict().keys()
    # the mode may come from the environment
    monkeypatch.setenv('TUTEL_B200_FP8', 'block')
    assert FusedExpertsNetwork(128, 128, 2, 1, fp8_wgrad=True).fp8_wgrad
    assert LlamaFFNNetwork(128, 128, 2, 1, fp8_wgrad=True).fp8_wgrad
    with pytest.raises(ValueError, match='fp8_wgrad'):
        FusedExpertsNetwork(128, 128, 2, 1, fp8='row', fp8_wgrad=True)


@pytest.mark.parametrize('kind', ['ffn', 'llama_ffn'])
def test_cpu_layer_with_the_option_takes_the_16_bit_path(monkeypatch, kind):
    from tutel_b200 import moe
    calls = []
    for name in ('fused_relu_ffn_block_fp8', 'fused_glu_ffn_block_fp8'):
        monkeypatch.setattr(BF, name, lambda *a, **k: calls.append(a))

    def run(wgrad):
        experts = {'type': kind, 'num_experts_per_device': 2, 'hidden_size_per_expert': 128, 'fp8': 'block',
                   'fp8_wgrad': wgrad}
        if kind == 'ffn':
            experts['activation_fn'] = lambda t: F.relu(t)
        torch.manual_seed(0)
        layer = moe.moe_layer(gate_type={'type': 'top', 'k': 1}, model_dim=128, experts=experts, seeds=(1, 1, 1),
                              shared_experts={'num_experts': 1})
        assert layer.experts.fp8_wgrad == wgrad and layer.shared_experts.fp8_wgrad == wgrad
        x = torch.randn(2, 16, 128, generator=torch.Generator().manual_seed(2), requires_grad=True)
        y = layer(x)
        y.float().sum().backward()
        return y, x.grad, [p.grad for p in layer.parameters()]

    y, dx, grads = run(True)
    y0, dx0, grads0 = run(False)
    assert not calls and torch.isfinite(y).all()
    assert torch.equal(y, y0) and torch.equal(dx, dx0)
    assert all((a is None and b is None) or torch.equal(a, b) for a, b in zip(grads, grads0))


@pytest.mark.parametrize('expert', ['ffn', 'llama_ffn'])
def test_layer_wgrad_reference_changes_only_the_weight_gradient_bounds(expert):
    """tests/layer_wgrad_reference.py: without fp8 its expert backward is layer_reference's exactly; with fp8, dx and
    the bias gradients are the same and the weight gradients keep their values under wider (e4m3 operand) bounds."""
    import layer_reference as LR
    import layer_wgrad_reference as LW
    gen = torch.Generator().manual_seed(4)
    T, M, H = 40, 16, 24

    def t(*shape):
        return torch.randn(*shape, generator=gen, dtype=torch.float64)
    cfg = LR.Config(E=2, k=1, dtype=torch.bfloat16, logit_dtype=torch.float32, expert=expert,
                    act='relu' if expert == 'ffn' else 'silu', fp8='row')
    if expert == 'ffn':
        w = [t(H, M), t(H), t(H, M), t(M)]
        saved = (LR.B(t(T, M)), LR.B(t(T, H)), LR.B(t(T, H).clamp_min(0)))
    else:
        w = [t(M, H), t(M, H), t(H, M)]
        saved = (LR.B(t(T, M)), LR.B(t(T, H)), LR.B(t(T, H)), LR.B(t(T, H)))
    dout = LR.B(t(T, M))
    wgrad_slots = [0, 2] if expert == 'ffn' else [0, 1, 2]
    for fp8 in (False, True):
        dx, dws = LR.expert_backward(cfg, w, saved, dout, torch.bfloat16, fp8, torch.bfloat16)
        dx2, dws2 = LW.expert_backward(cfg, w, saved, dout, torch.bfloat16, fp8, torch.bfloat16)
        assert torch.equal(dx.v, dx2.v) and torch.equal(dx.err, dx2.err)
        for i, (a, b) in enumerate(zip(dws, dws2)):
            if a is None:
                assert b is None
                continue
            assert torch.equal(a.v, b.v)
            if fp8 and i in wgrad_slots:
                assert bool((b.err >= a.err).all()) and bool((b.err > a.err).any())
            else:
                assert torch.equal(a.err, b.err)
    assert LR.expert_backward is not LW.expert_backward
