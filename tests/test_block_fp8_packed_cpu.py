"""Block-fp8 experts on the expert-packed layout (``fp8_packed``) on the CPU: the option is refused where it cannot apply,
the CPU definitions of the packed launch modes (block-mapped GEMM, ragged-K weight-gradient GEMM, bounded quantisers)
agree with per-segment compositions of the existing references, CPU layers never take the packed path, and the option
leaves the state dict alone."""
import pytest
import torch
import torch.nn.functional as F

from tutel_b200.ops import block_fp8 as BF


def _ffn(**kw):
    from tutel_b200.models.experts.ffn import FusedExpertsNetwork
    args = dict(model_dim=256, hidden_size_per_expert=384, num_experts_per_device=4, sharded_count=1,
                activation_fn=F.relu, fp8='block', fp8_packed=True)
    args.update(kw)
    return FusedExpertsNetwork(**args)


def _llama(**kw):
    from tutel_b200.models.experts.llama_ffn import LlamaFFNNetwork
    args = dict(model_dim=256, hidden_size_per_expert=384, num_experts_per_device=4, sharded_count=1, fp8='block',
                fp8_packed=True)
    args.update(kw)
    return LlamaFFNNetwork(**args)


@pytest.mark.parametrize('case', ['ffn row', 'ffn mx', 'ffn off', 'ffn gelu', 'ffn silu', 'ffn model_dim', 'ffn hidden',
                                  'ffn output_dim', 'ffn weight_format', 'llama row', 'llama off', 'llama fp8_block',
                                  'llama model_dim', 'llama hidden'])
def test_refusals(case, monkeypatch):
    monkeypatch.delenv('TUTEL_B200_FP8', raising=False)
    build, kw, match = {
        'ffn row': (_ffn, dict(fp8='row'), "needs fp8='block'"),
        'ffn mx': (_ffn, dict(fp8='mx'), "needs fp8='block'"),
        'ffn off': (_ffn, dict(fp8=None), "needs fp8='block'"),
        'ffn gelu': (_ffn, dict(activation_fn=F.gelu), 'ReLU only'),
        'ffn silu': (_ffn, dict(activation_fn=F.silu), 'ReLU only'),
        'ffn model_dim': (_ffn, dict(model_dim=192), 'multiples of 128'),
        'ffn hidden': (_ffn, dict(hidden_size_per_expert=320), 'multiples of 128'),
        'ffn output_dim': (_ffn, dict(output_dim=200), 'multiples of 128'),
        'ffn weight_format': (_ffn, dict(weight_format='fp8_block'), 'no stored weight format'),
        'llama row': (_llama, dict(fp8='row'), "needs fp8='block'"),
        'llama off': (_llama, dict(fp8=None), "needs fp8='block'"),
        'llama fp8_block': (_llama, dict(weight_format='fp8_block'), 'inference-only'),
        'llama model_dim': (_llama, dict(model_dim=192), 'multiples of 128'),
        'llama hidden': (_llama, dict(hidden_size_per_expert=320), 'multiples of 128'),
    }[case]
    with pytest.raises(ValueError, match=match):
        build(**kw)


def test_option_from_the_environment(monkeypatch):
    monkeypatch.setenv('TUTEL_B200_FP8', 'block')
    assert _ffn(fp8=None).fp8_packed and _llama(fp8=None).fp8_packed
    monkeypatch.setenv('TUTEL_B200_FP8', 'row')
    with pytest.raises(ValueError, match="needs fp8='block'"):
        _ffn(fp8=None)


def test_default_is_off_and_repr():
    from tutel_b200.models.experts.ffn import FusedExpertsNetwork
    m = FusedExpertsNetwork(256, 384, 4, 1, activation_fn=F.relu, fp8='block')
    assert not m.fp8_packed and 'fp8_packed' not in m.extra_repr()
    assert 'fp8_packed=True' in _ffn().extra_repr() and 'fp8_packed=True' in _llama(fp8_wgrad=True).extra_repr()


@pytest.mark.parametrize('build', [_ffn, _llama], ids=['ffn', 'llama_ffn'])
def test_supports_packed_is_false_on_cpu(build):
    m = build().bfloat16()
    assert not m.supports_packed(torch.zeros(256, 256, dtype=torch.bfloat16))


def test_state_dict_is_unchanged_by_the_option():
    from tutel_b200 import moe
    for kind in ('ffn', 'llama_ffn'):
        def make(packed):
            experts = {'type': kind, 'num_experts_per_device': 4, 'hidden_size_per_expert': 256, 'fp8': 'block'}
            if packed:
                experts['fp8_packed'] = True
            if kind == 'ffn':
                experts['activation_fn'] = F.relu
            return moe.moe_layer(gate_type={'type': 'top', 'k': 2, 'capacity_factor': 0}, model_dim=128, experts=experts,
                                 seeds=(1, 2, 3), shared_experts={'num_experts': 1})
        a, b = make(True), make(False)
        sa, sb = a.state_dict(), b.state_dict()
        assert list(sa) == list(sb), kind
        for n in sa:
            assert sa[n].shape == sb[n].shape and sa[n].dtype == sb[n].dtype and torch.equal(sa[n], sb[n]), (kind, n)
        b.load_state_dict(sa)
        assert a.shared_experts.fp8_packed, 'shared experts inherit the option'


# ------------------------------------------------------------------------------------------------------------------
# CPU definitions of the packed launch modes
# ------------------------------------------------------------------------------------------------------------------
COUNTS = [0, 1, 127, 128, 129, 255, 300]


def _layout(counts):
    """seg_off, block_expert, block_rows (as ops/packed.py defines them) and R for per-expert row counts, built on the
    host.  R leaves a spare 128-row tail past seg_off[E], as packed_rows does."""
    seg = [0]
    for c in counts:
        seg.append(seg[-1] + -(-c // 128) * 128)
    R = seg[-1] + 256
    block_expert, block_rows = [0] * (R // 128), [0] * (R // 128)
    for e, c in enumerate(counts):
        for j in range(-(-c // 128)):
            block_expert[seg[e] // 128 + j] = e
            block_rows[seg[e] // 128 + j] = min(128, c - 128 * j)
    i32 = lambda v: torch.tensor(v, dtype=torch.int32)      # noqa: E731
    return i32(seg), i32(block_expert), i32(block_rows), R


def _pack(xp, counts, seg, R):
    """[E, C, K] padded -> [R, K] packed; rows past seg_off[E] are NaN (never initialised in a real buffer)."""
    out = torch.full((R, xp.size(-1)), float('nan'), dtype=xp.dtype)
    for e, c in enumerate(counts):
        n = -(-c // 128) * 128
        out[int(seg[e]):int(seg[e]) + n] = 0
        out[int(seg[e]):int(seg[e]) + c] = xp[e, :c]
    return out


def _unpack(t, counts, seg, C):
    out = torch.zeros(len(counts), C, t.size(-1), dtype=t.dtype)
    for e, c in enumerate(counts):
        out[e, :c] = t[int(seg[e]):int(seg[e]) + c]
    return out


def _close(what, got, want):
    """Equal up to the fp32 summation order of the CPU matmul inside one 128-deep K step, one bf16 rounding apart."""
    g, w = got.float(), want.float()
    tol = 2.0 ** -7 * w.abs() + 1e-6 * w.abs().max() + 1e-30
    assert bool(((g - w).abs() <= tol).all()), '%s: max |diff| %g' % (what, float((g - w).abs().max()))


def _padded(E, C, K, counts, seed):
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(E, C, K, generator=gen)
    for e, c in enumerate(counts):
        x[e, c:] = 0
    return x.bfloat16()


def test_bounded_quantisers_match_the_unbounded_ones_below_the_bound():
    counts = COUNTS[:4]
    seg, _, _, R = _layout(counts)
    x = _pack(_padded(len(counts), 256, 256, counts, 0), counts, seg, R)
    used = seg[-1:]
    q, s = BF.quantize_act(x, live_rows=used)
    n = int(used)
    qr, sr = BF.quantize_act_reference(x[:n].unsqueeze(0))
    assert q.shape == (1, R, 256) and s.shape == (1, 2, R)
    assert torch.equal(q[:, :n].view(torch.uint8), qr.view(torch.uint8)) and torch.equal(s[:, :, :n], sr[:, :, :n])
    got = BF.quantize_act_dual(x, live_rows=used)
    want = BF.quantize_act_dual_reference(x[:n].unsqueeze(0))
    assert torch.equal(got[0][:, :n].view(torch.uint8), want[0].view(torch.uint8))
    assert torch.equal(got[2][:, :, :n].view(torch.uint8), want[2].view(torch.uint8))
    assert torch.equal(got[3][:, :n // 128], want[3])
    col = BF.quantize_act_dual(x, rowwise=False, live_rows=used)
    assert col[0] is None and torch.equal(col[2].view(torch.uint8), got[2].view(torch.uint8))
    assert torch.isfinite(got[3]).all(), 'the NaN rows past the bound are not read'


@pytest.mark.parametrize('epi', ['none', 'bias', 'relu', 'relu_bwd', 'glu', 'glu_bwd'])
def test_block_mapped_gemm_matches_the_grouped_reference(epi):
    counts = COUNTS
    E, C, K, N = len(counts), 384, 256, 256
    seg, bexp, brows, R = _layout(counts)
    xp = _padded(E, C, K, counts, 1)
    xq, xs = BF.quantize_act(xp)
    pq, ps = BF.quantize_act(_pack(xp, counts, seg, R), live_rows=seg[-1:])
    gen = torch.Generator().manual_seed(2)
    w = (torch.randn(E, N, K, generator=gen) * K ** -0.5).bfloat16()
    q1, s1, _, _ = BF.quantize_weight(w)
    kw, code, act = {}, BF.EPI_NONE, 'silu'
    if epi in ('bias', 'relu'):
        kw['bias'] = torch.randn(E, N, generator=gen).bfloat16()
        code = BF.EPI_RELU if epi == 'relu' else BF.EPI_NONE
    if epi == 'relu_bwd':
        code, kw['aux'] = BF.EPI_RELU_BWD, _padded(E, C, N, counts, 3)
    if epi == 'glu':
        code, act = BF.EPI_GLU, 'gelu'
        q1, s1 = BF.quantize_glu_weight(*(torch.randn(2, E, K, N // 2, generator=gen) * K ** -0.5).bfloat16().unbind(0))[2:]
    if epi == 'glu_bwd':
        code, act = BF.EPI_GLU_BWD, 'silu'
        kw['aux'], kw['aux2'] = _padded(E, C, N, counts, 4), _padded(E, C, N, counts, 5)
    counts_t = torch.tensor(counts, dtype=torch.int32)
    want = BF.block_fp8_gemm(xq, xs, q1, s1, epilogue=code, act=act, row_counts=counts_t, **kw)
    pkw = dict(kw)
    for k in ('aux', 'aux2'):
        if k in pkw:
            pkw[k] = _pack(pkw[k], counts, seg, R).nan_to_num(0.0)
    got = BF.block_fp8_gemm(pq, ps, q1, s1, epilogue=code, act=act, row_counts=brows, b_group_map=bexp, **pkw)
    assert len(got) == len(want)
    for i, (g, wt) in enumerate(zip(got, want)):
        assert g.shape == (R, wt.size(-1))
        _close('%s output %d' % (epi, i), _unpack(g, counts, seg, C), wt)
        for e, c in enumerate(counts):           # padding rows inside the segments are exact zeros
            end = int(seg[e + 1])
            assert bool((g[int(seg[e]) + c:end] == 0).all()), (epi, i, e)


@pytest.mark.parametrize('split', [False, True])
def test_ragged_wgrad_matches_per_expert_padding(split):
    counts = COUNTS
    E, C, M, N = len(counts), 384, 256, 256
    seg, _, _, R = _layout(counts)
    a, b = _padded(E, C, M, counts, 6), _padded(E, C, N, counts, 7)
    _, _, aT, saT = BF.quantize_act_dual(a, rowwise=False)
    _, _, bT, sbT = BF.quantize_act_dual(b, rowwise=False)
    want = BF.wgrad_gemm(aT, saT, bT, sbT, split=N // 2 if split else None)
    _, _, paT, psaT = BF.quantize_act_dual(_pack(a, counts, seg, R), rowwise=False, live_rows=seg[-1:])
    _, _, pbT, psbT = BF.quantize_act_dual(_pack(b, counts, seg, R), rowwise=False, live_rows=seg[-1:])
    got = BF.wgrad_gemm(paT, psaT, pbT, psbT, split=N // 2 if split else None, k_offsets=seg)
    assert len(got) == len(want)
    for g, wt in zip(got, want):
        assert g.shape == wt.shape
        _close('wgrad', g, wt)
        assert bool((g[0] == 0).all()), 'an expert with no tokens gets zeros'
