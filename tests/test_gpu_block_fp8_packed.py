"""Block-fp8 experts on the expert-packed layout (``fp8_packed``): the packed launch modes of csrc/gemm_block_fp8.cu
against the grouped launches on the same data, both expert autograd functions against the padded buffer, and whole
dropless training steps against the padded path (``capacity_factor=-E``) and the fp64 layer reference.

Why the packed and padded results are equal: activation quantisation is row-local (1 x 128 tiles), every expert segment
starts on a 128-row boundary and padding rows are zero, so each row tile holds the rows, scales and K order it holds in
the padded layout; the 128 x 1 column tiles of the weight-gradient operands are the padded layout's too, and padded K
blocks only add zero products.  Bias gradients are column sums in another fp32 order (compared under a bound), and
``dW2`` of an ``ffn`` with an fc1 bias under ``fp8_wgrad`` differs in the last bits: the padded path's padding rows of
``act`` hold relu(b1) and enter the column scales of ``act^T``, the packed path's are zero (compared against the fp64
bound instead)."""
import pytest
import torch
import torch.nn.functional as F

import layer_reference as LR
import layer_wgrad_reference as LW

pytestmark = pytest.mark.gpu


def _bits(t):
    return t.view(torch.int16)


def _routing(counts, seed=0):
    """A k = 1 routing with the given per-expert counts, tokens in random order -> (idx [1, S], loc [1, S], counts)."""
    g = torch.Generator().manual_seed(seed)
    idx = torch.repeat_interleave(torch.arange(len(counts)), torch.tensor(counts))
    idx = idx[torch.randperm(idx.numel(), generator=g)]
    loc = torch.zeros_like(idx)
    for e in range(len(counts)):
        loc[idx == e] = torch.arange(counts[e])
    i32 = lambda t: t.to(torch.int32).cuda()       # noqa: E731
    return i32(idx.view(1, -1)), i32(loc.view(1, -1)), i32(torch.tensor(counts))


def _layout(counts, seed=0):
    from tutel_b200.ops.packed import PackedLayout
    return PackedLayout.build(*_routing(counts, seed))


def _pack(xp, counts, layout, fill=float('nan')):
    """[E, C, K] padded (zero past the counts) -> [R, K] packed; rows past seg_off[E] hold ``fill``."""
    seg = layout.seg_off.cpu().tolist()
    out = torch.full((layout.R, xp.size(-1)), fill, dtype=xp.dtype, device=xp.device)
    for e, c in enumerate(counts):
        out[seg[e]:seg[e + 1]] = 0
        out[seg[e]:seg[e] + c] = xp[e, :c]
    return out


def _unpack(t, counts, layout, C):
    seg = layout.seg_off.cpu().tolist()
    out = torch.zeros(len(counts), C, t.size(-1), dtype=t.dtype, device=t.device)
    for e, c in enumerate(counts):
        out[e, :c] = t[seg[e]:seg[e] + c]
    return out


def _padded(E, C, K, counts, seed, scale=1.0):
    g = torch.Generator(device='cuda').manual_seed(seed)
    x = torch.randn(E, C, K, device='cuda', generator=g) * scale
    for e, c in enumerate(counts):
        x[e, c:] = 0
    return x.bfloat16()


def _segment_padding_is_zero(what, t, counts, layout):
    seg = layout.seg_off.cpu().tolist()
    for e, c in enumerate(counts):
        assert bool((t[seg[e] + c:seg[e + 1]] == 0).all()), '%s: padding rows of expert %d' % (what, e)


def _live_equal(what, got, want, counts, layout):
    C = want.size(1)
    assert torch.equal(_bits(_unpack(got, counts, layout, C)), _bits(want)), what
    _segment_padding_is_zero(what, got, counts, layout)


EDGE = [0, 1, 127, 128, 129, 255, 1500, 40]                  # one expert holds most tokens


def _skewed(E, S, seed):
    g = torch.Generator().manual_seed(seed)
    w = torch.rand(E, generator=g) ** 4 + 0.01
    w[0] += w.sum()
    c = (w / w.sum() * S).long()
    c[1], c[2] = 0, 1
    return c.tolist()


# name -> (counts, K, N): every K from 128 to 4096; E = 64 gives more row tiles than SMs and partial last tiles
SHAPES = {
    'edge K128': (EDGE, 128, 256),
    'edge K4096': (EDGE, 4096, 512),
    'E64 K512': (_skewed(64, 6000, 1), 512, 1024),
}


# ------------------------------------------------------------------------------------------------------------------
# kernels
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('shape', list(SHAPES))
@pytest.mark.parametrize('epi', ['none', 'bias', 'bias_relu', 'relu_bwd', 'glu', 'glu_bwd'])
def test_block_mapped_gemm(epi, shape):
    """Live rows bit for bit the grouped launch on [E, C, K]; padding rows inside segments exactly zero (also under
    bias + ReLU); NaN operand rows and scales past seg_off[E] reach no live output."""
    from tutel_b200.ops import block_fp8 as BF
    counts, K, N = SHAPES[shape]
    E, C = len(counts), max(counts)
    layout = _layout(counts)
    xp = _padded(E, C, K, counts, 1)
    xq, xs = BF.quantize_act(xp)
    pq, ps = BF.quantize_act(_pack(xp, counts, layout), live_rows=layout.used_rows)
    used = int(layout.seg_off[-1])
    pq.view(torch.uint8)[:, used:] = 0x7F                      # e4m3 NaN
    ps[:, :, used:] = float('nan')
    g = torch.Generator(device='cuda').manual_seed(2)
    kw, code, act = {}, BF.EPI_NONE, 'silu'
    if epi == 'glu':
        code, act = BF.EPI_GLU, 'silu'
        w1, w2 = (torch.randn(2, E, K, N // 2, device='cuda', generator=g) * K ** -0.5).bfloat16().unbind(0)
        qb, sb = BF.quantize_glu_weight(w1, w2)[2:]
    else:
        w = (torch.randn(E, N, K, device='cuda', generator=g) * K ** -0.5).bfloat16()
        qb, sb = BF.quantize_weight(w)[:2]
    if epi in ('bias', 'bias_relu'):
        kw['bias'] = torch.randn(E, N, device='cuda', generator=g).bfloat16().abs()      # positive: relu(b) != 0
        code = BF.EPI_RELU if epi == 'bias_relu' else BF.EPI_NONE
    if epi == 'relu_bwd':
        code, kw['aux'] = BF.EPI_RELU_BWD, _padded(E, C, N, counts, 3)
    if epi == 'glu_bwd':
        code = BF.EPI_GLU_BWD
        kw['aux'], kw['aux2'] = _padded(E, C, N, counts, 4), _padded(E, C, N, counts, 5)
    want = BF.block_fp8_gemm(xq, xs, qb, sb, epilogue=code, act=act, row_counts=layout.counts, **kw)
    pkw = {k: (_pack(v, counts, layout) if k.startswith('aux') else v) for k, v in kw.items()}
    got = BF.block_fp8_gemm(pq, ps, qb, sb, epilogue=code, act=act, row_counts=layout.block_rows,
                            b_group_map=layout.block_expert, **pkw)
    assert len(got) == len(want)
    for i, (gt, wt) in enumerate(zip(got, want)):
        assert gt.shape == (layout.R, wt.size(-1))
        _live_equal('%s %s output %d' % (epi, shape, i), gt, wt, counts, layout)


@pytest.mark.parametrize('dual', [False, True], ids=['rowwise', 'dual'])
def test_bounded_quantisers(dual):
    """Bit for bit the unbounded launch below seg_off[E]; NaN rows past it change nothing."""
    from tutel_b200.ops import block_fp8 as BF
    counts = _skewed(64, 6000, 2)
    layout = _layout(counts)
    used = int(layout.seg_off[-1])
    assert layout.R - used >= 128, 'the buffer has rows past the used ones'
    xp = _padded(64, max(counts), 1024, counts, 6)
    nan, zero = _pack(xp, counts, layout), _pack(xp, counts, layout, fill=0.0)
    if not dual:
        q, s = BF.quantize_act(nan, live_rows=layout.used_rows)
        qr, sr = BF.quantize_act(zero.unsqueeze(0))
        assert torch.equal(q.view(torch.uint8)[:, :used], qr.view(torch.uint8)[:, :used])
        assert torch.equal(s[:, :, :used], sr[:, :, :used])
        return
    for rowwise in (True, False):
        got = BF.quantize_act_dual(nan, rowwise=rowwise, live_rows=layout.used_rows)
        want = BF.quantize_act_dual(zero.unsqueeze(0), rowwise=rowwise)
        if rowwise:
            assert torch.equal(got[0].view(torch.uint8)[:, :used], want[0].view(torch.uint8)[:, :used])
            assert torch.equal(got[1][:, :, :used], want[1][:, :, :used])
        assert torch.equal(got[2].view(torch.uint8)[:, :, :used], want[2].view(torch.uint8)[:, :, :used])
        assert torch.equal(got[3][:, :used // 128], want[3][:, :used // 128])


@pytest.mark.parametrize('split', [False, True], ids=['single', 'split'])
@pytest.mark.parametrize('shape', ['edge', 'E64'])
def test_ragged_wgrad(shape, split):
    """Bit for bit the padded launch on per-expert zero-padded operands; empty experts get exact zeros."""
    from tutel_b200.ops import block_fp8 as BF
    counts = EDGE if shape == 'edge' else _skewed(64, 6000, 3)
    E, C = len(counts), max(counts)
    M, N = (512, 1024) if shape == 'edge' else (256, 512)
    layout = _layout(counts)
    a, b = _padded(E, C, M, counts, 7), _padded(E, C, N, counts, 8)
    sp = N // 2 if split else None
    want = BF.wgrad_gemm(*BF.quantize_act_dual(a, rowwise=False)[2:], *BF.quantize_act_dual(b, rowwise=False)[2:], split=sp)
    pa = BF.quantize_act_dual(_pack(a, counts, layout), rowwise=False, live_rows=layout.used_rows)[2:]
    pb = BF.quantize_act_dual(_pack(b, counts, layout), rowwise=False, live_rows=layout.used_rows)[2:]
    got = BF.wgrad_gemm(*pa, *pb, split=sp, k_offsets=layout.seg_off)
    assert len(got) == len(want)
    for gt, wt in zip(got, want):
        assert torch.equal(_bits(gt), _bits(wt))
        for e, c in enumerate(counts):
            if c == 0:
                assert bool((gt[e] == 0).all())


# ------------------------------------------------------------------------------------------------------------------
# expert autograd functions
# ------------------------------------------------------------------------------------------------------------------
def _bias_bound(ref, rows):
    return 2.0 ** -8 * ref.abs().float() + (rows + 16) * 2.0 ** -24 * ref.abs().float().max() + 1e-7


def _rel(a, b):
    return float((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-30))


def _run(fn, x, params, dy):
    x = x.detach().clone().requires_grad_(True)
    ps = [None if p is None else p.detach().clone().requires_grad_(True) for p in params]
    y = fn(x, *ps)
    y.backward(dy)
    return y.detach(), x.grad, [None if p is None else p.grad for p in ps]


@pytest.mark.parametrize('wgrad', [False, True], ids=['bf16_wgrad', 'fp8_wgrad'])
@pytest.mark.parametrize('expert', ['ffn', 'ffn_nobias', 'llama_ffn'])
def test_expert_functions_with_layout(expert, wgrad):
    from tutel_b200.ops import block_fp8 as BF
    counts = [300, 0, 1, 127, 128, 129, 255, 40]
    E, C, M, H = len(counts), max(counts), 256, 384
    layout = _layout(counts, seed=4)
    g = torch.Generator(device='cuda').manual_seed(9)
    rnd = lambda *s, sc=1.0: (torch.randn(*s, device='cuda', generator=g) * sc).bfloat16()      # noqa: E731
    xp, dyp = _padded(E, C, M, counts, 10), _padded(E, C, M, counts, 11)
    if expert == 'llama_ffn':
        params = [rnd(E, M, H, sc=M ** -0.5), rnd(E, M, H, sc=M ** -0.5), rnd(E, H, M, sc=H ** -0.5)]
        fn = lambda lay: (lambda x, w1, w2, w3: BF.fused_glu_ffn_block_fp8(x, w1, w2, w3, 'silu', wgrad, layout=lay))  # noqa: E731
        names = ['w1', 'w2', 'w3']
    else:
        biases = expert == 'ffn'
        params = [rnd(E, H, M, sc=M ** -0.5), rnd(E, H, sc=0.5) if biases else None, rnd(E, H, M, sc=H ** -0.5),
                  rnd(E, M, sc=0.5) if biases else None]
        fn = lambda lay: (lambda x, w1, b1, w2, b2: BF.fused_relu_ffn_block_fp8(x, w1, b1, w2, b2, wgrad, layout=lay))  # noqa: E731
        names = ['w1', 'b1', 'w2', 'b2']
    # the padded buffer as the padded dispatch leaves it (zero rows past the counts)
    y_r, dx_r, gr_r = _run(fn(None), xp, params, dyp)
    y, dx, gr = _run(fn(layout), _pack(xp, counts, layout), params, _pack(dyp, counts, layout))
    _live_equal('y', y, _zero_past(y_r, counts), counts, layout)
    _live_equal('dx', dx, _zero_past(dx_r, counts), counts, layout)
    for n, a, b in zip(names, gr, gr_r):
        if a is None:
            assert b is None
            continue
        if n.startswith('b'):
            assert bool(((a.float() - b.float()).abs() <= _bias_bound(b, C)).all()), n
        elif expert == 'ffn' and wgrad and n == 'w2':
            # relu(b1) in the padded act^T scales: last-bit differences only (the layer test checks it against fp64)
            assert 0 < _rel(a, b) < 2.0 ** -6, (n, _rel(a, b))
        else:
            assert torch.equal(_bits(a), _bits(b)), n


def _zero_past(t, counts):
    t = t.clone()
    for e, c in enumerate(counts):
        t[e, c:] = 0
    return t


# ------------------------------------------------------------------------------------------------------------------
# the layer
# ------------------------------------------------------------------------------------------------------------------
def _layer(expert, E=8, k=2, gate='softmax', wgrad=False, packed=True, shared=False, biases=True, M=256, H=512, seed=1):
    from tutel_b200 import moe
    spec = {'type': 'top', 'k': k, 'capacity_factor': 0}
    if gate == 'sigmoid':
        spec.update(scoring_func='sigmoid', n_group=4, topk_group=2, routed_scaling_factor=2.5)
    experts = {'type': expert, 'num_experts_per_device': E, 'hidden_size_per_expert': H, 'fp8': 'block'}
    if packed:
        experts['fp8_packed'] = True
    if wgrad:
        experts['fp8_wgrad'] = True
    if expert == 'ffn':
        experts.update(activation_fn=lambda t: F.relu(t), has_fc1_bias=biases, has_fc2_bias=biases)
    torch.manual_seed(seed)
    layer = moe.moe_layer(gate_type=spec, model_dim=M, experts=experts, seeds=(seed, seed + 1, seed + 2),
                          shared_experts={'num_experts': 1} if shared else None).cuda().bfloat16()
    with torch.no_grad():
        if gate == 'sigmoid':
            layer.gates[0].e_score_correction_bias.copy_(torch.linspace(-0.05, 0.05, E))
        w = layer.gates[0].wg.weight                       # skewed routing: a few experts get most tokens
        w.mul_(4.0)
        w[: max(E // 8, 1)] += 0.5
        if expert == 'llama_ffn':                          # unit-scale hidden activations (the default init gives ~1e-4)
            for n, p in layer.named_parameters():
                if 'W_fc' in n:
                    p.normal_(0, M ** -0.5 if 'fc3' not in n else H ** -0.5)
    return layer


def _loss(y):
    w = torch.linspace(-1, 1, y.size(-1), device=y.device, dtype=torch.float32)
    return (y.float() * w).sum() / y.size(0) + 0.5 * y.l_aux.float()


def _step(layer, x, cf):
    for p in layer.parameters():
        p.grad = None
    xx = x.detach().clone().requires_grad_(True)
    y = layer(xx, capacity_factor=cf)
    _loss(y).backward()
    grads = {n: p.grad.clone() for n, p in layer.named_parameters() if p.grad is not None}
    return y.detach(), y.l_aux.detach(), xx.grad.clone(), grads, layer.dispatch_count.clone()


def _recorded_step(layer, x):
    with LR.recording(layer) as recs:
        params = LR.snapshot(layer)
        for p in layer.parameters():
            p.grad = None
        xx = x.detach().clone().requires_grad_(True)
        _loss(layer(xx)).backward()
        torch.cuda.synchronize()
        return LR.make_step(layer, recs[-1], xx, params, xx.grad)


def _took_packed(layer, x, **fwd):
    from tutel_b200.ops import routing
    calls = []
    orig = routing._packed_critical
    routing._packed_critical = lambda *a: calls.append(1) or orig(*a)
    try:
        y = layer(x, **fwd)
    finally:
        routing._packed_critical = orig
    return bool(calls), y


# (expert, gate, k, E, shared, wgrad, fp64 check)
LAYER_CASES = [
    ('ffn', 'softmax', 2, 8, False, False, True),
    ('ffn', 'softmax', 2, 8, False, True, True),
    ('ffn', 'sigmoid', 1, 8, True, False, False),
    ('ffn', 'sigmoid', 8, 64, False, True, False),
    ('llama_ffn', 'softmax', 2, 8, False, False, True),
    ('llama_ffn', 'softmax', 2, 8, False, True, True),
    ('llama_ffn', 'sigmoid', 8, 64, True, False, False),
    ('llama_ffn', 'sigmoid', 1, 8, True, True, False),
]


@pytest.mark.parametrize('expert,gate,k,E,shared,wgrad,fp64', LAYER_CASES,
                         ids=['%s-%s-k%d-E%d-%s-%s' % (c[0], c[1], c[2], c[3], 'shared' if c[4] else 'routed',
                                                      'fp8wgrad' if c[5] else 'bf16wgrad') for c in LAYER_CASES])
def test_layer_step_matches_padded(expert, gate, k, E, shared, wgrad, fp64):
    layer = _layer(expert, E, k, gate, wgrad, shared=shared)
    S = 512
    x = torch.randn(S, 256, device='cuda', dtype=torch.bfloat16, generator=torch.Generator(device='cuda').manual_seed(5))
    took, _ = _took_packed(layer, x)
    assert took, 'the dropless block-fp8 step did not take the packed path'
    y, l_aux, dx, grads, counts = _step(layer, x, None)
    y_r, l_r, dx_r, grads_r, counts_r = _step(layer, x, -E)
    assert torch.equal(counts, counts_r)
    assert 4 * int(counts.max()) > 5 * k * S // E, 'routing is not skewed'
    assert torch.equal(_bits(y), _bits(y_r))
    assert torch.equal(l_aux, l_r)
    assert torch.equal(_bits(dx), _bits(dx_r))
    assert grads.keys() == grads_r.keys()
    for n in grads:
        if 'bias' in n and 'e_score' not in n:
            bound = _bias_bound(grads_r[n], int(counts.max()) if 'shared' not in n else S)
            assert bool(((grads[n].float() - grads_r[n].float()).abs() <= bound).all()), n
        elif expert == 'ffn' and wgrad and n == 'experts.batched_fc2_w':
            assert _rel(grads[n], grads_r[n]) < 2.0 ** -6, n       # checked against fp64 below
        else:
            assert torch.equal(grads[n], grads_r[n]), n
    if fp64 or (expert == 'ffn' and wgrad):
        st = _recorded_step(layer, x)
        assert st.layout is not None, 'the recorded step did not take the packed layout'
        cfg = LR.config_of(layer, x)
        cfg.fp8 = 'row'
        (LW if wgrad else LR).check_step(cfg, st)


def test_ffn_without_biases_has_equal_fp8_weight_gradients():
    layer = _layer('ffn', wgrad=True, biases=False)
    x = torch.randn(512, 256, device='cuda', dtype=torch.bfloat16)
    _, _, dx, grads, _ = _step(layer, x, None)
    _, _, dx_r, grads_r, _ = _step(layer, x, -8)
    assert torch.equal(_bits(dx), _bits(dx_r))
    for n in grads:
        if 'bias' not in n:
            assert torch.equal(grads[n], grads_r[n]), n


@pytest.mark.parametrize('expert', ['ffn', 'llama_ffn'])
def test_no_host_sync(expert):
    layer = _layer(expert, wgrad=True)
    x = torch.randn(512, 256, device='cuda', dtype=torch.bfloat16, requires_grad=True)
    _step(layer, x, None)                  # warm-up (lazy initialisation, weight copies)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        y = layer(x)
        _loss(y).backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()


@pytest.mark.parametrize('wgrad', [False, True], ids=['bf16_wgrad', 'fp8_wgrad'])
@pytest.mark.parametrize('expert', ['ffn', 'llama_ffn'])
def test_graphed_train_step_equals_eager(expert, wgrad):
    from tutel_b200.utils.graph import GraphedTrainStep
    xs = [torch.randn(512, 256, device='cuda', dtype=torch.bfloat16) for _ in range(4)]

    def make():
        layer = _layer(expert, wgrad=wgrad, gate='sigmoid', seed=3)
        opt = torch.optim.SGD(layer.parameters(), lr=0.05)

        def step(x):
            opt.zero_grad(set_to_none=True)
            loss = _loss(layer(x))
            loss.backward()
            opt.step()                     # the next step re-quantises the updated weights
            return loss.detach()
        return layer, step

    assert _took_packed(make()[0], xs[0].clone().requires_grad_(True))[0], 'the step does not take the packed path'
    eager_layer, eager_step = make()
    eager = [eager_step(x).clone() for x in [xs[0]] * 3 + xs]
    graph_layer, graph_step = make()
    fast = GraphedTrainStep(graph_step, xs[0], warmup=3)
    graphed = [fast(x).clone() for x in xs]
    for i, (a, b) in enumerate(zip(eager[3:], graphed)):
        assert torch.equal(a, b), i
    for (n, p), (_, q) in zip(eager_layer.state_dict().items(), graph_layer.state_dict().items()):
        assert torch.equal(p, q), n


@pytest.mark.parametrize('variant', ['option_off', 'fp16', 'no_grad', 'megablocks'])
def test_fallbacks_take_the_padded_path(variant):
    layer = _layer('ffn', packed=variant != 'option_off')
    x = torch.randn(512, 256, device='cuda', dtype=torch.bfloat16)
    if variant == 'fp16':
        layer, x = layer.half(), x.half()
    if variant == 'no_grad':
        with torch.no_grad():
            took, y = _took_packed(layer, x)
    elif variant == 'megablocks':
        with torch.no_grad():
            took, y = _took_packed(layer, x, megablocks_size=1)
    else:
        took, y = _took_packed(layer, x.requires_grad_(True))
        _loss(y).backward()
    assert not took, 'an ineligible configuration took the packed path'
    assert torch.isfinite(y.detach().float()).all()
