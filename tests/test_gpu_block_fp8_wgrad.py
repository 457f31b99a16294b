"""Block-scaled fp8 weight gradients (``fp8_wgrad``): the dual quantiser and the weight-gradient GEMM of
csrc/gemm_block_fp8.cu against tests/block_fp8_wgrad_reference.py, and the experts and layer with the option against
``fp8='block'`` (bit for bit where they must agree) and tests/layer_wgrad_reference.py.

* dual quantiser, bit for bit: R = 1, 127, 129, 300; zero, tiny, NaN and +-inf blocks; its row-wise half against
  ``block_fp8_quantize_act``;
* the GEMM element by element against the fp64 bound: K = 128 ... 16384 tokens (200 through the quantiser), M and N up
  to 14336 / 4096, G = 1, 8, 64, more tiles than SMs, one CTA walking many tiles, the split output with H % 256 != 0;
* both FFNs stage by stage, whole layer steps, graph replay, host synchronisation, saved bytes and a short training run.
"""
import pytest
import torch
import torch.nn.functional as F

import block_fp8_reference as R
import block_fp8_wgrad_reference as W
import dispatch_reference as D
import layer_reference as LR
import layer_wgrad_reference as LW

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module', autouse=True)
def _report():
    yield
    print('\nblock fp8 wgrad normalised errors: %s; C_BLOCK %g' % (
        {k: round(v, 4) for k, v in sorted(R.OBSERVED.items())}, R.C_BLOCK))


def _ext():
    from tutel_b200.ops import backend
    return backend.require_ext()


def _bits(t):
    return t.view(torch.int16)


def _check_dual(what, got, x):
    wq, ws, wqT, wsT = W.quantize_act_dual(x)
    q, s, qT, sT = got
    R.check_scales(what + ' column scales', sT, wsT)
    R.check_bytes(what + ' columns', qT, wqT)
    if q is not None:
        R.check_scales(what + ' row scales', s, ws)
        R.check_bytes(what + ' rows', q, wq)


# ------------------------------------------------------------------------------------------------------------------
# dual quantiser
# ------------------------------------------------------------------------------------------------------------------
def _special(G, rows, K, seed=0):
    """Random values spread over 2^+-20 per column block, plus an all-zero column block, a column below 448 * FLT_MIN,
    a row of tiny values, NaN and +-inf."""
    gen = torch.Generator().manual_seed(seed)
    spread = torch.exp2(torch.randint(-20, 20, (G, rows, K // 128, 1), generator=gen).float())
    x = (torch.randn(G, rows, K // 128, 128, generator=gen) * spread).view(G, rows, K)
    x[0, :, :128] = 0
    if K >= 256:
        x[0, :, 130] = torch.randn(rows, generator=gen) * 1e-37
        x[0, 0, 128:256] = torch.randn(128, generator=gen) * 1e-37
    x[G - 1, rows - 1, 7] = float('nan')
    x[G - 1, rows - 1, 9] = float('-nan')
    if rows > 1:
        x[G - 1, rows // 2, 3] = float('inf')
        x[G - 1, rows // 2, K - 1] = float('-inf')
    return x.bfloat16().cuda()


@pytest.mark.parametrize('G,rows,K', [(1, 1, 128), (1, 127, 256), (3, 129, 384), (2, 300, 512), (2, 2048, 256)])
def test_dual_quantiser_is_bit_exact(G, rows, K):
    x = _special(G, rows, K, seed=rows + K)
    what = 'dual G=%d R=%d K=%d' % (G, rows, K)
    got = _ext().block_fp8_quantize_act_dual(x, True)
    _check_dual(what, got, x)
    q, s = _ext().block_fp8_quantize_act(x)
    assert torch.equal(got[0].view(torch.uint8), q.view(torch.uint8)), what + ': row-wise bytes'
    assert torch.equal(got[1].view(torch.int32), s.view(torch.int32)), what + ': row-wise scales'
    qT, sT = _ext().block_fp8_quantize_act_dual(x, False)
    assert torch.equal(qT.view(torch.uint8), got[2].view(torch.uint8)) and torch.equal(sT, got[3]), what + ': column-only'


# ------------------------------------------------------------------------------------------------------------------
# weight-gradient GEMM
# ------------------------------------------------------------------------------------------------------------------
def _operands(G, M, N, K, seed=0):
    aq, sa, _, _ = R.operands(G, M, 128, K, seed=seed, device='cuda')
    bq, sb, _, _ = R.operands(G, N, 128, K, seed=seed + 1, device='cuda')
    return aq, sa, bq, sb


def _wgrad(aq, sa, bq, sb, split=0, max_ctas=0):
    out = _ext().block_fp8_wgrad_gemm(aq, sa, bq, sb, split, max_ctas)
    return out[0] if split == 0 else torch.cat(out, dim=2)


# (G, M, N, K, split, max_ctas): (8, 1024, 1024, ...) is 512 tiles; max_ctas 1 walks every tile on one CTA (the
# 6-stage ring wraps mid-tile for K = 384); the flagship shapes are 14336 x 4096 and 4096 x 14336 over 2048 tokens.
WGRAD_CASES = [
    (1, 128, 128, 128, 0, 0), (3, 256, 384, 384, 0, 1), (64, 128, 256, 128, 0, 0), (8, 1024, 1024, 2048, 0, 0),
    (2, 256, 512, 16384, 0, 5), (1, 14336, 4096, 2048, 0, 0), (1, 4096, 14336, 2048, 0, 0),
    (3, 256, 768, 384, 384, 0), (8, 512, 1280, 2048, 640, 7),
]


@pytest.mark.parametrize('G,M,N,K,split,max_ctas', WGRAD_CASES)
def test_wgrad_gemm_matches_fp64_reference(G, M, N, K, split, max_ctas):
    aq, sa, bq, sb = _operands(G, M, N, K, seed=M + N + K)
    what = 'wgrad: G=%d M=%d N=%d K=%d split=%d max_ctas=%d' % (G, M, N, K, split, max_ctas)
    d = _wgrad(aq, sa, bq, sb, split, max_ctas)
    R.check(what, d, W.ref_wgrad(aq, sa, bq, sb))
    if split:
        outs = _ext().block_fp8_wgrad_gemm(aq, sa, bq, sb, split, 0)
        assert len(outs) == 2 and all(t.shape == (G, M, split) and t.is_contiguous() for t in outs)
    if G * M * N <= 8 * 1024 * 1024:          # a fixed K order and no atomics: another CTA count gives the same bits
        assert torch.equal(_bits(_wgrad(aq, sa, bq, sb, split, (max_ctas % 5) + 2)), _bits(d)), what


@pytest.mark.parametrize('G,tokens,M,N', [(2, 1, 256, 384), (2, 200, 256, 384), (1, 129, 128, 256), (8, 2048, 512, 256)])
def test_wgrad_of_quantised_activations(G, tokens, M, N):
    """``dW = a^T b`` from the dual quantiser's column-wise outputs, with partial last token blocks."""
    gen = torch.Generator(device='cuda').manual_seed(tokens)
    a = torch.randn(G, tokens, M, generator=gen, device='cuda').bfloat16()
    b = (torch.randn(G, tokens, N, generator=gen, device='cuda') * 1e-3).bfloat16()
    aqT, asT = _ext().block_fp8_quantize_act_dual(a, False)
    bqT, bsT = _ext().block_fp8_quantize_act_dual(b, False)
    what = 'wgrad quantised: G=%d tokens=%d M=%d N=%d' % (G, tokens, M, N)
    R.check(what, _wgrad(aqT, asT, bqT, bsT), W.ref_wgrad(aqT, asT, bqT, bsT))


def test_wgrad_refusals():
    aq, sa, bq, sb = _operands(1, 256, 256, 256)

    def refused(match, *args):
        with pytest.raises(RuntimeError, match=match):
            _ext().block_fp8_wgrad_gemm(*args)
        torch.cuda.synchronize()

    refused('e4m3 operands', aq.view(torch.uint8), sa, bq, sb, 0, 0)
    refused('scale arrays', aq, sa, bq, sb.transpose(1, 2).contiguous(), 0, 0)
    refused('multiples of 128', aq[:, :192].contiguous(), sa[:, :, :192].contiguous(), bq, sb, 0, 0)
    refused('split', aq, sa, bq, sb, 64, 0)
    refused('split', aq, sa, bq, sb, 256, 0)
    buf = torch.zeros(1 + aq.numel(), dtype=torch.uint8, device='cuda')
    refused('16-byte aligned', buf[1:].view(torch.float8_e4m3fn).view(aq.shape), sa, bq, sb, 0, 0)
    with pytest.raises(RuntimeError):
        _ext().block_fp8_quantize_act_dual(torch.zeros(1, 4, 96, dtype=torch.bfloat16, device='cuda'), True)
    R.check('wgrad: after refusals', _wgrad(aq, sa, bq, sb), W.ref_wgrad(aq, sa, bq, sb))


# ------------------------------------------------------------------------------------------------------------------
# expert FFNs, stage by stage
# ------------------------------------------------------------------------------------------------------------------
class _Recorder:
    """Records every launch of ``name`` in ops.block_fp8 (operands and outputs)."""

    def __init__(self, monkeypatch, name):
        from tutel_b200.ops import block_fp8
        self.calls = []
        real = getattr(block_fp8, name)

        def f(*a, **kw):
            out = real(*a, **kw)
            self.calls.append((a, kw, out))
            return out
        monkeypatch.setattr(block_fp8, name, f)


def _check_rowwise(what, q, s, x):
    wq, ws = R.quantize_act(x)
    R.check_scales(what + ' scales', s, ws)
    R.check_bytes(what, q, wq)


def _half(r, sl):
    return R.Ref(r.val[..., sl], r.acc[..., sl], r.S[..., sl], r.other[..., sl])


def _wref(a, b):
    """fp64 bound of ``a^T b`` on the column-wise quantisation of a and b (both [E, C, *])."""
    aqT, asT = W.quantize_act_dual(a)[2:]
    bqT, bsT = W.quantize_act_dual(b)[2:]
    return W.ref_wgrad(aqT, asT, bqT, bsT)


def _check_wgrad_call(what, call, a, b):
    (aqT, asT, bqT, bsT) = call[0][:4]
    _check_dual(what + ' A', (None, None, aqT, asT), a)
    _check_dual(what + ' B', (None, None, bqT, bsT), b)


def _leaves(*ts):
    return [t.detach().clone().requires_grad_() for t in ts]


@pytest.mark.parametrize('E,C,M,H,Mo', [(2, 200, 256, 384, 128), (3, 77, 384, 256, 512)])
def test_relu_ffn_stage_by_stage(monkeypatch, E, C, M, H, Mo):
    from tutel_b200.ops import block_fp8
    g = torch.Generator(device='cuda').manual_seed(C)
    x = torch.randn(E, C, M, generator=g, device='cuda').bfloat16()
    w1 = (torch.randn(E, H, M, generator=g, device='cuda') * M ** -0.5).bfloat16()
    w2 = (torch.randn(E, H, Mo, generator=g, device='cuda') * H ** -0.5).bfloat16()
    b1 = (torch.randn(E, H, generator=g, device='cuda') * 0.1).bfloat16()
    b2 = (torch.randn(E, Mo, generator=g, device='cuda') * 0.1).bfloat16()
    dy = torch.randn(E, C, Mo, generator=g, device='cuda').bfloat16()
    base = _leaves(x, w1, b1, w2, b2)
    y0 = block_fp8.fused_relu_ffn_block_fp8(*base)
    y0.backward(dy)
    leaves = _leaves(x, w1, b1, w2, b2)
    gemms = _Recorder(monkeypatch, 'block_fp8_gemm')
    wgrads = _Recorder(monkeypatch, 'wgrad_gemm')
    y = block_fp8.fused_relu_ffn_block_fp8(*leaves, wgrad=True)
    y.backward(dy)
    what = 'E=%d C=%d M=%d H=%d Mo=%d' % (E, C, M, H, Mo)
    (c_act, c_y, c_dh, c_dx), (c_dw2, c_dw1) = gemms.calls, wgrads.calls
    with torch.no_grad():
        act, dh = c_act[2][0], c_dh[2][0]
        _check_rowwise('x', c_act[0][0], c_act[0][1], x)
        _check_rowwise('act', c_y[0][0], c_y[0][1], act)
        _check_rowwise('dy', c_dh[0][0], c_dh[0][1], dy)
        _check_rowwise('dh', c_dx[0][0], c_dx[0][1], dh)
        _check_wgrad_call('dW2 ' + what, c_dw2, act, dy)
        _check_wgrad_call('dW1 ' + what, c_dw1, dh, x)
        R.check('dw2: ' + what, leaves[3].grad, _wref(act, dy))
        R.check('dw1: ' + what, leaves[1].grad, _wref(dh, x))
        # everything but the weight gradients is that of fp8='block'
        assert torch.equal(_bits(y), _bits(y0)), what
        for i, name in ((0, 'dx'), (2, 'db1'), (4, 'db2')):
            assert torch.equal(_bits(leaves[i].grad), _bits(base[i].grad)), name + ' ' + what
        D.check_colsum('db1 ' + what, leaves[2].grad, dh)
        D.check_colsum('db2 ' + what, leaves[4].grad, dy)


@pytest.mark.parametrize('act', ['silu', 'gelu'])
@pytest.mark.parametrize('E,C,M,H,Mo', [(2, 200, 256, 384, 256), (3, 77, 384, 256, 128)])
def test_glu_ffn_stage_by_stage(monkeypatch, act, E, C, M, H, Mo):
    from tutel_b200.ops import block_fp8
    g_ = torch.Generator(device='cuda').manual_seed(C + H)
    x = torch.randn(E, C, M, generator=g_, device='cuda').bfloat16()
    w1 = (torch.randn(E, M, H, generator=g_, device='cuda') * M ** -0.5).bfloat16()
    w2 = (torch.randn(E, M, H, generator=g_, device='cuda') * M ** -0.5).bfloat16()
    w3 = (torch.randn(E, H, Mo, generator=g_, device='cuda') * H ** -0.5).bfloat16()
    dy = torch.randn(E, C, Mo, generator=g_, device='cuda').bfloat16()
    base = _leaves(x, w1, w2, w3)
    y0 = block_fp8.fused_glu_ffn_block_fp8(*base, act)
    y0.backward(dy)
    leaves = _leaves(x, w1, w2, w3)
    gemms = _Recorder(monkeypatch, 'block_fp8_gemm')
    wgrads = _Recorder(monkeypatch, 'wgrad_gemm')
    y = block_fp8.fused_glu_ffn_block_fp8(*leaves, act, wgrad=True)
    y.backward(dy)
    what = '%s E=%d C=%d M=%d H=%d Mo=%d' % (act, E, C, M, H, Mo)
    (c_glu, c_y, c_dh, c_dx), (c_dw3, c_dw12) = gemms.calls, wgrads.calls
    with torch.no_grad():
        h, dgu = c_glu[2][0], c_dh[2][0]
        _check_rowwise('x', c_glu[0][0], c_glu[0][1], x)
        _check_rowwise('h', c_y[0][0], c_y[0][1], h)
        _check_rowwise('dy', c_dh[0][0], c_dh[0][1], dy)
        _check_rowwise('dgu', c_dx[0][0], c_dx[0][1], dgu)
        _check_wgrad_call('dW3 ' + what, c_dw3, h, dy)
        _check_wgrad_call('dW1|dW2 ' + what, c_dw12, x, dgu)
        assert c_dw12[1].get('split') == H
        R.check('dw3: ' + what, leaves[3].grad, _wref(h, dy))
        r12 = _wref(x, dgu)
        R.check('dw1: ' + what, leaves[1].grad, _half(r12, slice(0, H)))
        R.check('dw2: ' + what, leaves[2].grad, _half(r12, slice(H, 2 * H)))
        assert torch.equal(_bits(y), _bits(y0)), what
        assert torch.equal(_bits(leaves[0].grad), _bits(base[0].grad)), 'dx ' + what


# ------------------------------------------------------------------------------------------------------------------
# the layer
# ------------------------------------------------------------------------------------------------------------------
def _layer(expert, wgrad=True, fp8='block', gate='softmax', shared=False, M=256, H=512, E=8, seed=1, biases=True):
    from tutel_b200 import moe
    spec = {'type': 'top', 'k': 2, 'capacity_factor': 1.0}
    if gate == 'sigmoid':
        spec.update(scoring_func='sigmoid', n_group=4, topk_group=2, routed_scaling_factor=2.5)
    experts = {'type': expert, 'num_experts_per_device': E, 'hidden_size_per_expert': H, 'fp8': fp8}
    if wgrad:
        experts['fp8_wgrad'] = True
    if expert == 'ffn':
        experts.update(activation_fn=lambda t: F.relu(t), has_fc1_bias=biases, has_fc2_bias=biases)
    torch.manual_seed(seed)
    layer = moe.moe_layer(gate_type=spec, model_dim=M, experts=experts, seeds=(seed, seed + 1, seed + 2),
                          shared_experts={'num_experts': 1} if shared else None).cuda().bfloat16()
    if gate == 'sigmoid':
        with torch.no_grad():
            layer.gates[0].e_score_correction_bias.copy_(torch.linspace(-0.05, 0.05, E))
    if expert == 'llama_ffn':
        with torch.no_grad():          # unit-scale hidden activations (the default init gives ~1e-4)
            for n, p in layer.named_parameters():
                if 'W_fc' in n:
                    p.normal_(0, M ** -0.5 if 'fc3' not in n else H ** -0.5)
    return layer


def _loss(y):
    w = torch.linspace(-1, 1, y.size(-1), device=y.device, dtype=torch.float32)
    return (y.float() * w).sum() / y.size(0) + 0.5 * y.l_aux.float()


def _step(layer, x, opt):
    with LR.recording(layer) as recs:
        params = LR.snapshot(layer)
        opt.zero_grad(set_to_none=True)
        xx = x.detach().clone().requires_grad_(True)
        _loss(layer(xx)).backward()
        torch.cuda.synchronize()
        st = LR.make_step(layer, recs[-1], xx, params, xx.grad)
        opt.step()
    return st


def _x(S=512, M=256, seed=0):
    g = torch.Generator(device='cuda').manual_seed(seed)
    return torch.randn(2, S // 2, M, device='cuda', generator=g).bfloat16()


@pytest.mark.parametrize('shared', [False, True], ids=['routed', 'shared'])
@pytest.mark.parametrize('gate', ['softmax', 'sigmoid'])
@pytest.mark.parametrize('expert', ['ffn', 'llama_ffn'])
def test_layer_steps(expert, gate, shared):
    """Two steps with an SGD update of the expert weights in between (step 2 runs on re-quantised weights; the gate is
    left alone, so that its scores stay unsaturated).  Each step starts the ``fp8='block'`` twin from the option's
    weights: y, l_aux, dx and the gate's gradients are bit for bit the twin's; every gradient, the expert weights'
    included, is within the fp64 bound with e4m3 weight-gradient operands."""
    layer = _layer(expert, gate=gate, shared=shared)
    twin = _layer(expert, wgrad=False, gate=gate, shared=shared)

    def expert_params(m):
        return [p for n, p in m.named_parameters() if 'gate' not in n]
    opt = torch.optim.SGD(expert_params(layer), lr=0.5)
    opt_twin = torch.optim.SGD(expert_params(twin), lr=0.5)
    what = '%s %s %s' % (expert, gate, 'shared' if shared else 'routed')
    for i in range(2):
        x = _x(seed=i)
        twin.load_state_dict(layer.state_dict())
        st = _step(layer, x, opt)
        tw = _step(twin, x, opt_twin)
        cfg = LR.config_of(layer, x)
        cfg.fp8 = 'row'
        LW.check_step(cfg, st)
        assert torch.equal(_bits(st.y), _bits(tw.y)), '%s step %d: y' % (what, i)
        assert torch.equal(st.l_aux, tw.l_aux), '%s step %d: l_aux' % (what, i)
        assert torch.equal(_bits(st.dx), _bits(tw.dx)), '%s step %d: dx' % (what, i)
        assert torch.equal(st.dlogits, tw.dlogits), '%s step %d: dlogits' % (what, i)
        for n, gr in st.grads.items():
            if 'gate' in n or 'bias' in n:
                assert (gr is None and tw.grads[n] is None) or torch.equal(gr, tw.grads[n]), '%s step %d: %s' % (what, i, n)
        assert any(not torch.equal(gr, tw.grads[n]) for n, gr in st.grads.items() if gr is not None and ('fc' in n)), \
            what + ': the expert weight gradients come from the e4m3 GEMM'


@pytest.mark.parametrize('expert', ['ffn', 'llama_ffn'])
def test_graphed_train_step_equals_eager(expert):
    from tutel_b200.utils.graph import GraphedTrainStep
    xs = [torch.randn(512, 256, device='cuda', dtype=torch.bfloat16) for _ in range(4)]

    def make():
        layer = _layer(expert, seed=3, biases=False)
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
    for i, (a, b) in enumerate(zip(eager[3:], graphed)):
        assert torch.equal(a, b), i
    for (n, p), (_, q) in zip(eager_layer.state_dict().items(), graph_layer.state_dict().items()):
        assert torch.equal(p, q), n


@pytest.mark.parametrize('expert', ['ffn', 'llama_ffn'])
def test_no_host_sync(expert):
    layer = _layer(expert)
    x = _x().requires_grad_(True)
    _loss(layer(x)).backward()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        _loss(layer(x)).backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()


@pytest.mark.parametrize('expert', ['ffn', 'llama_ffn'])
def test_saved_bytes_are_fewer(expert):
    def saved(wgrad):
        layer = _layer(expert, wgrad=wgrad)
        x = _x(S=1024).requires_grad_(True)
        total = [0]

        def pack(t):
            total[0] += t.numel() * t.element_size()
            return t
        with torch.autograd.graph.saved_tensors_hooks(pack, lambda t: t):
            y = layer(x)
        _loss(y).backward()
        return total[0]
    with_opt, without = saved(True), saved(False)
    print('\nsaved for backward (%s): block %d bytes, block + fp8_wgrad %d bytes' % (expert, without, with_opt))
    assert with_opt < without


@pytest.mark.parametrize('expert', ['ffn', 'llama_ffn'])
def test_training_converges_like_block(expert):
    """A seeded teacher-student regression, 50 SGD steps in bf16, ``block`` and ``block + fp8_wgrad``: the option moves
    the final loss by at most twice what ``block`` moves it from bf16 (plus 0.1 % of the bf16 loss)."""
    M = 256
    gen = torch.Generator(device='cuda').manual_seed(11)
    A = torch.randn(M, M, generator=gen, device='cuda') * M ** -0.5
    B = torch.randn(M, M, generator=gen, device='cuda') * M ** -0.5
    xs = [torch.randn(1024, M, generator=gen, device='cuda') for _ in range(50)]
    x_eval = torch.randn(2048, M, generator=gen, device='cuda')

    def teacher(x):
        return torch.tanh(x @ A) @ B

    def run(fp8, wgrad):
        layer = _layer(expert, wgrad=wgrad, fp8=fp8, seed=5)
        opt = torch.optim.SGD(layer.parameters(), lr=0.2 if expert == 'ffn' else 0.5)
        for x in xs:
            opt.zero_grad(set_to_none=True)
            y = layer(x.bfloat16())
            loss = F.mse_loss(y.float(), teacher(x)) + 0.01 * y.l_aux.float()
            loss.backward()
            opt.step()
        with torch.no_grad():
            return float(F.mse_loss(layer(x_eval.bfloat16()).float(), teacher(x_eval)))
    l_bf16, l_block, l_wgrad = run(None, False), run('block', False), run('block', True)
    print('\n%s final loss: bf16 %.6f, block %.6f, block + fp8_wgrad %.6f' % (expert, l_bf16, l_block, l_wgrad))
    assert abs(l_wgrad - l_block) <= 2 * abs(l_block - l_bf16) + 1e-3 * l_bf16
