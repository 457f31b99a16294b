"""Block-scaled fp8 kernels (csrc/gemm_block_fp8.cu) and experts (``fp8='block'``) against the references of
tests/block_fp8_reference.py and tests/layer_reference.py.

* quantisers, bit for bit: zero, tiny, NaN and +-inf tiles, partial row tiles, and the transposed / SwiGLU weight
  copies as exact rearrangements of the forward copy;
* the GEMM against the fp64 reference with its per-element bound: M around tile edges, K from 128 to 14336, up to 8
  groups, more tiles than SMs, K steps that wrap the 6-stage ring mid-tile, every epilogue, scale exponents over +-30;
* promotion: the block GEMM against the row-scaled e4m3 GEMM on the same operands with all scales 1;
* both expert FFNs stage by stage, whole layer training steps, CUDA-graph replay, host synchronisation, the weight
  cache, and which path each configuration takes.
"""
import pytest
import torch
import torch.nn.functional as F

import block_fp8_reference as R
import dispatch_reference as D
import gemm_reference as GR
import layer_reference as LR

pytestmark = pytest.mark.gpu
PROMOTION = {}


@pytest.fixture(scope='module', autouse=True)
def _report():
    yield
    print('\nblock fp8 normalised errors: %s; C_BLOCK %g; promotion (max|err| block / row, all scales 1): %s' % (
        {k: round(v, 4) for k, v in sorted(R.OBSERVED.items())}, R.C_BLOCK, PROMOTION))


def _ext():
    from tutel_b200.ops import backend
    return backend.require_ext()


def _bits(t):
    return t.view(torch.int16)


# ------------------------------------------------------------------------------------------------------------------
# quantisers
# ------------------------------------------------------------------------------------------------------------------
def _special(G, R_, K, seed=0):
    """Random 1 x 128 tiles spread over 2^+-20, plus a zero tile, a tile of values below 448 * FLT_MIN, a tile with NaN
    and one with +-inf (where the shape has room)."""
    gen = torch.Generator().manual_seed(seed)
    spread = torch.exp2(torch.randint(-20, 20, (G, R_, K // 128, 1), generator=gen).float())
    x = (torch.randn(G, R_, K // 128, 128, generator=gen) * spread).view(G, R_, K)
    x[0, 0, :128] = 0
    x[0, 0, 5] = -0.0
    if K >= 256:
        x[0, 0, 128:256] = torch.randn(128, generator=gen) * 1e-37
    x[G - 1, R_ - 1, 7] = float('nan')
    x[G - 1, R_ - 1, 9] = float('-nan')
    if R_ > 1:
        x[G - 1, R_ // 2, 3] = float('inf')
        x[G - 1, R_ // 2, K - 1] = float('-inf')
    return x.bfloat16()


@pytest.mark.parametrize('G,rows,K', [(1, 1, 128), (1, 127, 256), (3, 129, 384), (2, 300, 512), (1, 128, 1024)])
def test_quantize_act_is_bit_exact(G, rows, K):
    x = _special(G, rows, K, seed=rows).cuda()
    q, s = _ext().block_fp8_quantize_act(x)
    wq, ws = R.quantize_act(x)
    R.check_scales('act scales %s' % ((G, rows, K),), s, ws)
    R.check_bytes('act %s' % ((G, rows, K),), q, wq, x)
    assert bool((s[:, :, rows:] == 0).all()), 'pad rows must have scale 0'


def _weight_values(G, R_, C, seed):
    x = _special(G, R_, C, seed).float()
    # one whole 128 x 128 block of tiny values, and one of zeros
    x[0, :128, :128] = torch.randn(128, 128) * 1e-37
    if C > 128:
        x[0, :128, 128:256] = 0
    return x.bfloat16()


@pytest.mark.parametrize('G,rows,cols', [(1, 128, 128), (3, 256, 384), (2, 384, 256)])
def test_quantize_weight_both_orientations(G, rows, cols):
    w = _weight_values(G, rows, cols, seed=cols).cuda()
    q, s, qT, sT = _ext().block_fp8_quantize_weight(w)
    wq, ws = R.quantize_weight(w)
    R.check_scales('weight scales', s, ws)
    R.check_bytes('weight', q, wq, w)
    # the transposed copy is the forward copy transposed, byte for byte, with transposed scales
    assert torch.equal(qT.view(torch.uint8), q.view(torch.uint8).transpose(1, 2).contiguous())
    assert torch.equal(sT, s.transpose(1, 2).contiguous())


@pytest.mark.parametrize('G,M,H', [(1, 128, 128), (2, 256, 384)])
def test_quantize_glu_weight_layouts(G, M, H):
    w1 = _weight_values(G, M, H, seed=1).cuda()
    w2 = _weight_values(G, M, H, seed=2).cuda() * 3
    qcat, scat, qglu, sglu = _ext().block_fp8_quantize_glu_weight(w1, w2)
    (q1, s1), (q2, s2) = R.quantize_weight(w1), R.quantize_weight(w2)
    R.check_bytes('glu cat', qcat, torch.cat([q1, q2], dim=2))
    R.check_scales('glu cat scales', scat, torch.cat([s1, s2], dim=2))
    n = torch.arange(2 * H, device='cuda')
    which, col = R.glu_rows(n, H)
    qt = torch.stack([q1.transpose(1, 2), q2.transpose(1, 2)])           # [2, G, H, M]
    R.check_bytes('glu interleaved', qglu, qt[which, :, col].transpose(0, 1).contiguous())
    st = torch.stack([s1.transpose(1, 2), s2.transpose(1, 2)])           # [2, G, H / 128, M / 128]
    R.check_scales('glu interleaved scales', sglu, st[which[::64], :, col[::64] // 128].transpose(0, 1).contiguous())


# ------------------------------------------------------------------------------------------------------------------
# GEMM
# ------------------------------------------------------------------------------------------------------------------
def _gemm(aq, sa, bq, sb, bias=None, aux=None, aux2=None, epilogue=R.EPI_NONE, act='silu', max_ctas=0):
    return _ext().block_fp8_gemm(aq, sa, bq, sb, bias, aux, aux2, epilogue, R.ACT[act], max_ctas)


# (G, M, N, K, max_ctas).  K = 640, 768, 896 are 5, 6 (= STAGES) and 7 K steps: with several tiles per CTA the ring wraps
# mid-tile; (8, 1024, 1024, ...) is 512 tiles, more than an H100 has SMs.
CASES = [
    (1, 1, 128, 128, 0), (3, 1, 384, 4096, 1), (1, 127, 1152, 640, 3), (3, 127, 128, 896, 7),
    (1, 129, 128, 14336, 3), (3, 129, 384, 768, 7), (2, 300, 256, 896, 0), (1, 300, 384, 128, 2),
    (8, 1024, 1024, 896, 0), (8, 257, 256, 4096, 5), (1, 9 * 128 + 5, 1152, 896, 0), (2, 17 * 128, 384, 14336, 0),
]


@pytest.mark.parametrize('G,M,N,K,max_ctas', CASES)
def test_gemm_matches_fp64_reference(G, M, N, K, max_ctas):
    aq, sa, bq, sb = R.operands(G, M, N, K, seed=M + N + K, device='cuda')
    what = 'gemm: G=%d M=%d N=%d K=%d max_ctas=%d' % (G, M, N, K, max_ctas)
    r = R.ref_gemm(aq, sa, bq, sb)
    d = _gemm(aq, sa, bq, sb, max_ctas=max_ctas)[0]
    R.check(what, d, r[0])
    bias, aux = R.bias_aux(r[0].val)
    for epi, b, name in ((R.EPI_NONE, bias, 'bias'), (R.EPI_RELU, bias, 'bias+relu'), (R.EPI_RELU, None, 'relu'),
                         (R.EPI_RELU_BWD, None, 'relu_bwd')):
        a_ = aux if epi == R.EPI_RELU_BWD else None
        got = _gemm(aq, sa, bq, sb, bias=b, aux=a_, epilogue=epi, max_ctas=max_ctas)
        R.check_all('%s %s' % (what, name), got, R.ref_gemm(aq, sa, bq, sb, bias=b, aux=a_, epilogue=epi))
        if epi == R.EPI_RELU_BWD:
            assert torch.equal(_bits(got[0]), _bits(torch.where(aux > 0, d, torch.zeros_like(d))))
    # a fixed K order and no atomics: another CTA count gives the same bits
    if G * M * N <= 8 * 1024 * 1024:
        assert torch.equal(_bits(_gemm(aq, sa, bq, sb, max_ctas=(max_ctas % 5) + 1)[0]), _bits(d)), what


@pytest.mark.parametrize('act', ['silu', 'gelu', 'relu'])
@pytest.mark.parametrize('G,M,N,K', [(2, 300, 256, 896), (1, 129, 768, 4096), (8, 127, 256, 128)])
def test_gemm_glu_epilogues(act, G, M, N, K):
    aq, sa, bq, sb = R.operands(G, M, N, K, spread=3, seed=K + M, device='cuda', glu=True)
    what = 'glu: %s G=%d M=%d N=%d K=%d' % (act, G, M, N, K)
    outs = _gemm(aq, sa, bq, sb, epilogue=R.EPI_GLU, act=act)
    R.check_all(what, outs, R.ref_gemm(aq, sa, bq, sb, epilogue=R.EPI_GLU, act=act))
    # backward: acc = dh [G, M, N'] with g, u of that shape (plain B scales)
    aq, sa, bq, sb = R.operands(G, M, N, K, spread=3, seed=K + M + 1, device='cuda')
    g = (torch.randn(G, M, N, device='cuda') * 2).bfloat16()
    u = torch.randn(G, M, N, device='cuda').bfloat16()
    outs = _gemm(aq, sa, bq, sb, aux=g, aux2=u, epilogue=R.EPI_GLU_BWD, act=act)
    assert outs[0].shape == (G, M, 2 * N)
    R.check_all('glu_bwd: ' + what, outs, R.ref_gemm(aq, sa, bq, sb, aux=g, aux2=u, epilogue=R.EPI_GLU_BWD, act=act))


def test_gemm_refusals():
    aq, sa, bq, sb = R.operands(1, 128, 384, 256, device='cuda')

    def refused(match, *args, **kw):
        with pytest.raises(RuntimeError, match=match):
            _gemm(*args, **kw)
        torch.cuda.synchronize()

    refused('e4m3 operands', aq.view(torch.uint8), sa, bq, sb)
    refused('scale arrays', aq, sa[:, :1].contiguous(), bq, sb)
    refused('scale arrays', aq, sa, bq, sb.transpose(1, 2).contiguous())
    refused('N must be a multiple of 128', aq, sa, bq[:, :192].contiguous(), torch.ones(1, 2, 2, device='cuda'))
    a192 = aq[..., :192].contiguous()
    refused('K must be a multiple of 128', a192, sa[:, :2].contiguous(), bq[..., :192].contiguous(), sb[:, :, :2].contiguous())
    buf = torch.zeros(1 + aq.numel(), dtype=torch.uint8, device='cuda')
    refused('16-byte aligned', buf[1:].view(torch.float8_e4m3fn).view(aq.shape), sa, bq, sb)
    refused('aux', aq, sa, bq, sb, epilogue=R.EPI_RELU_BWD)
    refused('aux2', aq, sa, bq, sb, aux=torch.zeros(1, 128, 384, dtype=torch.bfloat16, device='cuda'), epilogue=R.EPI_GLU_BWD)
    refused('aux must be a contiguous bf16', aq, sa, bq, sb, aux=torch.zeros(1, 128, 384, device='cuda'), epilogue=R.EPI_RELU_BWD)
    refused('bias must be a contiguous bf16', aq, sa, bq, sb, bias=torch.zeros(1, 256, dtype=torch.bfloat16, device='cuda'))
    refused('unknown epilogue', aq, sa, bq, sb, epilogue=7)
    with pytest.raises(RuntimeError):
        _ext().block_fp8_quantize_act(torch.zeros(1, 4, 96, dtype=torch.bfloat16, device='cuda'))
    with pytest.raises(RuntimeError):
        _ext().block_fp8_quantize_weight(torch.zeros(1, 128, 128, dtype=torch.float16, device='cuda'))
    R.check('gemm: after refusals', _gemm(aq, sa, bq, sb)[0], R.ref_gemm(aq, sa, bq, sb)[0])


@pytest.mark.parametrize('K', [4096, 14336])
def test_promotion_beats_row_scaled_accumulation(K):
    """The same e4m3 operands with every scale 1: the block GEMM (fp32 promotion every 128 K) and the row-scaled GEMM
    (the whole K in the tensor core's accumulator) compute the same exact product; the block GEMM's largest error
    against fp64 must be the smaller."""
    from tutel_b200.ops import gemm
    G, M, N = 1, 512, 512
    gen = torch.Generator(device='cuda').manual_seed(K)
    a = (torch.randn(G, M, K, generator=gen, device='cuda') * 64).clamp(-448, 448).to(torch.float8_e4m3fn)
    b = (torch.randn(G, N, K, generator=gen, device='cuda') * 64).clamp(-448, 448).to(torch.float8_e4m3fn)
    exact = a.double() @ b.double().transpose(1, 2)
    ones_a = torch.ones(G, K // 128, M, device='cuda')
    ones_b = torch.ones(G, N // 128, K // 128, device='cuda')
    blk = _gemm(a, ones_a, b, ones_b)[0]
    row = gemm.raw_gemm(a, b, out_dtype=torch.float32, scale_a=torch.ones(G, M, device='cuda'),
                        scale_b=torch.ones(G, N, device='cuda'))
    # compare before the bf16 rounding of the block kernel's output: both errors in units of max |ref|
    e_blk = float((blk.double() - exact).abs().max()) / float(exact.abs().max())
    e_row = float((row.double() - exact).abs().max()) / float(exact.abs().max())
    # the block kernel rounds to bf16: measure its accumulation error net of that rounding
    rnd = float(GR.half_ulp(exact.abs(), torch.bfloat16).max()) / float(exact.abs().max())
    PROMOTION[K] = {'block': e_blk, 'block_rounding': rnd, 'row_fp32_out': e_row}
    blk32 = R.ref_gemm(a.view(torch.uint8), ones_a, b.view(torch.uint8), ones_b)[0]
    R.check('promotion K=%d' % K, blk, blk32)
    # both kernels' accumulation error: the block kernel's is what is left after its bf16 rounding
    net_blk = float(((blk.double() - exact).abs() - GR.half_ulp(exact, torch.bfloat16)).clamp_min(0).max())
    net_row = float((row.double() - exact).abs().max())
    PROMOTION[K]['ratio'] = net_blk / net_row if net_row else float('nan')
    assert net_blk < net_row, PROMOTION[K]


# ------------------------------------------------------------------------------------------------------------------
# expert FFNs, stage by stage
# ------------------------------------------------------------------------------------------------------------------
def _check_copy(what, q, s, x):
    """q, s must be the activation quantisation of x, bit for bit."""
    wq, ws = R.quantize_act(x)
    R.check_scales(what + ' scales', s, ws)
    R.check_bytes(what, q, wq)


class _Recorder:
    """Records every block_fp8_gemm launch (its operands and outputs)."""

    def __init__(self, monkeypatch):
        from tutel_b200.ops import block_fp8
        self.calls = []
        real = block_fp8.block_fp8_gemm

        def f(*a, **kw):
            out = real(*a, **kw)
            self.calls.append((a, kw, out))
            return out
        monkeypatch.setattr(block_fp8, 'block_fp8_gemm', f)


@pytest.mark.parametrize('E,C,M,H,Mo', [(2, 200, 256, 384, 128), (3, 77, 384, 256, 512)])
def test_relu_ffn_stage_by_stage(monkeypatch, E, C, M, H, Mo):
    from tutel_b200.ops import block_fp8
    g = torch.Generator(device='cuda').manual_seed(C)
    x = torch.randn(E, C, M, generator=g, device='cuda').bfloat16().requires_grad_()
    w1 = (torch.randn(E, H, M, generator=g, device='cuda') * M ** -0.5).bfloat16().requires_grad_()
    w2 = (torch.randn(E, H, Mo, generator=g, device='cuda') * H ** -0.5).bfloat16().requires_grad_()
    b1 = (torch.randn(E, H, generator=g, device='cuda') * 0.1).bfloat16().requires_grad_()
    b2 = (torch.randn(E, Mo, generator=g, device='cuda') * 0.1).bfloat16().requires_grad_()
    rec = _Recorder(monkeypatch)
    y = block_fp8.fused_relu_ffn_block_fp8(x, w1, b1, w2, b2)
    dy = torch.randn(y.shape, generator=g, device='cuda').bfloat16()
    y.backward(dy)
    what = 'E=%d C=%d M=%d H=%d Mo=%d' % (E, C, M, H, Mo)
    (c_act, c_y, c_dh, c_dx) = rec.calls
    with torch.no_grad():
        q1, s1 = R.quantize_weight(w1)
        q2, s2 = R.quantize_weight(w2)
        act = c_act[2][0]
        # each launch's operands: the quantisation of the stage's real input, and the right weight copy
        _check_copy('x', c_act[0][0], c_act[0][1], x)
        R.check_bytes('W1', c_act[0][2], q1)
        _check_copy('act', c_y[0][0], c_y[0][1], act)
        R.check_bytes('W2^T', c_y[0][2], q2.transpose(1, 2).contiguous())
        R.check_scales('W2^T scales', c_y[0][3], s2.transpose(1, 2).contiguous())
        _check_copy('dy', c_dh[0][0], c_dh[0][1], dy)
        R.check_bytes('W2', c_dh[0][2], q2)
        dh = c_dh[2][0]
        _check_copy('dh', c_dx[0][0], c_dx[0][1], dh)
        R.check_bytes('W1^T', c_dx[0][2], q1.transpose(1, 2).contiguous())
        R.check_scales('W1^T scales', c_dx[0][3], s1.transpose(1, 2).contiguous())
        # each stage against its fp64 reference
        xq, xs = R.quantize_act(x)
        R.check('act: ' + what, act, R.ref_gemm(xq, xs, q1, s1, bias=b1, epilogue=R.EPI_RELU)[0])
        aq, as_ = R.quantize_act(act)
        R.check('y: ' + what, y, R.ref_gemm(aq, as_, q2.transpose(1, 2).contiguous(), s2.transpose(1, 2).contiguous(), bias=b2)[0])
        dq, ds = R.quantize_act(dy)
        R.check('dh: ' + what, dh, R.ref_gemm(dq, ds, q2, s2, aux=act, epilogue=R.EPI_RELU_BWD)[0])
        hq, hs = R.quantize_act(dh)
        R.check('dx: ' + what, x.grad, R.ref_gemm(hq, hs, q1.transpose(1, 2).contiguous(), s1.transpose(1, 2).contiguous())[0])
        GR.check(GR.ref_gemm(dh, x, a_mn=True, b_mn=True), w1.grad, what='dw1: ' + what)
        GR.check(GR.ref_gemm(act, dy, a_mn=True, b_mn=True), w2.grad, what='dw2: ' + what)
        D.check_colsum('db1 ' + what, b1.grad, dh)
        D.check_colsum('db2 ' + what, b2.grad, dy)


@pytest.mark.parametrize('act', ['silu', 'gelu'])
@pytest.mark.parametrize('E,C,M,H,Mo', [(2, 200, 256, 384, 256), (3, 77, 384, 256, 128)])
def test_glu_ffn_stage_by_stage(monkeypatch, act, E, C, M, H, Mo):
    from tutel_b200.ops import block_fp8
    g_ = torch.Generator(device='cuda').manual_seed(C + H)
    x = torch.randn(E, C, M, generator=g_, device='cuda').bfloat16().requires_grad_()
    w1 = (torch.randn(E, M, H, generator=g_, device='cuda') * M ** -0.5).bfloat16().requires_grad_()
    w2 = (torch.randn(E, M, H, generator=g_, device='cuda') * M ** -0.5).bfloat16().requires_grad_()
    w3 = (torch.randn(E, H, Mo, generator=g_, device='cuda') * H ** -0.5).bfloat16().requires_grad_()
    rec = _Recorder(monkeypatch)
    y = block_fp8.fused_glu_ffn_block_fp8(x, w1, w2, w3, act)
    dy = torch.randn(y.shape, generator=g_, device='cuda').bfloat16()
    y.backward(dy)
    what = '%s E=%d C=%d M=%d H=%d Mo=%d' % (act, E, C, M, H, Mo)
    (c_glu, c_y, c_dh, c_dx) = rec.calls
    with torch.no_grad():
        (q1, s1), (q2, s2), (q3, s3) = R.quantize_weight(w1), R.quantize_weight(w2), R.quantize_weight(w3)
        h, g, u = c_glu[2]
        _check_copy('x', c_glu[0][0], c_glu[0][1], x)
        xq, xs = R.quantize_act(x)
        qglu, sglu = c_glu[0][2], c_glu[0][3]
        # the forward operand: gate / up columns interleaved every 64 (checked against W1^T / W2^T by its reference)
        n = torch.arange(2 * H, device='cuda')
        which, col = R.glu_rows(n, H)
        R.check_bytes('W1|W2 interleaved', qglu, torch.stack([q1.transpose(1, 2), q2.transpose(1, 2)])[which, :, col].transpose(0, 1).contiguous())
        R.check_all('glu: ' + what, [h, g, u], R.ref_gemm(xq, xs, qglu, sglu, epilogue=R.EPI_GLU, act=act))
        _check_copy('h', c_y[0][0], c_y[0][1], h)
        hq, hs = R.quantize_act(h)
        q3t, s3t = q3.transpose(1, 2).contiguous(), s3.transpose(1, 2).contiguous()
        R.check_bytes('W3^T', c_y[0][2], q3t)
        R.check('y: ' + what, y, R.ref_gemm(hq, hs, q3t, s3t)[0])
        _check_copy('dy', c_dh[0][0], c_dh[0][1], dy)
        R.check_bytes('W3', c_dh[0][2], q3)
        dgu = c_dh[2][0]
        dq, ds = R.quantize_act(dy)
        R.check_all('dgu: ' + what, [dgu], R.ref_gemm(dq, ds, q3, s3, aux=g, aux2=u, epilogue=R.EPI_GLU_BWD, act=act))
        _check_copy('dgu', c_dx[0][0], c_dx[0][1], dgu)
        R.check_bytes('[W1 W2]', c_dx[0][2], torch.cat([q1, q2], dim=2))
        R.check_scales('[W1 W2] scales', c_dx[0][3], torch.cat([s1, s2], dim=2))
        gq, gs = R.quantize_act(dgu)
        R.check('dx: ' + what, x.grad, R.ref_gemm(gq, gs, torch.cat([q1, q2], dim=2), torch.cat([s1, s2], dim=2))[0])
        dg, du = dgu[..., :H], dgu[..., H:]
        GR.check(GR.ref_gemm(x, dg, a_mn=True, b_mn=True), w1.grad, what='dw1: ' + what)
        GR.check(GR.ref_gemm(x, du, a_mn=True, b_mn=True), w2.grad, what='dw2: ' + what)
        GR.check(GR.ref_gemm(h, dy, a_mn=True, b_mn=True), w3.grad, what='dw3: ' + what)


# ------------------------------------------------------------------------------------------------------------------
# the layer
# ------------------------------------------------------------------------------------------------------------------
def _layer(expert, fp8='block', act=F.relu, M=256, H=512, E=8, cf=1.0, seed=1, dtype=torch.bfloat16, biases=True):
    from tutel_b200 import moe
    if expert == 'llama_ffn':
        experts = {'type': 'llama_ffn', 'num_experts_per_device': E, 'hidden_size_per_expert': H, 'fp8': fp8,
                   'activation_fn': act if act is not F.relu else F.silu}
    else:
        experts = {'type': 'ffn', 'num_experts_per_device': E, 'hidden_size_per_expert': H, 'fp8': fp8,
                   'activation_fn': lambda t: act(t), 'has_fc1_bias': biases, 'has_fc2_bias': biases}
    torch.manual_seed(seed)
    layer = moe.moe_layer(gate_type={'type': 'top', 'k': 2, 'capacity_factor': cf}, model_dim=M, experts=experts,
                          seeds=(seed, seed + 1, seed + 2)).cuda().to(dtype)
    if expert == 'llama_ffn':
        with torch.no_grad():          # unit-scale hidden activations (the default init gives ~1e-4)
            for n, p in layer.named_parameters():
                if 'W_fc' in n:
                    p.normal_(0, M ** -0.5 if 'fc3' not in n else H ** -0.5)
    return layer


def _loss(y, t=None):
    w = torch.linspace(-1, 1, y.size(-1), device=y.device, dtype=torch.float32)
    return (y.float() * w).sum() / y.size(0) + 0.5 * y.l_aux.float()


def _steps(layer, x, steps=1, graphed=False, lr=0.0):
    from tutel_b200.utils.graph import GraphedTrainStep
    opt = torch.optim.SGD(layer.parameters(), lr=lr)
    t = torch.zeros(1, device='cuda')

    def step_fn(xx, tt):
        opt.zero_grad(set_to_none=True)
        xx.grad = None
        loss = _loss(layer(xx))
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


def _x(S=512, M=256, seed=0):
    g = torch.Generator(device='cuda').manual_seed(seed)
    return torch.randn(2, S // 2, M, device='cuda', generator=g).bfloat16().requires_grad_(True)


class _Spy:
    def __init__(self, monkeypatch):
        from tutel_b200.ops import block_fp8
        self.calls = {'relu': 0, 'glu': 0}
        for name, key in (('fused_relu_ffn_block_fp8', 'relu'), ('fused_glu_ffn_block_fp8', 'glu')):
            real = getattr(block_fp8, name)

            def f(*a, _real=real, _key=key, **kw):
                self.calls[_key] += 1
                return _real(*a, **kw)
            monkeypatch.setattr(block_fp8, name, f)


@pytest.mark.parametrize('expert', ['ffn', 'llama_ffn'])
def test_layer_training_steps_match_fp64_reference(monkeypatch, expert):
    """Two steps with an SGD update in between; the e4m3 operand bound of the row recipe (row / column maxima, never
    below a block's maximum) covers block scales.  Step 2 runs on re-quantised weights."""
    spy = _Spy(monkeypatch)
    layer = _layer(expert)
    x = _x()
    steps = _steps(layer, x, steps=2, lr=0.5)
    assert spy.calls['relu' if expert == 'ffn' else 'glu'] == 2
    for st in steps:
        cfg = LR.config_of(layer, x)
        cfg.fp8 = 'row'
        LR.check_step(cfg, st)


@pytest.mark.parametrize('expert', ['ffn', 'llama_ffn'])
def test_graphed_train_step_equals_eager(expert):
    """Several SGD steps replayed from a ``GraphedTrainStep`` give the eager losses and weights bit for bit (weight
    copies are re-quantised inside the graph).  The ffn experts have no biases here: their gradients are fp32 atomic
    column sums, whose order is not fixed."""
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
    eager = [eager_step(x).clone() for x in [xs[0]] * 3 + xs]      # the same warm-up the graph runs
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
    x = _x()
    _loss(layer(x)).backward()                 # warm-up (lazy initialisation, weight copies)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        _loss(layer(x)).backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()


@pytest.mark.parametrize('update', ['optimizer_step', 'no_grad_inplace'])
@pytest.mark.parametrize('expert', ['ffn', 'llama_ffn'])
def test_weight_copies_follow_updates(update, expert):
    """After an update the next forward equals that of a fresh layer holding the new weights, bit for bit."""
    layer = _layer(expert)
    x = _x()
    y0 = layer(x)
    if update == 'optimizer_step':
        opt = torch.optim.SGD(layer.parameters(), lr=1.0)
        _loss(y0).backward()
        opt.step()
    else:
        with torch.no_grad():
            for p in layer.parameters():
                p.mul_(-0.5)
    with torch.no_grad():
        y = layer(x)
        fresh = _layer(expert, seed=7)
        fresh.load_state_dict(layer.state_dict())
        assert torch.equal(_bits(y), _bits(fresh(x)))
        assert not torch.equal(_bits(y), _bits(y0.detach()))


def test_paths_and_fallbacks(monkeypatch):
    spy = _Spy(monkeypatch)
    x = torch.randn(2, 100, 256, device='cuda', dtype=torch.bfloat16)

    def ffn(act=F.relu, H=256, dtype=torch.bfloat16):
        from tutel_b200.models.experts.ffn import FusedExpertsNetwork
        return FusedExpertsNetwork(model_dim=256, hidden_size_per_expert=H, num_experts_per_device=2, sharded_count=1,
                                   activation_fn=lambda t: act(t), fp8='block').cuda().to(dtype)

    def run(ex, xx, **kw):
        return ex.compute(xx, ex.batched_fc1_w, ex.batched_fc1_bias, ex.batched_fc2_w, ex.batched_fc2_bias, **kw)

    run(ffn(), x)
    assert spy.calls['relu'] == 1
    for ex, xx, why in ((ffn(act=F.gelu), x, 'GELU'), (ffn(act=F.silu), x, 'SiLU'), (ffn(H=192), x, 'H % 128'),
                        (ffn(dtype=torch.float16), x.half(), 'fp16'), (ffn(dtype=torch.float32), x.float(), 'fp32')):
        run(ex, xx)
        assert spy.calls['relu'] == 1, why
    run(ffn(), x, row_counts=torch.tensor([3, 5], dtype=torch.int32, device='cuda'))
    assert spy.calls['relu'] == 1, 'row_counts'
    assert not ffn().supports_packed(x)

    xl = _x(S=256)
    _layer('llama_ffn')(xl)
    assert spy.calls['glu'] == 1
    _layer('llama_ffn', act=F.gelu)(xl)
    assert spy.calls['glu'] == 2, 'GELU has an epilogue'
    for layer, xx, why in ((_layer('llama_ffn', act=lambda t: torch.tanh(t)), xl, 'custom activation'),
                           (_layer('llama_ffn', H=192), xl, 'H % 128'),
                           (_layer('llama_ffn', dtype=torch.float16), xl.half(), 'fp16')):
        layer(xx)
        assert spy.calls['glu'] == 2, why
    with torch.no_grad():                      # dropless decoding: the 16-bit kernels
        _layer('llama_ffn')(xl[:1, :4], megablocks_size=1)
    assert spy.calls['glu'] == 2, 'dropless decoding'
    assert not _layer('llama_ffn').experts.supports_packed(xl)
    # a dropless training step stays on the padded layout (supports_packed is False) and takes the block path
    for expert, key in (('ffn', 'relu'), ('llama_ffn', 'glu')):
        layer = _layer(expert, cf=0.0)
        before = spy.calls[key]
        with LR.recording(layer) as recs:
            y = layer(_x())
        assert getattr(recs[-1]['crit'], 'layout', None) is None, expert
        assert spy.calls[key] == before + 1, expert
        _loss(y).backward()
