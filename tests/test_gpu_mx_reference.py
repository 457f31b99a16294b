"""MX block-scaled fp8 kernels (csrc/gemm_mx.cu) against the references of tests/mx_reference.py.

* quantisers, bit for bit: special values, row tails, groups, K % 128 != 0 for the transposing kernel, and every
  positive bf16 / fp16 value as a block maximum;
* the GEMM against the fp64 reference with its per-element bound, at shapes that give partial 8-tile bands, K steps
  that wrap the 6-stage ring at a different step on each tile, persistent CTAs that walk many tiles, every epilogue,
  and scale exponents that differ from block to block; bit-identical results across launch hints, CTA counts and
  repeated launches; the launcher's and the binding's refusals;
* ``FusedReluFFNMx`` stage by stage, each output against the reference of its own stage built from its real inputs;
* the expert layer's path selection and its MX weight cache.
"""
import pytest
import torch
import torch.nn.functional as F

import dispatch_reference as D
import gemm_reference as GR
import mx_reference as R

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module', autouse=True)
def _report():
    yield
    print('\nmx normalised errors: %s; C_ACC[e4m3] %g; gemm_reference (bf16 weight gradients): %s; colsum: %s' % (
        {k: round(v, 4) for k, v in sorted(R.OBSERVED.items())}, R.C_MMA,
        {str(k): round(v, 4) for k, v in GR.OBSERVED.items()}, D.OBSERVED.get('colsum')))


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip('needs an H100')


def _ext():
    from tutel_b200.ops import backend
    return backend.require_ext()


def _q(t):
    """Reference quantisation of a CUDA tensor [G, R, K]: (e4m3 bytes, scales)."""
    q, sf, _ = R.quantize(t)
    return q, sf


# ------------------------------------------------------------------------------------------------------------------
# quantisers
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16])
@pytest.mark.parametrize('G,rows,K', [(1, 1, 128), (1, 127, 256), (3, 129, 384), (2, 300, 512), (1, 130, 1024)])
def test_mx_quantize_is_bit_exact(dtype, G, rows, K):
    _need_gpu()
    x = R.special_values(dtype, G, rows, K, seed=rows).cuda()
    q, sf = _ext().mx_quantize(x)
    R.check_quantized('mx_quantize %s' % ((G, rows, K),), q, sf, x)


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16])
def test_mx_quantize_every_positive_value_as_block_maximum(dtype):
    _need_gpu()
    x = R.every_positive(dtype).cuda()
    q, sf = _ext().mx_quantize(x)
    R.check_quantized('mx_quantize, every positive %s' % dtype, q, sf, x)
    # the transposing kernel computes the exponent on its own: the same values as its columns
    rows = x.size(1) - x.size(1) % 128
    xt = x[:, :rows].transpose(1, 2).contiguous()                                   # [1, 128, rows]
    q, sf = _ext().mx_quantize_transpose(xt)
    R.check_quantized('mx_quantize_transpose, every positive %s' % dtype, q, sf, x[:, :rows])


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16])
@pytest.mark.parametrize('G,rows,K', [(1, 128, 64), (3, 256, 192), (2, 384, 256), (1, 128, 320)])
def test_mx_quantize_transpose_is_bit_exact(dtype, G, rows, K):
    """x [G, rows, K] -> the MX copy of x^T [G, K, rows]; with K % 128 != 0 the pad rows of the scales are byte 0."""
    _need_gpu()
    xt = R.special_values(dtype, G, K, rows, seed=K).cuda()                         # the operand: [G, K, rows]
    x = xt.transpose(1, 2).contiguous()
    q, sf = _ext().mx_quantize_transpose(x)
    assert q.shape == (G, K, rows)
    R.check_quantized('mx_quantize_transpose %s' % ((G, rows, K),), q, sf, xt)


# ------------------------------------------------------------------------------------------------------------------
# GEMM
# ------------------------------------------------------------------------------------------------------------------
def _gemm(aq, sfa, bq, sfb, bias=None, aux=None, epilogue=R.EPI_NONE, block_n=0, cta_group=0, max_ctas=0):
    return _ext().mx_gemm(aq, sfa, bq, sfb, bias, aux, epilogue, block_n, cta_group, max_ctas)


def _bits(t):
    return t.view(torch.int16)


# (G, M, N, K, max_ctas).  M = 9 * 128 + 5 and 17 * 128 leave a partial band of 8 row tiles; K = 640, 768, 896 are 5, 6
# (= STAGES) and 7 K steps, 4096 and 14336 are 32 and 112: with several tiles per CTA the ring wraps mid-tile.
CASES = [
    (1, 1, 128, 128, 0), (3, 1, 384, 4096, 1), (1, 127, 1152, 640, 3), (3, 127, 128, 896, 7),
    (1, 128, 384, 768, 1), (3, 128, 1152, 128, 0), (1, 129, 128, 14336, 3), (3, 129, 384, 768, 7),
    (1, 9 * 128 + 5, 1152, 896, 0), (3, 9 * 128 + 5, 384, 640, 3), (1, 9 * 128 + 5, 128, 4096, 7),
    (1, 17 * 128, 384, 14336, 0), (3, 17 * 128, 1152, 768, 7), (1, 17 * 128, 128, 896, 1), (3, 9 * 128 + 5, 1152, 4096, 0),
]


@pytest.mark.parametrize('G,M,N,K,max_ctas', CASES)
def test_mx_gemm_matches_fp64_reference(G, M, N, K, max_ctas):
    _need_gpu()
    aq, sfa, bq, sfb = R.operands(G, M, N, K, seed=M + N + K, device='cuda')
    r = R.ref_gemm(aq, sfa, bq, sfb)
    what = 'gemm: G=%d M=%d N=%d K=%d max_ctas=%d' % (G, M, N, K, max_ctas)
    d = _gemm(aq, sfa, bq, sfb, max_ctas=max_ctas)
    R.check(what, d, r)
    bias, aux = R.bias_aux(r.val)
    for epi, b, name in ((R.EPI_NONE, bias, 'bias'), (R.EPI_RELU, bias, 'bias+relu'), (R.EPI_RELU, None, 'relu'),
                         (R.EPI_RELU_BWD, None, 'relu_bwd')):
        got = _gemm(aq, sfa, bq, sfb, bias=b, aux=aux if epi == R.EPI_RELU_BWD else None, epilogue=epi, max_ctas=max_ctas)
        R.check('%s %s' % (what, name), got, R.ref_gemm(aq, sfa, bq, sfb, bias=b, aux=aux, epilogue=epi))
        if epi == R.EPI_RELU_BWD:          # the mask alone: the plain result where aux > 0, exactly 0 elsewhere
            assert torch.equal(_bits(got), _bits(torch.where(aux > 0, d, torch.zeros_like(d))))
    # no atomics and a fixed K order: every CTA count and a second launch give the same bits
    for m in sorted({0, 1, 3, 7} - {max_ctas}) if M * N * G <= 384 * 1152 else [max_ctas]:
        assert torch.equal(_bits(_gemm(aq, sfa, bq, sfb, max_ctas=m)), _bits(d)), (what, m)


@pytest.mark.parametrize('G,M,N,K', [(1, 300, 384, 896), (3, 9 * 128 + 5, 1152, 4096)])
def test_mx_gemm_is_exact_on_integer_operands(G, M, N, K):
    """Integers in [-8, 8] with exponents in [-2, 2]: every partial sum is exact in fp32, so the output is the bf16
    rounding of the exact result.  This is the check a kernel that rounded partial sums to bf16 would fail."""
    _need_gpu()
    ops = R.integer_operands(G, M, N, K, seed=K, device='cuda')
    R.check_exact('gemm, integer operands', _gemm(*ops), *ops)
    R.check_exact('gemm, integer operands, max_ctas=3', _gemm(*ops, max_ctas=3), *ops)


def test_mx_gemm_at_extreme_scale_exponents():
    """ea + eb from about -120 to +116, with elements small enough that fp32 does not overflow; the smallest results
    are fp32 subnormals."""
    _need_gpu()
    G, M, N, K = 2, 257, 384, 640
    gen = torch.Generator(device='cuda').manual_seed(11)

    def small(rows):
        b = torch.randint(0, 0x39, (G, rows, K), generator=gen, device='cuda', dtype=torch.int32)
        b = b | (torch.randint(0, 2, b.shape, generator=gen, device='cuda', dtype=torch.int32) << 7)
        return b.to(torch.uint8).view(torch.float8_e4m3fn)
    aq, bq = small(M), small(N)
    ea = torch.randint(-60, 59, (G, M, K // 32), generator=gen, device='cuda', dtype=torch.int32)
    eb = torch.where(torch.arange(N, device='cuda').view(1, N, 1) % 2 == 0, -60, 58).expand(G, N, K // 32)
    sfa, sfb = R.pack(ea), R.pack(eb.to(torch.int32).contiguous())
    A = R.dequantize(aq, sfa)
    assert float(A.abs().max()) > 2.0 ** 50 and float(A[A != 0].abs().min()) < 2.0 ** -60
    r = R.ref_gemm(aq, sfa, bq, sfb)
    R.check('gemm: extreme scales', _gemm(aq, sfa, bq, sfb), r)
    R.check('gemm: extreme scales, max_ctas=5', _gemm(aq, sfa, bq, sfb, max_ctas=5), r)


def test_mx_gemm_hints_and_relaunch_are_bit_identical():
    """block_n / cta_group are hints: every accepted combination runs the same kernel and gives the same bits."""
    _need_gpu()
    G, M, N, K = 2, 300, 1024, 768
    aq, sfa, bq, sfb = R.operands(G, M, N, K, seed=5, device='cuda')
    bias, aux = R.bias_aux(R.ref_gemm(aq, sfa, bq, sfb).val)
    for epi in (R.EPI_NONE, R.EPI_RELU, R.EPI_RELU_BWD):
        kw = dict(bias=bias if epi != R.EPI_RELU_BWD else None, aux=aux if epi == R.EPI_RELU_BWD else None, epilogue=epi)
        base = _gemm(aq, sfa, bq, sfb, **kw)
        R.check('gemm: hints epi=%d' % epi, base, R.ref_gemm(aq, sfa, bq, sfb, **kw))
        for bn, cg in ((128, 1), (256, 1), (256, 2), (0, 2), (128, 0), (0, 1)):
            for m in (0, 4):
                assert torch.equal(_bits(_gemm(aq, sfa, bq, sfb, block_n=bn, cta_group=cg, max_ctas=m, **kw)), _bits(base)), \
                    (epi, bn, cg, m)
        assert torch.equal(_bits(_gemm(aq, sfa, bq, sfb, **kw)), _bits(base))


def test_mx_gemm_refusals():
    _need_gpu()
    from tutel_b200.ops import mx
    aq, sfa, bq, sfb = R.operands(1, 128, 384, 256, device='cuda')

    def refused(match, *args, **kw):
        with pytest.raises(RuntimeError, match=match):
            _gemm(*args, **kw)
        torch.cuda.synchronize()

    # K and N not multiples of 128 (scale arrays of the matching size, so that the launcher is the one refusing)
    a192 = aq[..., :192].contiguous()
    refused('K must be a multiple of 128', a192, sfa[:512].contiguous(), bq[..., :192].contiguous(), sfb[:3 * 512].contiguous())
    b192 = bq[:, :192].contiguous()
    refused('N must be a multiple of 128', aq, sfa, b192, torch.zeros(2 * 2 * 512, dtype=torch.uint8, device='cuda'))
    # misaligned operands: contiguous views 1 byte into a buffer
    buf = torch.zeros(1 + aq.numel(), dtype=torch.uint8, device='cuda')
    a_off = buf[1:].view(torch.float8_e4m3fn).view(aq.shape)
    refused('16-byte aligned', a_off, sfa, bq, sfb)
    sbuf = torch.zeros(1 + sfb.numel(), dtype=torch.uint8, device='cuda')
    refused('16-byte aligned', aq, sfa, bq, sbuf[1:])
    # ReLU backward without aux, and with a misaligned aux
    refused('aux', aq, sfa, bq, sfb, epilogue=R.EPI_RELU_BWD)
    abuf = torch.zeros(1 + 128 * 384, dtype=torch.bfloat16, device='cuda')
    refused('aux', aq, sfa, bq, sfb, aux=abuf[1:].view(1, 128, 384), epilogue=R.EPI_RELU_BWD)
    refused('aux must be a contiguous bf16', aq, sfa, bq, sfb, aux=torch.zeros(1, 128, 384, device='cuda'),
            epilogue=R.EPI_RELU_BWD)
    # bias of the wrong shape or dtype, and misaligned
    refused('bias must be a contiguous bf16', aq, sfa, bq, sfb, bias=torch.zeros(1, 256, dtype=torch.bfloat16, device='cuda'))
    refused('bias must be a contiguous bf16', aq, sfa, bq, sfb, bias=torch.zeros(1, 384, dtype=torch.float16, device='cuda'))
    bbuf = torch.zeros(1 + 384, dtype=torch.bfloat16, device='cuda')
    refused('bias must be 16-byte aligned', aq, sfa, bq, sfb, bias=bbuf[1:].view(1, 384))
    # tile-shape hints that cannot hold
    refused('block_n 256 needs N % 256 == 0', aq, sfa, bq, sfb, block_n=256)
    refused('CTA pairs need block_n 256', aq, sfa, bq, sfb, block_n=128, cta_group=2)
    refused('block_n must be 0, 128 or 256', aq, sfa, bq, sfb, block_n=64)
    refused('cta_group must be 0, 1 or 2', aq, sfa, bq, sfb, cta_group=3)
    # the binding: scale arrays of the wrong size, operands of the wrong type
    refused('scale arrays', aq, sfa[:512].contiguous(), bq, sfb)
    refused('e4m3 operands', aq.view(torch.uint8), sfa, bq, sfb)
    with pytest.raises(ValueError):
        mx.mx_quantize(torch.zeros(1, 4, 96, dtype=torch.bfloat16, device='cuda'))
    # after all that the kernel still runs
    R.check('gemm: after refusals', _gemm(aq, sfa, bq, sfb), R.ref_gemm(aq, sfa, bq, sfb))


# ------------------------------------------------------------------------------------------------------------------
# FusedReluFFNMx, stage by stage
# ------------------------------------------------------------------------------------------------------------------
def _ffn_params(E, C, M, H, Mo, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    x = torch.randn(E, C, M, generator=g, device='cuda').bfloat16().requires_grad_()
    w1 = (torch.randn(E, H, M, generator=g, device='cuda') * M ** -0.5).bfloat16().requires_grad_()
    w2 = (torch.randn(E, H, Mo, generator=g, device='cuda') * H ** -0.5).bfloat16().requires_grad_()
    b1 = (torch.randn(E, H, generator=g, device='cuda') * 0.1).bfloat16().requires_grad_()
    b2 = (torch.randn(E, Mo, generator=g, device='cuda') * 0.1).bfloat16().requires_grad_()
    return x, w1, b1, w2, b2


def _check_forward(what, x, w1, b1, w2, b2, act, y):
    """act = relu(x W1^T + b1) from x and w1 [E, H, M]; y = act W2 + b2 from the kernel's act and w2 [E, H, Mo]."""
    with torch.no_grad():
        R.check('act: ' + what, act, R.ref_gemm(*_q(x), *_q(w1), bias=b1, epilogue=R.EPI_RELU))
        R.check('y: ' + what, y, R.ref_gemm(*_q(act), *_q(w2.transpose(1, 2).contiguous()), bias=b2))


@pytest.mark.parametrize('E,C,M,H,Mo', [(2, 200, 256, 384, 128), (3, 77, 384, 256, 512)])
def test_mx_ffn_stage_by_stage(E, C, M, H, Mo):
    _need_gpu()
    from tutel_b200.ops import mx
    x, w1, b1, w2, b2 = _ffn_params(E, C, M, H, Mo, seed=C)
    y = mx.fused_relu_ffn_mx(x, w1, b1, w2, b2)
    saved_act = y.grad_fn.saved_tensors[3]
    dy = torch.randn(y.shape, generator=torch.Generator(device='cuda').manual_seed(1), device='cuda').bfloat16()
    y.backward(dy)
    what = 'E=%d C=%d M=%d H=%d Mo=%d' % (E, C, M, H, Mo)
    with torch.no_grad():
        # the intermediates, recomputed with the public ops: the MX GEMM is deterministic
        act = mx.mx_linear(x, w1, 'nk', b1, mx.EPI_RELU)
        assert torch.equal(_bits(act), _bits(mx.mx_linear(x, w1, 'nk', b1, mx.EPI_RELU)))
        assert torch.equal(_bits(act), _bits(saved_act))
        dh = mx.mx_linear(dy, w2, 'nk', None, mx.EPI_RELU_BWD, aux=act)
        assert torch.equal(_bits(dh), _bits(mx.mx_linear(dy, w2, 'nk', None, mx.EPI_RELU_BWD, aux=act)))
        _check_forward(what, x, w1, b1, w2, b2, act, y)
        # dh = (dy W2^T) masked by act: W2 [E, H, Mo] is the 'nk' operand of this product
        R.check('dh: ' + what, dh, R.ref_gemm(*_q(dy), *_q(w2), aux=act, epilogue=R.EPI_RELU_BWD))
        # dx = dh W1: the transposed copy of w1, [E, M, H]
        R.check('dx: ' + what, x.grad, R.ref_gemm(*_q(dh), *_q(w1.transpose(1, 2).contiguous())))
        # weight gradients: 16-bit GEMMs on the master operands
        r = GR.ref_gemm(dh, x, a_mn=True, b_mn=True)
        GR.check(r, w1.grad, what='dw1: ' + what)
        r = GR.ref_gemm(act, dy, a_mn=True, b_mn=True)
        GR.check(r, w2.grad, what='dw2: ' + what)
        D.check_colsum('db1 ' + what, b1.grad, dh)
        D.check_colsum('db2 ' + what, b2.grad, dy)


# ------------------------------------------------------------------------------------------------------------------
# the expert layer: path selection and the weight cache
# ------------------------------------------------------------------------------------------------------------------
def _experts(act=F.relu, M=256, H=256, E=2, seed=0):
    from tutel_b200.models.experts.ffn import FusedExpertsNetwork
    torch.manual_seed(seed)
    ex = FusedExpertsNetwork(model_dim=M, hidden_size_per_expert=H, num_experts_per_device=E, sharded_count=1,
                             activation_fn=lambda t: act(t), fp8='mx').cuda().bfloat16()
    with torch.no_grad():
        for p in ex.parameters():
            p.normal_(0, M ** -0.5)
    return ex


def _params(ex):
    return ex.batched_fc1_w, ex.batched_fc1_bias, ex.batched_fc2_w, ex.batched_fc2_bias


class _Spy:
    def __init__(self, monkeypatch):
        from tutel_b200.ops import mx
        self.calls = 0
        real = mx.fused_relu_ffn_mx

        def f(*a, **kw):
            self.calls += 1
            return real(*a, **kw)
        monkeypatch.setattr(mx, 'fused_relu_ffn_mx', f)


def test_mx_expert_takes_the_mx_path_exactly_when_it_can(monkeypatch):
    _need_gpu()
    from tutel_b200.ops import mx
    x = torch.randn(2, 100, 256, device='cuda', dtype=torch.bfloat16)
    spy = _Spy(monkeypatch)
    ex = _experts()
    assert mx.can_use_mx(x, ex.batched_fc1_w, ex.batched_fc2_w)
    y = ex.compute(x, *_params(ex))
    assert spy.calls == 1
    act = y.grad_fn.saved_tensors[3]
    _check_forward('layer', x, *_params(ex), act, y)
    for ex, why in ((_experts(act=F.gelu), 'GELU'), (_experts(H=192), 'H % 128 != 0')):
        ex.compute(x, *_params(ex))
        assert spy.calls == 1, why
    # dropless decoding: per-expert row counts
    ex.compute(x, *_params(_experts()), row_counts=torch.tensor([3, 5], dtype=torch.int32, device='cuda'))
    assert spy.calls == 1, 'row_counts'


def test_mx_layer_in_dropless_decoding_does_not_take_the_mx_path(monkeypatch):
    _need_gpu()
    from tutel_b200 import moe
    torch.manual_seed(3)
    layer = moe.moe_layer(gate_type={'type': 'top', 'k': 2, 'capacity_factor': 0.0}, model_dim=256,
                          experts={'type': 'ffn', 'num_experts_per_device': 4, 'hidden_size_per_expert': 256,
                                   'activation_fn': lambda t: F.relu(t), 'fp8': 'mx'}, seeds=(1, 1, 1)).cuda().bfloat16()
    spy = _Spy(monkeypatch)
    x = torch.randn(1, 4, 256, device='cuda', dtype=torch.bfloat16)
    with torch.no_grad():
        layer(x, megablocks_size=1)
    assert spy.calls == 0
    layer(torch.randn(2, 128, 256, device='cuda', dtype=torch.bfloat16))          # padded training forward: taken
    assert spy.calls == 1


@pytest.mark.parametrize('update', ['load_state_dict', 'optimizer_step', 'no_grad_inplace', 'data_write'])
def test_mx_expert_follows_updated_weights(update):
    """After each way of changing the weights, the next forward is the reference of the new weights (the MX weight
    cache is not stale)."""
    _need_gpu()
    from tutel_b200.ops import gemm
    ex, other = _experts(seed=0), _experts(seed=1)
    x = torch.randn(2, 100, 256, device='cuda', dtype=torch.bfloat16)
    y0 = ex.compute(x, *_params(ex))                                              # fills the cache
    if update == 'load_state_dict':
        ex.load_state_dict(other.state_dict())
    elif update == 'optimizer_step':
        opt = torch.optim.SGD(ex.parameters(), lr=1.0)
        y0.float().pow(2).mean().backward()
        opt.step()
    elif update == 'no_grad_inplace':
        with torch.no_grad():
            for p in ex.parameters():
                p.mul_(-0.5)
    else:
        for p, q in zip(ex.parameters(), other.parameters()):
            p.data.copy_(q.data)
        gemm.invalidate_fp8_cache()
    y = ex.compute(x, *_params(ex))
    act = y.grad_fn.saved_tensors[3]
    _check_forward(update, x, *_params(ex), act, y)
    assert not torch.equal(y, y0)
