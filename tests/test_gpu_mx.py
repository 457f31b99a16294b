"""MX block-scaled fp8 kernels (csrc/gemm_mx.cu) against their PyTorch definition (tutel_b200/ops/mx.py)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip('needs an H100')


@pytest.mark.parametrize('shape', [(1, 128, 256), (2, 300, 512), (3, 64, 1024)])
@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16])
def test_mx_quantize_kernel_matches_definition(shape, dtype):
    _need_gpu()
    from tutel_b200.ops import mx
    torch.manual_seed(0)
    x = (torch.randn(*shape, device='cuda') * torch.exp(2 * torch.randn(shape[0], shape[1], 1, device='cuda'))).to(dtype)
    x[0, 0, :40] = 0
    q, sf = mx.mx_quantize(x)
    rq, rsf = mx.mx_quantize_reference(x)
    assert torch.equal(q.view(torch.uint8), rq.view(torch.uint8))
    assert torch.equal(sf, rsf)


@pytest.mark.parametrize('G,M,N,K,bn,cg', [(1, 128, 128, 128, 128, 1), (2, 200, 384, 512, 128, 1), (1, 256, 512, 1024, 256, 1),
                                           (1, 256, 512, 1024, 256, 2), (1, 100, 256, 256, 256, 2), (2, 1000, 1024, 2048, 0, 0)])
def test_mx_gemm_is_exact_on_exactly_representable_operands(G, M, N, K, bn, cg):
    """Small integers x powers of two: every product and partial sum is exact in fp32, so the tensor-core result must
    equal the fp32 matmul of the dequantised operands bit for bit (after the bf16 rounding of the output) - this pins
    the scale layout (row / column -> word of the atom, K block -> byte) and the descriptors."""
    _need_gpu()
    from tutel_b200.ops import mx
    g = torch.Generator().manual_seed(M + N)
    a = torch.randint(-3, 4, (G, M, K), generator=g).float().cuda()
    b = torch.randint(-3, 4, (G, N, K), generator=g).float().cuda()
    ea = torch.randint(-2, 3, (G, M, K // 32), generator=g, dtype=torch.int32).cuda()
    eb = torch.randint(-2, 3, (G, N, K // 32), generator=g, dtype=torch.int32).cuda()
    aq, bq = a.to(torch.float8_e4m3fn), b.to(torch.float8_e4m3fn)
    sa, sb = mx.pack_scales(ea), mx.pack_scales(eb)
    ref = torch.matmul(mx.mx_dequantize(aq, sa), mx.mx_dequantize(bq, sb).transpose(1, 2))
    y = mx.mx_gemm(aq, sa, bq, sb, block_n=bn, cta_group=cg)
    assert torch.equal(y.float(), ref.to(torch.bfloat16).float())


def test_mx_quantize_transpose_kernel_matches_definition():
    _need_gpu()
    from tutel_b200.ops import mx
    torch.manual_seed(3)
    w = (torch.randn(2, 256, 192, device='cuda') * torch.exp(torch.randn(2, 1, 192, device='cuda'))).to(torch.bfloat16)
    q, sf = mx.mx_quantize_transpose(w)                               # [2, 192, 256] quantised along the 256
    rq, rsf = mx.mx_quantize_reference(w.transpose(1, 2).contiguous())
    assert q.shape == (2, 192, 256)
    assert torch.equal(q.view(torch.uint8), rq.view(torch.uint8))
    assert torch.equal(sf, rsf)


@pytest.mark.parametrize('bn,cg', [(128, 1), (256, 1), (256, 2)])
def test_mx_gemm_epilogues(bn, cg):
    _need_gpu()
    from tutel_b200.ops import mx
    torch.manual_seed(4)
    G, M, N, K = 2, 300, 512, 256
    a = torch.randn(G, M, K, device='cuda', dtype=torch.bfloat16)
    b = torch.randn(G, N, K, device='cuda', dtype=torch.bfloat16)
    bias = torch.randn(G, N, device='cuda', dtype=torch.bfloat16)
    aux = torch.randn(G, M, N, device='cuda', dtype=torch.bfloat16)
    aux[0, 0, :8] = 0                                                  # zero (and -0) activations pass no gradient
    aux[0, 1, :8] = -0.0
    aq, sa = mx.mx_quantize(a)
    bq, sb = mx.mx_quantize(b)
    acc = torch.matmul(mx.mx_dequantize(aq, sa), mx.mx_dequantize(bq, sb).transpose(1, 2))
    plain = mx.mx_gemm(aq, sa, bq, sb, block_n=bn, cta_group=cg).float()
    assert float((plain - acc).abs().max() / acc.abs().max()) < 8e-3
    want = torch.relu(acc + bias.float().unsqueeze(1))
    got = mx.mx_gemm(aq, sa, bq, sb, bias=bias, epilogue=mx.EPI_RELU, block_n=bn, cta_group=cg).float()
    assert float((got - want).abs().max() / want.abs().max()) < 8e-3 and float(got.min()) >= 0
    got = mx.mx_gemm(aq, sa, bq, sb, aux=aux, epilogue=mx.EPI_RELU_BWD, block_n=bn, cta_group=cg).float()
    assert torch.equal(got, torch.where(aux > 0, plain, torch.zeros_like(plain)))
    # a persistent grid smaller than the tile count walks the same tiles
    few = mx.mx_gemm(aq, sa, bq, sb, block_n=bn, cta_group=cg, max_ctas=4).float()
    assert torch.equal(few, plain)


def test_mx_ffn_forward_and_gradients_close_to_fp32():
    _need_gpu()
    from tutel_b200.ops import mx
    torch.manual_seed(2)
    E, C, M, H = 2, 256, 512, 1024
    x = torch.randn(E, C, M, device='cuda', dtype=torch.bfloat16, requires_grad=True)
    w1 = (torch.randn(E, H, M, device='cuda') * M ** -0.5).to(torch.bfloat16).requires_grad_()
    w2 = (torch.randn(E, H, M, device='cuda') * H ** -0.5).to(torch.bfloat16).requires_grad_()
    b1 = (torch.randn(E, H, device='cuda') * 0.1).to(torch.bfloat16).requires_grad_()
    b2 = (torch.randn(E, M, device='cuda') * 0.1).to(torch.bfloat16).requires_grad_()
    y = mx.fused_relu_ffn_mx(x, w1, b1, w2, b2)
    dy = torch.randn_like(y)
    y.backward(dy)
    got = [y] + [t.grad for t in (x, w1, b1, w2, b2)]
    xf, w1f, b1f, w2f, b2f = (t.detach().float().requires_grad_() for t in (x, w1, b1, w2, b2))
    ref = torch.matmul(torch.relu(torch.matmul(xf, w1f.transpose(1, 2)) + b1f.unsqueeze(1)), w2f) + b2f.unsqueeze(1)
    ref.backward(dy.float())
    want = [ref] + [t.grad for t in (xf, w1f, b1f, w2f, b2f)]
    # y, dw2, db2 do not pass through the ReLU mask: plain quantisation error.  dx, dw1, db1 do: the mask comes from the
    # fp8 forward, so a few per cent of the entries near zero flip against the fp32 oracle and each flip costs a whole
    # entry (measured ~0.16 relative, the same as the row-scaled fp8 path) - the direction must still agree.
    for name, g, w in zip(('y', 'dx', 'dw1', 'db1', 'dw2', 'db2'), got, want):
        g = g.detach().float()
        w = w.detach()
        rel = float((g - w).norm() / w.norm())
        cos = float((g * w).sum() / (g.norm() * w.norm()))
        if name in ('y', 'dw2', 'db2'):
            assert rel < 0.07, (name, rel)
        else:
            assert rel < 0.3 and cos > 0.96, (name, rel, cos)


def test_moe_layer_with_mx_experts_trains_like_bf16():
    _need_gpu()
    from tutel_b200 import moe
    outs = {}
    for mode in (None, 'mx'):
        torch.manual_seed(5)
        layer = moe.moe_layer(gate_type={'type': 'top', 'k': 2}, model_dim=256,
                              experts={'type': 'ffn', 'num_experts_per_device': 2, 'hidden_size_per_expert': 512,
                                       'activation_fn': lambda t: torch.nn.functional.relu(t), **({'fp8': mode} if mode else {})},
                              seeds=(1, 1, 1)).cuda().to(torch.bfloat16)
        assert layer.experts.mx == (mode == 'mx')
        x = torch.randn(4, 128, 256, device='cuda', dtype=torch.bfloat16, requires_grad=True)
        y = layer(x)
        (y.float().pow(2).mean() + layer.l_aux).backward()
        outs[mode] = (y.detach().float(), x.grad.float(), layer.experts.batched_fc1_w.grad.float())
    for i, (a, b) in enumerate(zip(outs[None], outs['mx'])):
        rel = float((a - b).norm() / a.norm())
        cos = float((a * b).sum() / (a.norm() * b.norm()))
        assert (rel < 0.08) if i == 0 else (rel < 0.3 and cos > 0.96), (i, rel, cos)
