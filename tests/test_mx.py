"""MX block-scaled fp8 number format (CPU): the PyTorch definition the sm_90a kernels are tested against."""
import pytest
import torch

from tutel_b200.ops import mx


def test_scale_layout_round_trip_and_atom_offsets():
    G, R, K = 2, 200, 256
    e = torch.randint(-20, 20, (G, R, K // 32), dtype=torch.int32)
    sf = mx.pack_scales(e)
    assert sf.numel() == G * (K // 128) * 2 * 512
    assert torch.equal(mx.unpack_scales(sf, G, R, K), e)
    # spot-check the documented byte offset
    g, r, k = 1, 171, 200
    RT = 2
    off = ((g * (K // 128) + k // 128) * RT + r // 128) * 512 + (r % 32) * 16 + ((r % 128) // 32) * 4 + (k % 128) // 32
    assert int(sf[off]) == int(e[g, r, k // 32]) + 127
    # padded rows carry byte 0, which decodes to a scale of 0
    r = 250
    off = ((0 * (K // 128) + 0) * RT + r // 128) * 512 + (r % 32) * 16 + ((r % 128) // 32) * 4
    assert int(sf[off]) == 0


def test_quantise_dequantise_error_bound_and_outlier_locality():
    torch.manual_seed(0)
    x = torch.randn(1, 64, 256)
    x[0, 3, 7] = 1000.0                       # one outlier: only its own 32-block loses resolution
    q, sf = mx.mx_quantize_reference(x)
    y = mx.mx_dequantize(q, sf)
    e = mx.unpack_scales(sf, 1, 64, 256)
    amax = x.abs().view(1, 64, 8, 32).amax(-1)
    # every block is scaled into e4m3's finite range without overflow, using at least half of it
    scaled = amax / torch.exp2(e.float())
    assert float(scaled.max()) <= 448.0 and float(scaled[amax > 0].min()) > 224.0 - 1e-3
    # e4m3 has 3 mantissa bits: relative error <= 2^-4 for normal values, absolute error bounded by the block scale
    err = (y - x).abs().view(1, 64, 8, 32)
    bound = torch.maximum(x.abs().view(1, 64, 8, 32) * 2.0 ** -4, torch.exp2(e.float()).unsqueeze(-1) * 2.0 ** -9)
    assert bool((err <= bound + 1e-12).all())
    # A per-row scale (the other fp8 mode of this framework) pushes the small entries of an outlier row into e4m3's
    # subnormals once the row spans more than ~2^15; per-block scales keep their full 3-bit mantissa.
    x = torch.randn(1, 4, 256) * 0.004
    x[0, 1, 7] = 1000.0
    q, sf = mx.mx_quantize_reference(x)
    mx_err = (mx.mx_dequantize(q, sf) - x).abs()[0, 1, 32:]
    s_row = x[0, 1].abs().max() / 448.0
    row_err = ((x[0, 1] / s_row).to(torch.float8_e4m3fn).float() * s_row - x[0, 1]).abs()[32:]
    assert float(mx_err.mean()) * 4 < float(row_err.mean())


def test_mx_gemm_cpu_definition_matches_float_matmul():
    torch.manual_seed(1)
    a, b = torch.randn(2, 48, 128), torch.randn(2, 128, 128)
    aq, sa = mx.mx_quantize(a)
    bq, sb = mx.mx_quantize(b)
    y = mx.mx_gemm(aq, sa, bq, sb).float()
    ref = torch.matmul(a, b.transpose(1, 2))
    assert float((y - ref).abs().max() / ref.abs().max()) < 0.06
    with pytest.raises(ValueError):
        mx.mx_quantize(torch.randn(1, 4, 96))


def test_expert_fp8_modes_select_row_or_mx_paths(monkeypatch):
    """fp8=True / 'row' -> row-scaled e4m3 (eligible for the fused engine); fp8='mx' -> MX block scales (unfused path)."""
    from tutel_b200.models.experts.ffn import FusedExpertsNetwork
    kw = dict(model_dim=128, hidden_size_per_expert=256, num_experts_per_device=2, sharded_count=1)
    for arg, want in ((None, (False, False)), (False, (False, False)), (True, (True, False)), ('row', (True, False)), ('mx', (False, True))):
        ex = FusedExpertsNetwork(fp8=arg, **kw)
        assert (ex.fp8, ex.mx) == want, arg
    monkeypatch.setenv('TUTEL_B200_FP8', 'mx')
    ex = FusedExpertsNetwork(**kw)
    assert ex.mx and not ex.fp8
    monkeypatch.setenv('TUTEL_B200_FP8', '1')
    ex = FusedExpertsNetwork(**kw)
    assert ex.fp8 and not ex.mx
    with pytest.raises(AssertionError):
        FusedExpertsNetwork(fp8='int4', **kw)
    # on CPU the MX path is never taken: the layer computes in the model dtype
    x = torch.randn(2, 8, 128)
    assert not mx.can_use_mx(x, ex.batched_fc1_w, ex.batched_fc2_w)


def test_mx_epilogues_of_the_cpu_definition():
    torch.manual_seed(5)
    a, b = torch.randn(1, 16, 128), torch.randn(1, 128, 128)
    bias, aux = torch.randn(1, 128), torch.randn(1, 16, 128)
    aq, sa = mx.mx_quantize(a)
    bq, sb = mx.mx_quantize(b)
    acc = torch.matmul(mx.mx_dequantize(aq, sa), mx.mx_dequantize(bq, sb).transpose(1, 2))
    relu = mx.mx_gemm(aq, sa, bq, sb, bias=bias, epilogue=mx.EPI_RELU).float()
    assert torch.allclose(relu, torch.relu(acc + bias.unsqueeze(1)).bfloat16().float())
    bwd = mx.mx_gemm(aq, sa, bq, sb, aux=aux, epilogue=mx.EPI_RELU_BWD).float()
    assert torch.equal(bwd, torch.where(aux > 0, acc, torch.zeros_like(acc)).bfloat16().float())
    # the transposing quantiser is the plain one applied to the transpose
    w = torch.randn(2, 128, 256)
    q, sf = mx.mx_quantize_transpose(w)
    rq, rsf = mx.mx_quantize_reference(w.transpose(1, 2).contiguous())
    assert torch.equal(q.view(torch.uint8), rq.view(torch.uint8)) and torch.equal(sf, rsf)
