"""The references of the MX kernels (tests/mx_reference.py) on CPU.

A plain-torch fp32 emulation of each kernel passes its check, and each near miss - one plausible kernel bug - is
rejected by the check that guards it.  The CPU definition in tutel_b200/ops/mx.py agrees with the reference bit for bit,
over every positive bf16 and fp16 value as a block maximum and over the special values.
"""
import pytest
import torch

import mx_reference as R
from tutel_b200.ops import mx

F448 = torch.tensor(1.0 / 448.0, dtype=torch.float32)    # the kernels' fp32 constant 1.0f / 448.0f


# ------------------------------------------------------------------------------------------------------------------
# quantiser
# ------------------------------------------------------------------------------------------------------------------
def emulate_quantize(x, miss=None):
    """mx_quantize_kernel in fp32: amax by fmaxf (NaN ignored), e from the bits of amax * (1/448), q = e4m3(x * 2^-e)."""
    G, Rn, K = x.shape
    f = x.float()
    a = f.abs()
    a = torch.where(torch.isnan(a), torch.zeros_like(a), a)
    amax = a.view(G, Rn, K // 32, 32).amax(-1)
    bits = (amax * F448).view(torch.int32)
    e = ((bits >> 23) & 0xFF) - 127
    if miss != 'floor':
        e = e + ((bits & 0x7FFFFF) != 0).to(torch.int32)
    e = e.clamp(-127, 126)
    v = f * torch.ldexp(torch.ones_like(e, dtype=torch.float32), -e).repeat_interleave(32, -1)
    q = v.clamp(-448, 448).to(torch.float8_e4m3fn).view(torch.uint8)
    if miss == 'truncate':                  # round toward zero: one code down wherever RN rounded up in magnitude
        up = q.view(torch.float8_e4m3fn).float().abs() > v.abs()
        q = torch.where(up & ~torch.isnan(v), q - 1, q)
    off = R.scale_offsets(G, Rn, K)
    if miss == 'swap_offsets':              # (r % 128) / 32 and (k % 128) / 32 trade places inside the 16-byte word
        r = torch.arange(Rn).view(1, Rn, 1)
        k = torch.arange(K // 32).view(1, 1, -1) * 32
        off = off - ((r % 128) // 32) * 4 - (k % 128) // 32 + ((k % 128) // 32) * 4 + (r % 128) // 32
    sf = torch.zeros(G * (K // 128) * ((Rn + 127) // 128) * 512, dtype=torch.uint8)
    sf[off.reshape(-1)] = (e + 127).to(torch.uint8).reshape(-1)
    return q, sf


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16])
def test_quantizer_emulation_and_cpu_definition_match_reference(dtype):
    for x in (R.special_values(dtype), R.every_positive(dtype)):
        R.check_quantized('emulation', *emulate_quantize(x), x)
        q, sf = mx.mx_quantize_reference(x)
        R.check_quantized('ops.mx definition', q, sf, x)
        assert torch.equal(mx.block_exponents_reference(x), R.block_exponents(x))


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16])
def test_exponent_range_and_nan_contract(dtype):
    x = R.special_values(dtype)
    e = R.block_exponents(x)
    nonzero = x.float().nan_to_num(0.0).abs().view(*e.shape, 32).amax(-1) > 0
    assert bool((e[nonzero] >= -126).all() and (e[nonzero] <= 126).all()) and bool((e[~nonzero] == -127).all())
    assert int(e[0, 2, 0]) == int(R.block_exponents(torch.where(torch.isnan(x), torch.zeros_like(x), x))[0, 2, 0])
    q, _, nan = R.quantize(x)
    assert bool(nan[0, 2, 7]) and int(q[0, 2, 7]) & 0x7F == 0x7F
    assert int(q[0, 1, 64 + 3]) == 0x7E and int(q[0, 1, 96 + 5]) == 0xFE            # +-inf saturate to +-448
    assert int(q[0, 0, 40]) == 0x80                                                 # -0 stays -0
    if dtype == torch.bfloat16:                                                     # below 448 * 2^-126: clamped
        tiny = torch.zeros(1, 1, 128, dtype=dtype)
        tiny[0, 0, 0] = 2.0 ** -130
        assert int(R.block_exponents(tiny)[0, 0, 0]) == -126


@pytest.mark.parametrize('miss', ['floor', 'truncate', 'swap_offsets'])
def test_quantizer_near_misses_are_rejected(miss):
    x = R.special_values(torch.bfloat16)
    with pytest.raises(AssertionError, match='differ'):
        R.check_quantized(miss, *emulate_quantize(x, miss), x)


def test_byte_zero_decodes_to_zero_in_reference_and_cpu_definition():
    q = torch.full((1, 4, 128), 1.0).to(torch.float8_e4m3fn)
    e = torch.zeros(1, 4, 4, dtype=torch.int32)
    e[0, 1, 2] = -127
    sf = R.pack(e)
    assert torch.equal(sf, mx.pack_scales(e))
    want = torch.ones(1, 4, 128, dtype=torch.float64)
    want[0, 1, 64:96] = 0
    assert torch.equal(R.dequantize(q, sf), want)
    assert torch.equal(mx.mx_dequantize(q, sf).double(), want)


# ------------------------------------------------------------------------------------------------------------------
# GEMM
# ------------------------------------------------------------------------------------------------------------------
def _scales(sf, G, rows, K):
    """fp32 scales [G, rows padded to 128, K / 32] as ue8m0_to_float decodes them (byte 0 -> 0)."""
    b = R.scale_bytes(sf, G, -(-rows // 128) * 128, K)
    return torch.where(b == 0, torch.zeros_like(b, dtype=torch.float32),
                       torch.ldexp(torch.ones_like(b, dtype=torch.float32), b - 127))


def emulate_gemm(aq, sfa, bq, sfb, bias=None, aux=None, epilogue=R.EPI_NONE, miss=None):
    """mx_gemm_kernel in fp32: per 32-element block the exact products summed in fp32, times sa * sb, folded into an
    fp32 accumulator; bias / ReLU / ReLU-backward in fp32; one RN rounding to bf16."""
    G, M, K = aq.shape
    N = bq.size(1)
    a, b = aq.float(), bq.float()
    sa, sb = _scales(sfa, G, M, K), _scales(sfb, G, N, K)
    rows, cols = torch.arange(M), torch.arange(N)
    if miss == 'row_plus_8':
        rows = rows ^ 8                 # the other row of the thread's pair (r0, r0 + 8)
    if miss == 'col_xor_1':
        cols = cols ^ 1
    sa, sb = sa[:, rows], sb[:, cols]
    acc = torch.zeros(G, M, N)
    nkb = K // 32 - (4 if miss == 'drop_last_step' else 0)
    for kb in range(nkb):
        k = slice(32 * kb, 32 * kb + 32)
        part = a[..., k] @ b[..., k].transpose(1, 2)
        skb = kb ^ 1 if miss == 'neighbour_block' else (kb - kb % 4 if miss == 'per_128' else kb)
        t = part * (sa[:, :, skb, None] * sb[:, None, :, skb])
        if miss == 'bf16_partials':
            t = t.bfloat16().float()
        acc = acc + t
    if bias is not None and miss != 'bias_after_relu':
        acc = acc + bias.float().unsqueeze(1)
    if epilogue == R.EPI_RELU:
        acc = acc.clamp_min(0)
        if miss == 'bias_after_relu':
            acc = acc + bias.float().unsqueeze(1)
    if epilogue == R.EPI_RELU_BWD:
        keep = aux.float() >= 0 if miss == 'mask_ge' else aux.float() > 0
        acc = torch.where(keep, acc, torch.zeros_like(acc))
    return acc.bfloat16()


SHAPE = (2, 160, 256, 512)          # a partial 128-row tile, two column tiles, four K steps


@pytest.mark.parametrize('epilogue,with_bias', [(R.EPI_NONE, False), (R.EPI_NONE, True), (R.EPI_RELU, True),
                                                (R.EPI_RELU, False), (R.EPI_RELU_BWD, False)])
def test_gemm_emulation_passes(epilogue, with_bias):
    G, M, N, K = SHAPE
    aq, sfa, bq, sfb = R.operands(G, M, N, K)
    bias, aux = R.bias_aux(R.ref_gemm(aq, sfa, bq, sfb).val)
    bias = bias if with_bias else None
    r = R.ref_gemm(aq, sfa, bq, sfb, bias=bias, aux=aux, epilogue=epilogue)
    assert R.check('emulation', emulate_gemm(aq, sfa, bq, sfb, bias, aux, epilogue), r) <= 1.0


def test_gemm_emulation_passes_at_extreme_scales():
    """ea + eb from about -120 to +116 with small elements: nothing overflows in fp32, and the smallest results are
    fp32 subnormals."""
    G, M, N, K = 1, 128, 128, 256
    gen = torch.Generator().manual_seed(7)
    aq = (torch.randint(0, 0x39, (G, M, K), generator=gen) | (torch.randint(0, 2, (G, M, K), generator=gen) << 7))
    bq = (torch.randint(0, 0x39, (G, N, K), generator=gen) | (torch.randint(0, 2, (G, N, K), generator=gen) << 7))
    aq, bq = aq.to(torch.uint8).view(torch.float8_e4m3fn), bq.to(torch.uint8).view(torch.float8_e4m3fn)
    ea = torch.randint(-60, 59, (G, M, K // 32), generator=gen, dtype=torch.int32)
    eb = torch.where(torch.arange(N).view(1, N, 1) % 2 == 0, torch.full((G, N, K // 32), -60, dtype=torch.int32),
                     torch.full((G, N, K // 32), 58, dtype=torch.int32))
    sfa, sfb = R.pack(ea), R.pack(eb)
    r = R.ref_gemm(aq, sfa, bq, sfb)
    assert R.check('emulation, extreme scales', emulate_gemm(aq, sfa, bq, sfb), r) <= 1.0


def test_gemm_emulation_is_exact_on_exactly_representable_operands():
    G, M, N, K = SHAPE
    ops = R.integer_operands(G, M, N, K)
    R.check_exact('emulation', emulate_gemm(*ops), *ops)


def test_bf16_partials_are_rejected_by_the_exact_check():
    """Rounding each block's partial sum to bf16 costs at most 2^-9 of it, which the fp8 tensor core's own error bound
    allows (module docstring of mx_reference); on exactly representable operands it changes the result."""
    G, M, N, K = SHAPE
    ops = R.integer_operands(G, M, N, K)
    with pytest.raises(AssertionError, match='exact check'):
        R.check_exact('bf16_partials', emulate_gemm(*ops, miss='bf16_partials'), *ops)


GEMM_MISSES = ['neighbour_block', 'row_plus_8', 'col_xor_1', 'drop_last_step', 'per_128', 'bias_after_relu', 'mask_ge']


@pytest.mark.parametrize('miss', GEMM_MISSES)
def test_gemm_near_misses_are_rejected(miss):
    G, M, N, K = SHAPE
    aq, sfa, bq, sfb = R.operands(G, M, N, K)
    bias, aux = R.bias_aux(R.ref_gemm(aq, sfa, bq, sfb).val)
    epilogue = {'bias_after_relu': R.EPI_RELU, 'mask_ge': R.EPI_RELU_BWD}.get(miss, R.EPI_NONE)
    bias = bias if miss == 'bias_after_relu' else None
    r = R.ref_gemm(aq, sfa, bq, sfb, bias=bias, aux=aux, epilogue=epilogue)
    d = emulate_gemm(aq, sfa, bq, sfb, bias, aux, epilogue, miss)
    with pytest.raises(AssertionError, match='not exactly 0' if miss == 'mask_ge' else 'outside the bound'):
        R.check(miss, d, r)


def test_cpu_definition_of_the_gemm_passes():
    """ops.mx.mx_gemm on CPU (fp32 matmul of the dequantised operands) is within the kernel's bound."""
    G, M, N, K = SHAPE
    aq, sfa, bq, sfb = R.operands(G, M, N, K, spread=10)
    bias, aux = R.bias_aux(R.ref_gemm(aq, sfa, bq, sfb).val)
    for epi in (R.EPI_NONE, R.EPI_RELU, R.EPI_RELU_BWD):
        r = R.ref_gemm(aq, sfa, bq, sfb, bias=bias, aux=aux, epilogue=epi)
        assert R.check('ops.mx definition', mx.mx_gemm(aq, sfa, bq, sfb, bias=bias, aux=aux, epilogue=epi), r) <= 1.0
