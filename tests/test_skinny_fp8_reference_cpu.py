"""The fp64 references of the weight-only fp8 skinny kernels (tests/skinny_fp8_reference.py) on CPU.

A plain-torch fp32 emulation of each kernel's arithmetic (16-bit x, e4m3 weights, scales applied to finished dot
products, layer 2 summed per 128-unit hidden slice) passes the checker, and each near miss - one plausible kernel bug -
is rejected.
"""
import pytest
import torch

import skinny_fp8_reference as R

SLICE = 128                 # hidden units per block (kHS8 in csrc/skinny_gemm.cu)
ROWS = 12
COUNTS = [0, 1, 2, 3, 5, 9, ROWS, ROWS + 7]


def _inputs(K, H, N, glu, dtype=torch.bfloat16, seed=0):
    gen = torch.Generator().manual_seed(seed)
    G = len(COUNTS)
    x = torch.randn(G, ROWS, K, generator=gen).to(dtype)
    if glu:
        w = [torch.randn(G, H, K, generator=gen) * K ** -0.5, torch.randn(G, H, K, generator=gen) * K ** -0.5,
             torch.randn(G, N, H, generator=gen) * H ** -0.5]
        return x, [R.quantize(t) for t in w], None
    w = [torch.randn(G, H, K, generator=gen) * K ** -0.5, torch.randn(G, N, H, generator=gen) * H ** -0.5]
    b = (torch.randn(G, H, generator=gen).to(dtype), torch.randn(G, N, generator=gen).to(dtype))
    return x, [R.quantize(t) for t in w], b


def _act(name, t):
    return R._FN[name](t)


def _w8a8(x):
    s = (x.float().abs().amax(-1, keepdim=True) / 448.0).clamp(min=1e-12)
    return (x.float() / s).to(torch.float8_e4m3fn).float() * s


def _dequant32(q, s, miss):
    if miss == 'scale_axis':
        return q.float() * s.unsqueeze(-2)          # the row scale applied along the columns
    return q.float() * s.unsqueeze(-1)


def _layer2(h, q, s, miss):
    """y = sum over 128-unit slices of (h[:, slice] @ q[:, slice]^T) * s, in fp32, as the blocks' atomics add it."""
    H = h.size(-1)
    y = torch.zeros(h.size(0), h.size(1), q.size(1))
    stop = H - H % SLICE if miss == 'drop_tail' and H % SLICE else H
    qf = _dequant32(q, s, miss) if miss == 'scale_axis' else q.float()
    for h0 in range(0, stop, SLICE):
        part = h[..., h0:h0 + SLICE] @ qf[..., h0:h0 + SLICE].transpose(1, 2)
        if miss not in ('no_out_scale', 'scale_axis'):
            part = part * s.unsqueeze(-2)
        y += part
    return y


def emulate_ffn(x, q1, s1, b1, q2t, s2, b2, act, miss=None):
    xf = _w8a8(x) if miss == 'w8a8' else x.float()
    w1 = _dequant32(q1, s1, miss) if miss == 'scale_axis' else None
    pre = (xf @ w1.transpose(1, 2)) if w1 is not None else (xf @ q1.float().transpose(1, 2)) * s1.unsqueeze(-2)
    h = _act(act, pre + b1.float().unsqueeze(1))
    if miss == 'h_bf16':
        h = h.bfloat16().float()
    y = _layer2(h, q2t, s2, miss) + b2.float().unsqueeze(1)
    return _mask(y)


def emulate_glu(x, q1t, s1, q2t, s2, q3t, s3, act, miss=None):
    xf = _w8a8(x) if miss == 'w8a8' else x.float()
    if miss == 'scale_axis':
        g, u = xf @ _dequant32(q1t, s1, miss).transpose(1, 2), xf @ _dequant32(q2t, s2, miss).transpose(1, 2)
    else:
        g = (xf @ q1t.float().transpose(1, 2)) * s1.unsqueeze(-2)
        u = (xf @ q2t.float().transpose(1, 2)) * s2.unsqueeze(-2)
    if miss == 'swap':
        g, u = u, g
    h = _act(act, g) * u
    if miss == 'h_bf16':
        h = h.bfloat16().float()
    return _mask(_layer2(h, q3t, s3, miss))


def _mask(y):
    rows = torch.arange(y.size(1)).view(1, -1, 1)
    return torch.where(rows < torch.tensor(COUNTS).clamp(max=y.size(1)).view(-1, 1, 1), y, torch.zeros(()))


# K, H, N multiples of 16 but not of the slice: two whole slices and a 16-unit partial one
SHAPE = (208, 272, 144)
# The wrong scale axis needs the right length (square), and the bf16 rounding of h (2^-9 relative, random sign) shows
# over the (K + H) * 2^-24 bound when K is small: one whole slice and a partial one.
MISS_SHAPES = {'scale_axis': (96, 96, 96), 'h_bf16': (32, 144, 64)}


@pytest.mark.parametrize('act', ['relu', 'gelu', 'silu'])
@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16])
def test_ffn_emulation_passes(act, dtype):
    x, [(q1, s1), (q2, s2)], (b1, b2) = _inputs(*SHAPE, glu=False, dtype=dtype)
    ref, bound = R.ffn_reference(x, q1, s1, b1, q2, s2, b2, act)
    assert R.check(emulate_ffn(x, q1, s1, b1, q2, s2, b2, act), ref, bound, torch.tensor(COUNTS)) <= 1.0


@pytest.mark.parametrize('act', ['relu', 'gelu', 'silu'])
@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16])
def test_glu_emulation_passes(act, dtype):
    x, [(q1, s1), (q2, s2), (q3, s3)], _ = _inputs(*SHAPE, glu=True, dtype=dtype)
    ref, bound = R.glu_reference(x, q1, s1, q2, s2, q3, s3, act)
    assert R.check(emulate_glu(x, q1, s1, q2, s2, q3, s3, act), ref, bound, torch.tensor(COUNTS)) <= 1.0


def test_ffn_without_biases_matches_reference_without_biases():
    x, [(q1, s1), (q2, s2)], (b1, b2) = _inputs(*SHAPE, glu=False)
    ref, bound = R.ffn_reference(x, q1, s1, None, q2, s2, None, 'relu')
    y = emulate_ffn(x, q1, s1, torch.zeros_like(b1), q2, s2, torch.zeros_like(b2), 'relu')
    assert R.check(y, ref, bound, torch.tensor(COUNTS)) <= 1.0


MISSES = ['w8a8', 'scale_axis', 'no_out_scale', 'drop_tail', 'h_bf16']


@pytest.mark.parametrize('miss', MISSES)
def test_ffn_near_misses_are_rejected(miss):
    shape = MISS_SHAPES.get(miss, SHAPE)
    x, [(q1, s1), (q2, s2)], (b1, b2) = _inputs(*shape, glu=False)
    ref, bound = R.ffn_reference(x, q1, s1, b1, q2, s2, b2, 'relu')
    with pytest.raises(AssertionError, match='bound'):
        R.check(emulate_ffn(x, q1, s1, b1, q2, s2, b2, 'relu', miss), ref, bound, torch.tensor(COUNTS))


@pytest.mark.parametrize('miss', MISSES + ['swap'])
def test_glu_near_misses_are_rejected(miss):
    shape = MISS_SHAPES.get(miss, SHAPE)
    x, [(q1, s1), (q2, s2), (q3, s3)], _ = _inputs(*shape, glu=True)
    ref, bound = R.glu_reference(x, q1, s1, q2, s2, q3, s3, 'silu')
    with pytest.raises(AssertionError, match='bound'):
        R.check(emulate_glu(x, q1, s1, q2, s2, q3, s3, 'silu', miss), ref, bound, torch.tensor(COUNTS))


def test_nonzero_rows_past_the_count_are_rejected():
    x, [(q1, s1), (q2, s2), (q3, s3)], _ = _inputs(*SHAPE, glu=True)
    ref, bound = R.glu_reference(x, q1, s1, q2, s2, q3, s3, 'silu')
    y = emulate_glu(x, q1, s1, q2, s2, q3, s3, 'silu')
    y[3, 3] = ref[3, 3].float()                      # a row at the count, with the right values
    with pytest.raises(AssertionError, match='past the count'):
        R.check(y, ref, bound, torch.tensor(COUNTS))
