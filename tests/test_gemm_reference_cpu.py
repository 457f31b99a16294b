"""The fp64 GEMM reference and its per-element bound (tests/gemm_reference.py) on CPU.

An emulation of the kernel's arithmetic (exact products, fp32 sums, fp32 epilogue, one rounding to the output dtype)
must pass the check, and each of a set of near misses - kernels that are subtly wrong - must fail it.  This keeps the
bound honest: it is loose enough for a correct kernel and tight enough to catch these mistakes.
"""
import pytest
import torch

import gemm_reference as R

G_, M_, N_, K_ = 3, 328, 264, 200


def _data(dtype=torch.bfloat16, seed=0, K=K_):
    gen = torch.Generator().manual_seed(seed)
    rnd = lambda *s: (torch.randn(*s, generator=gen) * 0.5)   # noqa: E731
    a, b, b2 = rnd(G_, M_, K), rnd(G_, N_, K), rnd(G_, N_, K)
    bias, aux, aux2 = rnd(G_, N_) * 4, rnd(G_, M_, N_) * 4, rnd(G_, M_, N_) * 4
    if dtype in (torch.float8_e4m3fn, torch.float8_e5m2):
        top = 448.0 if dtype == torch.float8_e4m3fn else 57344.0
        sa, sb = a.abs().amax(-1) / top, b.abs().amax(-1) / top
        a, b = (a / sa[..., None]).to(dtype), (b / sb[..., None]).to(dtype)
        return dict(a=a, b=b, b2=None, bias=bias.bfloat16(), aux=aux.bfloat16(), aux2=aux2.bfloat16(), scale_a=sa, scale_b=sb)
    return dict(a=a.to(dtype), b=b.to(dtype), b2=b2.to(dtype), bias=bias.to(dtype), aux=aux.to(dtype), aux2=aux2.to(dtype),
                scale_a=None, scale_b=None)


def _gelu(x, tanh=False):
    return torch.nn.functional.gelu(x, approximate='tanh' if tanh else 'none')


def _emulate(t, epilogue, out_dtype, act=R.ACT_SILU, alpha=1.0, row_counts=None, miss=None):
    """What the kernel computes: exact products summed in fp32, the epilogue in fp32, one rounding to out_dtype.
    ``miss`` selects a near miss.  Returns (d, d2, colsum)."""
    a, b = t['a'].float(), t['b'].float()
    if miss == 'drop_k_block':
        a = a.clone()
        a[..., 64:128] = 0
    acc = a @ b.transpose(1, 2)
    if t['scale_a'] is not None:
        sb = t['scale_b'].roll(1, dims=-1) if miss == 'shift_scale_b' else t['scale_b']
        acc = acc * (t['scale_a'][:, :, None] * sb[:, None, :])
    if miss == 'round_acc':
        acc = acc.to(out_dtype).float()
    bias = t['bias'].float()[:, None, :]
    d2 = None
    if epilogue == R.EPI_NONE:
        v = acc * alpha
    elif epilogue == R.EPI_BIAS:
        v = acc + bias
    elif epilogue == R.EPI_BIAS_RELU:
        v = torch.relu(acc) + bias if miss == 'bias_after_act' else torch.relu(acc + bias)
    elif epilogue == R.EPI_BIAS_GELU:
        d2 = acc + bias
        v = _gelu(d2, tanh=miss == 'tanh_gelu')
    elif epilogue == R.EPI_BIAS_SILU:
        d2 = acc + bias
        v = torch.nn.functional.silu(d2)
    elif epilogue == R.EPI_RELU_BWD:
        v = torch.where(t['aux'].float() > 0, acc, torch.zeros(()))
    elif epilogue == R.EPI_ADD:
        v = acc + t['aux'].float()
    elif epilogue == R.EPI_ACT_BWD:
        v = acc * R.act_grad(t['aux'].float(), act)
    elif epilogue == R.EPI_GLU:
        g, u = acc, t['a'].float() @ t['b2'].float().transpose(1, 2)
        v = R.act_fn(g, act) * u
        d2 = (g, u)
    elif epilogue == R.EPI_GLU_BWD:
        g, u = t['aux'].float(), t['aux2'].float()
        v = acc * u * R.act_grad(g, act)
        d2 = acc * R.act_fn(g, act)
    rows = torch.arange(M_).view(1, M_, 1)
    valid = rows < (row_counts.view(-1, 1, 1) if row_counts is not None else M_)
    if miss == 'colsum_all_rows':
        valid = torch.ones_like(valid)
    colsum = torch.where(valid, v, torch.zeros(())).sum(1)
    if isinstance(d2, tuple):
        d2 = tuple(x.to(out_dtype) for x in d2)
    elif d2 is not None:
        d2 = d2.to(out_dtype)
    return v.to(out_dtype), d2, colsum


def _ref(t, epilogue, out_dtype, act=R.ACT_SILU, alpha=1.0, row_counts=None):
    return R.ref_gemm(t['a'], t['b'], epilogue=epilogue, alpha=alpha, bias=t['bias'], aux=t['aux'], aux2=t['aux2'],
                      b2=t['b2'] if epilogue == R.EPI_GLU else None, act=act, scale_a=t['scale_a'], scale_b=t['scale_b'],
                      row_counts=row_counts, out_dtype=out_dtype, want_pre=True)


def _check(r, epilogue, out, row_counts=None):
    d, d2, cs = out
    if epilogue == R.EPI_GLU:
        R.check(r, d, d2=d2[0], d3=d2[1])
    else:
        R.check(r, d, d2=d2, colsum=cs)


CASES = [(R.EPI_NONE, R.ACT_SILU), (R.EPI_BIAS, R.ACT_SILU), (R.EPI_BIAS_RELU, R.ACT_SILU), (R.EPI_BIAS_GELU, R.ACT_SILU),
         (R.EPI_BIAS_SILU, R.ACT_SILU), (R.EPI_RELU_BWD, R.ACT_SILU), (R.EPI_ADD, R.ACT_SILU), (R.EPI_ACT_BWD, R.ACT_GELU),
         (R.EPI_ACT_BWD, R.ACT_SILU), (R.EPI_ACT_BWD, R.ACT_RELU), (R.EPI_GLU, R.ACT_GELU), (R.EPI_GLU, R.ACT_SILU),
         (R.EPI_GLU, R.ACT_RELU), (R.EPI_GLU_BWD, R.ACT_GELU), (R.EPI_GLU_BWD, R.ACT_SILU), (R.EPI_GLU_BWD, R.ACT_RELU)]


@pytest.mark.parametrize('dtype,out_dtype', [(torch.bfloat16, torch.bfloat16), (torch.float16, torch.float16),
                                             (torch.bfloat16, torch.float32)])
@pytest.mark.parametrize('epilogue,act', CASES)
def test_emulated_kernel_passes(epilogue, act, dtype, out_dtype):
    t = _data(dtype)
    _check(_ref(t, epilogue, out_dtype, act), epilogue, _emulate(t, epilogue, out_dtype, act))


@pytest.mark.parametrize('dtype', [torch.float8_e4m3fn, torch.float8_e5m2])
@pytest.mark.parametrize('epilogue', [R.EPI_NONE, R.EPI_BIAS, R.EPI_BIAS_RELU, R.EPI_RELU_BWD, R.EPI_ADD])
def test_emulated_fp8_kernel_passes(epilogue, dtype):
    t = _data(dtype)
    _check(_ref(t, epilogue, torch.bfloat16), epilogue, _emulate(t, epilogue, torch.bfloat16))


def test_emulated_row_counts_and_alpha_pass():
    t = _data()
    rc = torch.tensor([0, 129, 400], dtype=torch.int32)
    _check(_ref(t, R.EPI_RELU_BWD, torch.bfloat16, row_counts=rc), R.EPI_RELU_BWD,
           _emulate(t, R.EPI_RELU_BWD, torch.bfloat16, row_counts=rc))
    _check(_ref(t, R.EPI_NONE, torch.float32, alpha=0.375), R.EPI_NONE, _emulate(t, R.EPI_NONE, torch.float32, alpha=0.375))


def test_bound_is_much_tighter_than_allclose():
    # on outputs of magnitude up to 4, as in the allclose checks of the 16-bit GEMM tests (atol 0.1, rtol 2e-2), the
    # per-element bound is at least 10x tighter, and its accumulation part is a small fraction of the final rounding
    t = _data()
    r = _ref(t, R.EPI_BIAS, torch.bfloat16)
    v = r.outs['d'].val
    tol = R.tolerance(r, 'd')
    small = v.abs() <= 4
    assert float((tol / (0.1 + 2e-2 * v.abs()))[small].max()) <= 0.1
    assert float((R.C_ACC[torch.bfloat16] * r.outs['d'].acc / R.half_ulp(v, torch.bfloat16))[v.abs() >= 1].max()) <= 0.1


NEAR_MISSES = [
    ('tanh_gelu', R.EPI_BIAS_GELU, torch.bfloat16, torch.float32, R.ACT_SILU),
    ('round_acc', R.EPI_BIAS, torch.bfloat16, torch.bfloat16, R.ACT_SILU),
    ('round_acc', R.EPI_BIAS, torch.float16, torch.float16, R.ACT_SILU),
    ('bias_after_act', R.EPI_BIAS_RELU, torch.bfloat16, torch.bfloat16, R.ACT_SILU),
    ('shift_scale_b', R.EPI_BIAS, torch.float8_e4m3fn, torch.bfloat16, R.ACT_SILU),
    ('drop_k_block', R.EPI_NONE, torch.bfloat16, torch.bfloat16, R.ACT_SILU),
    ('colsum_all_rows', R.EPI_RELU_BWD, torch.bfloat16, torch.bfloat16, R.ACT_SILU),
]


@pytest.mark.parametrize('miss,epilogue,dtype,out_dtype,act', NEAR_MISSES, ids=[m[0] + '-' + str(m[3])[6:] for m in NEAR_MISSES])
def test_near_miss_is_rejected(miss, epilogue, dtype, out_dtype, act):
    t = _data(dtype)
    rc = torch.tensor([300, 129, 200], dtype=torch.int32) if miss == 'colsum_all_rows' else None
    r = _ref(t, epilogue, out_dtype, act, row_counts=rc)
    _check(r, epilogue, _emulate(t, epilogue, out_dtype, act, row_counts=rc))      # the faithful emulation passes ...
    with pytest.raises(AssertionError):                                              # ... and the near miss does not
        _check(r, epilogue, _emulate(t, epilogue, out_dtype, act, row_counts=rc, miss=miss))


def test_half_ulp():
    x = torch.tensor([1.0, 1.5, 3.0, -3.0, 0.0, 2.0 ** -130, 65504.0], dtype=torch.float64)
    assert R.half_ulp(x, torch.bfloat16).tolist() == [2.0 ** -8, 2.0 ** -8, 2.0 ** -7, 2.0 ** -7, 2.0 ** -134, 2.0 ** -134, 2.0 ** 7]
    assert R.half_ulp(x[:5], torch.float16).tolist() == [2.0 ** -11, 2.0 ** -11, 2.0 ** -10, 2.0 ** -10, 2.0 ** -25]
    assert R.half_ulp(x[:2], torch.float32).tolist() == [2.0 ** -24, 2.0 ** -24]
