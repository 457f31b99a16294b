"""The stage checkers of tests/expert_ffn_reference.py on the CPU: the real FusedReluFFN, FusedReluFFNFp8, FusedGLUFFN and
GroupedLinear run on fp32 fakes of the ops they launch and pass; near misses, each one small change to an op or to what
one launch receives, are rejected by the check that guards them.  fp32 emulations of the 16-bit skinny kernels, in their
reduction order, pass their bounds; four near misses do not."""
import math

import pytest
import torch

import expert_ffn_reference as R
import gemm_reference as GR
from tutel_b200.ops import gemm as G


# ----------------------------------------------------------------------------------------------------------------
# fp32 fakes of the launches (the contracts in ops/gemm.py and csrc/gemm_sm90.h)
# ----------------------------------------------------------------------------------------------------------------
def _mat(a, b, a_mn, b_mn, scale_a=None, scale_b=None):
    A = a.float().transpose(1, 2) if a_mn else a.float()
    B = b.float() if b_mn else b.float().transpose(1, 2)
    acc = A @ B
    if scale_a is not None:
        acc = acc * scale_a.float().view(acc.size(0), -1, 1)
    if scale_b is not None:
        acc = acc * scale_b.float().view(acc.size(0), 1, -1)
    return acc


def _act(v, code):
    return GR.act_fn(v, code)


def _store(v, rc, dt, out=None):
    """Rows at or past the counts are left as they were; a fresh output holds garbage there (NaN and 3)."""
    if out is None:
        d = torch.full(v.shape, 3.0, dtype=dt)
        d[..., ::2] = math.nan
    else:
        d = out
    m = R._rows_mask(v, rc).unsqueeze(-1)
    d.copy_(torch.where(m, v.to(dt), d))
    return d


def fake_raw_gemm(a, b, *, a_mn=False, b_mn=False, epilogue=G.EPI_NONE, bias=None, aux=None, row_counts=None, out=None,
                  out_dtype=None, scale_a=None, scale_b=None, colsum=None, d2=None, act=0, **kw):
    if a.dim() == 2:
        a = a.unsqueeze(0)
    acc = _mat(a, b, a_mn, b_mn, scale_a, scale_b)
    dt = out_dtype or (a.dtype if a.element_size() > 1 else torch.bfloat16)
    if bias is not None:
        acc = acc + bias.float().view(acc.size(0), 1, -1)
    if epilogue in (G.EPI_NONE, G.EPI_BIAS):
        v = acc
    elif epilogue == G.EPI_BIAS_RELU:
        v = acc.clamp_min(0)
    elif epilogue in (G.EPI_BIAS_GELU, G.EPI_BIAS_SILU):
        v = _act(acc, GR.ACT_GELU if epilogue == G.EPI_BIAS_GELU else GR.ACT_SILU)
        if d2 is not None:
            _store(acc, row_counts, d2.dtype, d2)
    elif epilogue == G.EPI_RELU_BWD:
        v = torch.where(aux.float() > 0, acc, torch.zeros(()))
    elif epilogue == G.EPI_ACT_BWD:
        v = acc * GR.act_grad(aux.float(), act)
    elif epilogue == G.EPI_ADD:
        v = acc + aux.float()
    else:
        raise NotImplementedError(epilogue)
    if colsum is not None:
        colsum += torch.where(R._rows_mask(v, row_counts).unsqueeze(-1), v, torch.zeros(())).sum(1)
    return _store(v, row_counts, dt, out)


def fake_glu_gemm(a, b, b2, *, b_mn, act, save_pre=False, scale_a=None, scale_b=None, scale_b2=None, row_counts=None,
                  out_dtype=None, **kw):
    g, u = _mat(a, b, False, b_mn, scale_a, scale_b), _mat(a, b2, False, b_mn, scale_a, scale_b2)
    dt = out_dtype or (a.dtype if a.element_size() > 1 else torch.bfloat16)
    h = _act(g, G.ACT_CODES[act]) * u
    return (_store(h, row_counts, dt),) + ((_store(g, row_counts, dt), _store(u, row_counts, dt)) if save_pre else (None, None))


def fake_glu_gemm_bwd(dy, w, g, u, *, b_mn, act, row_counts=None, scale_a=None, scale_b=None, **kw):
    dh = _mat(dy, w, False, b_mn, scale_a, scale_b)
    code = G.ACT_CODES[act]
    gf, uf = g.float(), u.float()
    return (_store(dh * uf * GR.act_grad(gf, code), row_counts, g.dtype),
            _store(dh * _act(gf, code), row_counts, g.dtype))


def fake_quantize_rows(x):
    return R.quantize_rows_reference(x.contiguous())


def fake_fp8_operand(w, transpose):
    return G.quantize_rows((w.transpose(1, 2) if transpose else w).contiguous())


@pytest.fixture
def fakes(monkeypatch):
    for name, f in (('raw_gemm', fake_raw_gemm), ('glu_gemm', fake_glu_gemm), ('glu_gemm_bwd', fake_glu_gemm_bwd),
                    ('quantize_rows', fake_quantize_rows), ('fp8_operand', fake_fp8_operand)):
        monkeypatch.setattr(G, name, f)
    return monkeypatch


def tamper(monkeypatch, name, index, fn):
    """Call ``index`` (counted from 0 over the whole test) of op ``name`` runs ``fn(real, args, kw)`` instead."""
    real, n = getattr(G, name), [0]

    def op(*args, **kw):
        i = n[0]
        n[0] += 1
        return fn(real, args, kw) if i == index else real(*args, **kw)
    monkeypatch.setattr(G, name, op)


# ----------------------------------------------------------------------------------------------------------------
# cases
# ----------------------------------------------------------------------------------------------------------------
E, T, M, H, MO = 3, 150, 64, 48, 40           # T: one full 128-row tile and a partial one
COUNTS = torch.tensor([150, 1, 0], dtype=torch.int32)


def _t(*shape, scale=1.0, dtype=torch.bfloat16, seed=0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(dtype)


def _ffn_inputs(dtype=torch.bfloat16, bias=True, Mo=MO, H=H):
    x = _t(E, T, M, dtype=dtype, seed=1)
    w1, w2 = _t(E, H, M, scale=M ** -0.5, dtype=dtype, seed=2), _t(E, H, Mo, scale=H ** -0.5, dtype=dtype, seed=3)
    b1 = _t(E, H, scale=0.1, dtype=dtype, seed=4) if bias else None
    b2 = _t(E, Mo, scale=0.1, dtype=dtype, seed=5) if bias else None
    dy = _t(E, T, Mo, dtype=dtype, seed=6)
    return x, w1, b1, w2, b2, dy


def run_ffn(act='relu', fp8=False, rc=None, dtype=torch.bfloat16, bias=True, needs=(True,) * 5, Mo=MO, H=H):
    x, w1, b1, w2, b2, dy = _ffn_inputs(dtype, bias, Mo, H)
    ins = [t.requires_grad_(n) if t is not None else None for t, n in zip((x, w1, b1, w2, b2), needs)]
    with R.Recorder() as rec:
        y = G.fused_relu_ffn_fp8(*ins, rc) if fp8 else G.fused_act_ffn(*ins, rc, act)
        grads = y.grad_fn.apply(dy)
    R.check_fused_ffn(rec.take(), *[t.detach() if t is not None else None for t in ins], y.detach(), act=act, row_counts=rc,
                      dy=dy, grads=grads[:5], needs=needs, fp8=fp8, what='ffn %s fp8=%s' % (act, fp8))


def run_glu(act='silu', fp8=False, dtype=torch.bfloat16, needs=(True,) * 4):
    x = _t(E, T, M, dtype=dtype, seed=1)
    ws = [_t(E, M, H, scale=M ** -0.5, dtype=dtype, seed=2), _t(E, M, H, scale=M ** -0.5, dtype=dtype, seed=3),
          _t(E, H, M, scale=H ** -0.5, dtype=dtype, seed=4)]
    dy = _t(E, T, M, dtype=dtype, seed=5)
    ins = [t.requires_grad_(n) for t, n in zip([x] + ws, needs)]
    with R.Recorder() as rec:
        y = G.fused_glu_ffn(*ins, act, fp8)
        grads = y.grad_fn.apply(dy)
    R.check_glu_ffn(rec.take(), *[t.detach() for t in ins], y.detach(), act=act, fp8=fp8, dy=dy, grads=grads[:4],
                    needs=needs, what='glu %s fp8=%s' % (act, fp8))


def run_linear(layout='nk', bias=True, fp8=False, rc=None, needs=(True,) * 3):
    x = _t(E, T, M, seed=1)
    N = 48
    w = _t(E, N, M, scale=M ** -0.5, seed=2) if layout == 'nk' else _t(E, M, N, scale=M ** -0.5, seed=2)
    b = _t(E, N, scale=0.1, seed=3) if bias else None
    dy = _t(E, T, N, seed=4)
    ins = [t.requires_grad_(n) if t is not None else None for t, n in zip((x, w, b), needs)]
    with R.Recorder() as rec:
        y = G.GroupedLinear.apply(*ins, layout, rc, fp8)
        grads = y.grad_fn.apply(dy)
    R.check_grouped_linear(rec.take(), *[t.detach() if t is not None else None for t in ins], y.detach(), layout=layout,
                           fp8=fp8, row_counts=rc, dy=dy, grads=grads[:3], needs=needs, what='linear %s' % layout)


# ----------------------------------------------------------------------------------------------------------------
# the real functions on the fakes pass
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('act', ['relu', 'gelu', 'silu'])
@pytest.mark.parametrize('rc', [None, COUNTS])
@pytest.mark.parametrize('bias', [True, False])
def test_fused_ffn_passes(fakes, act, rc, bias):
    run_ffn(act, rc=rc, bias=bias)


@pytest.mark.parametrize('needs', [(True, False, False, False, False), (False, True, True, True, True),
                                   (False, False, False, True, False)])
def test_fused_ffn_partial_gradients_pass(fakes, needs):
    run_ffn('gelu', needs=needs, rc=COUNTS, dtype=torch.float16)


@pytest.mark.parametrize('rc', [None, COUNTS])
@pytest.mark.parametrize('needs', [(True,) * 5, (True, False, False, False, False), (False, True, True, True, True)])
def test_fused_ffn_fp8_passes(fakes, rc, needs):
    run_ffn(fp8=True, rc=rc, needs=needs)


@pytest.mark.parametrize('act', ['silu', 'relu', 'gelu'])
@pytest.mark.parametrize('fp8', [False, True])
def test_glu_ffn_passes(fakes, act, fp8):
    run_glu(act, fp8)


@pytest.mark.parametrize('needs', [(True, False, False, False), (False, True, True, True)])
def test_glu_ffn_partial_gradients_pass(fakes, needs):
    run_glu('silu', False, torch.float16, needs)


@pytest.mark.parametrize('layout', ['nk', 'kn'])
@pytest.mark.parametrize('bias', [True, False])
@pytest.mark.parametrize('fp8', [False, True])
@pytest.mark.parametrize('rc', [None, COUNTS])
def test_grouped_linear_passes(fakes, layout, bias, fp8, rc):
    run_linear(layout, bias, fp8, rc)


def test_quantize_reference_is_the_kernel_formula():
    """s = max|row| * fp32(1/448), q = e4m3(x * fp32(1/s)): the largest element maps to 448, zero rows get s = 1."""
    x = torch.tensor([[3.0, -7.5, 0.25, 1e-3], [0.0, 0.0, 0.0, 0.0], [math.nan, 2.0, -1.0, 0.5]])
    q, s = R.quantize_rows_reference(x)
    assert s[1] == 1.0 and float(q[0, 1]) == -448.0 and float(q[2, 1]) == 448.0 and bool(torch.isnan(q[2, 0].float()))
    assert s[0] == torch.tensor(7.5) * torch.tensor(1.0 / 448.0)


# ----------------------------------------------------------------------------------------------------------------
# near misses
# ----------------------------------------------------------------------------------------------------------------
def _fails(match, run):
    with pytest.raises(AssertionError, match=match):
        run()


def test_near_miss_dw2_from_act_before_the_zero_tail(fakes):
    acts = []
    tamper(fakes, 'raw_gemm', 0, lambda real, a, kw: acts.append(real(*a, **kw)) or acts[0])
    tamper(fakes, 'raw_gemm', 3, lambda real, a, kw: real(acts[0], *a[1:], **kw))     # the dw2 launch
    _fails('dw2', lambda: run_ffn(rc=COUNTS))


def test_near_miss_relu_backward_mask_from_dy(fakes):
    def dh(real, a, kw):
        out = real(*a, **dict(kw, epilogue=G.EPI_NONE, aux=None))
        return torch.where(torch.nan_to_num(out.float()) > 0, out, torch.zeros((), dtype=out.dtype))
    tamper(fakes, 'raw_gemm', 2, dh)
    _fails('dh', lambda: run_ffn())


def test_near_miss_db1_summed_over_rows_past_the_counts(fakes):
    x, w1, b1, w2, b2, dy = _ffn_inputs()
    # the dh launch sees every row of dy (not zero-tailed) and sums all of them into db1
    tamper(fakes, 'raw_gemm', 2, lambda real, a, kw: real(dy, *a[1:], **dict(kw, row_counts=None)))
    _fails('colsum', lambda: run_ffn(rc=COUNTS))


def test_near_miss_one_experts_db2_dropped(fakes):
    def cs(real, a, kw):
        out = real(*a, **kw).clone()
        out[1] = 0
        return out
    tamper(fakes, 'column_sums', 0, cs)
    _fails('db2', lambda: run_ffn())


def test_near_miss_w1t_fp8_copy_scaled_per_row_of_w1(fakes):
    def per_row(real, a, kw):          # W1 [E, M, M]: W1^T needs one scale per column of W1, not per row
        q, s = G.quantize_rows(a[0].contiguous())
        return q.transpose(1, 2).contiguous(), s
    tamper(fakes, 'fp8_operand', 3, per_row)       # W1, W2^T (forward), W2, W1^T (backward)
    _fails('W1\\^T', lambda: run_ffn(fp8=True, H=M))


def test_near_miss_glu_dx_without_its_du_term(fakes):
    tamper(fakes, 'raw_gemm', 5, lambda real, a, kw: kw['aux'].clone())       # forward y, dw3, dw1, dw2, dx.1, dx
    _fails('dx', lambda: run_glu())


def test_near_miss_glu_backward_with_g_and_u_swapped(fakes):
    tamper(fakes, 'glu_gemm_bwd', 0, lambda real, a, kw: real(a[0], a[1], a[3], a[2], **kw))
    _fails('dg', lambda: run_glu())


def test_near_miss_dw1_of_two_experts_swapped(fakes):
    def dw1(real, a, kw):
        out = real(*a, **kw).clone()
        out[[0, 1]] = out[[1, 0]]
        return out
    tamper(fakes, 'raw_gemm', 5, dw1)            # act, y, dh, dw2, dx, dw1
    _fails('dw1', lambda: run_ffn())


@pytest.mark.parametrize('ulps', [3, -2])
def test_near_miss_a_few_ulps_in_the_last_partial_row_tile(fakes, ulps):
    def dx(real, a, kw):
        out = real(*a, **kw).clone()
        v = out[0, T - 1, 5].float()
        out[0, T - 1, 5] = (v + ulps * 2 * GR.half_ulp(v.double(), torch.bfloat16).float()).to(out.dtype)
        return out
    tamper(fakes, 'raw_gemm', 4, dx)
    _fails('dx', lambda: run_ffn('silu'))


def test_near_miss_grouped_linear_ignores_the_counts_in_the_backward(fakes):
    """What GroupedLinear did before it zero-tailed dy: rows of dy past the counts reached dw and db."""
    x = _t(E, T, M, seed=1)
    dy = _t(E, T, 48, seed=4)
    tamper(fakes, 'raw_gemm', 2, lambda real, a, kw: real(a[0], dy, **kw))      # y, dx, dw (nk: dy^T x)
    _fails('dw', lambda: run_linear('kn', rc=COUNTS))


def test_recorder_rejects_a_different_launch_order(fakes):
    x, w1, b1, w2, b2, dy = _ffn_inputs()
    with R.Recorder() as rec:
        y = G.fused_relu_ffn_fp8(x, w1, b1, w2, b2)
    calls = rec.take().calls
    assert [c.name for c in calls] == ['quantize_rows', 'fp8_operand', 'raw_gemm'] * 2
    check = lambda cs: R.check_fused_ffn(R.Calls(cs), x, w1, b1, w2, b2, y, fp8=True)      # noqa: E731
    check(calls)
    _fails('expected call 0 to be quantize_rows, got fp8_operand', lambda: check([calls[1], calls[0]] + calls[2:]))
    _fails('made no more calls', lambda: check(calls[:4]))
    _fails('unexpected extra calls', lambda: check(calls + calls[-1:]))


# ----------------------------------------------------------------------------------------------------------------
# skinny kernels: fp32 emulations in the kernels' reduction order
# ----------------------------------------------------------------------------------------------------------------
def _fma(acc, a, b):
    return (acc.double() + a.double() * b.double()).float()


def _butterfly(acc):
    """Five xor-shuffle levels over the last dim (32 lanes); every lane ends with the sum."""
    lanes = torch.arange(32)
    for o in (16, 8, 4, 2, 1):
        acc = acc + acc[..., lanes ^ o]
    return acc[..., 0]


def emulate_skinny_ffn(x, w1, b1, w2, b2, act, counts, h_dtype=None, bias_every_slice=False, drop_last_slice=False):
    V = R._vec(x.dtype)
    G_, Rw, K = x.shape
    H, N = w1.size(1), w2.size(2)
    Kp = -(-K // (32 * V)) * 32 * V
    xs = torch.nn.functional.pad(x.float(), (0, Kp - K)).view(G_, Rw, 1, -1, 32, V)
    ws = torch.nn.functional.pad(w1.float(), (0, Kp - K)).view(G_, 1, H, -1, 32, V)
    acc = torch.zeros(G_, Rw, H, 32)
    for m in range(xs.size(3)):
        for q in range(V):
            acc = _fma(acc, xs[:, :, :, m, :, q], ws[:, :, :, m, :, q])
    pre = _butterfly(acc)
    if b1 is not None:
        pre = pre + b1.float().view(G_, 1, H)
    h = R._FN[act](pre)
    if h_dtype is not None:
        h = h.to(h_dtype).float()
    y = torch.zeros(G_, Rw, N)
    slices = list(range(0, H, R.HS))
    if drop_last_slice:
        slices = slices[:-1]
    for s, h0 in enumerate(slices):
        part = torch.zeros(G_, Rw, N)
        for j in range(h0, min(H, h0 + R.HS)):
            part = _fma(part, h[:, :, j:j + 1], w2[:, j:j + 1, :].float())
        if b2 is not None and (s == 0 or bias_every_slice):
            part = part + b2.float().view(G_, 1, N)
        y = y + part
    return zero_rows(y, counts)


def emulate_skinny_gemm(x, w, bias, kn, relu, counts, drop_relu=False):
    G_, Rw, K = x.shape
    W = w.float() if kn else w.float().transpose(1, 2)                  # [G, K, N]
    if kn:
        acc = torch.zeros(G_, Rw, W.size(2))
        for k in range(K):
            acc = _fma(acc, x[:, :, k:k + 1].float(), W[:, k:k + 1, :])
    else:
        Kp = -(-K // 32) * 32
        xs = torch.nn.functional.pad(x.float(), (0, Kp - K)).view(G_, Rw, 1, -1, 32)
        ws = torch.nn.functional.pad(W.transpose(1, 2), (0, Kp - K)).view(G_, 1, W.size(2), -1, 32)
        lanes = torch.zeros(G_, Rw, W.size(2), 32)
        for m in range(xs.size(3)):
            lanes = _fma(lanes, xs[:, :, :, m], ws[:, :, :, m])
        acc = _butterfly(lanes)
    if bias is not None:
        acc = acc + bias.float().unsqueeze(1)
    if relu and not drop_relu:
        acc = acc.clamp_min(0)
    return zero_rows(acc.to(x.dtype), counts)


def zero_rows(y, counts):
    return R.zero_tail(y, counts.clamp(max=y.size(1)))


SK_COUNTS = torch.tensor([0, 1, 2, 3, 5, 9], dtype=torch.int32)


def _skinny_ffn_inputs(K, H, N, dtype, seed=0):
    Gn, Rw = SK_COUNTS.numel(), 9
    x = _t(Gn, Rw, K, dtype=dtype, seed=seed)
    w1, w2 = _t(Gn, H, K, scale=K ** -0.5, dtype=dtype, seed=seed + 1), _t(Gn, H, N, scale=H ** -0.5, dtype=dtype, seed=seed + 2)
    b1, b2 = _t(Gn, H, scale=0.5, dtype=dtype, seed=seed + 3), _t(Gn, N, scale=0.5, dtype=dtype, seed=seed + 4)
    return x, w1, b1, w2, b2


@pytest.mark.parametrize('act', ['relu', 'gelu', 'silu'])
@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float32])
def test_skinny_ffn_emulation_passes(act, dtype):
    x, w1, b1, w2, b2 = _skinny_ffn_inputs(264, 136, 40, dtype)          # a partial 64-unit slice
    for bias in (True, False):
        bb1, bb2 = (b1, b2) if bias else (None, None)
        y = emulate_skinny_ffn(x, w1, bb1, w2, bb2, act, SK_COUNTS)
        ref, bound = R.skinny_ffn_reference(x, w1, bb1, w2, bb2, act)
        assert R.check_skinny('skinny_ffn emulation', y, ref, bound, SK_COUNTS) <= 1.0


@pytest.mark.parametrize('miss', ['bias_every_slice', 'drop_last_slice'])
def test_skinny_ffn_near_misses(miss):
    x, w1, b1, w2, b2 = _skinny_ffn_inputs(264, 136, 40, torch.bfloat16)
    y = emulate_skinny_ffn(x, w1, b1, w2, b2, 'silu', SK_COUNTS, **{miss: True})
    ref, bound = R.skinny_ffn_reference(x, w1, b1, w2, b2, 'silu')
    _fails('outside the bound', lambda: R.check_skinny('skinny_ffn ' + miss, y, ref, bound, SK_COUNTS))


def test_skinny_ffn_rejects_bf16_hidden_activations_at_bench_dims():
    """At M = 4096, H = 14336 the bound is far below a bf16 rounding of h, which the loose (K + H) form lets through.
    The pre-activations are 1.x + 0.375 bf16 ulp, so every rounding goes the same way."""
    K, H, N = 4096, 14336, 16
    g = torch.Generator().manual_seed(7)
    x = torch.zeros(1, 1, K, dtype=torch.bfloat16)
    x[0, 0, :2] = 1
    w1 = torch.zeros(1, H, K, dtype=torch.bfloat16)
    w1[0, :, 0] = (1 + torch.randint(0, 128, (H,), generator=g) / 128.0).bfloat16()
    w1[0, :, 1] = 3 * 2.0 ** -10
    w1[0, :, 2:] = (torch.randn(H, K - 2, generator=g) * 2.0 ** -20).bfloat16()     # a dense first layer, ~no effect on h
    w2 = (torch.rand(1, H, N, generator=g) / H).bfloat16()
    counts = torch.tensor([1], dtype=torch.int32)
    ref, bound = R.skinny_ffn_reference(x, w1, None, w2, None, 'relu')
    assert R.check_skinny('skinny_ffn emulation', emulate_skinny_ffn(x, w1, None, w2, None, 'relu', counts),
                          ref, bound, counts) <= 1.0
    bad = emulate_skinny_ffn(x, w1, None, w2, None, 'relu', counts, h_dtype=torch.bfloat16)
    _fails('outside the bound', lambda: R.check_skinny('skinny_ffn bf16 h', bad, ref, bound, counts))
    ref, loose = R.skinny_ffn_reference(x, w1, None, w2, None, 'relu', loose=True)
    assert bool(((bad.double() - ref).abs() <= loose).all()), 'the loose bound was expected to miss this'


@pytest.mark.parametrize('kn', [False, True])
@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16, torch.float32])
def test_skinny_gemm_emulation_passes_and_missing_relu_fails(kn, dtype):
    Gn, Rw, K, N = SK_COUNTS.numel(), 9, 2100 if not kn else 300, 72        # nk: two 1024 chunks and a partial one
    x = _t(Gn, Rw, K, dtype=dtype, seed=3)
    w = _t(Gn, K, N, scale=K ** -0.5, dtype=dtype, seed=4) if kn else _t(Gn, N, K, scale=K ** -0.5, dtype=dtype, seed=4)
    b = _t(Gn, N, scale=0.5, dtype=dtype, seed=5)
    for bias, relu in ((b, True), (None, False)):
        y = emulate_skinny_gemm(x, w, bias, kn, relu, SK_COUNTS)
        ref, bound = R.skinny_gemm_reference(x, w, bias, kn, relu)
        assert R.check_skinny('skinny_gemm emulation', y, ref, bound, SK_COUNTS) <= 1.0
    y = emulate_skinny_gemm(x, w, b, kn, True, SK_COUNTS, drop_relu=True)
    ref, bound = R.skinny_gemm_reference(x, w, b, kn, True)
    _fails('outside the bound', lambda: R.check_skinny('skinny_gemm without relu', y, ref, bound, SK_COUNTS))
