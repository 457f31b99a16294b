"""The expert autograd functions of ops/gemm.py stage by stage, and the 16-bit skinny decode kernels, against the fp64
references of tests/expert_ffn_reference.py.

* ``FusedReluFFN`` (ReLU / GELU / SiLU), ``FusedReluFFNFp8``, ``FusedGLUFFN`` (16 bit and fp8) and ``GroupedLinear``:
  every launch's output, the e4m3 copies bit for bit, the returned gradients' values and dtypes, ``None`` for inputs
  that asked for none, at T off the 128-row tile with 1-row and empty experts, N off 128 / 256, K off 64, G = 1 and
  G > 1, bf16 and fp16, with and without biases, non-contiguous and expanded ``dy``;
* rows past ``row_counts``: NaN in x for forward-only calls (valid rows must stay within bound), finite garbage in x
  and dy for backward calls (gradients must be those of the valid rows alone);
* one case at the benchmark's dimensions (M = 4096, H = 14336);
* the two expert modules: which function each configuration takes, and its output;
* ``skinny_ffn`` / ``skinny_gemm`` at counts around the 1-, 2- and 4-row passes, partial slices and chunks, K at the
  staging limit.
"""
import math

import pytest
import torch
import torch.nn.functional as F

import dispatch_reference as D
import expert_ffn_reference as R
import gemm_reference as GR

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module', autouse=True)
def _report():
    yield
    print('\nexpert FFN normalised errors per stage (<= C_ACC: bf16/fp16 %g, e4m3 %g): %s; colsum: %s' % (
        GR.C_ACC[torch.bfloat16], GR.C_ACC[torch.float8_e4m3fn],
        {k: round(v, 3) for k, v in sorted(R.OBSERVED.items())}, D.OBSERVED.get('colsum')))


def G_():
    from tutel_b200.ops import gemm
    return gemm


def _gen(seed):
    return torch.Generator(device='cuda').manual_seed(seed)


def _rand(shape, seed, scale=1.0, dtype=torch.bfloat16):
    return (torch.randn(shape, generator=_gen(seed), device='cuda') * scale).to(dtype)


def _counts(vals):
    return None if vals is None else torch.tensor(vals, dtype=torch.int32, device='cuda')


def _fill_past(t, rc, value):
    """Rows of t at or past the counts set to ``value`` (NaN, or finite garbage when None)."""
    if rc is None:
        return t
    past = ~R._rows_mask(t, rc)
    g = _rand(t.shape, 99, 3.0, t.dtype) if value is None else torch.full_like(t, value)
    return torch.where(past.unsqueeze(-1), g, t)


def _dy(y, seed, kind):
    if kind == 'expanded':          # the gradient of y.sum()
        return torch.ones((), dtype=y.dtype, device='cuda').expand_as(y)
    d = _rand(y.shape, seed, 1.0, y.dtype)
    if kind == 'strided':           # every other column of a wider buffer
        wide = torch.zeros(list(y.shape[:-1]) + [2 * y.size(-1)], dtype=y.dtype, device='cuda')
        wide[..., ::2] = d
        return wide[..., ::2]
    return d


def _leaves(ts, needs):
    return [None if t is None else t.detach().requires_grad_(n) for t, n in zip(ts, needs)]


def _det(ts):
    return [None if t is None else t.detach() for t in ts]


ALL5, X_ONLY5, W_ONLY5 = (True,) * 5, (True, False, False, False, False), (False, True, True, True, True)


# ----------------------------------------------------------------------------------------------------------------
# FusedReluFFN / FusedReluFFNFp8
# ----------------------------------------------------------------------------------------------------------------
def run_ffn(E, T, M, H, Mo, act='relu', dtype=torch.bfloat16, bias=True, rc=None, fp8=False, needs=ALL5, dy_kind='dense',
            seed=0):
    G = G_()
    x = _rand((E, T, M), seed + 1, 1.0, dtype)
    w1, w2 = _rand((E, H, M), seed + 2, M ** -0.5, dtype), _rand((E, H, Mo), seed + 3, H ** -0.5, dtype)
    b1 = _rand((E, H), seed + 4, 0.1, dtype) if bias else None
    b2 = _rand((E, Mo), seed + 5, 0.1, dtype) if bias else None
    rc = _counts(rc)
    grad = any(needs)
    x = _fill_past(x, rc, None if grad else math.nan)
    ins = _leaves((x, w1, b1, w2, b2), needs)
    what = 'ffn %s %s E=%d T=%d M=%d H=%d Mo=%d bias=%s rc=%s fp8=%s needs=%s dy=%s' % (
        act, dtype, E, T, M, H, Mo, bias, None if rc is None else rc.tolist(), fp8, needs, dy_kind)
    with R.Recorder() as rec:
        if grad:
            y = G.fused_relu_ffn_fp8(*ins, rc) if fp8 else G.fused_act_ffn(*ins, rc, act)
            dy = _fill_past(_dy(y, seed + 6, dy_kind), rc, None) if dy_kind != 'expanded' else _dy(y, 0, dy_kind)
            grads = y.grad_fn.apply(dy)[:5]
        else:
            with torch.no_grad():
                y = G.fused_relu_ffn_fp8(*ins, rc) if fp8 else G.fused_act_ffn(*ins, rc, act)
            dy = grads = None
    R.check_fused_ffn(rec.take(), *_det(ins), y.detach(), act=act, row_counts=rc, dy=dy, grads=grads, needs=needs,
                      fp8=fp8, what=what)


FFN_CASES = [
    # E, T, M, H, Mo, act, dtype, bias, counts
    (2, 200, 264, 392, 200, 'relu', torch.bfloat16, True, None),
    (1, 77, 136, 264, 136, 'relu', torch.float16, False, None),
    (3, 300, 256, 136, 264, 'gelu', torch.bfloat16, True, [300, 1, 0]),
    (2, 130, 200, 256, 128, 'silu', torch.float16, True, [129, 1]),
    (1, 129, 328, 200, 72, 'silu', torch.bfloat16, False, [128]),
    (4, 64, 64, 520, 64, 'gelu', torch.float16, False, [0, 64, 1, 33]),
]


@pytest.mark.parametrize('E,T,M,H,Mo,act,dtype,bias,rc', FFN_CASES)
def test_fused_ffn_stage_by_stage(E, T, M, H, Mo, act, dtype, bias, rc):
    run_ffn(E, T, M, H, Mo, act, dtype, bias, rc)


@pytest.mark.parametrize('needs', [X_ONLY5, W_ONLY5, (False, False, False, True, True)])
@pytest.mark.parametrize('act', ['relu', 'silu'])
def test_fused_ffn_partial_gradients(needs, act):
    run_ffn(2, 150, 136, 200, 72, act, torch.bfloat16, True, [150, 3], needs=needs)


@pytest.mark.parametrize('dy_kind', ['strided', 'expanded'])
@pytest.mark.parametrize('fp8', [False, True])
def test_fused_ffn_dy_layouts(dy_kind, fp8):
    run_ffn(2, 160, 256, 384, 128, 'relu', torch.bfloat16, True, None, fp8=fp8, dy_kind=dy_kind)


@pytest.mark.parametrize('act,fp8', [('relu', False), ('gelu', False), ('silu', False), ('relu', True)])
def test_fused_ffn_forward_only_nan_past_the_counts(act, fp8):
    run_ffn(3, 200, 256, 384, 128, act, torch.bfloat16, True, [200, 1, 0], fp8=fp8, needs=(False,) * 5)


FP8_CASES = [
    # E, T, M, H, Mo, dtype, bias, counts
    (2, 200, 256, 384, 128, torch.bfloat16, True, None),
    (3, 130, 144, 272, 208, torch.float16, False, [130, 1, 0]),
    (1, 64, 512, 128, 512, torch.bfloat16, True, [40]),
]


@pytest.mark.parametrize('E,T,M,H,Mo,dtype,bias,rc', FP8_CASES)
@pytest.mark.parametrize('needs', [ALL5, X_ONLY5, W_ONLY5])
def test_fused_ffn_fp8_stage_by_stage(E, T, M, H, Mo, dtype, bias, rc, needs):
    run_ffn(E, T, M, H, Mo, 'relu', dtype, bias, rc, fp8=True, needs=needs)


def test_fused_ffn_at_the_benchmark_dimensions():
    """dx accumulates over K = 14336."""
    run_ffn(2, 200, 4096, 14336, 4096, 'relu', torch.bfloat16, True, [200, 3])


# ----------------------------------------------------------------------------------------------------------------
# FusedGLUFFN
# ----------------------------------------------------------------------------------------------------------------
def run_glu(E, T, M, H, act='silu', dtype=torch.bfloat16, fp8=False, needs=(True,) * 4, rc=None, dy_kind='dense', seed=10):
    G = G_()
    x = _rand((E, T, M), seed + 1, 1.0, dtype)
    ws = [_rand((E, M, H), seed + 2, M ** -0.5, dtype), _rand((E, M, H), seed + 3, M ** -0.5, dtype),
          _rand((E, H, M), seed + 4, H ** -0.5, dtype)]
    rc = _counts(rc)
    grad = any(needs)
    x = _fill_past(x, rc, math.nan)
    ins = _leaves([x] + ws, needs)
    what = 'glu %s %s E=%d T=%d M=%d H=%d fp8=%s needs=%s rc=%s dy=%s' % (act, dtype, E, T, M, H, fp8, needs,
                                                                          None if rc is None else rc.tolist(), dy_kind)
    with R.Recorder() as rec:
        if grad:
            y = G.fused_glu_ffn(*ins, act, fp8)
            dy = _dy(y, seed + 5, dy_kind)
            grads = y.grad_fn.apply(dy)[:4]
        else:
            with torch.no_grad():
                y = G.fused_glu_ffn(*ins, act, fp8, rc)
            dy = grads = None
    R.check_glu_ffn(rec.take(), *_det(ins), y.detach(), act=act, fp8=fp8, row_counts=rc, dy=dy, grads=grads, needs=needs,
                    what=what)


@pytest.mark.parametrize('E,T,M,H,act,dtype,fp8', [
    (2, 200, 264, 392, 'silu', torch.bfloat16, False),
    (1, 77, 136, 200, 'gelu', torch.float16, False),
    (3, 130, 256, 136, 'relu', torch.bfloat16, False),
    (2, 200, 256, 384, 'silu', torch.bfloat16, True),
    (1, 130, 144, 272, 'relu', torch.float16, True),
])
def test_glu_ffn_stage_by_stage(E, T, M, H, act, dtype, fp8):
    run_glu(E, T, M, H, act, dtype, fp8)


@pytest.mark.parametrize('needs', [(True, False, False, False), (False, True, True, True)])
@pytest.mark.parametrize('fp8', [False, True])
def test_glu_ffn_partial_gradients(needs, fp8):
    run_glu(2, 150, 128, 256, 'silu', torch.bfloat16, fp8, needs)


@pytest.mark.parametrize('dy_kind', ['strided', 'expanded'])
def test_glu_ffn_dy_layouts(dy_kind):
    run_glu(2, 150, 128, 256, 'silu', torch.bfloat16, False, dy_kind=dy_kind)


@pytest.mark.parametrize('fp8', [False, True])
def test_glu_ffn_forward_only_nan_past_the_counts(fp8):
    run_glu(3, 200, 256, 384, 'silu', torch.bfloat16, fp8, (False,) * 4, rc=[200, 1, 0])


# ----------------------------------------------------------------------------------------------------------------
# GroupedLinear
# ----------------------------------------------------------------------------------------------------------------
def run_linear(E, T, K, N, layout, bias, fp8=False, rc=None, needs=(True,) * 3, dtype=torch.bfloat16, dy_kind='dense',
               seed=20):
    G = G_()
    x = _rand((E, T, K), seed + 1, 1.0, dtype)
    w = _rand((E, N, K) if layout == 'nk' else (E, K, N), seed + 2, K ** -0.5, dtype)
    b = _rand((E, N), seed + 3, 0.1, dtype) if bias else None
    rc = _counts(rc)
    grad = any(needs)
    x = _fill_past(x, rc, None if grad else math.nan)
    ins = _leaves((x, w, b), needs)
    what = 'linear %s %s E=%d T=%d K=%d N=%d bias=%s fp8=%s rc=%s needs=%s' % (
        layout, dtype, E, T, K, N, bias, fp8, None if rc is None else rc.tolist(), needs)
    with R.Recorder() as rec:
        if grad:
            y = G.GroupedLinear.apply(*ins, layout, rc, fp8)
            dy = _fill_past(_dy(y, seed + 4, dy_kind), rc, None) if dy_kind != 'expanded' else _dy(y, 0, dy_kind)
            grads = y.grad_fn.apply(dy)[:3]
        else:
            with torch.no_grad():
                y = G.GroupedLinear.apply(*ins, layout, rc, fp8)
            dy = grads = None
    R.check_grouped_linear(rec.take(), *_det(ins), y.detach(), layout=layout, fp8=fp8, row_counts=rc, dy=dy, grads=grads,
                           needs=needs, what=what)


@pytest.mark.parametrize('layout', ['nk', 'kn'])
@pytest.mark.parametrize('bias', [True, False])
@pytest.mark.parametrize('fp8', [False, True])
def test_grouped_linear_stage_by_stage(layout, bias, fp8):
    run_linear(2, 200, 256 if fp8 else 264, 208 if fp8 else 200, layout, bias, fp8, dtype=torch.float16 if bias else torch.bfloat16)


@pytest.mark.parametrize('layout', ['nk', 'kn'])
@pytest.mark.parametrize('fp8', [False, True])
def test_grouped_linear_rows_past_the_counts(layout, fp8):
    """Backward: finite garbage in x and dy past the counts must not reach dw and db."""
    run_linear(3, 200, 256, 144, layout, True, fp8, rc=[200, 1, 0])


@pytest.mark.parametrize('layout', ['nk', 'kn'])
def test_grouped_linear_forward_only_nan_past_the_counts(layout):
    run_linear(3, 200, 256, 144, layout, True, False, rc=[130, 1, 0], needs=(False,) * 3)


@pytest.mark.parametrize('needs', [(True, False, False), (False, True, True)])
@pytest.mark.parametrize('dy_kind', ['strided', 'expanded'])
def test_grouped_linear_partial_gradients_and_dy_layouts(needs, dy_kind):
    run_linear(1, 130, 136, 72, 'kn', True, needs=needs, dy_kind=dy_kind)


# ----------------------------------------------------------------------------------------------------------------
# the expert modules: which function each configuration takes, and its output
# ----------------------------------------------------------------------------------------------------------------
class _Spy:
    ENTRIES = ('fused_act_ffn', 'fused_relu_ffn_fp8', 'fused_glu_ffn', 'grouped_linear', 'skinny_ffn', 'skinny_ffn_fp8',
               'skinny_linear', 'skinny_glu_ffn', 'skinny_glu_ffn_fp8')

    def __init__(self, monkeypatch):
        G = G_()
        self.names = []
        for n in self.ENTRIES:
            monkeypatch.setattr(G, n, self._wrap(n, getattr(G, n)))

    def _wrap(self, name, real):
        def f(*a, **kw):
            self.names.append(name)
            return real(*a, **kw)
        return f


FFN_MODULE_CASES = [
    # act, dtype, fp8, M, H, row counts, grad -> expected entry points
    ('relu', torch.bfloat16, False, 256, 384, None, True, ['fused_act_ffn']),
    ('gelu', torch.float16, False, 256, 384, [100, 7], True, ['fused_act_ffn']),
    ('relu', torch.bfloat16, True, 256, 384, None, True, ['fused_relu_ffn_fp8']),
    ('relu', torch.bfloat16, True, 264, 384, None, True, ['fused_act_ffn']),                # M % 16 != 0: 16 bit
    ('silu', torch.bfloat16, True, 256, 384, None, True, ['fused_act_ffn']),                # fp8 is ReLU only
    ('tanh', torch.bfloat16, False, 256, 384, [100, 7], True, ['grouped_linear', 'grouped_linear']),
    ('tanh', torch.float16, False, 256, 384, None, False, ['grouped_linear', 'grouped_linear']),
]


@pytest.mark.parametrize('act,dtype,fp8,M,H,rc,grad,expect', FFN_MODULE_CASES)
def test_ffn_module_takes_the_expected_function(monkeypatch, act, dtype, fp8, M, H, rc, grad, expect):
    from tutel_b200.models.experts.ffn import FusedExpertsNetwork
    torch.manual_seed(0)
    fn = {'relu': F.relu, 'gelu': F.gelu, 'silu': F.silu, 'tanh': torch.tanh}[act]
    ex = FusedExpertsNetwork(model_dim=M, hidden_size_per_expert=H, num_experts_per_device=2, sharded_count=1,
                             activation_fn=lambda t: fn(t), fp8=fp8).cuda().to(dtype)
    T = 100
    rc = _counts(rc)
    x = _fill_past(_rand((2, T, M), 5, 1.0, dtype), rc, None)
    spy = _Spy(monkeypatch)
    params = (ex.batched_fc1_w, ex.batched_fc1_bias, ex.batched_fc2_w, ex.batched_fc2_bias)
    with R.Recorder() as rec, torch.set_grad_enabled(grad):
        y = ex.compute(x, *params, row_counts=rc)
    assert spy.names == expect, (spy.names, expect)
    calls = rec.take()
    w1, b1, w2, b2 = _det(params)
    what = 'ffn module %s %s fp8=%s' % (act, dtype, fp8)
    if expect[0] in ('fused_act_ffn', 'fused_relu_ffn_fp8'):
        R.check_fused_ffn(calls, x, w1, b1, w2, b2, y.detach(), act=act, row_counts=rc, fp8=expect[0] != 'fused_act_ffn',
                          what=what)
        return
    # GroupedLinear, the activation in torch, GroupedLinear
    with torch.no_grad():
        c1 = R.Calls(calls.calls[:1])
        h = calls.calls[0].out
        R.check_grouped_linear(c1, x, w1, b1, h, 'nk', row_counts=rc, what=what + ' fc1')
        c2 = R.Calls(calls.calls[1:])
        R.check_grouped_linear(c2, fn(h), w2, b2, y.detach(), 'kn', row_counts=rc, what=what + ' fc2')


LLAMA_MODULE_CASES = [
    # act, dtype, fp8, M, H, grad -> expected entry points
    ('silu', torch.bfloat16, False, 256, 384, True, ['fused_glu_ffn']),
    ('gelu', torch.float16, False, 136, 200, True, ['fused_glu_ffn']),
    ('silu', torch.bfloat16, True, 256, 384, True, ['fused_glu_ffn']),
    ('silu', torch.bfloat16, True, 264, 384, True, ['fused_glu_ffn']),                      # M % 16 != 0: 16 bit
    ('tanh', torch.bfloat16, False, 256, 384, True, ['grouped_linear'] * 3),
    ('tanh', torch.bfloat16, True, 256, 384, False, ['grouped_linear'] * 3),
]


@pytest.mark.parametrize('act,dtype,fp8,M,H,grad,expect', LLAMA_MODULE_CASES)
def test_llama_module_takes_the_expected_function(monkeypatch, act, dtype, fp8, M, H, grad, expect):
    from tutel_b200.models.experts.llama_ffn import LlamaFFNNetwork
    from tutel_b200.parallel import communicate as C
    torch.manual_seed(0)
    fn = {'silu': F.silu, 'gelu': F.gelu, 'tanh': torch.tanh}[act]
    ex = LlamaFFNNetwork(M, H, 2, 1, activation_fn=(lambda t: fn(t)) if act != 'silu' else F.silu, fp8=fp8).cuda().to(dtype)
    with torch.no_grad():
        for p in ex.parameters():
            p.normal_(0, M ** -0.5)
    x = _rand((2, 100, M), 6, 1.0, dtype)

    class Ctx:
        group = None
    spy = _Spy(monkeypatch)
    with R.Recorder() as rec, torch.set_grad_enabled(grad):
        y = ex(x, Ctx())
    assert spy.names == expect, (spy.names, expect)
    calls = rec.take()
    w1, w2, w3 = (C.zero_gather(getattr(ex, n).detach(), full_shape=ex.full_shapes[n], group=None)
                  for n in ('W_fc1', 'W_fc2', 'W_fc3'))
    what = 'llama module %s %s fp8=%s M=%d' % (act, dtype, fp8, M)
    if expect == ['fused_glu_ffn']:
        R.check_glu_ffn(calls, x, w1, w2, w3, y.detach(), act=act, fp8=fp8 and M % 16 == 0, what=what)
        return
    per = 3 if fp8 else 1
    cs = calls.calls
    with torch.no_grad():
        y1, y2 = cs[per - 1].out, cs[2 * per - 1].out
        R.check_grouped_linear(R.Calls(cs[:per]), x, w1, None, y1, 'kn', fp8=fp8, what=what + ' fc1')
        R.check_grouped_linear(R.Calls(cs[per:2 * per]), x, w2, None, y2, 'kn', fp8=fp8, what=what + ' fc2')
        R.check_grouped_linear(R.Calls(cs[2 * per:]), fn(y1) * y2, w3, None, y.detach(), 'kn', fp8=fp8, what=what + ' fc3')


# ----------------------------------------------------------------------------------------------------------------
# 16-bit skinny kernels
# ----------------------------------------------------------------------------------------------------------------
SK_ROWS = 12
SK_COUNTS = [0, 1, 2, 3, 5, 9, SK_ROWS, SK_ROWS + 7]     # idle, 1- / 2-row passes, a padded 4-row pass, several, cap, above
SK_ACTS = {'relu': 1, 'gelu': 2, 'silu': 3}


@pytest.fixture(scope='module')
def C():
    from tutel_b200.ops import backend
    return backend.require_ext()


@pytest.mark.parametrize('K,H,N', [(256, 200, 136), (264, 136, 40), (6336, 72, 64)])    # partial slices; K at the limit
@pytest.mark.parametrize('act,dtype', [('relu', torch.float32), ('silu', torch.bfloat16), ('gelu', torch.float16),
                                       ('relu', torch.bfloat16)])
@pytest.mark.parametrize('bias', ['both', 'none', 'b1', 'b2'])
def test_skinny_ffn_matches_fp64_reference(C, K, H, N, act, dtype, bias):
    G = G_()
    counts = _counts(SK_COUNTS)
    E = counts.numel()
    x = _rand((E, SK_ROWS, K), 1, 1.0, dtype)
    w1, w2 = _rand((E, H, K), 2, K ** -0.5, dtype), _rand((E, H, N), 3, H ** -0.5, dtype)
    b1 = _rand((E, H), 4, 0.5, dtype) if bias in ('both', 'b1') else None
    b2 = _rand((E, N), 5, 0.5, dtype) if bias in ('both', 'b2') else None
    if K == 6336:
        with torch.no_grad():
            assert G.can_use_skinny_ffn(x, w1, w2, act) and not G.can_use_skinny_ffn(
                torch.zeros(1, 1, K + 8, dtype=dtype, device='cuda'), torch.zeros(1, H, K + 8, dtype=dtype, device='cuda'),
                w2[:1], act)
    y = C.skinny_ffn(x, w1, b1, w2, b2, counts, SK_ACTS[act])
    assert y.dtype == torch.float32 and y.shape == (E, SK_ROWS, N)
    ref, bound = R.skinny_ffn_reference(x, w1, b1, w2, b2, act)
    R.check_skinny('skinny_ffn', y, ref, bound, counts)


@pytest.mark.parametrize('kn', [False, True])
@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize('bias,relu', [(True, True), (False, False), (True, False)])
def test_skinny_gemm_matches_fp64_reference(C, kn, dtype, bias, relu):
    """K over two 1024-element chunks and a partial one, more than 8 rows, partial column blocks (64 nk / 256 kn)."""
    counts = _counts(SK_COUNTS)
    E, K, N = counts.numel(), 2300, 328
    x = _rand((E, SK_ROWS, K), 7, 1.0, dtype)
    w = _rand((E, K, N) if kn else (E, N, K), 8, K ** -0.5, dtype)
    b = _rand((E, N), 9, 0.5, dtype) if bias else None
    y = C.skinny_gemm(x, w, b, counts, kn, relu)
    assert y.dtype == dtype and y.shape == (E, SK_ROWS, N)
    ref, bound = R.skinny_gemm_reference(x, w, b, kn, relu)
    R.check_skinny('skinny_gemm', y, ref, bound, counts)
