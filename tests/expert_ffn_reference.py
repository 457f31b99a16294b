"""Stage-by-stage fp64 checks of the expert autograd functions in tutel_b200/ops/gemm.py, and fp64 references with
per-element bounds for the 16-bit skinny decode kernels (csrc/skinny_gemm.cu).  Plain torch: runs on the CPU or the GPU.

``Recorder`` wraps the module-level ops the autograd functions call (``raw_gemm``, ``glu_gemm``, ``glu_gemm_bwd``,
``quantize_rows``, ``fp8_operand`` - which ``fp8_weight`` goes through - and ``column_sums``) and records every
outermost call with its arguments and outputs, so the intermediates that are never returned (act / pre, dh, g / u / h,
dg / du, the first dx partial, every e4m3 copy) can be checked.

Each ``check_*`` function states its function's stages as math and checks them in launch order with
``gemm_reference.ref_gemm`` / ``check``.  A stage's reference is built only from the test's own tensors (x, weights,
biases, dy, row counts) and from intermediates that an earlier stage has already checked: nothing the code under test
passed between its launches is trusted.  A different launch order fails with the name of the op that was expected.
Every e4m3 operand must be bit-identical to ``quantize_rows_reference`` of the right tensor in the right orientation.
"""
import math
from dataclasses import dataclass
from typing import Any, Dict, List, Optional

import pytest
import torch

import dispatch_reference as D
import gemm_reference as GR

U = 2.0 ** -24
OPS = ('raw_gemm', 'glu_gemm', 'glu_gemm_bwd', 'quantize_rows', 'fp8_operand', 'column_sums')
ACT = {'relu': GR.ACT_RELU, 'gelu': GR.ACT_GELU, 'silu': GR.ACT_SILU}
FWD_EPI = {'relu': GR.EPI_BIAS_RELU, 'gelu': GR.EPI_BIAS_GELU, 'silu': GR.EPI_BIAS_SILU}
# largest normalised error seen per stage: (|err| - output rounding - evaluation term) / accumulation term
OBSERVED: Dict[str, float] = {}


# ----------------------------------------------------------------------------------------------------------------
# recorder
# ----------------------------------------------------------------------------------------------------------------
@dataclass
class Call:
    name: str
    args: tuple
    kw: dict
    out: Any


class Recorder:
    """``with Recorder() as rec:`` records the outermost calls of the ops in ``OPS`` (calls an op makes to another op,
    such as ``fp8_operand``'s own ``quantize_rows``, are part of the outer call)."""

    def __init__(self):
        from tutel_b200.ops import gemm
        self.module = gemm
        self.calls: List[Call] = []
        self._depth = 0
        self._mp = None

    def __enter__(self):
        self._mp = pytest.MonkeyPatch()
        for name in OPS:
            self._mp.setattr(self.module, name, self._wrap(name, getattr(self.module, name)))
        return self

    def __exit__(self, *exc):
        self._mp.undo()
        return False

    def _wrap(self, name, real):
        def op(*args, **kw):
            self._depth += 1
            try:
                out = real(*args, **kw)
            finally:
                self._depth -= 1
            if self._depth == 0:
                self.calls.append(Call(name, args, kw, out))
            return out
        return op

    def take(self) -> 'Calls':
        """The calls recorded so far, as a queue; the recorder starts a new list."""
        calls, self.calls = self.calls, []
        return Calls(calls)


class Calls:
    def __init__(self, calls: List[Call]):
        self.calls = list(calls)
        self.i = 0

    def next(self, name: str, what: str) -> Call:
        assert self.i < len(self.calls), '%s: expected a %s call, the function made no more calls (%s)' % (
            what, name, self.names())
        c = self.calls[self.i]
        assert c.name == name, '%s: expected call %d to be %s, got %s (%s)' % (what, self.i, name, c.name, self.names())
        self.i += 1
        return c

    def done(self, what: str):
        assert self.i == len(self.calls), '%s: unexpected extra calls %s' % (what, [c.name for c in self.calls[self.i:]])

    def names(self):
        return [c.name for c in self.calls]


# ----------------------------------------------------------------------------------------------------------------
# references
# ----------------------------------------------------------------------------------------------------------------
def zero_tail(t: torch.Tensor, counts: Optional[torch.Tensor]) -> torch.Tensor:
    if counts is None:
        return t
    rows = torch.arange(t.size(1), device=t.device).view(1, -1, 1)
    return torch.where(rows < counts.to(t.device).long().view(-1, 1, 1), t, torch.zeros((), dtype=t.dtype, device=t.device))


def quantize_rows_reference(t: torch.Tensor):
    """The row quantisation of csrc/moe_kernels.h, in fp32 as the kernels compute it: s = max(max|row| * fp32(1/448),
    FLT_MIN) (1 for an all-zero row), q = e4m3_rn(x * fp32(1 / s)).  NaN elements do not count towards the maximum."""
    f = t.float()
    a = torch.where(torch.isnan(f), torch.zeros_like(f), f.abs()).amax(-1)
    s = torch.where(a > 0, (a * torch.tensor(1.0 / 448.0, dtype=torch.float32, device=f.device)).clamp_min(2.0 ** -126),
                    torch.ones_like(a))
    inv = torch.ones((), dtype=torch.float32, device=f.device) / s
    return (f * inv.unsqueeze(-1)).to(torch.float8_e4m3fn), s


def _rows_mask(t, counts):
    if counts is None:
        return torch.ones(t.shape[:-1], dtype=torch.bool, device=t.device)
    rows = torch.arange(t.size(1), device=t.device).view(1, -1)
    return rows < counts.to(t.device).long().view(-1, 1)


def check_quantized(what: str, got, src: torch.Tensor, counts=None):
    """``got = (q, s)`` must be the bytes and scales of quantize_rows_reference(src), on the rows below the counts."""
    q, s = got
    wq, ws = quantize_rows_reference(src)
    assert q.dtype == torch.float8_e4m3fn and q.shape == wq.shape and s.shape == ws.shape, (what, q.dtype, q.shape, s.shape)
    m = _rows_mask(src, counts)
    bad_s = (s.float() != ws) & m
    assert not bool(bad_s.any()), '%s: %d row scales differ from max|row| / 448, first at %s' % (
        what, int(bad_s.sum()), tuple(int(i) for i in bad_s.nonzero()[0]))
    bad_q = (q.view(torch.uint8) != wq.view(torch.uint8)) & m.unsqueeze(-1)
    assert not bool(bad_q.any()), '%s: %d e4m3 bytes differ from the row quantisation, first at %s' % (
        what, int(bad_q.sum()), tuple(int(i) for i in bad_q.nonzero()[0]))


def _observe(name: str, r: GR.Ref, key: str, out: torch.Tensor):
    v = GR.normalised_error(r, key, out)
    if not math.isinf(v):
        name = '%s %s' % (name, 'e4m3' if r.in_dtype == torch.float8_e4m3fn else '16-bit')
        OBSERVED[name] = max(OBSERVED.get(name, -math.inf), v)


def stage(name: str, what: str, r: GR.Ref, d, d2=None, d3=None, colsum=None):
    GR.check(r, d, d2, d3, colsum=colsum, what='%s: %s' % (name, what))
    for key, out, sub in (('d', d, ''), ('d2', d2, '.2'), ('d3', d3, '.3')):
        if out is not None and key in r.outs:
            _observe(name + sub, r, key, out)


def _no_grad(what, name, g):
    assert g is None, '%s: %s was computed although it was not asked for' % (what, name)


def _zero_rows_past(what, name, t, counts):
    if counts is not None:
        past = ~_rows_mask(t, counts)
        assert bool((t[past] == 0).all()), '%s: %s rows past the counts are not zero' % (what, name)


def _wgrad(name, what, a, b, got, a_mn=True, b_mn=True):
    assert got.dtype == a.dtype, '%s: %s dtype %s' % (what, name, got.dtype)
    stage(name, what, GR.ref_gemm(a, b, a_mn=a_mn, b_mn=b_mn, out_dtype=a.dtype), got)


def _colsum(name, what, got, src, dtype):
    assert got.dtype == dtype, '%s: %s dtype %s' % (what, name, got.dtype)
    D.check_colsum('%s %s' % (name, what), got, src)


def _qcopy(calls, what, label, src, counts=None):
    c = calls.next('quantize_rows', '%s (%s)' % (what, label))
    check_quantized('%s: e4m3 %s' % (what, label), c.out, src, counts)
    return c.out


def _wcopy(calls, what, label, w):
    c = calls.next('fp8_operand', '%s (%s)' % (what, label))
    check_quantized('%s: e4m3 %s' % (what, label), c.out, w.contiguous())
    return c.out


# ----------------------------------------------------------------------------------------------------------------
# FusedReluFFN (relu / gelu / silu) and FusedReluFFNFp8
# ----------------------------------------------------------------------------------------------------------------
def check_fused_ffn(calls: Calls, x, w1, b1, w2, b2, y, act='relu', row_counts=None, dy=None, grads=None,
                    needs=(True,) * 5, fp8=False, what=''):
    """y = act(x W1^T + b1) W2 + b2 with w1 [G, H, M], w2 [G, H, Mout]; ``grads`` is what the backward returned for
    (x, w1, b1, w2, b2) given ``dy`` and ``needs`` (the inputs that asked for a gradient)."""
    dt, rc = x.dtype, row_counts
    with torch.no_grad():
        if fp8:
            xq, sx = _qcopy(calls, what, 'x', x, rc)
            q1, s1 = _wcopy(calls, what, 'W1', w1)
            c = calls.next('raw_gemm', what + ' (act)')
            at = c.out
            r = GR.ref_gemm(xq, q1, epilogue=GR.EPI_BIAS_RELU, bias=b1, scale_a=sx, scale_b=s1, row_counts=rc, out_dtype=dt)
            stage('act', what, r, at)
            aq, sa = _qcopy(calls, what, 'act', at, rc)
            q2, s2 = _wcopy(calls, what, 'W2^T', w2.transpose(1, 2))
            c = calls.next('raw_gemm', what + ' (y)')
            r = GR.ref_gemm(aq, q2, epilogue=GR.EPI_BIAS, bias=b2, scale_a=sa, scale_b=s2, row_counts=rc, out_dtype=dt)
            pre = None
        else:
            c = calls.next('raw_gemm', what + ' (act)')
            at, pre = c.out, c.kw.get('d2')
            r = GR.ref_gemm(x, w1, epilogue=FWD_EPI[act], bias=b1, row_counts=rc, out_dtype=dt, want_pre=pre is not None)
            stage('act', what, r, at, d2=pre)
            c = calls.next('raw_gemm', what + ' (y)')
            r = GR.ref_gemm(at, w2, b_mn=True, epilogue=GR.EPI_BIAS, bias=b2, row_counts=rc, out_dtype=dt)
        assert y.dtype == dt
        stage('y', what, r, y)
        if dy is None:
            calls.done(what)
            return
        # ---- backward: dy past the counts is ignored ----
        dyz = zero_tail(dy, rc)
        dx, dw1, db1, dw2, db2 = grads
        want_db1 = b1 is not None and needs[2]
        if fp8:
            dyq, sdy = _qcopy(calls, what, 'dy', dyz)
            q2, s2 = _wcopy(calls, what, 'W2', w2)
            c = calls.next('raw_gemm', what + ' (dh)')
            r = GR.ref_gemm(dyq, q2, epilogue=GR.EPI_RELU_BWD, aux=at, scale_a=sdy, scale_b=s2, row_counts=rc, out_dtype=dt)
        else:
            c = calls.next('raw_gemm', what + ' (dh)')
            if act == 'relu':
                r = GR.ref_gemm(dyz, w2, epilogue=GR.EPI_RELU_BWD, aux=at, row_counts=rc, out_dtype=dt)
            else:
                r = GR.ref_gemm(dyz, w2, epilogue=GR.EPI_ACT_BWD, aux=pre, act=ACT[act], row_counts=rc, out_dtype=dt)
        dh, colsum = c.out, c.kw.get('colsum')
        if want_db1:
            assert colsum is not None and colsum.dtype == torch.float32, what + ': db1 is not the fused fp32 column sum'
        stage('dh', what, r, dh, colsum=colsum if want_db1 else None)
        dhz, actz = zero_tail(dh, rc), zero_tail(at, rc)
        if needs[3]:
            _wgrad('dw2', what, actz, dyz, calls.next('raw_gemm', what + ' (dw2)').out)
            _wgrad('dw2', what, actz, dyz, dw2)
        else:
            _no_grad(what, 'dw2', dw2)
        if b2 is not None and needs[4]:
            calls.next('column_sums', what + ' (db2)')
            _colsum('db2', what, db2, dyz, dt)
        else:
            _no_grad(what, 'db2', db2)
        if needs[0]:
            if fp8:
                hq, sh = _qcopy(calls, what, 'dh', dhz)
                q1t, s1t = _wcopy(calls, what, 'W1^T', w1.transpose(1, 2))
                r = GR.ref_gemm(hq, q1t, scale_a=sh, scale_b=s1t, row_counts=rc, out_dtype=dt)
            else:
                r = GR.ref_gemm(dhz, w1, b_mn=True, row_counts=rc, out_dtype=dt)
            calls.next('raw_gemm', what + ' (dx)')
            assert dx.dtype == dt
            stage('dx', what, r, dx)
            _zero_rows_past(what, 'dx', dx, rc)
        else:
            _no_grad(what, 'dx', dx)
        if needs[1]:
            calls.next('raw_gemm', what + ' (dw1)')
            _wgrad('dw1', what, dhz, x, dw1)
        else:
            _no_grad(what, 'dw1', dw1)
        if want_db1:
            assert db1.dtype == dh.dtype and torch.equal(db1, colsum.to(dh.dtype)), what + ': db1 is not the fused colsum'
        else:
            _no_grad(what, 'db1', db1)
        calls.done(what)


# ----------------------------------------------------------------------------------------------------------------
# FusedGLUFFN (16 bit and fp8)
# ----------------------------------------------------------------------------------------------------------------
def check_glu_ffn(calls: Calls, x, w1, w2, w3, y, act='silu', fp8=False, row_counts=None, dy=None, grads=None,
                  needs=(True,) * 4, what=''):
    """(h, g, u) = GLU(x W1, x W2); y = h W3 with w1, w2 [G, M, H], w3 [G, H, Mout]."""
    dt, rc, a = x.dtype, row_counts, ACT[act]
    with torch.no_grad():
        if fp8:
            xq, sx = _qcopy(calls, what, 'x', x, rc)
            q1, s1 = _wcopy(calls, what, 'W1^T', w1.transpose(1, 2))
            q2, s2 = _wcopy(calls, what, 'W2^T', w2.transpose(1, 2))
            q3, s3 = _wcopy(calls, what, 'W3^T', w3.transpose(1, 2))
            c = calls.next('glu_gemm', what + ' (h, g, u)')
            r = GR.ref_gemm(xq, q1, b2=q2, epilogue=GR.EPI_GLU, act=a, scale_a=sx, scale_b=s1, scale_b2=s2, row_counts=rc,
                            out_dtype=dt, want_pre=True)
        else:
            c = calls.next('glu_gemm', what + ' (h, g, u)')
            r = GR.ref_gemm(x, w1, b_mn=True, b2=w2, epilogue=GR.EPI_GLU, act=a, row_counts=rc, out_dtype=dt, want_pre=True)
        h, g, u = c.out
        stage('h', what, r, h, d2=g, d3=u)
        if fp8:
            hq, sh = _qcopy(calls, what, 'h', h, rc)
            c = calls.next('raw_gemm', what + ' (y)')
            r = GR.ref_gemm(hq, q3, scale_a=sh, scale_b=s3, row_counts=rc, out_dtype=dt)
        else:
            c = calls.next('raw_gemm', what + ' (y)')
            r = GR.ref_gemm(h, w3, b_mn=True, row_counts=rc, out_dtype=dt)
        assert y.dtype == dt
        stage('y', what, r, y)
        if dy is None:
            calls.done(what)
            return
        dx, dw1, dw2, dw3 = grads
        if fp8:
            dyq, sdy = _qcopy(calls, what, 'dy', dy)
            q3n, s3n = _wcopy(calls, what, 'W3', w3)
            c = calls.next('glu_gemm_bwd', what + ' (dg, du)')
            r = GR.ref_gemm(dyq, q3n, epilogue=GR.EPI_GLU_BWD, aux=g, aux2=u, act=a, scale_a=sdy, scale_b=s3n, out_dtype=dt)
        else:
            c = calls.next('glu_gemm_bwd', what + ' (dg, du)')
            r = GR.ref_gemm(dy, w3, epilogue=GR.EPI_GLU_BWD, aux=g, aux2=u, act=a, out_dtype=dt)
        dg, du = c.out
        stage('dg', what, r, dg, d2=du)
        for i, (name, a_, b_, got) in enumerate((('dw3', h, dy, dw3), ('dw1', x, dg, dw1), ('dw2', x, du, dw2))):
            if needs[(3, 1, 2)[i]]:
                calls.next('raw_gemm', '%s (%s)' % (what, name))
                _wgrad(name, what, a_, b_, got)
            else:
                _no_grad(what, name, got)
        if needs[0]:
            if fp8:
                gq, sg = _qcopy(calls, what, 'dg', dg)
                uq, su = _qcopy(calls, what, 'du', du)
                q1n, s1n = _wcopy(calls, what, 'W1', w1)
                q2n, s2n = _wcopy(calls, what, 'W2', w2)
                c = calls.next('raw_gemm', what + ' (dx, dg term)')
                r = GR.ref_gemm(gq, q1n, scale_a=sg, scale_b=s1n, out_dtype=dt)
                stage('dx.1', what, r, c.out)
                calls.next('raw_gemm', what + ' (dx)')
                r = GR.ref_gemm(uq, q2n, epilogue=GR.EPI_ADD, aux=c.out, scale_a=su, scale_b=s2n, out_dtype=dt)
            else:
                c = calls.next('raw_gemm', what + ' (dx, dg term)')
                stage('dx.1', what, GR.ref_gemm(dg, w1, out_dtype=dt), c.out)
                calls.next('raw_gemm', what + ' (dx)')
                r = GR.ref_gemm(du, w2, epilogue=GR.EPI_ADD, aux=c.out, out_dtype=dt)
            assert dx.dtype == dt
            stage('dx', what, r, dx)
        else:
            _no_grad(what, 'dx', dx)
        calls.done(what)


# ----------------------------------------------------------------------------------------------------------------
# GroupedLinear
# ----------------------------------------------------------------------------------------------------------------
def check_grouped_linear(calls: Calls, x, w, b, y, layout='nk', fp8=False, row_counts=None, dy=None, grads=None,
                         needs=(True,) * 3, what=''):
    """y = x W^T + b (``'nk'``, w [G, N, K]) or x W + b (``'kn'``, w [G, K, N])."""
    dt, rc, kn = x.dtype, row_counts, layout == 'kn'
    with torch.no_grad():
        if fp8:
            xq, sx = _qcopy(calls, what, 'x', x, rc)
            wq, sw = _wcopy(calls, what, 'W^T' if kn else 'W', w.transpose(1, 2) if kn else w)
            calls.next('raw_gemm', what + ' (y)')
            r = GR.ref_gemm(xq, wq, epilogue=GR.EPI_BIAS, bias=b, scale_a=sx, scale_b=sw, row_counts=rc, out_dtype=dt)
        else:
            calls.next('raw_gemm', what + ' (y)')
            r = GR.ref_gemm(x, w, b_mn=kn, epilogue=GR.EPI_BIAS, bias=b, row_counts=rc, out_dtype=dt)
        assert y.dtype == dt
        stage('y', what, r, y)
        if dy is None:
            calls.done(what)
            return
        dyz = zero_tail(dy, rc)
        dx, dw, db = grads
        if needs[0]:
            calls.next('raw_gemm', what + ' (dx)')
            assert dx.dtype == dt
            stage('dx', what, GR.ref_gemm(dyz, w, b_mn=not kn, row_counts=rc, out_dtype=dt), dx)
            _zero_rows_past(what, 'dx', dx, rc)
        else:
            _no_grad(what, 'dx', dx)
        if needs[1]:
            calls.next('raw_gemm', what + ' (dw)')
            if kn:
                _wgrad('dw', what, zero_tail(x, rc), dyz, dw)
            else:
                _wgrad('dw', what, dyz, zero_tail(x, rc), dw)
        else:
            _no_grad(what, 'dw', dw)
        if b is not None and needs[2]:
            calls.next('column_sums', what + ' (db)')
            _colsum('db', what, db, dyz, dt)
        else:
            _no_grad(what, 'db', db)
        calls.done(what)


# ----------------------------------------------------------------------------------------------------------------
# 16-bit skinny kernels (csrc/skinny_gemm.cu): skinny_ffn_kernel, skinny_kernel
# ----------------------------------------------------------------------------------------------------------------
ACT_LIPSCHITZ = 1.13      # largest |act'|: 1 (ReLU), 1.0998 (SiLU), 1.1289 (erf-GELU)
SLACK = 1.01              # first-order n u sum|terms| bounds, widened for their second-order terms (n u < 2^-10 here)
HS = 64                   # hidden units per block of skinny_ffn_kernel (kHS)
_FN = {'relu': torch.relu, 'gelu': lambda v: 0.5 * v * (1 + torch.erf(v / math.sqrt(2))), 'silu': lambda v: v * torch.sigmoid(v)}


def _vec(dtype):
    return 4 if dtype == torch.float32 else 8        # elements per 16-byte load (WVec<T>::N)


def skinny_ffn_reference(x, w1, b1, w2, b2, act, loose=False):
    """y = act(x W1^T + b1) W2 + b2 (w1 [G, H, K], w2 [G, H, N]) in fp64 for skinny_ffn_kernel's fp32 output, and a
    bound from its reduction order:

    * layer 1: one warp per hidden unit, each lane an fmaf chain over ceil(K / 32V) * V elements, five shuffle levels
      and the bias add: ``e1 = (ceil(K / 32V) V + 6) u (sum|x w1| + |b1|)``; the activation passes e1 on with slope
      <= 1.13 and adds its own evaluation error (erff / __expf: ``2^-18 (|h| + |pre|)``);
    * layer 2: per 64-unit slice an fmaf chain of <= 64 terms, the bias (slice 0), then one fp32 atomic per slice:
      ``(64 + 1 + ceil(H / 64)) u (sum|h w2| + |b2|)``, plus ``sum_j |w2_j| e_h_j``.

    ``loose=True`` gives the (K + H) form of tests/skinny_fp8_reference.py instead, for comparison."""
    xd, w1d, w2d = x.double(), w1.double(), w2.double()
    G, K, H = x.size(0), x.size(2), w1.size(1)
    zero = torch.zeros((), dtype=torch.float64, device=x.device)
    b1d = b1.double().view(G, 1, H) if b1 is not None else zero
    b2d = b2.double().view(G, 1, -1) if b2 is not None else zero
    pre = xd @ w1d.transpose(1, 2) + b1d
    h = _FN[act](pre)
    y = h @ w2d + b2d
    s1 = xd.abs() @ w1d.abs().transpose(1, 2) + b1d.abs()
    if loose:
        terms = (ACT_LIPSCHITZ * s1 + h.abs()) @ w2d.abs() + b2d.abs()
        return y, U * y.abs() + (2.0 * (K + H) + 2) * U * terms
    V = _vec(x.dtype)
    n1 = math.ceil(K / (32 * V)) * V + 6
    eh = ACT_LIPSCHITZ * n1 * U * s1 + (GR.FN_REL * (h.abs() + pre.abs()) if act != 'relu' else 0.0)
    n2 = min(HS, H) + 1 + math.ceil(H / HS)
    bound = SLACK * (n2 * U * (h.abs() @ w2d.abs() + b2d.abs()) + eh @ w2d.abs())
    return y, bound


def skinny_gemm_reference(x, w, bias, kn, relu):
    """y = relu?(x W + b) (w [G, K, N] when ``kn``, else [G, N, K]) in fp64 for skinny_kernel, and a bound: the fmaf
    chain of a thread (``kn``: all K terms) or of a lane (``nk``: ceil(K / 32) + one per 1024-element chunk, then five
    shuffle levels), the bias add, and half an ulp of the output dtype at the largest value the result can take."""
    xd, wd = x.double(), w.double()
    W = wd if kn else wd.transpose(1, 2)
    K = x.size(2)
    b = bias.double().unsqueeze(1) if bias is not None else torch.zeros((), dtype=torch.float64, device=x.device)
    pre = xd @ W + b
    y = pre.clamp_min(0) if relu else pre
    n = (K if kn else math.ceil(K / 32) + math.ceil(K / 1024) + 5) + 1
    acc = SLACK * n * U * (xd.abs() @ W.abs() + b.abs())
    if x.dtype == torch.float32:
        return y, acc + U * (y.abs() + acc)
    return y, acc + GR.half_ulp(y.abs() + acc, x.dtype)


def check_skinny(name: str, y: torch.Tensor, ref: torch.Tensor, bound: torch.Tensor, counts: torch.Tensor) -> float:
    """Rows below each group's count within their bound, every other row exactly zero; returns max |err| / bound."""
    R = y.size(1)
    worst = 0.0
    for g, c in enumerate(counts.clamp(min=0, max=R).tolist()):
        if c > 0:
            err = (y[g, :c].double() - ref[g, :c]).abs()
            err = torch.where(torch.isnan(err), torch.full_like(err, math.inf), err)
            ratio = err / bound[g, :c].clamp_min(1e-300)
            i = tuple(int(v) for v in (ratio == ratio.max()).nonzero()[0])
            assert bool((err <= bound[g, :c]).all()), '%s: group %d, %d elements outside the bound, worst %.3g x at %s' % (
                name, g, int((err > bound[g, :c]).sum()), float(ratio.max()), i)
            worst = max(worst, float(ratio.max()))
        assert torch.count_nonzero(y[g, c:]) == 0, '%s: group %d rows at or past the count %d are not zero' % (name, g, c)
    OBSERVED[name] = max(OBSERVED.get(name, 0.0), worst)
    return worst
