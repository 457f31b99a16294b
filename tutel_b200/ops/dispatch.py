"""Sparse dispatch (encode) / combine (decode) with autograd - ``tutel.moe.fast_encode / fast_decode / fast_dispatcher``.

Reference behaviour: tutel/impls/fast_dispatch.py:16-136,209-221 (k scatter launches into a zero-filled fp32 buffer,
then casts).  Here:

* **encode** is a *slot-centric row gather*: one launch writes every row of the ``[E*C, M]`` buffer exactly once
  (token row, or zeros for padding) in the tensor's own dtype;
* **decode** sums all k choices of a token in one pass with fp32 accumulation;
* the two are each other's backward (encode.bwd = decode of the gradient buffer, decode.bwd = encode of the output
  gradient), gate gradients come from a fused row-dot kernel.

CPU tensors use the C++ loops of csrc/cpu_kernels.cpp (fp32/fp64) or an index_add/index_select torch fallback.
"""
from __future__ import annotations

from typing import Any, List, Optional, Sequence

import torch

from . import backend
from .routing import CriticalData, build_slot_map

_NATIVE_CUDA_DTYPES = (torch.float32, torch.float16, torch.bfloat16)


class DispatchPlan:
    """Routing decisions in kernel-friendly form (stacked ``[k, S]`` int32 ids / locations, inverse slot map)."""

    def __init__(self, E: int, C: int, idx_ks: torch.Tensor, loc_ks: torch.Tensor, slot_src: Optional[torch.Tensor] = None):
        self.E, self.C = int(E), int(C)
        self.idx_ks = idx_ks.contiguous()
        self.loc_ks = loc_ks.contiguous()
        self.k, self.S = int(idx_ks.size(0)), int(idx_ks.size(1))
        self._slot_src = slot_src
        self.valid_rows = None        # int32 [E]: when set, encode leaves rows past the per-expert count untouched
        self.layout = None            # PackedLayout (ops/packed.py): the buffer is the expert-packed [R, M]

    @property
    def slot_src(self) -> torch.Tensor:
        if self._slot_src is None:
            self._slot_src = build_slot_map(self.idx_ks, self.loc_ks, self.E, self.C)
        return self._slot_src

    @staticmethod
    def from_critical(crit) -> 'DispatchPlan':
        if isinstance(crit, CriticalData):
            plan = getattr(crit, '_plan', None)
            if plan is None:
                plan = DispatchPlan(crit[0], crit[4], crit.idx_ks, crit.loc_ks, crit._slot_src)
                if getattr(crit, 'skip_padding', False):
                    plan.valid_rows = crit[5]
                plan.layout = getattr(crit, 'layout', None)
                crit._plan = plan
            return plan
        E, indices_s, locations_s, _, capacity = crit[0], crit[1], crit[2], crit[3], crit[4]
        idx = torch.stack([x.to(torch.int32).view(-1) for x in indices_s])
        loc = torch.stack([x.to(torch.int32).view(-1) for x in locations_s])
        return DispatchPlan(E, capacity, idx, loc)


# ----------------------------------------------------------------------------------------------------------------
# raw (non-differentiable) kernels with CPU / torch fallbacks
# ----------------------------------------------------------------------------------------------------------------
def _native_cuda(t: torch.Tensor) -> bool:
    return t.is_cuda and t.dtype in _NATIVE_CUDA_DTYPES and backend.has_cuda_ext()


def _cpu_native(t: torch.Tensor) -> bool:
    return (not t.is_cuda) and t.dtype in (torch.float32, torch.float64) and backend.has_ext()


def _slots(plan: DispatchPlan):
    """flat slot index [k, S] (int64) and validity mask for the torch fallback paths."""
    valid = (plan.loc_ks < plan.C) & (plan.idx_ks >= 0)
    slot = plan.idx_ks.to(torch.int64) * plan.C + plan.loc_ks.to(torch.int64).clamp(max=max(plan.C - 1, 0))
    return slot, valid


def raw_encode(x: torch.Tensor, gates: Optional[torch.Tensor], plan: DispatchPlan) -> torch.Tensor:
    """x [S, M] -> [E*C, M];  row(slot) = gate * x[token(slot)]  or zeros."""
    if plan.layout is not None:
        from . import packed
        return packed.encode(x, gates, plan.layout)
    x = x.contiguous()
    M = x.size(1)
    if _native_cuda(x):
        out = torch.empty([plan.E * plan.C, M], dtype=x.dtype, device=x.device)
        g = None if gates is None else gates.to(torch.float32).contiguous()
        backend.count_launch()
        backend.require_ext().encode_rows(x, g, plan.slot_src, out, plan.k, plan.E, plan.C, 0, 0, 0, 0, 0, 0, plan.valid_rows)
        return out
    if _cpu_native(x):
        g = None if gates is None else gates.to(x.dtype).contiguous()
        return backend.ext().cpu_encode(x, g, plan.idx_ks, plan.loc_ks, plan.E, plan.C)
    work = x if x.dtype in (torch.float32, torch.float64) else x.float()
    out = torch.zeros([plan.E * plan.C, M], dtype=work.dtype, device=x.device)
    slot, valid = _slots(plan)
    for j in range(plan.k):
        rows = work[valid[j]] if gates is None else work[valid[j]] * gates[j][valid[j]].to(work.dtype).unsqueeze(1)
        out.index_copy_(0, slot[j][valid[j]], rows)
    return out.to(x.dtype)


def shared_weight(shared_logit: Optional[torch.Tensor], dtype: torch.dtype = torch.float32):
    """Per-token weight ``[S, 1]`` of the shared experts' output: sigmoid of the shared-gate logit computed in ``dtype``
    (fp32 as in the kernels, or fp64 for fp64 tensors), or None for weight 1."""
    if shared_logit is None:
        return None
    return torch.sigmoid(shared_logit.to(dtype).view(-1, 1))


def _add_shared(out: torch.Tensor, base: Optional[torch.Tensor], shared_logit: Optional[torch.Tensor]) -> torch.Tensor:
    """out + w_s * base in out's (fp32 or fp64) precision: the shared term of the torch combine paths."""
    if base is None:
        return out
    b = base.to(out.dtype).view_as(out)
    ws = shared_weight(shared_logit, out.dtype)
    return out + (b if ws is None else ws * b)


def _shared_args(base: Optional[torch.Tensor], shared_logit: Optional[torch.Tensor]):
    """The shared terms as the native kernels take them: contiguous base, fp32 logits [S]."""
    b = None if base is None else base.contiguous()
    sl = None if shared_logit is None else shared_logit.to(torch.float32).contiguous().view(-1)
    return b, sl


def raw_decode(buf: torch.Tensor, gates: Optional[torch.Tensor], plan: DispatchPlan, base: Optional[torch.Tensor] = None,
               shared_logit: Optional[torch.Tensor] = None) -> torch.Tensor:
    """buf [E*C, M] -> [S, M];  out[s] = sum_j gate_j[s] * buf[slot_j(s)]  (+ w_s * base[s]).

    ``base [S, M]`` (optional): the shared experts' output, added with weight w_s = 1, or sigmoid(shared_logit[s]) when
    ``shared_logit [S]`` is given; on CUDA in the same launch and with one rounding (csrc/moe_kernels.cu: decode_rows)."""
    if plan.layout is not None:
        from . import packed
        return packed.decode(buf.view(plan.layout.R, -1), gates, plan.idx_ks, plan.loc_ks, plan.layout, base, shared_logit)
    buf = buf.contiguous().view(plan.E * plan.C, -1)
    if _native_cuda(buf):
        g = None if gates is None else gates.to(torch.float32).contiguous()
        backend.count_launch()
        if base is None:
            return backend.require_ext().decode_rows(buf, g, plan.idx_ks, plan.loc_ks, plan.E, plan.C, 0, 0)
        b, sl = _shared_args(base, shared_logit)
        return backend.require_ext().decode_rows(buf, g, plan.idx_ks, plan.loc_ks, plan.E, plan.C, 0, 0, None, b, sl)
    if _cpu_native(buf):
        g = None if gates is None else gates.to(buf.dtype).contiguous()
        return _add_shared(backend.ext().cpu_decode(buf, g, plan.idx_ks, plan.loc_ks, plan.E, plan.C), base, shared_logit)
    work = buf if buf.dtype in (torch.float32, torch.float64) else buf.float()
    out = torch.zeros([plan.S, work.size(1)], dtype=work.dtype, device=buf.device)
    slot, valid = _slots(plan)
    for j in range(plan.k):
        rows = work.index_select(0, slot[j])
        w = valid[j].to(work.dtype) if gates is None else valid[j].to(work.dtype) * gates[j].to(work.dtype)
        out += rows * w.unsqueeze(1)
    return _add_shared(out, base, shared_logit).to(buf.dtype)


def raw_shared_grad(a: torch.Tensor, buf: Optional[torch.Tensor], plan: DispatchPlan, base: torch.Tensor,
                    shared_logit: torch.Tensor, routed: bool = True):
    """Backward of a combine with gated shared experts: ``(dgate [k, S] or None, d_base [S, M], d_shared_logit [S])`` with
    dgate as :func:`raw_gate_grad`, d_base = w_s * a[s] and d_shared_logit = w_s (1 - w_s) <a[s], base[s]> (fp32 on
    CUDA).  On CUDA one launch computes all three; ``routed=False`` skips the routed dots (``buf`` unused)."""
    if _native_cuda(a) and a.dtype == base.dtype and (not routed or a.dtype == buf.dtype):
        b, sl = _shared_args(base, shared_logit)
        a = a.contiguous()
        seg_off = None
        if routed and plan.layout is not None:
            bufv, seg_off = buf.contiguous().view(plan.layout.R, -1), plan.layout.seg_off
            E, C = plan.layout.E, plan.layout.R
        elif routed:
            bufv, E, C = buf.contiguous().view(plan.E * plan.C, -1), plan.E, plan.C
        else:
            bufv, E, C = None, plan.E, plan.C
        idx, loc = (plan.idx_ks, plan.loc_ks) if routed else (plan.idx_ks[:0], plan.loc_ks[:0])
        backend.count_launch()
        dg, d_base, d_sl = backend.require_ext().gate_grad(a, bufv, idx, loc, E, C, seg_off, b, sl)
        return (dg if routed else None), d_base, d_sl
    dg = raw_gate_grad(a, buf, plan) if routed else None
    work = a.double() if a.dtype == torch.float64 else a.float()
    ws = shared_weight(shared_logit, work.dtype)
    d_base = (ws * work).to(a.dtype)
    d_sl = (ws * (1 - ws)).view(-1) * (work * base.to(work.dtype)).sum(1)
    return dg, d_base, d_sl


def raw_gate_grad(a: torch.Tensor, buf: torch.Tensor, plan: DispatchPlan) -> torch.Tensor:
    """[k, S] row dots  <a[s], buf[slot_j(s)]>  (0 for dropped choices); fp32 on CUDA."""
    if plan.layout is not None:
        from . import packed
        return packed.gate_grad(a, buf.view(plan.layout.R, -1), plan.idx_ks, plan.loc_ks, plan.layout)
    a = a.contiguous()
    buf = buf.contiguous().view(plan.E * plan.C, -1)
    if _native_cuda(a) and a.dtype == buf.dtype:
        backend.count_launch()
        return backend.require_ext().gate_grad(a, buf, plan.idx_ks, plan.loc_ks, plan.E, plan.C)
    if _cpu_native(a) and a.dtype == buf.dtype:
        return backend.ext().cpu_gate_grad(a, buf, plan.idx_ks, plan.loc_ks, plan.E, plan.C)
    wa = a if a.dtype in (torch.float32, torch.float64) else a.float()
    wb = buf.to(wa.dtype)
    slot, valid = _slots(plan)
    return torch.stack([(wa * wb.index_select(0, slot[j])).sum(1) * valid[j].to(wa.dtype) for j in range(plan.k)])


# ----------------------------------------------------------------------------------------------------------------
# autograd
# ----------------------------------------------------------------------------------------------------------------
class GatingEncoder(torch.autograd.Function):
    """tokens [S, M] (+ optional gates [k, S]) -> dispatch buffer [E*C, M]."""

    @staticmethod
    def forward(ctx: Any, plan: DispatchPlan, x: torch.Tensor, gates: Optional[torch.Tensor]):
        ctx.plan = plan
        ctx.has_gates = gates is not None
        if ctx.has_gates:
            ctx.save_for_backward(x, gates)
        return raw_encode(x, gates, plan)

    @staticmethod
    def backward(ctx: Any, dbuf: torch.Tensor):
        plan = ctx.plan
        dbuf = dbuf.contiguous()
        if ctx.has_gates:
            x, gates = ctx.saved_tensors
            dx = raw_decode(dbuf, gates, plan)
            dg = raw_gate_grad(x, dbuf, plan).to(gates.dtype)
            return None, dx, dg
        return None, raw_decode(dbuf, None, plan), None


class GatingDecoder(torch.autograd.Function):
    """expert outputs [E*C, M] (+ optional gates [k, S]) -> tokens [S, M].

    Optional shared experts: ``base [S, M]`` (their output) is added with weight 1, or sigmoid(``shared_logit [S]``)
    per token, inside the same combine launch.  Backward: without the shared gate d_base is the output gradient itself
    (no launch); with it, d_base and d_shared_logit come from the gate-gradient launch (with zero routed choices when
    the routed gates were applied before the experts)."""

    @staticmethod
    def forward(ctx: Any, plan: DispatchPlan, buf: torch.Tensor, gates: Optional[torch.Tensor],
                base: Optional[torch.Tensor] = None, shared_logit: Optional[torch.Tensor] = None):
        ctx.plan = plan
        ctx.has_gates = gates is not None
        ctx.n_inputs = 3 if base is None else 5
        ctx.shared_gated = shared_logit is not None
        if ctx.has_gates or ctx.shared_gated:
            ctx.save_for_backward(buf if ctx.has_gates else None, gates, base if ctx.shared_gated else None, shared_logit)
        return raw_decode(buf, gates, plan, base, shared_logit)

    @staticmethod
    def backward(ctx: Any, dout: torch.Tensor):
        plan = ctx.plan
        dout = dout.contiguous()
        if ctx.n_inputs == 3:
            if ctx.has_gates:
                buf, gates = ctx.saved_tensors[:2]
                dbuf = raw_encode(dout, gates, plan).view_as(buf)
                dg = raw_gate_grad(dout, buf, plan).to(gates.dtype)
                return None, dbuf, dg
            return None, raw_encode(dout, None, plan), None
        dg = d_logit = None
        if ctx.shared_gated:
            buf, gates, base, shared_logit = ctx.saved_tensors
            dbuf = raw_encode(dout, gates, plan)
            dg, d_base, d_logit = raw_shared_grad(dout, buf, plan, base, shared_logit, routed=ctx.has_gates)
            d_logit = d_logit.to(shared_logit.dtype).view_as(shared_logit)
        else:
            gates = ctx.saved_tensors[1] if ctx.has_gates else None
            dbuf = raw_encode(dout, gates, plan)
            if ctx.has_gates:
                dg = raw_gate_grad(dout, ctx.saved_tensors[0], plan)
            d_base = dout
        if ctx.has_gates:
            dbuf = dbuf.view_as(ctx.saved_tensors[0])
            dg = dg.to(gates.dtype)
        return None, dbuf, dg, d_base, d_logit


def _stack_gates(gates_s: Sequence[torch.Tensor]) -> torch.Tensor:
    return torch.stack([g.view(-1) for g in gates_s]) if len(gates_s) > 0 else None


class TutelMoeFastDispatcher:
    """Stateful encode/decode helper kept for API parity (tutel/impls/fast_dispatch.py:85-136)."""

    def __init__(self, num_global_experts, capacity, model_dim, dispatch_dtype):
        self.num_global_experts = int(num_global_experts)
        self.capacity = int(capacity)
        self.model_dim = int(model_dim)
        self.dtype = dispatch_dtype
        self.original_dtype = dispatch_dtype
        self.plan: Optional[DispatchPlan] = None
        self.gates: Optional[torch.Tensor] = None
        self.is_postscore = True

    def update(self, indices_, locations_, gates_, capacity=None, is_postscore=True, plan: Optional[DispatchPlan] = None,
               gates_ks: Optional[torch.Tensor] = None):
        self.capacity = int(capacity) if capacity else self.capacity
        self.is_postscore = is_postscore
        if plan is None:
            idx = torch.stack([x.to(torch.int32).view(-1) for x in indices_])
            loc = torch.stack([x.to(torch.int32).view(-1) for x in locations_])
            plan = DispatchPlan(self.num_global_experts, self.capacity, idx, loc)
        self.plan = plan
        self.gates = gates_ks if gates_ks is not None else _stack_gates(gates_)
        self.sample_size = plan.S
        self.indices_, self.locations_, self.gates_ = list(plan.idx_ks), list(plan.loc_ks), list(self.gates)

    def encode(self, data: torch.Tensor) -> torch.Tensor:
        gates = None if self.is_postscore else self.gates
        return GatingEncoder.apply(self.plan, data, gates)

    def decode(self, data: torch.Tensor, base: Optional[torch.Tensor] = None,
               shared_logit: Optional[torch.Tensor] = None) -> torch.Tensor:
        gates = self.gates if self.is_postscore else None
        if base is None:
            return GatingDecoder.apply(self.plan, data.reshape(self.plan.E * self.plan.C, -1), gates)
        return GatingDecoder.apply(self.plan, data.reshape(self.plan.E * self.plan.C, -1), gates, base, shared_logit)


fast_dispatcher = TutelMoeFastDispatcher


def _dispatcher_for(data: torch.Tensor, crit, is_postscore: bool) -> TutelMoeFastDispatcher:
    d = TutelMoeFastDispatcher(crit[0], crit[4], data.size(-1), data.dtype)
    if isinstance(crit, CriticalData):
        d.update(None, None, None, capacity=crit[4], is_postscore=is_postscore, plan=DispatchPlan.from_critical(crit),
                 gates_ks=crit.gates_ks)
    else:
        d.update(crit[1], crit[2], crit[3], capacity=crit[4], is_postscore=is_postscore)
    return d


def fast_encode(data: torch.Tensor, critical_data, is_postscore: bool = True) -> torch.Tensor:
    """[S, M] tokens -> [E, C, M] expert-major dispatch buffer."""
    assert data.is_contiguous(), 'Input tensor for encode/decode should be in contiguous memory format.'
    E = critical_data[0]
    return _dispatcher_for(data, critical_data, is_postscore).encode(data).view(E, -1, data.size(-1))


def fast_decode(data: torch.Tensor, critical_data, is_postscore: bool = True, base: Optional[torch.Tensor] = None,
                shared_logit: Optional[torch.Tensor] = None) -> torch.Tensor:
    """[E, C, M'] expert outputs -> [S, M'] tokens (weighted sum over the k choices).  ``base [S, M']`` (optional): the
    shared experts' output, added with weight 1 or sigmoid(``shared_logit [S]``) in the same combine."""
    assert data.is_contiguous(), 'Input tensor for encode/decode should be in contiguous memory format.'
    return _dispatcher_for(data, critical_data, is_postscore).decode(data, base, shared_logit).view(-1, data.size(-1))
