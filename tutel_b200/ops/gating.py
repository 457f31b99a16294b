"""Location scan helper kept for API parity (``tutel.moe.fast_cumsum_sub_one``, tutel/jit_kernels/gating.py:19-24).

The layer itself no longer scans one-hot masks: routing uses the fused histogram/scan/rank kernels of
csrc/moe_kernels.cu (see :mod:`tutel_b200.ops.routing`).
"""
import math

import torch


def _use_fast_cumsum() -> bool:
    import os
    return int(os.environ.get('FAST_CUMSUM', '1')) == 1       # same switch as the reference (jit_kernels/gating.py:11)


def fast_cumsum_sub_one(data: torch.Tensor, dim: int = 0) -> torch.Tensor:
    """``cumsum(data, dim=0) - 1`` of a 2-D mask.  CUDA tensors run the three-pass tile scan of csrc/gate_route.cu
    (int32 result, like the reference's ``tutel_ops.cumsum``); ``FAST_CUMSUM=0`` or CPU tensors use ``torch.cumsum``."""
    if data.dim() != 2 or dim != 0:
        raise Exception('Unimplemented fast_cumsum_sub_one() of data = %s and dim = %s' % (data.size(), dim))
    if data.is_cuda and _use_fast_cumsum() and not data.is_floating_point():
        from . import backend
        if backend.has_cuda_ext():
            backend.count_launch(3)
            return backend.require_ext().cumsum_sub_one(data)
    return torch.cumsum(data, dim=0) - 1


# ----------------------------------------------------------------------------------------------------------------
# Fused top-k gating (default on; TUTEL_B200_FUSED_GATE=0 restores the op-by-op formulation)
# ----------------------------------------------------------------------------------------------------------------
# The reference computes softmax, top-k, the one-hot masks, the GShard loss and the gate normalisation as ~15 separate
# PyTorch kernels per forward (tutel/impls/moe_layer.py:283-305, fast_dispatch.py:143-176, losses.py:12-19), and
# autograd adds as many again in backward.  Here: ONE kernel forward (one warp per token: softmax in registers,
# iterative arg-max, per-block partial sums for the loss) and ONE kernel backward (closed-form gradient of the
# normalised gates and of the loss through the softmax).  The pure-torch branch implements the same formulas and is
# what the CPU tests check against autograd of the unfused path.
def fused_gate_mode() -> str:
    """``TUTEL_B200_FUSED_GATE``: unset/``auto`` - fused kernels on CUDA, op-by-op elsewhere;  ``1`` - the fused formulation
    everywhere (its pure-torch branch on CPU, used by the tests);  ``0`` - always op by op."""
    import os
    v = os.environ.get('TUTEL_B200_FUSED_GATE', 'auto').lower()
    if v in ('0', 'off', 'false'):
        return 'off'
    return 'force' if v in ('1', 'on', 'true', 'force') else 'auto'


def fused_gate_enabled() -> bool:
    return fused_gate_mode() != 'off'


class FusedTopKGate(torch.autograd.Function):
    """``logits [S,E] -> (gates [k,S], l_aux)`` plus non-differentiable ``idx [k,S] int32``, ``top1 [S]`` (raw best score)."""

    @staticmethod
    def forward(ctx, logits: torch.Tensor, k: int, normalize: bool, want_loss: bool):
        S, E = logits.shape
        eps = float(torch.finfo(logits.dtype).eps)
        lf = logits.detach()
        if lf.dtype not in (torch.float32, torch.float64):
            lf = lf.to(torch.float32)
        # (the CUDA kernels live in FusedGateRoute below; this class is the same mathematics op by op)
        p = torch.softmax(lf, dim=1)
        top_sk, idx_sk = torch.topk(p, k, dim=1)
        idx, top = idx_sk.t().contiguous().to(torch.int32), top_sk.t().contiguous()
        me = p.sum(0)
        ce = torch.zeros([E], dtype=p.dtype, device=p.device)
        ce.scatter_add_(0, idx[0].to(torch.int64), torch.ones([S], dtype=p.dtype, device=p.device))
        gates = top
        if normalize and k > 1:
            gates = top / torch.clamp(top.sum(dim=0, keepdim=True), min=eps)
        l_aux = (me * ce).sum() * (E / float(S * S)) if want_loss else None
        ctx.save_for_backward(p, idx, top, ce)
        ctx.k, ctx.normalize, ctx.eps, ctx.in_dtype, ctx.want_loss = k, normalize, eps, logits.dtype, want_loss
        out_loss = l_aux.to(logits.dtype) if want_loss else torch.zeros((), dtype=logits.dtype, device=logits.device)
        idx_out, top1 = idx, top[0].to(logits.dtype)
        ctx.mark_non_differentiable(idx_out, top1)
        return gates.to(logits.dtype), out_loss, idx_out, top1

    @staticmethod
    def backward(ctx, dgates, dloss, _didx, _dtop1):
        p, idx, top, ce = ctx.saved_tensors
        S, E = p.shape
        k = ctx.k
        dg = (dgates if dgates is not None else torch.zeros_like(top)).to(p.dtype).contiguous()
        dl = dloss.to(p.dtype).reshape(1).contiguous() if (ctx.want_loss and dloss is not None) else None
        dr = dg
        if ctx.normalize and k > 1:
            D = top.sum(dim=0, keepdim=True)
            Dc = torch.clamp(D, min=ctx.eps)
            dot = (dg * top).sum(dim=0, keepdim=True)
            dr = dg / Dc - torch.where(D > ctx.eps, dot / (Dc * Dc), torch.zeros_like(dot))
        dp = torch.zeros_like(p)
        if dl is not None:
            dp += (dl * (E / float(S * S))) * ce.unsqueeze(0)
        dp.scatter_add_(1, idx.t().to(torch.int64), dr.t().contiguous())
        dlogits = p * (dp - (dp * p).sum(dim=1, keepdim=True))
        return dlogits.to(ctx.in_dtype), None, None, None


def fused_topk_gate(logits: torch.Tensor, k: int, normalize: bool = True, want_loss: bool = True):
    """Returns ``(idx_ks int32 [k,S], gates_ks [k,S], l_aux or None, top1 [S])``."""
    gates, l_aux, idx, top1 = FusedTopKGate.apply(logits, int(k), bool(normalize), bool(want_loss))
    return idx, gates, (l_aux if want_loss else None), top1


# ----------------------------------------------------------------------------------------------------------------
# Fused gate + routing on CUDA: logits -> everything the dispatch needs in TWO launches, backward in ONE
# ----------------------------------------------------------------------------------------------------------------
class FusedGateRoute(torch.autograd.Function):
    """``logits [S,E]`` -> differentiable ``(gates fp32 [k,S], l_aux)`` plus the routing decisions ``idx, loc [k,S]``,
    ``counts [E]``, ``slot_src [E*C]`` (or None when ``capacity`` is 0) and ``top1 [S]`` (csrc/gate_route.cu).

    The gates are kept in fp32 (they are consumed by fp32-accumulating kernels; the reference rounds them to the
    score dtype first), the loss is returned in the logits' dtype."""

    @staticmethod
    def forward(ctx, logits: torch.Tensor, k: int, normalize: bool, capacity: int):
        from . import backend
        lg = logits.detach().contiguous()
        eps = float(torch.finfo(logits.dtype).eps)
        backend.count_launch(2)
        out = backend.require_ext().gate_route_forward(lg, int(k), int(capacity), bool(normalize), eps)
        scores, idx, top, gates, loc, counts, ce, l_aux = out[:8]
        slot = out[8] if len(out) > 8 else None
        ctx.save_for_backward(scores, idx, top, ce)
        ctx.normalize, ctx.eps, ctx.like = bool(normalize), eps, lg.new_empty(0)
        top1 = top[0]
        ctx.mark_non_differentiable(idx, loc, counts, top1)
        if slot is not None:
            ctx.mark_non_differentiable(slot)
        ctx.has_slot = slot is not None
        res = (gates, l_aux, idx, loc, counts, top1)
        return res + ((slot,) if slot is not None else ())

    @staticmethod
    def backward(ctx, dgates, dloss, *_unused):
        from . import backend
        scores, idx, top, ce = ctx.saved_tensors
        dg = None if dgates is None else dgates.to(torch.float32).contiguous()
        dl = None if dloss is None else dloss.to(ctx.like.dtype).reshape(1)
        backend.count_launch()
        dlogits = backend.require_ext().gate_route_backward(scores, idx, top, dg, ce, dl, ctx.like, ctx.normalize, ctx.eps)
        return dlogits, None, None, None


def fused_gate_route_available(logits: torch.Tensor, k: int) -> bool:
    from . import backend
    return (logits.is_cuda and logits.dim() == 2 and logits.size(1) <= 512 and 1 <= k <= min(32, logits.size(1)) and
            logits.dtype in (torch.float32, torch.float16, torch.bfloat16) and logits.size(0) > 0 and
            k * logits.size(1) <= 4096 and backend.has_cuda_ext())


def fused_gate_route(logits: torch.Tensor, k: int, normalize: bool, capacity: int):
    """Returns ``(idx_ks, loc_ks, gates_ks fp32, l_aux, counts, top1, slot_src or None)``."""
    out = FusedGateRoute.apply(logits, int(k), bool(normalize), int(capacity))
    gates, l_aux, idx, loc, counts, top1 = out[:6]
    return idx, loc, gates, l_aux, counts, top1, (out[6] if len(out) > 6 else None)


# ----------------------------------------------------------------------------------------------------------------
# Sigmoid scoring with a selection bias and group-limited choice (DeepSeek-V3 / Kimi-K2 / GLM-4.5 / Moonlight routing)
# ----------------------------------------------------------------------------------------------------------------
def sigmoid_topk_gate(logits: torch.Tensor, bias: torch.Tensor, k: int, normalize: bool = True, n_group: int = 1,
                      topk_group: int = 1, scale: float = 1.0, want_loss: bool = True):
    """The definition of sigmoid routing, in plain torch (also the CPU / op-by-op path; autograd gives its backward).

    Per token s and expert e, in fp32:  score s_se = sigmoid(z_se), selection key s_se + b_e (a NaN key counts as
    -inf).  With ``n_group > 1`` group g holds experts [g E/n_group, (g+1) E/n_group), its score is the sum of its top
    min(2, E/n_group) keys, and only experts of the ``topk_group`` best groups (ties to the lower group id; a group
    whose score is NaN or -inf is never kept) may be chosen.  The ``k`` largest keys among those are chosen (ties to
    the lower id); a choice without a key above -inf gets id E and routes nowhere.  Gates use the scores without the
    bias: ``scale * r_j / max(sum_j r_j, eps)`` (``normalize`` and k > 1) or ``scale * r_j``.  The auxiliary loss is
    ``E / (k S^2) sum_e n_e sum_s s_se / T_s`` with n_e the (token, choice) pairs routed to e and T_s = sum_e s_se.

    Returns ``(idx int32 [k,S], gates fp32 (fp64 for fp64 logits) [k,S], l_aux (logits dtype) or None, counts n_e fp32 [E], top1 [S])``,
    top1 being each token's first-choice score."""
    S, E = logits.shape
    eps = float(torch.finfo(logits.dtype).eps)
    s = torch.sigmoid(logits if logits.dtype == torch.float64 else logits.float())     # (fp64 stays fp64: tests)
    neg_inf = torch.tensor(-math.inf, device=logits.device, dtype=s.dtype)
    with torch.no_grad():
        key = s + bias.to(s.dtype)
        key = torch.where(torch.isnan(key), neg_inf, key)
        if n_group > 1:
            gsz = E // n_group
            gs = key.view(S, n_group, gsz).topk(min(2, gsz), dim=2).values.sum(2)
            gs = torch.where(torch.isnan(gs), neg_inf, gs)
            order = torch.sort(gs, dim=1, descending=True, stable=True).indices[:, :topk_group]
            kept = torch.zeros_like(gs, dtype=torch.bool).scatter_(1, order, True) & (gs > -math.inf)
            key = torch.where(kept.repeat_interleave(gsz, dim=1), key, neg_inf)
        srt = torch.sort(key, dim=1, descending=True, stable=True)
        valid = srt.values[:, :k] > -math.inf
        ids = torch.where(valid, srt.indices[:, :k], torch.full_like(srt.indices[:, :k], E))       # [S, k]
        # (a scatter into E + 1 bins, the last one for choices that route nowhere: no host synchronisation on CUDA)
        counts = torch.zeros(E + 1, dtype=s.dtype, device=s.device).scatter_add_(
            0, ids.reshape(-1), torch.ones(ids.numel(), dtype=s.dtype, device=s.device))[:E]
    r = torch.where(valid, s.gather(1, ids.clamp(max=E - 1)), torch.zeros((), device=s.device, dtype=s.dtype))
    gates = r
    if normalize and k > 1:
        gates = r / torch.clamp(r.sum(dim=1, keepdim=True), min=eps)
    gates = gates * float(scale)
    l_aux = None
    if want_loss:
        l_aux = ((s / s.sum(dim=1, keepdim=True)).sum(0) * counts).sum() * (E / float(k * S * S))
        l_aux = l_aux.to(logits.dtype)
    return ids.t().contiguous().to(torch.int32), gates.t(), l_aux, counts, r[:, 0].detach()


class SigmoidGateRoute(torch.autograd.Function):
    """CUDA kernels of :func:`sigmoid_topk_gate` fused with routing, as :class:`FusedGateRoute`: ``logits [S,E]`` ->
    differentiable ``(gates fp32 [k,S], l_aux)`` plus ``idx, loc [k,S]``, ``counts [E]``, ``top1 [S]`` and the slot map
    (when ``capacity > 0``).  ``expert_load`` (fp32 [E] or None) accumulates the all-choice counts inside the routing
    launch."""

    @staticmethod
    def forward(ctx, logits, bias, k, normalize, capacity, n_group, topk_group, scale, expert_load):
        from . import backend
        lg = logits.detach().contiguous()
        eps = float(torch.finfo(logits.dtype).eps)
        backend.count_launch(2)
        out = backend.require_ext().sigmoid_gate_route_forward(lg, bias.detach(), int(k), int(capacity), bool(normalize),
                                                               eps, int(n_group), int(topk_group), float(scale),
                                                               expert_load)
        scores, idx, top, gates, loc, counts, ce, l_aux = out[:8]
        slot = out[8] if len(out) > 8 else None
        ctx.save_for_backward(scores, idx, top, ce)
        ctx.normalize, ctx.eps, ctx.scale, ctx.like = bool(normalize), eps, float(scale), lg.new_empty(0)
        top1 = top[0]
        ctx.mark_non_differentiable(idx, loc, counts, top1)
        if slot is not None:
            ctx.mark_non_differentiable(slot)
        res = (gates, l_aux, idx, loc, counts, top1)
        return res + ((slot,) if slot is not None else ())

    @staticmethod
    def backward(ctx, dgates, dloss, *_unused):
        from . import backend
        scores, idx, top, ce = ctx.saved_tensors
        dg = None if dgates is None else dgates.to(torch.float32).contiguous()
        dl = None if dloss is None else dloss.to(ctx.like.dtype).reshape(1)
        backend.count_launch()
        dlogits = backend.require_ext().sigmoid_gate_route_backward(scores, idx, top, dg, ce, dl, ctx.like, ctx.normalize,
                                                                   ctx.eps, ctx.scale)
        return dlogits, None, None, None, None, None, None, None, None


def sigmoid_gate_route_available(logits: torch.Tensor, k: int, n_group: int) -> bool:
    """The fused kernels' limits (those of :func:`fused_gate_route_available`, and at most 32 expert groups)."""
    return n_group <= 32 and fused_gate_route_available(logits, k)


def sigmoid_gate_route(logits, bias, k, normalize, capacity, n_group=1, topk_group=1, scale=1.0, expert_load=None):
    """Returns ``(idx_ks, loc_ks, gates_ks fp32, l_aux, counts, top1, slot_src or None)``."""
    out = SigmoidGateRoute.apply(logits, bias, int(k), bool(normalize), int(capacity), int(n_group), int(topk_group),
                                 float(scale), expert_load)
    gates, l_aux, idx, loc, counts, top1 = out[:6]
    return idx, loc, gates, l_aux, counts, top1, (out[6] if len(out) > 6 else None)


def expert_bias_update(bias: torch.Tensor, load: torch.Tensor, gamma: float) -> None:
    """Auxiliary-loss-free balancing step, in place: ``bias += gamma * sign(mean(load) - load)``, then ``load = 0``.
    The mean is ``sum(load) / E`` in fp32 (exact for integer loads below 2^24).  CUDA tensors take one launch."""
    if bias.is_cuda:
        from . import backend
        backend.count_launch()
        backend.require_ext().expert_bias_update(bias, load, float(gamma))
        return
    mean = load.sum() / load.numel()
    bias.add_(torch.sign(mean - load) * gamma)
    load.zero_()
