"""Top-k routing: expert ids, queue locations, gate values, capacity (``tutel.moe.top_k_routing``).

Semantics follow tutel/impls/fast_dispatch.py:143-204 exactly (stable token order, j-th choices queue behind all
(j-1)-th choices, drop rule ``location >= capacity``, capacity rules for positive / zero / negative factors and the
alignment round-up), but the implementation is different: no one-hot masks and no per-choice cumsum - a fused
histogram / scan / rank pass (csrc/moe_kernels.cu on CUDA, csrc/cpu_kernels.cpp on CPU) produces locations, the
per-expert counts and (on CUDA) the inverse slot->token map used by the gather-style encode kernel.
"""
from __future__ import annotations

import logging
from typing import List, Optional

import torch

from ..models import losses
from ..parallel.communicate import get_world_rank, simple_all_reduce
from . import backend


class CriticalData(tuple):
    """``(num_global_experts, indices_s, locations_s, gates_s, capacity, dispatch_count)`` plus cached stacked views.

    Behaves like the reference's plain tuple; the extra attributes let the kernels consume ``[k, S]`` tensors
    without re-stacking: ``idx_ks``, ``loc_ks`` (int32), ``gates_ks`` (differentiable), ``slot_src`` (lazy).
    ``layout``: the :class:`tutel_b200.ops.packed.PackedLayout` of a packed-mode routing (capacity 0), else None.
    """

    def __new__(cls, E, idx_ks, loc_ks, gates_ks, capacity, counts):
        k = idx_ks.size(0)
        self = super().__new__(cls, (E, [idx_ks[j] for j in range(k)], [loc_ks[j] for j in range(k)],
                                     [gates_ks[j] for j in range(k)], capacity, counts))
        self.idx_ks, self.loc_ks, self.gates_ks = idx_ks, loc_ks, gates_ks
        self._slot_src = None
        self.layout = None
        return self

    @property
    def slot_src(self) -> torch.Tensor:
        if self._slot_src is None:
            self._slot_src = build_slot_map(self.idx_ks, self.loc_ks, self[0], self[4])
        return self._slot_src


def _locations(idx_ks: torch.Tensor, E: int):
    """Stable queue positions for [k, S] expert ids -> (loc [k,S] int32, counts [E] int32)."""
    k, S = idx_ks.shape
    if idx_ks.is_cuda and backend.has_cuda_ext():
        backend.count_launch(3)
        loc, counts = backend.require_ext().route_locations(idx_ks, E, 0)[:2]
        return loc, counts
    if not idx_ks.is_cuda and backend.has_ext():
        loc, counts = backend.ext().cpu_route_locations(idx_ks.contiguous(), E)
        return loc, counts
    # pure-torch fallback: one-hot cumulative sums
    flat = idx_ks.reshape(-1).to(torch.int64)
    onehot = torch.zeros([k * S, E], dtype=torch.int32, device=idx_ks.device)
    onehot.scatter_(1, flat.unsqueeze(1), 1)
    pos = torch.cumsum(onehot, dim=0) - 1
    loc = pos.gather(1, flat.unsqueeze(1)).view(k, S).to(torch.int32)
    return loc, onehot.sum(0).to(torch.int32)


def build_slot_map(idx_ks: torch.Tensor, loc_ks: torch.Tensor, E: int, C: int) -> torch.Tensor:
    """int32 [E*C]: ``token * k + choice`` occupying each slot, -1 for padding."""
    k, S = idx_ks.shape
    if idx_ks.is_cuda and backend.has_cuda_ext():
        backend.count_launch()
        return backend.require_ext().build_slot_map(idx_ks.contiguous(), loc_ks.contiguous(), E, C)
    slot = torch.full([E * C], -1, dtype=torch.int32, device=idx_ks.device)
    valid = (loc_ks < C) & (idx_ks >= 0)
    tok = torch.arange(S, device=idx_ks.device, dtype=torch.int32).unsqueeze(0) * k + \
        torch.arange(k, device=idx_ks.device, dtype=torch.int32).unsqueeze(1)
    slot[(idx_ks.to(torch.int64) * C + loc_ks.to(torch.int64))[valid]] = tok[valid]
    return slot


def extract_critical(scores: torch.Tensor, top_k: int, loss_fn=losses.gshard_loss, capacity_factor: float = 1.0,
                     batch_prioritized_routing: bool = False, normalize_gate: bool = True, alignment: int = 1,
                     group=None, inequivalent_tokens: bool = False, _fused=None, packed: bool = False):
    """``_fused`` (internal): ``(idx_ks, gates_ks, l_aux, top1)`` from :func:`tutel_b200.ops.gating.fused_topk_gate` -
    top-k selection, gate normalisation and the auxiliary loss were then already computed by the fused kernel.

    ``packed`` (dropless on one GPU, CUDA): no capacity is computed - nothing is read back to the host - and the result
    carries the :class:`tutel_b200.ops.packed.PackedLayout` built from the device counts; its capacity field is 0."""
    num_global_experts = int(scores.size(1))
    top_k_original, top_k = top_k, min(top_k, num_global_experts)
    if _fused is None:
        topk_indices = torch.topk(scores, top_k, dim=1).indices                     # [S, k]
        idx_ks = topk_indices.t().contiguous().to(torch.int32)                      # [k, S]
        gates_ks = scores.gather(1, topk_indices).t()                               # [k, S], differentiable
        l_loss = loss_fn(scores, topk_indices) if loss_fn is not None else None
        confidence = None
    else:
        idx_ks, gates_ks, l_loss, confidence = _fused

    if batch_prioritized_routing:
        # tokens claim slots in order of decreasing confidence instead of batch order
        if confidence is None:
            confidence = scores.max(dim=1)[0]
        order = (-confidence).argsort(dim=0)
        loc_sorted, counts = _locations(idx_ks[:, order].contiguous(), num_global_experts)
        loc_ks = torch.empty_like(loc_sorted)
        loc_ks[:, order] = loc_sorted
    else:
        loc_ks, counts = _locations(idx_ks, num_global_experts)

    if _fused is None and top_k > 1 and normalize_gate:
        denom = torch.clamp(gates_ks.sum(dim=0, keepdim=True), min=torch.finfo(gates_ks.dtype).eps)
        gates_ks = gates_ks / denom

    if packed:
        return _packed_critical(num_global_experts, idx_ks, loc_ks, gates_ks, counts), l_loss

    num_samples = _num_samples(int(scores.size(0)), scores.device, group, inequivalent_tokens)
    capacity = _capacity(num_samples, num_global_experts, top_k, top_k_original, capacity_factor, counts, group, alignment)

    return CriticalData(num_global_experts, idx_ks, loc_ks, gates_ks, capacity, counts), l_loss


def _packed_critical(E, idx_ks, loc_ks, gates_ks, counts) -> CriticalData:
    from .packed import PackedLayout
    crit = CriticalData(E, idx_ks, loc_ks, gates_ks, 0, counts)
    crit.layout = PackedLayout.build(idx_ks, loc_ks, counts)
    crit._slot_src = crit.layout.slot_src
    return crit


def _num_samples(local: int, device, group, inequivalent_tokens: bool) -> int:
    if not inequivalent_tokens:
        return local
    t = torch.tensor(local, device=device)
    return int(simple_all_reduce(t, group=group, op=torch.distributed.ReduceOp.MAX))


def _capacity(num_samples, num_global_experts, top_k, top_k_original, capacity_factor, counts, group, alignment) -> int:
    """Slots per expert and source rank (tutel/impls/fast_dispatch.py:182-200): a positive factor is a static multiple
    of the even share, zero means "as large as the fullest expert anywhere" (dropless), a negative factor caps that."""
    samples_per_expert = (num_samples + num_global_experts - 1) // num_global_experts
    if capacity_factor > 0:
        capacity = top_k * int(capacity_factor * samples_per_expert)
    else:
        capacity = int(simple_all_reduce(counts.max(), group=group, op=torch.distributed.ReduceOp.MAX))
        if capacity_factor < 0:
            capacity = min(capacity, top_k * int(-capacity_factor * samples_per_expert))
    remainder = capacity % alignment
    if remainder > 0:
        capacity = capacity + alignment - remainder
    if logging.getLogger().isEnabledFor(logging.INFO) and get_world_rank(group) == 0:
        logging.info('Capacity = %s, real-time capacity-factor for top-%s = %s', capacity, top_k_original,
                     capacity / max(top_k * samples_per_expert, 1))
    return capacity


def fused_extract_critical(logits: torch.Tensor, top_k: int, capacity_factor: float = 1.0, normalize_gate: bool = True,
                           alignment: int = 1, group=None, inequivalent_tokens: bool = False, rows_bound: int = 0,
                           sigmoid: Optional[dict] = None, packed: bool = False):
    """CUDA fast path of :func:`extract_critical` for GShard-loss top-k gates: softmax, top-k, gate normalisation, the
    auxiliary loss, queue locations, counts and the inverse slot map come out of TWO kernel launches
    (:func:`tutel_b200.ops.gating.fused_gate_route`); with a positive capacity factor nothing touches the host.

    ``sigmoid``: sigmoid scoring instead (:func:`tutel_b200.ops.gating.sigmoid_gate_route`), a dict with ``bias``,
    ``n_group``, ``topk_group``, ``scale`` and ``expert_load`` (or None).

    ``packed``: dropless into the expert-packed layout (see :func:`extract_critical`): no capacity, no host read."""
    from .gating import fused_gate_route, sigmoid_gate_route
    E = int(logits.size(1))
    top_k_original, top_k = top_k, min(top_k, E)
    if packed:
        if sigmoid is None:
            idx, loc, gates, l_aux, counts, _top1, _ = fused_gate_route(logits, top_k, normalize_gate, 0)
        else:
            idx, loc, gates, l_aux, counts, _top1, _ = sigmoid_gate_route(logits, k=top_k, normalize=normalize_gate,
                                                                          capacity=0, **sigmoid)
        return _packed_critical(E, idx, loc, gates, counts), l_aux
    num_samples = _num_samples(int(logits.size(0)), logits.device, group, inequivalent_tokens)
    static_cap = _capacity(num_samples, E, top_k, top_k_original, capacity_factor, None, group, alignment) if capacity_factor > 0 else 0
    if capacity_factor <= 0 and rows_bound > 0:
        # Dropless without the host round trip (the reference reads the fullest expert's count back, tutel/impls/
        # fast_dispatch.py:192-193): a token never picks an expert twice, so `num_samples` rows per expert always suffice.
        # The buffers are sized for that bound and every kernel downstream skips rows past the device-side counts.
        static_cap = rows_bound if capacity_factor == 0 else min(rows_bound, top_k * int(-capacity_factor * ((num_samples + E - 1) // E)))
        static_cap = (static_cap + alignment - 1) // alignment * alignment
        capacity_factor = 1.0          # (only selects the "capacity is already known" branch below)
    if sigmoid is None:
        idx, loc, gates, l_aux, counts, _top1, slot = fused_gate_route(logits, top_k, normalize_gate, static_cap)
    else:
        idx, loc, gates, l_aux, counts, _top1, slot = sigmoid_gate_route(logits, k=top_k, normalize=normalize_gate,
                                                                         capacity=static_cap, **sigmoid)
    capacity = static_cap if capacity_factor > 0 else \
        _capacity(num_samples, E, top_k, top_k_original, capacity_factor, counts, group, alignment)
    crit = CriticalData(E, idx, loc, gates, capacity, counts)
    crit._slot_src = slot
    crit.skip_padding = rows_bound > 0 and slot is not None     # bound-sized buffers: only rows below the counts are ever read
    return crit, l_aux


def get_dispatch_count(critical_data):
    return critical_data[-1]
