"""Bias-free linear top-k gate: ``logits = x @ wg^T`` with ``wg`` of shape ``[num_global_experts, model_dim]``
(API and state-dict key ``wg.weight`` as in tutel/gates/top.py:6-25).

``scoring_func='sigmoid'`` selects DeepSeek-V3-style routing (ops/gating.py, :func:`sigmoid_topk_gate`): sigmoid
scores, selection on score + ``e_score_correction_bias``, optionally limited to the best ``topk_group`` of ``n_group``
expert groups, gates scaled by ``routed_scaling_factor``.  The bias is not trained by gradient: with
``bias_update_speed > 0`` every training forward adds its per-expert counts to ``expert_load``, and after the
optimizer step the bias moves by ``bias_update_speed`` towards balance (auxiliary-loss-free load balancing).  With the
default 0 the bias is frozen and nothing is accumulated."""
import itertools
import weakref

import torch
import torch.nn.functional as F

# Sigmoid gates whose training forwards accumulated loads since their last update, keyed by creation number.  Updates
# run in creation order: each one may all-reduce over the gate's process group, and a model built the same way on
# every rank then pairs the same gates' collectives on every rank.
_PENDING = {}
_CREATED = itertools.count()
_HOOKED = [False]


def apply_pending_bias_updates():
    """Apply the bias update of every gate that ran a training forward since its last update, in creation order (an
    optimizer-step post-hook calls this; a step captured into a CUDA graph captures the updates with it)."""
    for key in sorted(_PENDING):
        gate = _PENDING.get(key, lambda: None)()
        if gate is None:
            _PENDING.pop(key, None)
        else:
            gate.update_bias()


def _ensure_step_hook():
    if _HOOKED[0]:
        return
    _HOOKED[0] = True
    from torch.optim.optimizer import register_optimizer_step_post_hook
    register_optimizer_step_post_hook(lambda *_: apply_pending_bias_updates())


class LinearTopKGate(torch.nn.Module):
    #: per-gate options that the MoE layer consumes itself (they only have to be accepted here)
    accepted_options = frozenset({'capacity_factor', 'gate_noise'})
    #: buffers kept in fp32 when the model is cast: a 16-bit bias would swallow increments of 1e-3
    _fp32_buffers = ('e_score_correction_bias', 'expert_load')

    def __init__(self, model_dim, num_global_experts, k=1, fp32_gate=False, scoring_func='softmax', n_group=1,
                 topk_group=1, routed_scaling_factor=1.0, bias_update_speed=0.0, **options):
        super().__init__()
        unknown = sorted(set(options) - self.accepted_options)
        if unknown:
            raise Exception('Unrecognized argument provided to Gating module: %s' % unknown[0])
        self.fp32_gate = bool(fp32_gate)
        self.top_k = min(int(k), num_global_experts)
        self.wg = torch.nn.Linear(model_dim, num_global_experts, bias=False, dtype=torch.float32 if self.fp32_gate else None)
        if scoring_func not in ('softmax', 'sigmoid'):
            raise ValueError("scoring_func must be 'softmax' or 'sigmoid', got %r" % (scoring_func,))
        self.scoring_func = scoring_func
        if scoring_func == 'softmax':
            if (n_group, topk_group, routed_scaling_factor, bias_update_speed) != (1, 1, 1.0, 0.0):
                raise ValueError('n_group, topk_group, routed_scaling_factor and bias_update_speed need '
                                 "scoring_func='sigmoid'")
            return
        E = num_global_experts
        self.n_group, self.topk_group = int(n_group), int(topk_group)
        if self.n_group < 1 or E % self.n_group != 0:
            raise ValueError('n_group (%d) must be positive and divide the number of experts (%d)' % (self.n_group, E))
        if not 1 <= self.topk_group <= self.n_group:
            raise ValueError('topk_group (%d) must be in [1, n_group = %d]' % (self.topk_group, self.n_group))
        self.routed_scaling_factor = float(routed_scaling_factor)
        self.bias_update_speed = float(bias_update_speed)
        if not self.bias_update_speed >= 0:
            raise ValueError('bias_update_speed (%r) must be >= 0' % (bias_update_speed,))
        self.check_top_k(self.top_k)
        self.register_buffer('e_score_correction_bias', torch.zeros(E, dtype=torch.float32))
        self.register_buffer('expert_load', torch.zeros(E, dtype=torch.float32), persistent=False)
        self.balance_group = None          # process group the loads are summed over (set by the MoE layer)
        self._created = next(_CREATED)
        _ensure_step_hook()

    def check_top_k(self, k):
        """A sigmoid gate must find ``k`` experts in its ``topk_group`` kept groups."""
        if self.scoring_func != 'sigmoid':
            return
        E = self.wg.weight.size(0)
        if not 1 <= k <= self.topk_group * E // self.n_group:
            raise ValueError('top_k (%d) must be in [1, topk_group * E / n_group = %d]' % (
                k, self.topk_group * E // self.n_group))

    def _apply(self, fn, recurse=True):
        keep = {n: self._buffers.pop(n) for n in self._fp32_buffers if n in self._buffers}
        try:
            super()._apply(fn, recurse)
        finally:
            for n, b in keep.items():
                t = fn(b)
                self._buffers[n] = t if t.dtype == torch.float32 else b.to(t.device)
        return self

    @property
    def balancing(self) -> bool:
        """Whether training forwards accumulate loads and the bias moves (``bias_update_speed > 0``)."""
        return self.bias_update_speed > 0

    def note_training_forward(self):
        """Called by the layer after a training forward added its counts to ``expert_load``."""
        _PENDING[self._created] = weakref.ref(self)

    @torch.no_grad()
    def update_bias(self):
        """``e_score_correction_bias += bias_update_speed * sign(mean(load) - load)`` with the loads summed over
        ``balance_group``, then ``expert_load = 0``.  No host synchronisation.  Nothing to do for a frozen bias."""
        _PENDING.pop(self._created, None)
        if not self.balancing:
            return
        load = self.expert_load
        group = self.balance_group
        if group is not None and torch.distributed.get_world_size(group) > 1:
            torch.distributed.all_reduce(load, group=group)
        from ...ops.gating import expert_bias_update
        expert_bias_update(self.e_score_correction_bias, load, self.bias_update_speed)

    def forward(self, x):
        if self.fp32_gate and self.wg.weight.dtype != torch.float32:
            self.wg.float()          # the surrounding model was cast (`.half()` / `.bfloat16()`): this gate stays fp32
        weight = self.wg.weight
        return F.linear(x.to(weight.dtype), weight)


Gate = LinearTopKGate
