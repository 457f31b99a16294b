"""The MoE layer (``tutel.moe.moe_layer``).

Public behaviour follows tutel/impls/moe_layer.py:42-365: constructor options, per-forward overrides
(``capacity_factor, top_k, a2a_ffn_overlap_degree, adaptive_r, megablocks_size, gate_index, reserve_dims,
inequivalent_tokens``), parallelism switching with an unchanged parameter layout, state-dict keys and tolerant
loading.  The execution engine underneath is new:

    routing   fused histogram/scan/rank kernels          (ops/routing.py, csrc/moe_kernels.cu)
    dispatch  slot-centric gather, native bf16/fp16      (ops/dispatch.py)
    exchange  in-kernel NVLink peer-to-peer pushes       (parallel/p2p.py)  or NCCL / Gloo
    experts   wgmma grouped GEMMs with fused epilogues (ops/gemm.py, csrc/gemm_sm90.cu)
    fused     dispatch+GEMM1 / GEMM2+combine over peer memory, tile-granular flags (parallel/fused.py)
"""
from __future__ import annotations

import importlib
import logging
import os
import re
from typing import Optional

import torch
import torch.distributed as dist
import torch.nn.functional as F
from torch import Tensor
from torch.nn import ModuleList

from ..ops.dispatch import fast_decode, fast_encode
from ..ops.gating import (fused_gate_mode, fused_gate_route_available, fused_topk_gate, sigmoid_gate_route_available,
                          sigmoid_topk_gate)
from ..ops.routing import extract_critical, fused_extract_critical, get_dispatch_count
from ..parallel import communicate as C
from ..parallel.overlap import a2a_ffn_overlap_forward
from ..utils.trace import stage


def _OVERLAP_ON_CPU() -> bool:
    """Testing hook: run the chunked a2a/FFN pipeline (parallel/overlap.py) on CPU tensors too (the reference only
    pipelines on CUDA, tutel/impls/moe_layer.py:344; on CPU it buys nothing but lets Gloo tests cover the logic)."""
    return os.environ.get('TUTEL_B200_OVERLAP_ON_CPU', '0') == '1'
from . import losses


def _autocast_dtype(tensor: Tensor) -> Optional[torch.dtype]:
    if not torch.is_autocast_enabled():
        return None
    kind = tensor.device.type
    if kind == 'cuda':
        return torch.get_autocast_gpu_dtype()
    if kind == 'cpu':
        return torch.get_autocast_cpu_dtype()
    return torch.get_autocast_dtype(kind)


def _parse_parallel_type(parallel_type: str, sharded_count: int, valid_rs):
    """'adaptive:N' | 'data' | 'model' | 'auto'  ->  adaptive degree r (moe_layer.py:131-143)."""
    if parallel_type.startswith('adaptive:'):
        r = min(max(int(parallel_type.split(':', 1)[1]), 0), sharded_count)
        if r not in valid_rs:
            raise Exception('Unexpected value of adaptive_degree: %d, expecting a candidate within %s.' % (r, valid_rs))
        return r
    if sharded_count == 1:
        return sharded_count
    if parallel_type == 'data':
        return 1
    if parallel_type == 'model':
        return sharded_count
    if parallel_type == 'auto':
        return 1
    raise Exception('Unrecognized parallel type specified: %s' % parallel_type)


class MOELayer(torch.nn.Module):
    """Mixture-of-Experts layer with switchable parallelism (H100-native engine)."""

    # ------------------------------------------------------------------------------------------------ statics
    @staticmethod
    def global_expert_count(num_local_experts, group=None):
        """Positive int: experts per GPU.  Negative int -Sh (or the fraction 1/Sh): one expert shared by Sh GPUs."""
        if not isinstance(num_local_experts, int):
            num_local_experts = -int(1 / (num_local_experts + 1e-5))
        world_size = C.get_world_size(group)
        if num_local_experts == 0:
            raise Exception('Invalid value of num_local_experts: %d' % num_local_experts)
        if num_local_experts > 0:
            return num_local_experts * world_size
        assert world_size % -num_local_experts == 0, \
            'Excepting %d devices to share an expert param, while global device count is %d.' % (-num_local_experts, world_size)
        return world_size // -num_local_experts

    # ------------------------------------------------------------------------------------------ checkpointing
    def _load_from_state_dict(self, state_dict, prefix, *args, **kwargs):
        key = prefix + '_num_global_experts'
        if key not in state_dict:
            logging.warning('Loading a legacy MoE checkpoint without `_num_global_experts`; it will be rewritten in the '
                            'self-describing format on the next save.')
            state_dict[key] = self._num_global_experts
        else:
            have, want = int(state_dict[key]), self.num_global_experts
            assert have == want, 'Failed to load state from checkpoint: the number of global experts mismatch (%s <- %s)' % (want, have)
        for name, param in self.experts.named_parameters():
            key = prefix + 'experts.' + name
            if key not in state_dict:
                logging.warning('Could not find parameter `%s` in state_dict, zero values will be filled into this parameter.' % key)
                state_dict[key] = torch.zeros_like(param)
            if state_dict[key].numel() == param.numel():
                state_dict[key] = state_dict[key].view(param.shape)
        return super()._load_from_state_dict(state_dict, prefix, *args, **kwargs)

    @property
    def num_global_experts(self):
        # The count also lives in the `_num_global_experts` buffer (state-dict compatibility with the reference, which reads
        # it back with int() - a device-to-host synchronisation in every forward once the module is on a GPU).  The Python
        # copy is what the hot path uses: no synchronisation, and forward passes can be captured in CUDA graphs.
        return self._n_global_experts

    # -------------------------------------------------------------------------------------------- construction
    def __init__(self, gate_type, model_dim: int, experts=None, scan_expert_func=None, result_func=None, group=None,
                 seeds=None, a2a_ffn_overlap_degree=1, is_postscore=True, batch_prioritized_routing=False,
                 normalize_gate=True, is_gshard_loss=True, parallel_type='adaptive:1', use_2dh=False, shared_experts=None,
                 **kwargs):
        """``shared_experts`` (optional): ``{'num_experts': n}`` adds shared experts that every token passes through,
        added to the routed output with weight 1 (DeepSeek-V2/V3, Kimi-K2, GLM-4.5, Moonlight, Llama-4).  n experts of
        ``hidden_size_per_expert`` H that are always selected with weight 1 are one dense expert of hidden size nH, of the
        routed experts' type (``ffn`` or ``llama_ffn``) and options, replicated on every rank: ``shared_experts.*``.
        ``'gate': True`` adds ``shared_expert_gate`` (``Linear(model_dim, 1, bias=False)``) and scales the shared output
        by sigmoid(x . w) per token (Qwen1.5/2-MoE).  The shared term is added inside the combine kernel.
        ``'weight_format': None | 'fp8_block' | 'int4'`` overrides the routed experts' stored weight format for the
        shared expert alone (``llama_ffn``), e.g. bf16 shared experts beside int4 routed ones as Kimi-K2-Thinking ships
        them; without the key the shared expert takes the routed experts' format."""
        super().__init__()
        assert model_dim % 2 == 0, 'Model_dim (%s) must be even value, while this Model_dim mod 2 > 0.' % model_dim
        if 'pad_samples' in kwargs:
            logging.warning('`pad_samples` option in Tutel Moe-layer has been deprecated, as Tutel always assumes `pad_samples=False` for better efficiency.')
            kwargs.pop('pad_samples')
        for k in kwargs:
            raise Exception('Unrecognized argument provided to Tutel Moe-layer: %s' % k)

        if group is None and dist.is_available() and dist.is_initialized():
            group = dist.group.WORLD
        self.group = group
        self.result_func = result_func
        self.skip_moe = int(os.environ.get('SKIP_MOE', '0')) != 0
        self.model_dim = model_dim
        self.world_size = C.get_world_size(self.group)

        experts = dict(experts or {})
        shared_spec = self._shared_spec(shared_experts, experts)
        local = experts.pop('count_per_node', None)
        local2 = experts.pop('num_experts_per_device', None)
        self.num_local_experts = local if local is not None else (local2 if local2 is not None else 1)
        if self.num_local_experts == -1:
            self.num_local_experts = 1
        self._n_global_experts = int(MOELayer.global_expert_count(self.num_local_experts, self.group))
        self.register_buffer('_num_global_experts', torch.tensor(self._n_global_experts))
        if self.num_global_experts < self.world_size:
            self.sharded_count = self.world_size // self.num_global_experts
            self.num_local_experts = 1
        else:
            self.sharded_count = 1

        self.auto_parallel, self.use_model_parallel = False, True
        self.valid_rs = [0] + [i for i in range(1, self.sharded_count + 1) if self.sharded_count % i == 0]
        self.adaptive_degree = _parse_parallel_type(parallel_type, self.sharded_count, self.valid_rs)

        self.is_postscore = is_postscore
        self.batch_prioritized_routing = batch_prioritized_routing or int(os.environ.get('BATCH_PRIO', 0)) != 0
        self.normalize_gate = normalize_gate
        self.is_gshard_loss = is_gshard_loss
        self.a2a_ffn_overlap_degree = a2a_ffn_overlap_degree
        self.use_2dh = use_2dh
        self.megablocks_size = 0
        self.dispatch_count = None
        self.protected_shape = None
        self.l_aux = None

        # ---- experts (RNG: seeds[1]) ----
        if seeds is not None and seeds[1] is not None:
            torch.manual_seed(seeds[1])
        self.experts = self._build_experts(dict(experts))
        if scan_expert_func is not None:
            for n, p in self.experts.named_parameters():
                scan_expert_func(n, p)
        for _, p in self.experts.named_parameters():
            setattr(p, '_tutel_expert', True)

        # ---- gates (RNG: seeds[0] + index) ----
        if isinstance(gate_type, str):
            assert re.match(r'^Top[0-9]+Gate$', gate_type), 'Unrecognized gate_type: %s' % gate_type
            top_k = int(gate_type[3:-4])
            logging.warning("gate_type value `%s` in Tutel Moe-layer has been deprecated, please use gate_type = {'type': 'top', 'k': %d} instead." % (gate_type, top_k))
            gate_type = {'type': 'top', 'k': top_k}
        gate_specs = gate_type if isinstance(gate_type, list) else [gate_type]
        gates = []
        for gi, spec in enumerate(gate_specs):
            spec = dict(spec)
            if seeds is not None and seeds[0] is not None:
                torch.manual_seed(seeds[0] + gi)
            gates.append(self._build_gate(spec))
        self.gates = ModuleList(gates)
        for gate in self.gates:
            if getattr(gate, 'scoring_func', 'softmax') == 'sigmoid':
                if not self.is_gshard_loss:
                    raise ValueError('is_gshard_loss=False is not supported with a sigmoid gate: the load-importance '
                                     'loss is defined on softmax scores')
                gate.balance_group = self.group

        # ---- shared experts (after the gates: the RNG stream of the experts and gates is unchanged; replicated
        # parameters, so with `seeds` they draw from the gates' stream, which is the same on every rank) ----
        self.shared_experts, self.shared_expert_gate = None, None
        if shared_spec is not None:
            spec = dict(experts, hidden_size_per_expert=experts['hidden_size_per_expert'] * shared_spec['num_experts'])
            if 'weight_format' in shared_spec:
                spec['weight_format'] = shared_spec['weight_format']
            self.shared_experts = self._build_experts(spec, num_experts_per_device=1, sharded_count=1)
            if shared_spec.get('gate', False):
                self.shared_expert_gate = torch.nn.Linear(model_dim, 1, bias=False)

        if seeds is not None and len(seeds) > 2 and seeds[2] is not None:
            torch.manual_seed(seeds[2])

    @staticmethod
    def _shared_spec(shared_experts, experts: dict):
        """Validated ``shared_experts`` option, or None."""
        if shared_experts is None:
            return None
        if not isinstance(shared_experts, dict):
            raise ValueError("shared_experts must be None or a dict like {'num_experts': 2, 'gate': False}")
        unknown = set(shared_experts) - {'num_experts', 'gate', 'weight_format'}
        if unknown:
            raise ValueError('Unrecognized shared_experts option(s): %s' % sorted(unknown))
        n = shared_experts.get('num_experts')
        if isinstance(n, bool) or not isinstance(n, int) or n < 1:
            raise ValueError('shared_experts: num_experts must be a positive int (got %r)' % (n,))
        kind = experts.get('type')
        if kind == 'custom':
            raise ValueError('shared_experts are not supported with custom experts: their hidden size cannot be derived')
        if kind not in ('ffn', 'llama_ffn'):
            raise ValueError("shared_experts need 'ffn' or 'llama_ffn' experts (got %r)" % (kind,))
        if 'hidden_size_per_expert' not in experts:
            raise ValueError('shared_experts need the routed experts\' hidden_size_per_expert')
        if 'weight_format' in shared_experts and shared_experts['weight_format'] not in (None, 'fp8_block', 'int4'):
            raise ValueError("shared_experts: weight_format must be None, 'fp8_block' or 'int4' (got %r)"
                             % (shared_experts['weight_format'],))
        return dict(shared_experts)

    def _build_experts(self, experts: dict, num_experts_per_device=None, sharded_count=None):
        kind = experts.pop('type')
        experts['model_dim'] = self.model_dim
        experts['num_experts_per_device'] = self.num_local_experts if num_experts_per_device is None else num_experts_per_device
        experts['sharded_count'] = self.sharded_count if sharded_count is None else sharded_count
        if kind == 'custom':
            factory = experts.pop('module')
        else:
            assert re.match(r'^[a-zA-Z0-9_]+$', kind), 'Expert type must only include digits, letters and underline characters.'
            try:
                factory = importlib.import_module('.experts.%s' % kind, __package__).ExpertModule
            except ModuleNotFoundError:
                raise Exception('Builtin expert type is not recognized: %s' % kind)
            if kind == 'ffn':
                assert 'fused_custom_fn' not in experts, '`fused_custom_fn` option for Tutel Moe-layer has been deprecated, please follows helloworld_from_scratch.py for custom construction instead.'
                assert 'implicit_dropout_p' not in experts, '`implicit_dropout_p` option for Tutel Moe-layer has been deprecated, please use torch.nn.Dropout(p=implicit_dropout_p) on custom activation_fn (for fc1_dropout) and after Tutel Moe-layer (for fc2_dropout) instead.'
        try:
            return factory(**experts)
        except TypeError as ex:
            if 'num_experts_per_device' not in str(ex):
                raise
            logging.warning('ExpertModule.__init__(.., local_experts, ..) has been deprecated, please rename `local_experts` to `num_experts_per_device` in init methods.')
            experts['local_experts'] = experts.pop('num_experts_per_device')
            return factory(**experts)

    def _build_gate(self, spec: dict):
        kind = spec.pop('type')
        assert re.match(r'^[a-zA-Z0-9_]+$', kind), 'Gate type must only include digits, letters and underline characters.'
        if kind == 'custom':
            factory = spec.pop('module')
        else:
            try:
                factory = importlib.import_module('.gates.%s' % kind, __package__).Gate
            except ModuleNotFoundError:
                raise Exception('Unrecognized gate_type: %s' % kind)
        gate = factory(model_dim=self.model_dim, num_global_experts=self.num_global_experts, **spec)
        if not hasattr(gate, 'gate_noise'):
            gate.gate_noise = spec.get('gate_noise', 0.0)
        if not hasattr(gate, 'capacity_factor'):
            gate.capacity_factor = spec.get('capacity_factor', float(os.environ.get('CAP_FACTOR', 1.0)))
        return gate

    def extra_repr(self):
        return 'Top-K(s) = %s, Total-Experts = %d [managed by %d device(s)],' % (
            ['k=%s, noise=%s' % (g.top_k, g.gate_noise) for g in self.gates], self.num_global_experts, self.world_size)

    def get_parameter_iterator(self, param_type):
        if param_type == 'gate':
            return self.gates.named_parameters()
        if param_type == 'local_experts':
            return self.experts.named_parameters()
        if param_type == 'shared_experts':
            mods = [m for m in (self.shared_experts, self.shared_expert_gate) if m is not None]
            return torch.nn.ModuleList(mods).named_parameters()
        raise Exception('Specified parameter type is not recognized: %s. Valid `param_type` includes: gate, local_experts, '
                        'shared_experts.' % param_type)

    # ------------------------------------------------------------------------------------------------- forward
    def expert_local(self, x, reserve_shape):
        y = self.experts(x.view(x.size(0), x.size(1), *reserve_shape), self)
        self.protected_shape = y.shape
        return y.reshape(y.size(0), y.size(1), -1)

    def _route(self, x, gctx, top_k, capacity_factor, a2a_ffn_overlap_degree, megablocks_size, inequivalent_tokens,
               packed=False):
        logits = gctx(x)
        if self.training and gctx.gate_noise > 0:
            logits_w_noise = logits + gctx.gate_noise * torch.randn_like(logits) / self.num_global_experts
        else:
            logits_w_noise = logits
        mega = max(megablocks_size, 1)
        alignment = (self.sharded_count * a2a_ffn_overlap_degree + mega - 1) // mega * mega
        if alignment > 256:
            alignment = (alignment + 127) // 128 * 128
        if getattr(gctx, 'scoring_func', 'softmax') == 'sigmoid':
            return self._route_sigmoid(x, logits, logits_w_noise, gctx, top_k, capacity_factor, alignment,
                                       megablocks_size, inequivalent_tokens, packed)
        fused_gate, gate_mode = None, fused_gate_mode()
        k_eff = min(top_k, self.num_global_experts)
        cuda_fused = (self.is_gshard_loss and gate_mode != 'off' and not self.batch_prioritized_routing and
                      fused_gate_route_available(logits_w_noise, k_eff))
        if cuda_fused or (self.is_gshard_loss and gate_mode == 'force' and logits_w_noise.dim() == 2):
            if cuda_fused:
                # CUDA: gate + routing in two launches, gate backward in one (ops/gating.py, csrc/gate_route.cu)
                cf = capacity_factor or gctx.capacity_factor
                bound = self._dropless_bound(logits_w_noise, x, cf, megablocks_size, inequivalent_tokens)
                crit, l_aux = fused_extract_critical(logits_w_noise, top_k, cf, self.normalize_gate, alignment, self.group,
                                                     inequivalent_tokens, rows_bound=bound, packed=packed)
                if getattr(crit, 'skip_padding', False) and not getattr(self.experts, 'rows_independent', False):
                    # experts that do not declare `rows_independent = True` may mix rows of the buffer: keep the zero padding
                    crit.skip_padding = False
                return logits.dtype, crit, l_aux
            # same formulas, op by op (CPU, batch-prioritised routing): one autograd node for softmax + top-k + loss
            fused_gate = fused_topk_gate(logits_w_noise, k_eff, self.normalize_gate, True)
            scores = logits_w_noise                # only its shape is read below
        else:
            scores = F.softmax(logits_w_noise, dim=1)
        if self.is_gshard_loss:
            loss_fn = losses.gshard_loss
        else:
            def loss_fn(gates, topk_ids):
                return losses.load_importance_loss(F.softmax(logits, dim=1), logits_w_noise.gather(index=topk_ids, dim=1),
                                                   self.num_global_experts, gctx.gate_noise)
        crit, l_aux = extract_critical(scores, top_k=top_k, loss_fn=loss_fn,
                                       capacity_factor=capacity_factor or gctx.capacity_factor,
                                       batch_prioritized_routing=self.batch_prioritized_routing,
                                       normalize_gate=self.normalize_gate, group=self.group, alignment=alignment,
                                       inequivalent_tokens=inequivalent_tokens, _fused=fused_gate, packed=packed)
        return logits.dtype, crit, l_aux

    def _dropless_bound(self, logits, x, cf, megablocks_size, inequivalent_tokens):
        """Single-GPU dropless inference: a worst-case row bound replaces the host read-back of the capacity."""
        if cf <= 0 and megablocks_size > 0 and self.world_size == 1 and not inequivalent_tokens:
            S = int(logits.size(0))
            budget = int(os.environ.get('TUTEL_B200_DROPLESS_BOUND_MB', 512)) << 20
            if S * self.num_global_experts * self.model_dim * x.element_size() <= budget:
                return S
        return 0

    def _route_sigmoid(self, x, logits, logits_w_noise, gctx, top_k, capacity_factor, alignment, megablocks_size,
                       inequivalent_tokens, packed=False):
        """Sigmoid scoring with the gate's selection bias and group limit (ops/gating.py).  Training forwards with
        gradients add their all-choice counts to the gate's ``expert_load`` for the next bias update."""
        k_eff = min(top_k, self.num_global_experts)
        gctx.check_top_k(k_eff)
        accumulate = gctx.balancing and gctx.training and torch.is_grad_enabled()
        load = gctx.expert_load if accumulate else None
        args = dict(bias=gctx.e_score_correction_bias, n_group=gctx.n_group, topk_group=gctx.topk_group,
                    scale=gctx.routed_scaling_factor)
        cf = capacity_factor or gctx.capacity_factor
        if (fused_gate_mode() != 'off' and not self.batch_prioritized_routing and
                sigmoid_gate_route_available(logits_w_noise, k_eff, gctx.n_group)):
            # CUDA: gate + routing in two launches (the loads are added inside the second), backward in one
            bound = self._dropless_bound(logits_w_noise, x, cf, megablocks_size, inequivalent_tokens)
            crit, l_aux = fused_extract_critical(logits_w_noise, top_k, cf, self.normalize_gate, alignment, self.group,
                                                 inequivalent_tokens, rows_bound=bound,
                                                 sigmoid=dict(args, expert_load=load), packed=packed)
            if getattr(crit, 'skip_padding', False) and not getattr(self.experts, 'rows_independent', False):
                crit.skip_padding = False
        else:
            idx, gates, l_aux, counts, top1 = sigmoid_topk_gate(logits_w_noise, k=k_eff, normalize=self.normalize_gate,
                                                                **args)
            if load is not None:
                load.add_(counts)
            crit, _ = extract_critical(logits_w_noise, top_k=top_k, loss_fn=None, capacity_factor=cf,
                                       batch_prioritized_routing=self.batch_prioritized_routing,
                                       normalize_gate=self.normalize_gate, group=self.group, alignment=alignment,
                                       inequivalent_tokens=inequivalent_tokens, _fused=(idx, gates, l_aux, top1),
                                       packed=packed)
        if accumulate:
            gctx.note_training_forward()
        return logits.dtype, crit, l_aux

    def update_expert_bias(self):
        """Apply the pending auxiliary-loss-free bias update of every sigmoid gate of this layer.  An optimizer-step
        post-hook does this after every ``torch.optim`` step; call it in loops that update parameters otherwise."""
        for gate in self.gates:
            if getattr(gate, 'scoring_func', 'softmax') == 'sigmoid':
                gate.update_bias()

    def forward(self, input: Tensor, gate_index=0, capacity_factor=None, top_k=None, a2a_ffn_overlap_degree=None,
                reserve_dims=1, inequivalent_tokens=False, adaptive_r=None, megablocks_size=0):
        if self.skip_moe:
            out = input
            out.l_aux = None
            return self.result_func(out) if self.result_func is not None else out
        if self.shared_experts is not None and reserve_dims != 1:
            raise ValueError('shared_experts need reserve_dims=1 (got %d): the shared experts run on [tokens, model_dim]'
                             % reserve_dims)

        # Let go of the previous call's auxiliary loss BEFORE building a new autograd graph: it is the one tensor of a step
        # that outlives it, and through it the gate weight's gradient accumulator - which remembers the stream it was
        # created on and would otherwise tie a step captured into a CUDA graph (utils/graph.py) to the eager warm-up stream.
        self.l_aux = None
        original_shape, original_dtype = input.shape, input.dtype
        assert len(original_shape) >= 2, 'Input data must be at least 2D tensor: (s)amples, .., (m)odel_dim'
        reserve_shape = original_shape[-reserve_dims:]
        x = input.reshape(-1, reserve_shape.numel())
        ac = _autocast_dtype(x)
        if ac is not None:
            x = x.to(ac)
        else:
            p = next(self.experts.parameters(), None)
            if p is not None:
                x = x.to(p.dtype)

        gctx = self.gates[gate_index]
        if a2a_ffn_overlap_degree is not None:
            self.a2a_ffn_overlap_degree = a2a_ffn_overlap_degree
        d = self.a2a_ffn_overlap_degree
        top_k = top_k or gctx.top_k
        if megablocks_size > 0 and (self.num_local_experts <= 1 or torch.is_grad_enabled() or self.world_size > 1):
            megablocks_size = 0
        packed = self._packed_eligible(x, gctx, capacity_factor, megablocks_size, reserve_dims)

        with stage('route'):
            if x.is_cuda or x.device.type == 'cpu':
                with torch.amp.autocast(x.device.type, enabled=False):
                    logits_dtype, crit, l_aux = self._route(x, gctx, top_k, capacity_factor, d, megablocks_size, inequivalent_tokens,
                                                            packed)
            else:
                logits_dtype, crit, l_aux = self._route(x, gctx, top_k, capacity_factor, d, megablocks_size, inequivalent_tokens,
                                                        packed)

        self.megablocks_size = megablocks_size
        self.dispatch_count = get_dispatch_count(crit)
        self.top_k = min(top_k, self.num_global_experts)      # choices per token of this call (experts size their paths by it)
        if adaptive_r is not None:
            self.adaptive_degree = adaptive_r

        x = x.contiguous()
        base, shared_logit = None, None
        if self.shared_experts is not None:
            with stage('shared'):
                base, shared_logit = self._shared_forward(x)
        y = None
        fused = None if packed else self._fused_engine(x, crit, d, reserve_dims)
        if packed:
            y = self._packed_forward(x, crit, base, shared_logit)
        elif fused is not None:
            with stage('fused'):
                y = fused.run(self, x, crit, base, shared_logit)
            self.protected_shape = y.shape
        else:
            with stage('encode'):
                y = fast_encode(x, crit, self.is_postscore)
            if self.adaptive_degree == 0:
                with stage('experts'):
                    y = self.expert_local(y, reserve_shape)
            else:
                sharded = self.num_global_experts < self.world_size
                if sharded:
                    if self.use_model_parallel:
                        y = y.repeat(1, self.adaptive_degree, 1).view(self.world_size, -1, y.size(2))
                    else:
                        y = y.view(self.world_size, -1, y.size(2))
                if d > 1 and (y.is_cuda or _OVERLAP_ON_CPU()):
                    with stage('overlap'):
                        y = a2a_ffn_overlap_forward(y, expert_fn=lambda t: self.expert_local(t, reserve_shape),
                                                    a2a_ffn_overlap_degree=d, use_2dh=self.use_2dh, group=self.group)
                else:
                    with stage('dispatch'):
                        y = C.all_to_all(y, 1, 0, use_2dh=self.use_2dh, group=self.group)
                    with stage('experts'):
                        y = self.expert_local(y, reserve_shape)
                    with stage('combine'):
                        y = C.all_to_all(y, 0, 1, use_2dh=self.use_2dh, group=self.group)
                if sharded:
                    if self.use_model_parallel:
                        y = torch.sum(y.view(self.num_global_experts, self.adaptive_degree, -1, y.size(2)), dim=1)
                    else:
                        y = y.view(self.num_global_experts, -1, y.size(2))
            with stage('decode'):
                y = fast_decode(y.contiguous(), crit, self.is_postscore, base, shared_logit)

        y = y.view(list(original_shape[:-reserve_dims]) + list(self.protected_shape[-reserve_dims:])).to(original_dtype)
        self.l_aux = y.l_aux = l_aux
        return self.result_func(y) if self.result_func is not None else y

    # ---------------------------------------------------------------------------------------- packed dropless
    def _packed_eligible(self, x, gctx, capacity_factor, megablocks_size, reserve_dims) -> bool:
        """Dropless training on one GPU runs on the expert-packed layout (ops/packed.py): every expert GEMM costs
        sum(count) rows instead of E * max(count), and nothing reads the counts back to the host.  Taken by forwards with
        gradients when the resolved capacity factor is exactly 0, on one GPU, outside bound-based dropless decoding
        (megablocks_size), with one reserved dim, 16-bit CUDA activations and experts that implement ``forward_packed``
        for them.  Inference forwards keep the padded and bound-based paths."""
        cf = capacity_factor or gctx.capacity_factor
        if not (cf == 0 and torch.is_grad_enabled() and self.world_size == 1 and megablocks_size == 0 and reserve_dims == 1 and x.is_cuda and
                x.dtype in (torch.float16, torch.bfloat16) and x.dim() == 2 and x.size(0) > 0):
            return False
        supports = getattr(self.experts, 'supports_packed', None)
        if not callable(getattr(self.experts, 'forward_packed', None)) or supports is None or not supports(x):
            return False
        from ..ops import backend
        return backend.has_cuda_ext()

    def _packed_forward(self, x, crit, base=None, shared_logit=None):
        from ..ops.dispatch import DispatchPlan, GatingDecoder, GatingEncoder
        plan = DispatchPlan.from_critical(crit)
        with stage('encode'):
            y = GatingEncoder.apply(plan, x, None if self.is_postscore else crit.gates_ks)
        with stage('experts'):
            y = self.experts.forward_packed(y, crit.layout, self)
        self.protected_shape = y.shape
        with stage('decode'):
            gates = crit.gates_ks if self.is_postscore else None
            if base is None:
                y = GatingDecoder.apply(plan, y, gates)
            else:
                y = GatingDecoder.apply(plan, y, gates, base, shared_logit)
        return y

    # ------------------------------------------------------------------------------------------------ shared experts
    def _shared_forward(self, x):
        """(shared experts' output [S, Mout], shared-gate logits [S] or None) for the tokens x [S, M].  The expert runs
        on x viewed as one expert's [1, S, M] block; no-grad forwards of up to 64 tokens on CUDA give it a device row
        count of S, so that it takes the dropless decoding kernels of its type (the weight-streaming skinny kernels)."""
        S = x.size(0)
        rows = _shared_rows(S, x.device) if (x.is_cuda and 0 < S <= 64 and not torch.is_grad_enabled()) else None
        base = self.shared_experts(x.view(1, S, x.size(1)), _SharedExpertContext(self, rows))
        base = base.reshape(S, -1)
        logit = None
        if self.shared_expert_gate is not None:
            w = self.shared_expert_gate.weight
            if x.is_cuda or x.device.type == 'cpu':           # the gate's rules (forward: _route runs without autocast)
                with torch.amp.autocast(x.device.type, enabled=False):
                    logit = F.linear(x.to(w.dtype), w)
            else:
                logit = F.linear(x.to(w.dtype), w)
            logit = logit.view(S)
        return base, logit

    # ------------------------------------------------------------------------------------------- fused engine
    def _fused_engine(self, x, crit, d, reserve_dims):
        """The NVLink-fused dispatch+GEMM / GEMM+combine engine, when this call is eligible for it."""
        if self.world_size <= 1 or not x.is_cuda or reserve_dims != 1:
            return None
        from ..parallel import fused
        return fused.engine_for(self, x, crit, d)


class _SharedExpertContext:
    """What an expert module reads from its layer, for the shared experts: one dense expert, not sharded, in this
    rank's replica.  ``rows`` (device int32 [1] or None) turns on the expert's dropless decoding path."""

    def __init__(self, layer: MOELayer, rows: Optional[Tensor]):
        self.group = layer.group
        self.model_dim = layer.model_dim
        self.num_global_experts = 1
        self.num_local_experts = 1
        self.sharded_count = 1
        self.adaptive_degree = 1
        self.top_k = 1
        self.megablocks_size = 1 if rows is not None else 0
        self.dispatch_count = rows


_SHARED_ROWS = {}


def _shared_rows(S: int, device) -> Tensor:
    """int32 [1] device tensor holding S (cached per device and S; not cached while a CUDA graph is being captured)."""
    key = (str(device), S)
    t = _SHARED_ROWS.get(key)
    if t is None:
        t = torch.full([1], S, dtype=torch.int32, device=device)
        if not torch.cuda.is_current_stream_capturing():
            _SHARED_ROWS[key] = t
    return t


moe_layer = MOELayer
