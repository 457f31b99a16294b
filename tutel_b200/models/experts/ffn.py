"""Batched two-layer feed-forward experts with optional hidden-dimension sharding.

Parameter names, shapes and initialisation order match the reference (tutel/experts/ffn.py:26-49) so that state
dicts, the re-sharding tools and the golden loss curves carry over:

    batched_fc1_w    [El, H/Sh, M]        batched_fc1_bias [El, H/Sh]
    batched_fc2_w    [El, H/Sh, Mout]     batched_fc2_bias [El, ceil(Mout/Sh)]

The compute path differs: on H100 both GEMMs (and their backward GEMMs) run on the wgmma grouped kernel with
bias/ReLU fused into the epilogue (:mod:`tutel_b200.ops.gemm`); the dropless "Megablocks" mode passes the per-expert
token counts to the kernel as a device tensor, so empty row tiles are skipped without the reference's host
synchronisation (tutel/custom/custom_kernel.cpp:874-889).
"""
import os

import torch
import torch.nn.functional as F

from ...ops import block_fp8 as BF8
from ...ops import gemm as G
from ...ops import mx as MX
from ...parallel import communicate as C
from . import dropless_row_counts


class FusedExpertsNetwork(torch.nn.Module):
    rows_independent = True      # each output row depends on its input row alone: dispatch may skip the zero padding

    def __init__(self, model_dim, hidden_size_per_expert, num_experts_per_device, sharded_count, activation_fn=None,
                 activation_fn_with_self=None, output_dim=None, has_fc1_bias=True, has_fc2_bias=True, fp8=None,
                 weight_format=None, fp8_wgrad=False, fp8_packed=False):
        super().__init__()
        if weight_format is not None:
            raise ValueError("ffn experts have no stored weight format (got weight_format=%r): the block-fp8 checkpoints "
                             "hold SwiGLU experts, use type 'llama_ffn'" % (weight_format,))
        self.skip_expert = int(os.environ.get('SKIP_EXPERT', '0')) != 0
        assert hidden_size_per_expert % sharded_count == 0, \
            "Can't evenly divide hidden_size_per_expert (%d) to %d slices." % (hidden_size_per_expert, sharded_count)
        self.model_dim = model_dim
        self.hidden_size_per_expert = hidden_size_per_expert
        self.local_experts = num_experts_per_device
        self.sharded_count = sharded_count
        self.hidden_size = hidden_size_per_expert // sharded_count
        self.output_dim = output_dim or model_dim
        # fp8=True / 'row' (or TUTEL_B200_FP8=1): forward and data-gradient expert GEMMs in e4m3 with per-row / per-channel
        # scales (also inside the fused engine).  fp8='mx' (TUTEL_B200_FP8=mx): OCP MX - e4m3 with one power-of-two scale
        # per 32 elements, applied by the tensor core (ops/mx.py, csrc/gemm_mx.cu); runs on the unfused path.
        # fp8='block' (TUTEL_B200_FP8=block): DeepSeek-V3 block scales - one fp32 scale per 1 x 128 activation tile and per
        # 128 x 128 weight block (ops/block_fp8.py, csrc/gemm_block_fp8.cu); ReLU experts, unfused path.
        mode = os.environ.get('TUTEL_B200_FP8', '0') if fp8 is None else fp8
        mode = str(mode).lower()
        assert mode in ('0', '1', 'true', 'false', 'none', 'row', 'mx', 'block'), \
            'fp8 must be a bool, "row", "mx" or "block" (got %r)' % (fp8,)
        self.fp8 = mode in ('1', 'true', 'row')
        self.mx = mode == 'mx'
        self.block = mode == 'block'
        # fp8_wgrad=True (with 'block' only): the weight-gradient GEMMs in block-scaled e4m3 too, on 128 x 1 token tiles
        # of the transposed activations; the backward keeps e4m3 x^T instead of bf16 x.  Outputs, dx and bias gradients
        # are those of fp8='block' bit for bit.
        if fp8_wgrad and not self.block:
            raise ValueError("fp8_wgrad=True needs fp8='block' (or TUTEL_B200_FP8=block); the resolved fp8 mode is %r" % (mode,))
        self.fp8_wgrad = bool(fp8_wgrad)

        if activation_fn_with_self is not None:
            assert activation_fn is None, 'Option `activation_fn_with_self` has been specified, please keep exactly one of them.'
            self.activation_fn = lambda x: activation_fn_with_self(x, self)
            self._act_kind = None
        else:
            self.activation_fn = activation_fn if activation_fn is not None else F.relu
            self._act_kind = G.classify_activation(self.activation_fn)
        # fp8_packed=True (with 'block' only): dropless training on one GPU runs the block-fp8 experts on the expert-packed
        # layout (ops/packed.py) instead of the padded one - no host read of the largest count, graph-capturable, and the
        # e4m3 GEMMs cover sum(roundup128(count)) rows instead of E * max(count).  An option for now: a follow-up may make
        # it the default for fp8='block' and delete it.
        if fp8_packed:
            if not self.block:
                raise ValueError("fp8_packed=True needs fp8='block' (or TUTEL_B200_FP8=block); the resolved fp8 mode is %r" % (mode,))
            if self._act_kind != 'relu':
                raise ValueError("fp8_packed=True: block-fp8 ffn experts run ReLU only; the activation here is %s"
                                 % (self._act_kind or 'custom',))
            if any(d % 128 for d in (model_dim, self.hidden_size, self.output_dim)):
                raise ValueError("fp8_packed=True needs model_dim, hidden_size_per_expert / sharded_count and output_dim "
                                 "to be multiples of 128 (got %d, %d, %d)" % (model_dim, self.hidden_size, self.output_dim))
        self.fp8_packed = bool(fp8_packed)

        El, Hs = num_experts_per_device, self.hidden_size
        self.batched_fc1_w = torch.nn.Parameter(torch.empty(El, Hs, model_dim))
        self.batched_fc2_w = torch.nn.Parameter(torch.empty(El, Hs, self.output_dim))
        if has_fc1_bias:
            self.batched_fc1_bias = torch.nn.Parameter(torch.empty(El, Hs))
        else:
            self.register_parameter('batched_fc1_bias', None)
        if has_fc2_bias:
            self.batched_fc2_bias = torch.nn.Parameter(torch.empty(El, (self.output_dim + sharded_count - 1) // sharded_count))
        else:
            self.register_parameter('batched_fc2_bias', None)
        self.reset_parameters()

    def reset_parameters(self):
        # Draw from the RNG in the same order as the reference (one fc1 then one fc2 Linear per local expert).
        with torch.no_grad():
            for i in range(self.local_experts):
                fc1 = torch.nn.Linear(self.model_dim, self.hidden_size, bias=self.batched_fc1_bias is not None)
                fc2 = torch.nn.Linear(self.hidden_size, self.output_dim, bias=self.batched_fc2_bias is not None)
                self.batched_fc1_w[i] = fc1.weight
                self.batched_fc2_w[i] = fc2.weight.t()
                if self.batched_fc1_bias is not None:
                    self.batched_fc1_bias[i] = fc1.bias
                if self.batched_fc2_bias is not None:
                    self.batched_fc2_bias[i] = fc2.bias[: self.batched_fc2_bias.size(-1)]

    def extra_repr(self):
        return 'model_dim=%d, hidden_size=%d, output_dim=%d, num_experts_per_device=%d. has_fc1_bias=%s, has_fc2_bias=%s.' % (
            self.batched_fc1_w.size(2), self.batched_fc1_w.size(1), self.batched_fc2_w.size(2), self.batched_fc1_w.size(0),
            self.batched_fc1_bias is not None, self.batched_fc2_bias is not None) + (' fp8_wgrad=True' if self.fp8_wgrad else '') + (
            ' fp8_packed=True' if self.fp8_packed else '')

    # ------------------------------------------------------------------------------------------------------------
    def materialize(self, ctx):
        """(w1, b1, w2, b2) for the layer's current parallel mode; biases come back as [G, n] or None.

        r = 0: every GPU gathers all experts (ZeRO-3 style, no all-to-all).  E < W: hidden slices are gathered over
        groups of Sh/r consecutive GPUs; the fc2 bias is gathered over all Sh sharers and scaled by 1/r because the
        r partial outputs are summed after the combine (reference: tutel/experts/ffn.py:83-112).
        """
        w1, w2, b1, b2 = self.batched_fc1_w, self.batched_fc2_w, self.batched_fc1_bias, self.batched_fc2_bias
        if ctx.adaptive_degree == 0:
            E = ctx.num_global_experts
            w1 = C.zero_gather(w1, group=ctx.group).view(E, -1, w1.size(2))
            w2 = C.zero_gather(w2, group=ctx.group).view(E, -1, w2.size(2))
            if b1 is not None:
                b1 = C.zero_gather(b1, group=ctx.group).view(E, -1)
            if b2 is not None:
                b2 = C.zero_gather(b2, group=ctx.group).view(E, -1)
        elif ctx.sharded_count > 1:
            mesh = C.get_world_size(ctx.group)
            if 1 < mesh < C.get_world_size():
                ctx.adaptive_degree = ctx.sharded_count
            group_size = ctx.sharded_count // ctx.adaptive_degree
            if group_size > 1:
                zero_group = C.create_groups_from_world(group_count=-group_size, parent_group=ctx.group).model_group
                w1 = C.zero_gather(w1, group=zero_group).view(1, -1, ctx.model_dim)
                w2 = C.zero_gather(w2, group=zero_group).view(1, -1, self.output_dim)
                if b1 is not None:
                    b1 = C.zero_gather(b1, group=zero_group).view(1, -1)
            if b2 is not None:
                sharers = C.create_groups_from_world(group_count=ctx.num_global_experts, parent_group=ctx.group).model_group
                b2 = C.zero_gather(b2, group=sharers).view(1, -1)
                if ctx.adaptive_degree > 1:
                    b2 = b2 * (1.0 / ctx.adaptive_degree)
        if b2 is not None and b2.size(-1) != self.output_dim:
            b2 = b2[:, : self.output_dim]
        return w1, b1, w2, b2

    def forward(self, x, ctx):
        if self.skip_expert:
            return x
        row_counts = dropless_row_counts(x, ctx)
        w1, b1, w2, b2 = self.materialize(ctx)
        return self.compute(x, w1, b1, w2, b2, row_counts)

    def supports_packed(self, x) -> bool:
        """The expert-packed layout (MOELayer's dropless path on one GPU) covers 16-bit ReLU / GELU / SiLU experts
        without fp8 / MX / block fp8, on weights of x's dtype, and with ``fp8_packed`` block-fp8 ReLU experts on bf16."""
        w1 = self.batched_fc1_w
        if self.block:
            return (self.fp8_packed and self._act_kind == 'relu' and x.is_cuda and x.dtype == torch.bfloat16 and
                    w1.dtype == x.dtype and self.sharded_count == 1 and
                    all(d % 128 == 0 for d in (self.model_dim, self.hidden_size, self.output_dim)))
        return (not self.fp8 and not self.mx and not self.block and self._act_kind in G.FWD_EPILOGUE and x.dtype in (torch.float16, torch.bfloat16)
                and w1.dtype == x.dtype and x.is_cuda and self.sharded_count == 1 and
                all(d % 8 == 0 for d in (self.model_dim, self.hidden_size, self.output_dim)))

    def forward_packed(self, x, layout, ctx):
        """x [R, M]: an expert-packed buffer (ops/packed.py) -> [R, Mout] in the same layout."""
        if self.skip_expert:
            return x
        w1, b1, w2, b2 = self.materialize(ctx)
        if self.block:
            return BF8.fused_relu_ffn_block_fp8(x, w1, b1, w2, b2, self.fp8_wgrad, layout=layout)
        return G.fused_act_ffn(x, w1, b1, w2, b2, None, self._act_kind, layout=layout)

    def compute(self, x, w1, b1, w2, b2, row_counts=None):
        lead = x.shape
        if x.dim() > 3:
            x = x.reshape(x.size(0), x.size(1), -1)
        if (row_counts is not None and self.fp8 and self._act_kind == 'relu' and
                G.can_use_skinny_ffn_fp8(x, w1, w2, self._act_kind)):
            # the same, streaming the cached e4m3 weight copies of the fp8 forward: half the bytes
            return G.skinny_ffn_fp8(x, w1, b1, w2, b2, row_counts, self._act_kind)
        if row_counts is not None and G.can_use_skinny_ffn(x, w1, w2, self._act_kind):
            # dropless decoder inference: a few tokens per expert -> ONE launch streams the active experts' weights once
            return G.skinny_ffn(x, w1, b1, w2, b2, row_counts, self._act_kind)
        if row_counts is not None and G.can_use_skinny(x, w1):
            relu = self._act_kind == 'relu'
            y = G.skinny_linear(x, w1, b1, 'nk', row_counts, relu=relu)
            if not relu:
                y = self.activation_fn(y)
            return G.skinny_linear(y, w2, b2, 'kn', row_counts)
        if self.mx and self._act_kind == 'relu' and row_counts is None and MX.can_use_mx(x, w1, w2):
            y = MX.fused_relu_ffn_mx(x, w1, b1, w2, b2)
        elif self.block and self._act_kind == 'relu' and row_counts is None and BF8.can_use_block_fp8(x, w1, w2):
            y = BF8.fused_relu_ffn_block_fp8(x, w1, b1, w2, b2, self.fp8_wgrad)
        elif self._act_kind in G.FWD_EPILOGUE and G.can_use_wgmma(x, w1) and G.can_use_wgmma(x, w2):
            if self.fp8 and self._act_kind == 'relu' and x.size(-1) % 16 == 0 and w1.size(1) % 16 == 0:
                y = G.fused_relu_ffn_fp8(x, w1, b1, w2, b2, row_counts)
            else:
                y = G.fused_act_ffn(x, w1, b1, w2, b2, row_counts, self._act_kind)
        else:
            y = G.grouped_linear(x, w1, b1, 'nk', row_counts)
            y = self.activation_fn(y)
            y = G.grouped_linear(y, w2, b2, 'kn', row_counts)
        if len(lead) > 3 and y.numel() == x.numel():
            y = y.view(lead)    # `reserve_dims > 1`: hand the trailing dims back in the caller's shape
        return y


ExpertModule = FusedExpertsNetwork
