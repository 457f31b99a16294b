"""SwiGLU ("LLaMA") experts with flat-sharded parameters (reference: tutel/experts/llama_ffn.py:7-48).

Each of the three matrices is stored as one flat shard of ``ceil(El*M*H / Sh)`` elements per GPU and re-assembled
over the ``Sh`` sharers each forward (ZeRO-style; gradient = reduce-scatter).  The three GEMMs run on the wgmma
grouped kernel when the dtype allows.  In dropless ("Megablocks") inference the per-expert token counts stay on the
device: up to 64 rows per expert the whole expert is one weight-streaming launch that reads only the active experts'
weights (csrc/skinny_gemm.cu), above that the wgmma kernels skip the rows past the counts.

``weight_format='fp8_block'`` stores the experts as the block-scaled e4m3 checkpoints of DeepSeek-V3, Kimi-K2, GLM-4.5,
Moonlight and Qwen3-FP8 do, 1 byte per weight plus one fp32 scale per 128 x 128 block, with no 16-bit master copy and
no parameters: inference only (``load_fp8_block_weights``, doc/CHECKPOINT.md).

``weight_format='int4'`` stores them as group-32 int4 (W4A16, the routed experts of Kimi-K2-Thinking), half a byte per
weight plus one bf16 scale per 32 input elements, under the same rules (``load_int4_weights``, ops/int4.py, doc/INT4.md).
"""
import torch

from ...ops import block_fp8 as BF8
from ...ops import gemm as G
from ...ops import int4 as I4
from ...parallel import communicate as C
from . import dropless_row_counts


class LlamaFFNNetwork(torch.nn.Module):
    rows_independent = True      # each output row depends on its input row alone: dispatch may skip the zero padding
    # weight_format='fp8_block': the stored buffers, kept e4m3 / fp32 by _apply
    FP8_BLOCK_BUFFERS = ('W_gate_up', 'W_gate_up_scale', 'W_down', 'W_down_scale')
    # weight_format='int4': the same four buffers, nibbles uint8 / scales bf16, kept so by the same _apply
    INT4_BUFFERS = FP8_BLOCK_BUFFERS

    def __init__(self, model_dim, hidden_size_per_expert, num_experts_per_device, sharded_count,
                 activation_fn=torch.nn.functional.silu, fp8=None, weight_format=None, fp8_wgrad=False, fp8_packed=False):
        super().__init__()
        import os
        self.weight_format = weight_format
        self.fp8_wgrad = bool(fp8_wgrad)
        self.fp8_packed = bool(fp8_packed)
        if weight_format is not None:
            if fp8_wgrad:
                raise ValueError("llama_ffn: fp8_wgrad=True is a training option; weight_format=%r experts have no "
                                 "weight gradients" % (weight_format,))
            if fp8_packed:
                raise ValueError("llama_ffn: fp8_packed=True is a training option (the packed layout runs dropless training "
                                 "steps); weight_format=%r experts are inference-only" % (weight_format,))
            self._init_fp8_block(model_dim, hidden_size_per_expert, num_experts_per_device, sharded_count,
                                 activation_fn, fp8, weight_format)
            return
        # fp8=True / 'row' (or TUTEL_B200_FP8=1 / true / row): e4m3 weights with per-row scales on every path, as in `ffn`.
        # fp8='block' (TUTEL_B200_FP8=block): DeepSeek-V3 block scales for the training GEMMs (ops/block_fp8.py); dropless
        # decoding keeps the 16-bit kernels.  OCP MX ('mx') has no SwiGLU kernel.
        mode = str(os.environ.get('TUTEL_B200_FP8', '0') if fp8 is None else fp8).lower()
        assert mode in ('0', '1', 'true', 'false', 'none', 'row', 'block'), \
            'llama_ffn: fp8 must be a bool, "row" or "block" (got %r); "mx" has no SwiGLU path' % (mode,)
        self.fp8 = mode in ('1', 'true', 'row')
        self.block = mode == 'block'
        # fp8_wgrad=True (with 'block' only): the weight-gradient GEMMs in block-scaled e4m3 too; see ffn.py
        if fp8_wgrad and not self.block:
            raise ValueError("llama_ffn: fp8_wgrad=True needs fp8='block' (or TUTEL_B200_FP8=block); the resolved fp8 mode "
                             "is %r" % (mode,))
        # fp8_packed=True (with 'block' only): dropless training on one GPU on the expert-packed layout; see ffn.py.  A
        # follow-up may make it the default for fp8='block' and delete the option.
        if fp8_packed and not self.block:
            raise ValueError("llama_ffn: fp8_packed=True needs fp8='block' (or TUTEL_B200_FP8=block); the resolved fp8 mode "
                             "is %r" % (mode,))
        if fp8_packed and (model_dim % 128 or hidden_size_per_expert % 128):
            raise ValueError("llama_ffn: fp8_packed=True needs model_dim and hidden_size_per_expert to be multiples of 128 "
                             "(got %d, %d)" % (model_dim, hidden_size_per_expert))
        self.sharded_count = sharded_count
        self.full_shapes = {
            'W_fc1': torch.Size([num_experts_per_device, model_dim, hidden_size_per_expert]),
            'W_fc2': torch.Size([num_experts_per_device, model_dim, hidden_size_per_expert]),
            'W_fc3': torch.Size([num_experts_per_device, hidden_size_per_expert, model_dim]),
        }
        for name, shape in self.full_shapes.items():
            shard = (shape.numel() + sharded_count - 1) // sharded_count
            setattr(self, name, torch.nn.Parameter(torch.empty(shard)))
        self.W_fc1_full_shape, self.W_fc2_full_shape, self.W_fc3_full_shape = (
            self.full_shapes['W_fc1'], self.full_shapes['W_fc2'], self.full_shapes['W_fc3'])
        self.activation_fn = activation_fn
        self.reset_parameters()

    def _init_fp8_block(self, M, H, E, sharded_count, activation_fn, fp8, weight_format):
        # Stored block-fp8 experts: exactly what the block GEMM's forward reads, one copy per weight (ops/block_fp8.py):
        #   W_gate_up [E, 2H, M] e4m3 (W1^T and W2^T interleaved every 64 rows) + W_gate_up_scale [E, 2H / 64, M / 128],
        #   W_down [E, M, H] e4m3 (the checkpoint's down_proj.weight orientation) + W_down_scale [E, M / 128, H / 128].
        #   int4: W_gate_up [E, 2H, M / 2] uint8 nibbles (interleaved the same way) + W_gate_up_scale [E, 2H, M / 32] bf16,
        #   W_down [E, M, H / 2] uint8 + W_down_scale [E, M, H / 32] bf16 (ops/int4.py).
        if weight_format not in ('fp8_block', 'int4'):
            raise ValueError("llama_ffn: weight_format must be None, 'fp8_block' or 'int4' (got %r)" % (weight_format,))
        if M % 128 or H % 128:
            raise ValueError("llama_ffn: weight_format=%r needs model_dim and hidden_size_per_expert to be "
                             "multiples of 128 (got %d, %d)" % (weight_format, M, H))
        if sharded_count != 1:
            raise ValueError("llama_ffn: weight_format=%r keeps whole experts on each GPU (sharded_count must be "
                             "1, got %d): use at least as many experts as GPUs" % (weight_format, sharded_count))
        if weight_format == 'int4':
            if fp8 is not None:
                raise ValueError("llama_ffn: weight_format='int4' runs bf16 activations on int4 weights; fp8 must be unset "
                                 "(got %r)" % (fp8,))
            self.fp8, self.block, self.sharded_count = False, False, sharded_count
            self.activation_fn = activation_fn
            self.model_dim, self.hidden_size = M, H
            self.register_buffer('W_gate_up', torch.full((E, 2 * H, M // 2), 0x88, dtype=torch.uint8))
            self.register_buffer('W_gate_up_scale', torch.ones(E, 2 * H, M // 32, dtype=torch.bfloat16))
            self.register_buffer('W_down', torch.full((E, M, H // 2), 0x88, dtype=torch.uint8))
            self.register_buffer('W_down_scale', torch.ones(E, M, H // 32, dtype=torch.bfloat16))
            return
        if fp8 is not None and str(fp8).lower() != 'block':
            raise ValueError("llama_ffn: weight_format='fp8_block' runs the block-scaled kernels; fp8 must be unset or "
                             "'block' (got %r)" % (fp8,))
        self.fp8, self.block, self.sharded_count = False, True, sharded_count
        self.activation_fn = activation_fn
        self.model_dim, self.hidden_size = M, H
        e4m3 = torch.float8_e4m3fn
        self.register_buffer('W_gate_up', torch.zeros(E, 2 * H, M, dtype=e4m3))
        self.register_buffer('W_gate_up_scale', torch.ones(E, 2 * H // 64, M // 128, dtype=torch.float32))
        self.register_buffer('W_down', torch.zeros(E, M, H, dtype=e4m3))
        self.register_buffer('W_down_scale', torch.ones(E, M // 128, H // 128, dtype=torch.float32))

    def _apply(self, fn, recurse=True):
        # .bfloat16() / .half() / .to(dtype) would cast the e4m3, fp32 and bf16 buffers (torch treats e4m3 as a floating
        # dtype): they only follow device moves.  An empty probe tells where fn sends them without converting them.
        keep = {n: self._buffers.pop(n) for n in self.FP8_BLOCK_BUFFERS if n in self._buffers}
        try:
            super()._apply(fn, recurse)
        finally:
            for n, b in keep.items():
                probe = fn(b.new_empty(0))
                self._buffers[n] = fn(b) if probe.dtype == b.dtype else b.to(probe.device)
        return self

    @torch.no_grad()
    def load_fp8_block_weights(self, gate, gate_scale, up, up_scale, down, down_scale):
        """Load block-scaled e4m3 experts in the checkpoint orientation, stacked over this module's E experts:
        ``gate``, ``up`` e4m3 [E, H, M] with scales fp32 [E, H / 128, M / 128], ``down`` e4m3 [E, M, H] with scale fp32
        [E, M / 128, H / 128]; the scales are HF's ``weight_scale_inv`` (``w ~= q * s`` per 128 x 128 block)."""
        if self.weight_format != 'fp8_block':
            raise ValueError("load_fp8_block_weights needs weight_format='fp8_block'")
        qglu, sglu, q3t, s3t = BF8.load_glu_weights(gate, gate_scale, up, up_scale, down, down_scale)
        for name, t in zip(self.FP8_BLOCK_BUFFERS, (qglu, sglu, q3t, s3t)):
            buf = getattr(self, name)
            if t.shape != buf.shape:
                raise ValueError('load_fp8_block_weights: %s is %s for this module, the checkpoint gives %s'
                                 % (name, tuple(buf.shape), tuple(t.shape)))
            buf.copy_(t)

    @torch.no_grad()
    def load_int4_weights(self, gate, gate_scale, up, up_scale, down, down_scale):
        """Load group-32 int4 experts in the checkpoint orientation, stacked over this module's E experts: ``gate``,
        ``up`` int8 [E, H, M] with values in [-8, 7] and scales bf16 [E, H, M / 32], ``down`` int8 [E, M, H] with scale
        bf16 [E, M, H / 32] (``w = q * s`` per 32 input elements; ``ops.int4.unpack_int32`` unpacks compressed-tensors
        ``weight_packed``)."""
        if self.weight_format != 'int4':
            raise ValueError("load_int4_weights needs weight_format='int4'")
        stored = I4.load_glu_weights(gate, gate_scale, up, up_scale, down, down_scale)
        for name, t in zip(self.INT4_BUFFERS, stored):
            buf = getattr(self, name)
            if t.shape != buf.shape:
                raise ValueError('load_int4_weights: %s is %s for this module, the checkpoint gives %s'
                                 % (name, tuple(buf.shape), tuple(t.shape)))
            buf.copy_(t)

    def export_int4_weights(self):
        """The six checkpoint tensors of ``load_int4_weights`` (gate, gate_scale, up, up_scale, down, down_scale) for a
        16-bit layer with whole experts, by the quantiser rule of ops/int4.py."""
        if self.weight_format is not None or self.sharded_count != 1:
            raise ValueError('export_int4_weights needs a 16-bit layer with whole experts (sharded_count == 1)')
        w1, w2, w3 = (getattr(self, n).view(self.full_shapes[n]) for n in ('W_fc1', 'W_fc2', 'W_fc3'))
        return I4.export_glu_weights(w1, w2, w3)

    def export_fp8_block_weights(self):
        """The inverse of ``load_fp8_block_weights`` for a bf16 layer (e.g. trained with ``fp8='block'``): the six
        checkpoint tensors (gate, gate_scale, up, up_scale, down, down_scale) of its whole experts."""
        if self.weight_format is not None or self.sharded_count != 1:
            raise ValueError('export_fp8_block_weights needs a 16-bit layer with whole experts (sharded_count == 1)')
        w1, w2, w3 = (getattr(self, n).view(self.full_shapes[n]) for n in ('W_fc1', 'W_fc2', 'W_fc3'))
        return BF8.export_glu_weights(w1, w2, w3)

    def reset_parameters(self):
        if self.weight_format is not None:
            return
        with torch.no_grad():
            for name in ('W_fc1', 'W_fc2', 'W_fc3'):
                getattr(self, name).normal_(0, 0.01)

    def _full(self, name, parent_group):
        param, shape = getattr(self, name), self.full_shapes[name]
        group = C.create_groups_from_world(group_count=-self.sharded_count, parent_group=parent_group).model_group
        # zero_gather drops the padding of the last shard and reshapes; with one sharer it is a pure view of the
        # parameter (no copies in either direction)
        return C.zero_gather(param, full_shape=shape, group=group)

    def _forward_stored(self, x, ctx):
        fmt = self.weight_format
        if torch.is_grad_enabled() and x.requires_grad:
            raise RuntimeError("llama_ffn: weight_format=%r experts are inference-only (no master weights and no "
                               "data-gradient copy); run the forward under torch.no_grad() or torch.inference_mode()" % fmt)
        if getattr(ctx, 'adaptive_degree', 1) == 0 and C.get_world_size(getattr(ctx, 'group', None)) > 1:
            raise ValueError("llama_ffn: weight_format=%r experts stay local; adaptive_r=0 (which gathers the "
                             "expert weights on every GPU) is not supported" % fmt)
        if x.dim() > 3:
            x = x.reshape(x.size(0), x.size(1), -1)
        kind = G.classify_activation(self.activation_fn)
        if kind not in BF8.ACT_CODES:
            raise ValueError("llama_ffn: weight_format=%r supports SiLU, GELU and ReLU activations" % fmt)
        if not BF8.can_use_stored_glu(x):
            raise ValueError("llama_ffn: weight_format=%r runs on bf16 activations [E, rows, M] (got %s %s); "
                             "convert the input or run under bf16 autocast" % (fmt, x.dtype, tuple(x.shape)))
        qglu, sglu, q3t, s3t = (getattr(self, n) for n in self.FP8_BLOCK_BUFFERS)
        row_counts = dropless_row_counts(x, ctx)
        # the rule of the 16-bit experts: one launch that streams the active experts' bytes when the average expert fits
        # in one pass of its rows, the GEMMs (which read each weight once) otherwise
        decode = row_counts is not None and x.size(1) * getattr(ctx, 'top_k', 1) <= G.SKINNY_PASS_ROWS * x.size(0)
        if fmt == 'int4':
            if decode and I4.can_use_skinny_glu_ffn_int4(x):
                return I4.skinny_glu_ffn_int4(x, qglu, sglu, q3t, s3t, row_counts, kind)
            return I4.glu_ffn_int4(x, qglu, sglu, q3t, s3t, kind, row_counts)
        if decode and BF8.can_use_skinny_glu_ffn_block_fp8(x):
            return BF8.skinny_glu_ffn_block_fp8(x, qglu, sglu, q3t, s3t, row_counts, kind)
        return BF8.glu_ffn_block_fp8_stored(x, qglu, sglu, q3t, s3t, kind, row_counts)

    def forward(self, x, ctx):
        if self.weight_format is not None:
            return self._forward_stored(x, ctx)
        w1, w2, w3 = (self._full(n, ctx.group) for n in ('W_fc1', 'W_fc2', 'W_fc3'))
        if x.dim() > 3:
            x = x.reshape(x.size(0), x.size(1), -1)
        kind = G.classify_activation(self.activation_fn)
        row_counts = dropless_row_counts(x, ctx)
        # The skinny kernel re-streams an expert's weights for every SKINNY_PASS_ROWS of its rows; the wgmma kernel reads
        # them once.  Where both run, the skinny one is taken when the average expert fits in one pass (tokens * top-k
        # <= SKINNY_PASS_ROWS * experts): on an H100 80GB HBM3 (700 W), 8 rows per Mixtral-sized expert took 2.9 ms skinny,
        # 1.2 ms wgmma.
        if row_counts is not None and G.can_use_skinny_glu_ffn(x, w1, w2, w3, kind) and (
                not G.can_use_wgmma(x, w1) or x.size(1) * getattr(ctx, 'top_k', 1) <= G.SKINNY_PASS_ROWS * x.size(0)):
            # dropless decoder inference: a few tokens per expert -> ONE launch streams the active experts' weights once
            # (with fp8: the cached e4m3 copies the wgmma fp8 forward uses, half the bytes)
            if self.fp8 and G.can_use_skinny_glu_ffn_fp8(x, w1, w2, w3, kind):
                return G.skinny_glu_ffn_fp8(x, w1, w2, w3, row_counts, kind)
            return G.skinny_glu_ffn(x, w1, w2, w3, row_counts, kind)
        if self.block and row_counts is None and kind in BF8.ACT_CODES and BF8.can_use_block_fp8(x, w1, w2, w3):
            return BF8.fused_glu_ffn_block_fp8(x, w1, w2, w3, kind, self.fp8_wgrad)
        if kind in G.ACT_CODES and G.can_use_wgmma(x, w1) and w3.size(-1) % 8 == 0:
            # gate/up GEMMs + activation + multiply in one dual-B wgmma launch; backward without elementwise passes
            return G.fused_glu_ffn(x, w1, w2, w3, kind, self.fp8 and x.size(-1) % 16 == 0 and w3.size(1) % 16 == 0,
                                   row_counts)
        # rows are independent here, so rows past the counts cost time but never reach the result
        y1 = G.grouped_linear(x, w1, None, 'kn', fp8=self.fp8)
        y2 = G.grouped_linear(x, w2, None, 'kn', fp8=self.fp8)
        return G.grouped_linear(self.activation_fn(y1) * y2, w3, None, 'kn', fp8=self.fp8)

    def supports_packed(self, x) -> bool:
        """The expert-packed layout (MOELayer's dropless path on one GPU) covers 16-bit experts without fp8 or block fp8,
        and with ``fp8_packed`` block-fp8 experts on bf16."""
        if self.weight_format is not None:
            return False
        M, H = self.full_shapes['W_fc1'][1], self.full_shapes['W_fc1'][2]
        if self.block:
            return (self.fp8_packed and x.is_cuda and x.dtype == torch.bfloat16 and self.W_fc1.dtype == x.dtype and
                    self.sharded_count == 1 and G.classify_activation(self.activation_fn) in BF8.ACT_CODES and
                    M % 128 == 0 and H % 128 == 0)
        return (not self.fp8 and not self.block and x.dtype in (torch.float16, torch.bfloat16) and self.W_fc1.dtype == x.dtype and x.is_cuda and
                self.sharded_count == 1 and G.classify_activation(self.activation_fn) in G.ACT_CODES and
                M % 8 == 0 and H % 8 == 0)

    def forward_packed(self, x, layout, ctx):
        """x [R, M]: an expert-packed buffer (ops/packed.py) -> [R, M] in the same layout."""
        w1, w2, w3 = (self._full(n, ctx.group) for n in ('W_fc1', 'W_fc2', 'W_fc3'))
        kind = G.classify_activation(self.activation_fn)
        if self.block:
            return BF8.fused_glu_ffn_block_fp8(x, w1, w2, w3, kind, self.fp8_wgrad, layout=layout)
        return G.fused_glu_ffn(x, w1, w2, w3, kind, False, None, layout=layout)

    def extra_repr(self):
        if self.weight_format is not None:
            return "weight_format=%r, %d experts, model_dim=%d, hidden=%d" % (
                self.weight_format, self.W_down.size(0), self.model_dim, self.hidden_size)
        return 'full shapes: %s, sharded_count=%d' % ({k: tuple(v) for k, v in self.full_shapes.items()}, self.sharded_count) + (
            ', fp8_wgrad=True' if self.fp8_wgrad else '') + (', fp8_packed=True' if self.fp8_packed else '')


ExpertModule = LlamaFFNNetwork
