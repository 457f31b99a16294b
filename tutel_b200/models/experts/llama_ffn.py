"""SwiGLU ("LLaMA") experts with flat-sharded parameters (reference: tutel/experts/llama_ffn.py:7-48).

Each of the three matrices is stored as one flat shard of ``ceil(El*M*H / Sh)`` elements per GPU and re-assembled
over the ``Sh`` sharers each forward (ZeRO-style; gradient = reduce-scatter).  The three GEMMs run on the wgmma
grouped kernel when the dtype allows.  In dropless ("Megablocks") inference the per-expert token counts stay on the
device: up to 64 rows per expert the whole expert is one weight-streaming launch that reads only the active experts'
weights (csrc/skinny_gemm.cu), above that the wgmma kernels skip the rows past the counts.
"""
import torch

from ...ops import block_fp8 as BF8
from ...ops import gemm as G
from ...parallel import communicate as C
from . import dropless_row_counts


class LlamaFFNNetwork(torch.nn.Module):
    rows_independent = True      # each output row depends on its input row alone: dispatch may skip the zero padding

    def __init__(self, model_dim, hidden_size_per_expert, num_experts_per_device, sharded_count,
                 activation_fn=torch.nn.functional.silu, fp8=None):
        super().__init__()
        import os
        # fp8=True / 'row' (or TUTEL_B200_FP8=1 / true / row): e4m3 weights with per-row scales on every path, as in `ffn`.
        # fp8='block' (TUTEL_B200_FP8=block): DeepSeek-V3 block scales for the training GEMMs (ops/block_fp8.py); dropless
        # decoding keeps the 16-bit kernels.  OCP MX ('mx') has no SwiGLU kernel.
        mode = str(os.environ.get('TUTEL_B200_FP8', '0') if fp8 is None else fp8).lower()
        assert mode in ('0', '1', 'true', 'false', 'none', 'row', 'block'), \
            'llama_ffn: fp8 must be a bool, "row" or "block" (got %r); "mx" has no SwiGLU path' % (mode,)
        self.fp8 = mode in ('1', 'true', 'row')
        self.block = mode == 'block'
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

    def reset_parameters(self):
        with torch.no_grad():
            for name in ('W_fc1', 'W_fc2', 'W_fc3'):
                getattr(self, name).normal_(0, 0.01)

    def _full(self, name, parent_group):
        param, shape = getattr(self, name), self.full_shapes[name]
        group = C.create_groups_from_world(group_count=-self.sharded_count, parent_group=parent_group).model_group
        # zero_gather drops the padding of the last shard and reshapes; with one sharer it is a pure view of the
        # parameter (no copies in either direction)
        return C.zero_gather(param, full_shape=shape, group=group)

    def forward(self, x, ctx):
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
            return BF8.fused_glu_ffn_block_fp8(x, w1, w2, w3, kind)
        if kind in G.ACT_CODES and G.can_use_wgmma(x, w1) and w3.size(-1) % 8 == 0:
            # gate/up GEMMs + activation + multiply in one dual-B wgmma launch; backward without elementwise passes
            return G.fused_glu_ffn(x, w1, w2, w3, kind, self.fp8 and x.size(-1) % 16 == 0 and w3.size(1) % 16 == 0,
                                   row_counts)
        # rows are independent here, so rows past the counts cost time but never reach the result
        y1 = G.grouped_linear(x, w1, None, 'kn', fp8=self.fp8)
        y2 = G.grouped_linear(x, w2, None, 'kn', fp8=self.fp8)
        return G.grouped_linear(self.activation_fn(y1) * y2, w3, None, 'kn', fp8=self.fp8)

    def supports_packed(self, x) -> bool:
        """The expert-packed layout (MOELayer's dropless path on one GPU) covers 16-bit experts without fp8 or block fp8."""
        M, H = self.full_shapes['W_fc1'][1], self.full_shapes['W_fc1'][2]
        return (not self.fp8 and not self.block and x.dtype in (torch.float16, torch.bfloat16) and self.W_fc1.dtype == x.dtype and x.is_cuda and
                self.sharded_count == 1 and G.classify_activation(self.activation_fn) in G.ACT_CODES and
                M % 8 == 0 and H % 8 == 0)

    def forward_packed(self, x, layout, ctx):
        """x [R, M]: an expert-packed buffer (ops/packed.py) -> [R, M] in the same layout."""
        w1, w2, w3 = (self._full(n, ctx.group) for n in ('W_fc1', 'W_fc2', 'W_fc3'))
        return G.fused_glu_ffn(x, w1, w2, w3, G.classify_activation(self.activation_fn), False, None, layout=layout)

    def extra_repr(self):
        return 'full shapes: %s, sharded_count=%d' % ({k: tuple(v) for k, v in self.full_shapes.items()}, self.sharded_count)


ExpertModule = LlamaFFNNetwork
