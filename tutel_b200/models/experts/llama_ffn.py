"""SwiGLU ("LLaMA") experts with flat-sharded parameters (reference: tutel/experts/llama_ffn.py:7-48).

Each of the three matrices is stored as one flat shard of ``ceil(El*M*H / Sh)`` elements per GPU and re-assembled
over the ``Sh`` sharers each forward (ZeRO-style; gradient = reduce-scatter).  The three GEMMs run on the wgmma
grouped kernel when the dtype allows.
"""
import torch

from ...ops import gemm as G
from ...parallel import communicate as C


class LlamaFFNNetwork(torch.nn.Module):
    def __init__(self, model_dim, hidden_size_per_expert, num_experts_per_device, sharded_count,
                 activation_fn=torch.nn.functional.silu, fp8=None):
        super().__init__()
        import os
        self.fp8 = bool(int(os.environ.get('TUTEL_B200_FP8', '0'))) if fp8 is None else bool(fp8)
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
        if kind in G.ACT_CODES and G.can_use_wgmma(x, w1) and w3.size(-1) % 8 == 0:
            # gate/up GEMMs + activation + multiply in one dual-B wgmma launch; backward without elementwise passes
            return G.fused_glu_ffn(x, w1, w2, w3, kind, self.fp8 and x.size(-1) % 16 == 0 and w3.size(1) % 16 == 0)
        y1 = G.grouped_linear(x, w1, None, 'kn', fp8=self.fp8)
        y2 = G.grouped_linear(x, w2, None, 'kn', fp8=self.fp8)
        return G.grouped_linear(self.activation_fn(y1) * y2, w3, None, 'kn', fp8=self.fp8)

    def extra_repr(self):
        return 'full shapes: %s, sharded_count=%d' % ({k: tuple(v) for k, v in self.full_shapes.items()}, self.sharded_count)


ExpertModule = LlamaFFNNetwork
