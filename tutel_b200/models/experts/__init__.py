"""Built-in experts: ``ffn`` (2-layer, biases, hidden-dim sharding) and ``llama_ffn`` (SwiGLU, flat-sharded)."""
import torch


def dropless_row_counts(x, ctx):
    """Rows of each expert's block of ``x [E, rows, ...]`` that hold tokens in dropless ("Megablocks") inference, as a
    device int32 [E] tensor, or None outside that mode: the layer's ``dispatch_count`` rounded up to whole blocks of
    ``megablocks_size`` rows and clamped to the buffer.  No host synchronisation."""
    if getattr(ctx, 'megablocks_size', 0) <= 0:
        return None
    mb = ctx.megablocks_size
    if mb == 1 and ctx.dispatch_count.dtype == torch.int32:
        return ctx.dispatch_count          # the kernels clamp to the buffer's rows themselves: no extra launches
    groups = torch.div(ctx.dispatch_count + (mb - 1), mb, rounding_mode='floor')
    return (torch.clamp(groups, max=x.size(1) // mb) * mb).to(torch.int32)
