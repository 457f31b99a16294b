"""Expert-packed token layout for dropless training on one GPU.

The padded dispatch buffer ``[E, C, M]`` gives every expert the fullest expert's row count, and dropless routing must
read that count back to the host to size it.  The packed buffer ``[R, M]`` instead stores expert ``e``'s tokens in
rows ``[seg_off[e], seg_off[e] + count[e])``, in the same queue order as the locations of the padded layout.  Each
segment starts on a multiple of 128 rows (the grouped GEMM's row tile), so no row tile and no 64-row K block of a
weight gradient ever spans two experts; the rows between the end of one expert's tokens and the next segment are
padding, and every padding row of every packed tensor is exactly zero.

``R = roundup(k S, 128) + 128 E`` bounds ``sum_e roundup128(count[e]) <= k S + 127 E`` for any routing, so every buffer
shape is known on the host and nothing reads the counts back.  Blocks past ``seg_off[E]`` are never written or read.

This module is the only place that computes segment offsets; :class:`PackedLayout` carries them to routing (the slot
map of the encode), the expert GEMMs (block-mapped B and ragged-K launches, ops/gemm.py) and the decode.
"""
from __future__ import annotations

import torch

from . import backend

BLOCK = 128     # rows per segment alignment: the row tile of the grouped GEMM (csrc/gemm_sm90.cu, Cfg::BM)


def packed_rows(S: int, k: int, E: int) -> int:
    """Rows of a packed buffer for S tokens with k choices over E experts (a static bound, see the module docstring)."""
    return (k * S + BLOCK - 1) // BLOCK * BLOCK + BLOCK * E


class PackedLayout:
    """Device descriptors of one routing's packed layout (all int32, built by csrc/moe_kernels.cu: packed_layout):

    * ``seg_off [E + 1]``: 128-aligned exclusive scan of the counts (``seg_off[E]`` = rows in use);
    * ``block_expert [R / 128]``: the expert of each 128-row block (0 for blocks past ``seg_off[E]``);
    * ``block_rows [R / 128]``: valid rows of each block, 0 past ``seg_off[E]``;
    * ``slot_src [R]``: ``token * k + choice`` stored in each row, -1 for padding.
    """

    def __init__(self, E: int, k: int, S: int, counts: torch.Tensor, seg_off: torch.Tensor, block_expert: torch.Tensor,
                 block_rows: torch.Tensor, slot_src: torch.Tensor):
        self.E, self.k, self.S = int(E), int(k), int(S)
        self.R = int(slot_src.numel())
        self.counts = counts
        self.seg_off, self.block_expert, self.block_rows, self.slot_src = seg_off, block_expert, block_rows, slot_src

    @property
    def used_rows(self) -> torch.Tensor:
        """``seg_off[E:]`` - a one-element device view: rows of the buffer that any kernel reads or writes."""
        return self.seg_off[self.E:]

    @staticmethod
    def build(idx_ks: torch.Tensor, loc_ks: torch.Tensor, counts: torch.Tensor) -> 'PackedLayout':
        """From the routing's expert ids / queue locations ``[k, S]`` and device counts ``[E]``, with no host read."""
        if not (idx_ks.is_cuda and backend.has_cuda_ext()):
            raise RuntimeError('PackedLayout.build: the packed layout is built by a CUDA kernel; CUDA tensors and the '
                               'native extension are required')
        k, S = int(idx_ks.size(0)), int(idx_ks.size(1))
        E = int(counts.numel())
        R = packed_rows(S, k, E)
        backend.count_launch(3)          # layout, -1 fill of the slot map, scatter
        seg_off, block_expert, block_rows, slot_src = backend.require_ext().packed_layout(
            idx_ks.to(torch.int32).contiguous(), loc_ks.to(torch.int32).contiguous(), counts.to(torch.int32).contiguous(), R)
        return PackedLayout(E, k, S, counts, seg_off, block_expert, block_rows, slot_src)


def encode(x: torch.Tensor, gates, layout: PackedLayout) -> torch.Tensor:
    """x [S, M] -> packed [R, M]: row r = gate * x[token(r)] or zeros for padding (the slot-centric gather of the padded
    layout, run over the R rows of ``slot_src``; rows past ``seg_off[E]`` are not written)."""
    x = x.contiguous()
    out = torch.empty([layout.R, x.size(1)], dtype=x.dtype, device=x.device)
    g = None if gates is None else gates.to(torch.float32).contiguous()
    backend.count_launch()
    backend.require_ext().encode_rows(x, g, layout.slot_src, out, layout.k, 1, layout.R, 0, 0, 0, 0, 0, 0, layout.used_rows)
    return out


def decode(buf: torch.Tensor, gates, idx_ks: torch.Tensor, loc_ks: torch.Tensor, layout: PackedLayout, base=None,
           shared_logit=None) -> torch.Tensor:
    """packed [R, M] -> [S, M]: out[s] = sum_j gate_j[s] * buf[seg_off[idx_j[s]] + loc_j[s]]  (+ w_s * base[s], the shared
    experts' term of ops/dispatch.py: raw_decode)."""
    g = None if gates is None else gates.to(torch.float32).contiguous()
    backend.count_launch()
    if base is None:
        return backend.require_ext().decode_rows(buf.contiguous(), g, idx_ks, loc_ks, layout.E, layout.R, 0, 0, layout.seg_off)
    sl = None if shared_logit is None else shared_logit.to(torch.float32).contiguous().view(-1)
    return backend.require_ext().decode_rows(buf.contiguous(), g, idx_ks, loc_ks, layout.E, layout.R, 0, 0, layout.seg_off,
                                             base.contiguous(), sl)


def gate_grad(a: torch.Tensor, buf: torch.Tensor, idx_ks: torch.Tensor, loc_ks: torch.Tensor,
              layout: PackedLayout) -> torch.Tensor:
    """[k, S] fp32 row dots <a[s], buf[seg_off[idx_j[s]] + loc_j[s]]>."""
    backend.count_launch()
    return backend.require_ext().gate_grad(a.contiguous(), buf.contiguous(), idx_ks, loc_ks, layout.E, layout.R,
                                           layout.seg_off)


def segment_colsum(x: torch.Tensor, layout: PackedLayout) -> torch.Tensor:
    """[R, N] -> [E, N]: column sums of each expert's segment (bias gradients; padding rows are zero), in x's dtype."""
    backend.count_launch(3)          # zero-fill of the fp32 accumulator, the kernel, the cast
    return backend.require_ext().grouped_colsum(x.contiguous(), layout.seg_off)
