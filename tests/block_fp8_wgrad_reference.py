"""References for the block-fp8 weight gradients (``fp8_wgrad``), built on tests/block_fp8_reference.py.  Plain torch:
runs on the CPU or the GPU.

Dual quantiser (exact).  The row-wise half is ``block_fp8_reference.quantize_act``.  The column-wise half is ``x^T``
``[G, K, Rp]`` (``Rp = roundup(R, 128)``) with one scale per column of x and 128-row block over the block's real rows
only, ``[G, Rp/128, K]``, by the same scale rule; pad bytes are 0.

Weight-gradient GEMM (bounded).  Both operands are column-wise copies, so B, like A, has one scale per row and K step
(``sb [G, K/128, N]``, the layout of ``sa``) instead of one per 128 x 128 block.  The kernel promotes each K step with
``acc = fmaf(part, sa[m] * sb[n], acc)``, so the bound of ``block_fp8_reference.ref_gemm`` holds unchanged with
``S_kb = |sa[m] sb[n]| sum_{k in kb} |a_k b_k|``: C_BLOCK per block, two fp32 roundings per promotion, the bf16 output
rounding.
"""
import torch

import block_fp8_reference as R


def quantize_act_dual(x: torch.Tensor):
    """x [G, R, K] -> (bytes, s) of ``quantize_act`` and the column-wise copy (qT bytes uint8 [G, K, Rp], sT fp32
    [G, Rp/128, K])."""
    G, Rows, K = x.shape
    Rp = -(-Rows // R.TILE) * R.TILE
    q, s = R.quantize_act(x)
    qT = torch.zeros(G, K, Rp, dtype=torch.uint8, device=x.device)
    sT = torch.empty(G, Rp // R.TILE, K, dtype=torch.float32, device=x.device)
    for rb in range(Rp // R.TILE):
        blk = x[:, rb * R.TILE:min(Rows, (rb + 1) * R.TILE)]                             # [G, rows, K], real rows
        sc = R.scale_of(R._amax(blk, 1))                                                  # [G, K]
        sT[:, rb] = sc
        qT[:, :, rb * R.TILE:rb * R.TILE + blk.size(1)] = R._q(blk, sc.unsqueeze(1)).transpose(1, 2)
    return q, s, qT, sT


def ref_wgrad(aq, sa, bq, sb) -> R.Ref:
    """Reference of one ``block_fp8_wgrad_gemm`` launch (before any split): aq [G, M, K] + sa [G, K/128, M],
    bq [G, N, K] + sb [G, K/128, N]."""
    A, B = R.deq_act(aq, sa), R.deq_act(bq, sb)
    acc, S, other = R._plain(A, B)
    return R.Ref(acc, R.C_BLOCK * S + other, S, other)
