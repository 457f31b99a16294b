"""Pure-torch reference of the expert-packed token layout (tutel_b200/ops/packed.py), written from its definition:

* expert e's rows are [seg_off[e], seg_off[e] + count[e]) in queue order (row seg_off[e] + loc holds the choice with
  location loc), segments start on multiples of 128 rows, ``R = roundup(k S, 128) + 128 E``;
* block b (rows [128 b, 128 b + 128)) belongs to the expert whose segment contains it, with
  ``min(128, seg_off[e] + count[e] - 128 b)`` valid rows, 0 past seg_off[E] (where the expert reads as 0);
* ``slot_src[r] = token * k + choice`` or -1; encode copies gate * x[token] into a row (zeros for padding), decode sums
  gate_j * buf[seg_off[idx_j] + loc_j] over the choices, gate gradients are the row dots with the same rows.
"""
from __future__ import annotations

import torch

BLOCK = 128


def packed_rows(S: int, k: int, E: int) -> int:
    return (k * S + BLOCK - 1) // BLOCK * BLOCK + BLOCK * E


def layout(idx_ks: torch.Tensor, loc_ks: torch.Tensor, counts: torch.Tensor, R: int):
    """(seg_off [E+1], block_expert [R/128], block_rows [R/128], slot_src [R]) as int32 CPU tensors."""
    idx, loc, counts = idx_ks.cpu().long(), loc_ks.cpu().long(), counts.cpu().long()
    E = counts.numel()
    k, S = idx.shape
    seg = [0]
    for e in range(E):
        seg.append(seg[-1] + (int(counts[e]) + BLOCK - 1) // BLOCK * BLOCK)
    assert seg[-1] <= R
    nb = R // BLOCK
    block_expert = torch.zeros(nb, dtype=torch.int32)
    block_rows = torch.zeros(nb, dtype=torch.int32)
    for e in range(E):
        for b in range(seg[e] // BLOCK, seg[e + 1] // BLOCK):
            block_expert[b] = e
            block_rows[b] = min(BLOCK, seg[e] + int(counts[e]) - b * BLOCK)
    slot = torch.full((R,), -1, dtype=torch.int32)
    for j in range(k):
        for s in range(S):
            e = int(idx[j, s])
            if 0 <= e < E:
                slot[seg[e] + int(loc[j, s])] = s * k + j
    return torch.tensor(seg, dtype=torch.int32), block_expert, block_rows, slot


def routing_from_counts(counts, k: int, S: int, seed: int = 0):
    """Expert ids / queue locations [k, S] (int32) whose per-expert totals are ``counts`` (sum(counts) == k S): each
    token's k choices are distinct experts when the counts allow it; locations follow the queue order of routing
    (all first choices in token order, then all second choices, ...)."""
    counts = [int(c) for c in counts]
    E = len(counts)
    assert sum(counts) == k * S
    g = torch.Generator().manual_seed(seed)
    pool = torch.cat([torch.full((c,), e, dtype=torch.long) for e, c in enumerate(counts)]) if sum(counts) else \
        torch.zeros(0, dtype=torch.long)
    pool = pool[torch.randperm(pool.numel(), generator=g)]
    idx = pool.view(k, S).clone()
    loc = torch.zeros_like(idx)
    seen = [0] * E
    for j in range(k):
        for s in range(S):
            e = int(idx[j, s])
            loc[j, s] = seen[e]
            seen[e] += 1
    return idx.to(torch.int32), loc.to(torch.int32)


def encode(x: torch.Tensor, gates, slot_src: torch.Tensor, k: int) -> torch.Tensor:
    """x [S, M] -> [R, M] (fp64): row r = gate * x[token] for slot_src[r] >= 0, else 0."""
    xs = x.cpu().double()
    slot = slot_src.cpu().long()
    out = torch.zeros(slot.numel(), xs.size(1), dtype=torch.float64)
    used = slot >= 0
    tok, j = slot[used] // k, slot[used] % k
    rows = xs[tok]
    if gates is not None:
        rows = rows * gates.cpu().double()[j, tok].unsqueeze(1)
    out[used] = rows
    return out


def rows_of(idx_ks, loc_ks, seg_off):
    """[k, S] packed row of each choice (int64), -1 for choices routed nowhere."""
    idx, loc, seg = idx_ks.cpu().long(), loc_ks.cpu().long(), seg_off.cpu().long()
    valid = idx >= 0
    return torch.where(valid, seg[idx.clamp_min(0)] + loc, torch.full_like(idx, -1))


def decode(buf: torch.Tensor, gates, idx_ks, loc_ks, seg_off) -> torch.Tensor:
    """buf [R, M] -> [S, M] (fp64), summing choices in order j = 0..k-1."""
    b = buf.cpu().double()
    rows = rows_of(idx_ks, loc_ks, seg_off)
    k, S = rows.shape
    out = torch.zeros(S, b.size(1), dtype=torch.float64)
    for j in range(k):
        w = (rows[j] >= 0).double()
        if gates is not None:
            w = w * gates.cpu().double()[j]
        out += b[rows[j].clamp_min(0)] * w.unsqueeze(1)
    return out


def gate_grad(a: torch.Tensor, buf: torch.Tensor, idx_ks, loc_ks, seg_off) -> torch.Tensor:
    """[k, S] fp64 row dots <a[s], buf[row_j(s)]> (0 for choices routed nowhere), and the bound sum_m |a| |buf|."""
    A, b = a.cpu().double(), buf.cpu().double()
    rows = rows_of(idx_ks, loc_ks, seg_off)
    val = torch.stack([(A * b[rows[j].clamp_min(0)]).sum(1) * (rows[j] >= 0).double() for j in range(rows.size(0))])
    mag = torch.stack([(A.abs() * b[rows[j].clamp_min(0)].abs()).sum(1) for j in range(rows.size(0))])
    return val, mag


def segment_colsum(x: torch.Tensor, seg_off: torch.Tensor):
    """[R, N] -> [E, N] fp64 column sums of each segment, and the same sums of |x|."""
    xs, seg = x.cpu().double(), seg_off.cpu().long()
    E = seg.numel() - 1
    val = torch.stack([xs[seg[e]:seg[e + 1]].sum(0) for e in range(E)])
    mag = torch.stack([xs[seg[e]:seg[e + 1]].abs().sum(0) for e in range(E)])
    return val, mag
