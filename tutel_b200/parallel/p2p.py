"""NVLink peer-to-peer transport: symmetric heap + in-kernel collectives.

This is the H100-native counterpart of the reference's private NCCL communicators and grouped ``ncclSend/ncclRecv``
all-to-alls (tutel/custom/custom_kernel.cpp:327-518).  Every rank owns an arena (``_C.SymmHeap``, CUDA IPC mapped into
all peers on the node); collectives are single kernels that *store* into the destination GPU's arena over NVLink and
publish completion with ``red.release.sys`` counters (csrc/p2p_kernels.cu).  ``torch.distributed`` is only used to
exchange the IPC handles.

Layout of the arena::

    [0, 4 MiB)                        counters: [0,16K) 64 slots x 4 arrays (ready / done / barrier / scratch),
                                      [16K, 4M) per-layer MoE arrival flags
    [4 MiB, 4 MiB + stage_bytes)      staging region shared by the generic collectives below
    [.. , heap_bytes)                 bump-allocated persistent buffers (MoE dispatch / combine buffers)
"""
from __future__ import annotations

import logging
import os
import socket
from typing import Dict, List, Optional, Sequence

import torch
import torch.distributed as dist

from ..ops import backend

_CTRL_BYTES = 4 << 20
_TRANSPORTS: Dict[int, Optional['P2PTransport']] = {}
_MAX_PEERS = 16


def _group_key(group) -> int:
    return 0 if group is None or group is dist.group.WORLD else id(group)


def _env_mode() -> str:
    return os.environ.get('TUTEL_B200_COMM', 'p2p').lower()


def transport_for(group) -> Optional['P2PTransport']:
    """Return the P2P transport of ``group`` (created collectively on first use) or None if NCCL must be used."""
    if _env_mode() in ('nccl', 'off', '0'):       # evaluated per call: tests and benchmarks switch transports at run time
        return None
    key = _group_key(group)
    if key in _TRANSPORTS:
        return _TRANSPORTS[key]
    t = None
    try:
        t = _create(group)
    except Exception as ex:  # noqa
        logging.warning('tutel_b200: P2P transport unavailable (%s); falling back to NCCL', ex)
        t = None
    _TRANSPORTS[key] = t
    return t


def _create(group) -> Optional['P2PTransport']:
    if _env_mode() in ('nccl', 'off', '0') or not backend.has_cuda_ext():
        return None
    if not (dist.is_available() and dist.is_initialized()):
        return None
    world = dist.get_world_size(group)
    if world <= 1 or world > _MAX_PEERS:
        return None
    if dist.get_backend(group) != 'nccl':
        return None
    # single NVLink domain check: same host, distinct devices, peer access possible
    me = (socket.gethostname(), torch.cuda.current_device())
    everyone = [None] * world
    dist.all_gather_object(everyone, me, group=group)
    ok = len({h for h, _ in everyone}) == 1 and len({d for _, d in everyone}) == world
    if ok:
        cur = torch.cuda.current_device()
        ok = all(d == cur or torch.cuda.can_device_access_peer(cur, d) for _, d in everyone)
    flags = [None] * world
    dist.all_gather_object(flags, bool(ok), group=group)
    if not all(flags):
        return None
    return P2PTransport(group)


class P2PTransport:
    def __init__(self, group):
        from .. import _C
        self.group = group
        self.rank = dist.get_rank(group)
        self.world = dist.get_world_size(group)
        self.device = torch.cuda.current_device()
        # The whole-world transport carries the fused MoE buffers (TUTEL_B200_HEAP_MB); sub-groups (model / data groups of
        # `create_groups_from_world`, ZeRO sharers, the two phases of the hierarchical all-to-all) get their own, smaller
        # arena, exchanged among the members only (TUTEL_B200_SUBHEAP_MB).
        self.is_world = group is None or group is dist.group.WORLD or self.world == dist.get_world_size()
        if self.is_world:
            heap_mb = int(os.environ.get('TUTEL_B200_HEAP_MB', 8192))
            stage_mb = int(os.environ.get('TUTEL_B200_STAGE_MB', 2048))
        else:
            heap_mb = int(os.environ.get('TUTEL_B200_SUBHEAP_MB', 1536))
            stage_mb = int(os.environ.get('TUTEL_B200_SUBSTAGE_MB', 1024))
        self.heap_bytes = heap_mb << 20
        self.stage_off = _CTRL_BYTES
        self.stage_bytes = min(stage_mb << 20, self.heap_bytes // 2)
        self._bump = self.stage_off + self.stage_bytes
        # staging = [bounce region for reductions / pool overflow | receive-buffer pool of the push collectives]
        self.bounce_bytes = self.stage_bytes // 4
        self.heap = _C.SymmHeap(self.heap_bytes, self.device)
        handles = [None] * self.world
        dist.all_gather_object(handles, self.heap.ipc_handle(), group=group)
        self.heap.open_peers(self.rank, handles)
        dist.barrier(group=group)
        self.peer_table = self.heap.peer_table_ptr()
        self.heap.set_pool(self.stage_off + self.bounce_bytes, self.stage_bytes - self.bounce_bytes)
        self._C = _C
        # counter slots (512 B each): mailboxes uint64[16] at +0, done uint32[16] at +128, barrier at +192, local scratch
        # at +256
        self._epochs: Dict[int, int] = {}
        self._fault = self._parse_fault(os.environ.get('TUTEL_B200_FAULT', ''))
        self._fault_calls = 0
        self._named: Dict[str, tuple] = {}
        self._next_slot = 2  # slot 0: generic push, slot 1: generic barrier/reduce
        # one-shot all-reduce: inbox 2 (parity) x W slots of _ONESHOT_BYTES, one flag per (parity, source, block)
        self._oneshot_inbox = self.alloc('__oneshot_inbox__', 2 * self.world * self._ONESHOT_BYTES)
        self._oneshot_flags = self.ctrl_alloc('__oneshot_flags__', 2 * self.world * int(_C.p2p_oneshot_max_blocks()) * 4)
        self._oneshot_epoch = 0
        # bound of every spin-wait in the kernels (a rank may legitimately be late: data loading, checkpointing)
        _C.set_spin_timeout(float(os.environ.get('TUTEL_B200_SPIN_TIMEOUT_SEC', 300)))

    # ---- fault injection (SURVEY 5.3: a dead peer must produce a diagnostic, not a hang) --------------------------
    def _parse_fault(self, spec: str):
        """``TUTEL_B200_FAULT=skip_push:rank=<r>:call=<n>``: rank r silently skips its n-th push collective (1-based)."""
        if not spec.startswith('skip_push'):
            return None
        opts = dict(kv.split('=') for kv in spec.split(':')[1:] if '=' in kv)
        if int(opts.get('rank', -1)) != self.rank:
            return None
        return int(opts.get('call', 1))

    def _fault_fires(self) -> bool:
        self._fault_calls += 1
        return self._fault_calls == self._fault

    # ---- arena management -------------------------------------------------------------------------------------
    def alloc(self, name: str, nbytes: int, align: int = 1024) -> int:
        """Persistent, collectively-called allocation; the same name returns the same offset (size may not grow)."""
        if name in self._named:
            off, size = self._named[name]
            if nbytes <= size:
                return off
            raise RuntimeError('tutel_b200 symmetric buffer %s cannot grow from %d to %d bytes' % (name, size, nbytes))
        off = (self._bump + align - 1) // align * align
        if off + nbytes > self.heap_bytes:
            raise RuntimeError('tutel_b200 symmetric heap exhausted (%d MiB); raise TUTEL_B200_HEAP_MB' % (self.heap_bytes >> 20))
        self._bump = off + nbytes
        self._named[name] = (off, nbytes)
        return off

    def can_alloc(self, nbytes: int, align: int = 1024) -> bool:
        return (self._bump + align - 1) // align * align + nbytes <= self.heap_bytes

    def new_counter_slot(self) -> int:
        s = self._next_slot
        self._next_slot += 1
        if 512 * (s + 1) > 16 << 10:
            raise RuntimeError('tutel_b200: out of counter slots')
        return s

    def ctrl_alloc(self, name: str, nbytes: int) -> int:
        """Zero-initialised counter storage inside the control area [16 KiB, 4 MiB)."""
        key = '__ctrl__' + name
        if key in self._named:
            return self._named[key][0]
        cur = getattr(self, '_ctrl_bump', 16 << 10)
        off = (cur + 127) // 128 * 128
        if off + nbytes > _CTRL_BYTES:
            raise RuntimeError('tutel_b200: control area exhausted')
        self._ctrl_bump = off + nbytes
        self._named[key] = (off, nbytes)
        return off

    def view(self, off: int, shape: Sequence[int], dtype: torch.dtype, rank: Optional[int] = None) -> torch.Tensor:
        r = self.rank if rank is None else rank
        return self.heap.tensor(r, off, list(shape), dtype, self.device)

    def owns(self, tensor: torch.Tensor) -> bool:
        """True when `tensor` lives inside this rank's arena (e.g. a zero-copy view of the staging region)."""
        base = self.heap.base_ptr(self.rank)
        return base <= tensor.data_ptr() < base + self.heap_bytes

    def base_ptr(self, rank: int) -> int:
        return self.heap.base_ptr(rank)

    def _next_epoch(self, slot: int) -> int:
        e = self._epochs.get(slot, 0) + 1
        self._epochs[slot] = e
        return e

    # ---- primitives -----------------------------------------------------------------------------------------
    def barrier(self, slot: int = 1) -> None:
        self._C.p2p_barrier(self.peer_table, 512 * slot + 192, self.rank, self.world, self._next_epoch(('b', slot)))

    def _blocks_per_peer(self, max_bytes: int) -> int:
        if max_bytes <= (64 << 10):
            return 1
        if max_bytes <= (1 << 20):
            return 4
        return max(8, min(74, 592 // self.world))     # ~4 CTAs per SM in total: enough bytes in flight for NVLink

    def collective(self, src: torch.Tensor, src_off: List[int], dst_off: List[int], nbytes: List[int], out_shape,
                   slot: int = 0) -> torch.Tensor:
        """Push-based collective with a zero-copy result: the receive buffer is taken from the arena pool, announced
        to the peers per call, and returned as a tensor (freed back to the pool when the tensor dies)."""
        if self._fault is not None and self._fault_fires():
            # fault injection (tests of the bounded-wait diagnostics): this rank "dies" for one collective - it neither
            # announces a receive buffer nor pushes, so the peers' kernels hit their spin timeout and report it
            return torch.zeros(list(out_shape), dtype=src.dtype, device=src.device)
        side = slot != 0 and slot == getattr(self, '_side_slot', None)
        blocks = self._blocks_per_peer(max(nbytes))
        if side:    # runs next to an expert GEMM: 128-thread blocks that co-reside with its CTAs, more of them instead
            blocks = min(4 * blocks, max(8, 1184 // self.world))
        return self._C.p2p_collective(self.heap, src, src_off, dst_off, nbytes, list(out_shape), 512 * slot,
                                      self._next_epoch(slot), blocks, self.stage_off, self.bounce_bytes, side)

    # ---- generic collectives (staging region; results are copied out so that callers may keep them) -------------
    def fits(self, nbytes: int) -> bool:
        # a rank whose pool is momentarily full receives into the bounce region (and copies out), so the size test
        # that every rank evaluates identically is against the bounce region
        return nbytes <= self.bounce_bytes

    def side_slot(self) -> int:
        """Counter slot (mailboxes / done counters / epoch sequence) reserved for collectives issued on a side stream
        (parallel/overlap.py): kernels sharing a slot must be serialised on one stream, and main-stream collectives
        (e.g. a `zero_gather` inside the expert function) may run while chunk exchanges are in flight."""
        if getattr(self, '_side_slot', None) is None:
            self._side_slot = self.new_counter_slot()
        return self._side_slot

    def all_to_all(self, x: torch.Tensor, copy: bool = True, slot: int = 0) -> torch.Tensor:
        nbytes = x.numel() * x.element_size()
        if not self.fits(nbytes) or nbytes % self.world:
            out = torch.empty_like(x)
            dist.all_to_all_single(out, x, group=self.group)
            return out
        chunk = nbytes // self.world
        return self.collective(x, [p * chunk for p in range(self.world)], [self.rank * chunk] * self.world,
                               [chunk] * self.world, x.shape, slot=slot)

    def all_gather(self, x: torch.Tensor) -> torch.Tensor:
        nbytes = x.numel() * x.element_size()
        if not self.fits(nbytes * self.world):
            out = torch.empty([self.world * x.numel()], device=x.device, dtype=x.dtype)
            dist.all_gather_into_tensor(out, x.view(-1), group=self.group)
            return out
        return self.collective(x, [0] * self.world, [self.rank * nbytes] * self.world, [nbytes] * self.world,
                               [self.world * x.numel()])

    def all_gather_v(self, x: torch.Tensor, sizes: List[int]) -> torch.Tensor:
        es = x.element_size()
        total = sum(sizes) * es
        if not self.fits(total):
            width = max(sizes)
            padded = torch.zeros([width], dtype=x.dtype, device=x.device)
            padded[: x.numel()] = x
            pieces = [torch.empty([width], dtype=x.dtype, device=x.device) for _ in sizes]
            dist.all_gather(pieces, padded, group=self.group)
            return torch.cat([p[:n] for p, n in zip(pieces, sizes)])
        my_off = sum(sizes[: self.rank]) * es
        n = sizes[self.rank] * es
        return self.collective(x, [0] * self.world, [my_off] * self.world, [n] * self.world, [sum(sizes)])

    def all_to_all_v(self, x: torch.Tensor, matrix: List[List[int]]) -> torch.Tensor:
        """``matrix[s][d]`` = elements rank s sends to rank d (known to every rank)."""
        es = x.element_size()
        in_list = matrix[self.rank]
        out_list = [matrix[s][self.rank] for s in range(self.world)]
        worst = max(sum(matrix[s][d] for s in range(self.world)) for d in range(self.world)) * es
        if not self.fits(worst):
            out = torch.empty([sum(out_list)], dtype=x.dtype, device=x.device)
            dist.all_to_all_single(out, x[: sum(in_list)], output_split_sizes=out_list, input_split_sizes=in_list,
                                   group=self.group)
            return out
        src_off, acc = [], 0
        for n in in_list:
            src_off.append(acc * es)
            acc += n
        dst_off = [sum(matrix[s][d] for s in range(self.rank)) * es for d in range(self.world)]
        return self.collective(x, src_off, dst_off, [n * es for n in in_list], [sum(out_list)])

    # ---- reductions ---------------------------------------------------------------------------------------------
    # <= _ONESHOT_BYTES: ONE kernel (push to every peer's inbox + flags + local reduce in rank order, ~1 NVLink round trip);
    # up to _REDUCE_MAX_BYTES: stage + barrier + pull-reduce + barrier.
    _ONESHOT_BYTES = 256 << 10      # inbox slot size
    _ONESHOT_LIMIT = 128 << 10      # measured cross-over with NCCL at 8 GPUs (64 KiB: 25 vs 28 us; 256 KiB: 34 vs 29 us)
    _REDUCE_MAX_BYTES = 4 << 20     # reduce-scatter through the staging region; must stay below bounce_bytes
    _ONESHOT_DTYPES = (torch.float32, torch.float16, torch.bfloat16, torch.int32, torch.int64)

    def supports_oneshot(self, x: torch.Tensor, op) -> bool:
        return (x.dtype in self._ONESHOT_DTYPES and op in (dist.ReduceOp.SUM, dist.ReduceOp.MAX) and
                0 < x.numel() * x.element_size() <= self._ONESHOT_LIMIT)

    def supports_reduce(self, x: torch.Tensor, op) -> bool:
        """All-reduce: the one-launch kernel up to _ONESHOT_LIMIT; beyond it NCCL (in-switch reduction) is at least as fast."""
        return self.supports_oneshot(x, op)

    def supports_reduce_scatter(self, x: torch.Tensor, op) -> bool:
        return (x.dtype in (torch.float32, torch.float16, torch.bfloat16) and op in (dist.ReduceOp.SUM, dist.ReduceOp.MAX)
                and x.numel() * x.element_size() <= self._REDUCE_MAX_BYTES and x.numel() > 0)

    def _stage(self, x: torch.Tensor) -> None:
        self.view(self.stage_off, [x.numel()], x.dtype).copy_(x.reshape(-1))

    def all_reduce(self, x: torch.Tensor, op=dist.ReduceOp.SUM, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Out-of-place all-reduce of a contiguous tensor (``out`` may be ``x`` itself)."""
        if out is None:
            out = torch.empty_like(x, memory_format=torch.contiguous_format)
        if self.supports_oneshot(x, op):
            if self._fault is not None and self._fault_fires():
                return out.copy_(x) if out is not x else out     # fault injection: this rank skips the collective
            src = x if x.is_contiguous() else x.contiguous()
            self._oneshot_epoch += 1
            backend.count_launch()
            self._C.p2p_allreduce_oneshot(src, out, self.peer_table, self._oneshot_inbox, self._ONESHOT_BYTES,
                                          self._oneshot_flags, self.rank, self.world, self._oneshot_epoch,
                                          op == dist.ReduceOp.MAX)
            return out
        self._stage(x)
        self.barrier()
        self._C.p2p_reduce_slice(out, self.peer_table, self.stage_off, 0, self.rank, self.world, op == dist.ReduceOp.MAX)
        self.barrier()
        return out

    def all_reduce_(self, x: torch.Tensor, op=dist.ReduceOp.SUM) -> torch.Tensor:
        if x.is_contiguous():
            return self.all_reduce(x, op, out=x)
        x.copy_(self.all_reduce(x.contiguous(), op))
        return x

    def reduce_scatter(self, x: torch.Tensor, op=dist.ReduceOp.SUM) -> torch.Tensor:
        self._stage(x)
        self.barrier()
        n = x.numel() // self.world
        out = torch.empty_like(x[: x.size(0) // self.world])
        self._C.p2p_reduce_slice(out, self.peer_table, self.stage_off, self.rank * n * x.element_size(), self.rank,
                                 self.world, op == dist.ReduceOp.MAX)
        self.barrier()
        return out
