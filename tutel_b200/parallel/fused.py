"""NVLink-fused expert-parallel engine: dispatch+GEMM1 and GEMM2+combine with no separate all-to-all.

This is the H100-native replacement of the reference's ``all_to_all -> experts -> all_to_all`` sequence
(tutel/impls/moe_layer.py:329-357) and of its chunked NCCL overlap scheduler (tutel/impls/overlap.py,
tutel/custom/custom_kernel.cpp:520-654).  Per forward pass and rank (W ranks, El local experts, capacity C):

  comm stream   encode kernel: gathers this rank's tokens slot by slot and *stores them straight into the
                destination expert GPU's receive buffer* ``IN[El, W(src), C, M]`` over NVLink, publishing an
                epoch flag per row chunk with ``st.release.sys``                       (csrc/moe_kernels.cu)
  main stream   GEMM1 (wgmma): its TMA producer ``ld.acquire.sys``-polls the flags of exactly the rows of the
                tile it is about to load, so tiles are multiplied as they arrive - own-rank rows first.
                GEMM2 (wgmma): the epilogue stores every output tile *directly into the source GPU's* combine
                buffer ``OUT[E, C, Mout]`` and bumps a ``red.release.sys`` counter per expert.
                decode kernel: acquires the counters of the experts a token used and sums its k rows.

Backward mirrors this (output gradients are dispatched, dgrad/wgrad GEMMs run as rows arrive, input gradients are
combined), so one training step issues 4 fused transfers and never calls NCCL for tokens.
``a2a_ffn_overlap_degree`` selects the flag granularity (rows per arrival flag = C / d, at least one MMA tile).

What the engine covers: ``ffn`` experts with ReLU / GELU / SiLU (bias or not, any ``output_dim``), gated ``llama_ffn``
experts, post- and pre-score gating, and experts sharded over several GPUs (E < W, every valid ``adaptive_r >= 1``):
sharding is expressed as a *virtual geometry* - one virtual expert per GPU that receives its share of the rows of
each of the r token copies - so the same kernels serve it (rows are replicated in the push, the r partial results are
summed in the decode).

Memory model.  Every forward or backward pass of a layer is one *transaction* on a ring of N (default 3) buffer sets
``(IN, OUT)`` in the symmetric heap that ALL layers with the same geometry share; transactions take the sets round
robin, in the same order on every rank.  A forward whose backward is still pending keeps a lease on its set (its
received rows feed the weight gradient, its combined rows the gate gradient).  When the ring wraps onto a leased set,
the lease is *spilled* - copied into ordinary tensors - one transaction ahead, on the communication stream in front of
that transaction's push.  Peers cannot write into a set before they have received this rank's rows of the preceding
transaction, which are pushed after the spill on the same stream, so no row that is still needed can be overwritten;
the arena is independent of the depth of the network (3 sets = 0.8 GB at the flagship shape).
"""
from __future__ import annotations

import logging
import os
import weakref
from typing import Any, Dict, List, Optional

import torch

from ..ops import backend
from ..ops import gemm as G
from ..ops.dispatch import DispatchPlan
from . import communicate as C_
from . import p2p

_FLAGS_PER_SEG = 64          # arrival flags per (expert, source) segment


def _enabled() -> bool:
    return os.environ.get('TUTEL_B200_FUSED', '1') not in ('0', 'off', 'false')


def _ring_size() -> int:
    return max(2, int(os.environ.get('TUTEL_B200_FUSED_SETS', 3)))


# ----------------------------------------------------------------------------------------------------------------
# geometry: what the kernels see (identical to the layer's own numbers unless experts are sharded)
# ----------------------------------------------------------------------------------------------------------------
class _Geometry:
    """W ranks, E (virtual) experts of which El live here, C rows per expert and source, k (virtual) choices."""

    def __init__(self, W, rank, E, El, C, k, M, H, Mo, es, copies=1, real_k=None):
        self.W, self.rank, self.E, self.El, self.C, self.k = W, rank, E, El, C, k
        self.M, self.H, self.Mo, self.es = M, H, Mo, es
        self.copies, self.real_k = copies, (real_k if real_k is not None else k)
        self.G = El * W                                    # GEMM groups: (local expert, source rank)
        self.width = max(M, Mo)

    def rows_quantum(self) -> int:
        """Buffer sets are sized for the next power of two >= C (at least 256 rows): a capacity that changes from call to
        call (dynamic / dropless capacity factors) re-uses a handful of rings instead of allocating one per distinct value."""
        q = 256
        while q < self.C:
            q *= 2
        return q

    def key(self):
        return (self.W, self.E, self.El, self.rows_quantum(), self.width, self.es)

    def set_bytes(self) -> int:
        return 2 * self.E * self.rows_quantum() * self.width * self.es


class _Plan:
    """Kernel-side routing tables of one call (virtual when experts are sharded)."""

    def __init__(self, idx_ks, loc_ks, slot_src):
        self.idx_ks, self.loc_ks, self.slot_src = idx_ks, loc_ks, slot_src


def _virtual_plan(plan: DispatchPlan, E: int, Sh: int, r: int) -> _Plan:
    """E real experts, each shared by Sh GPUs, tokens replicated r times (reference: the repeat / view / sum around the
    all-to-alls, tutel/impls/moe_layer.py:331-357).  GPU ``e*Sh + c*(Sh/r) + q`` receives rows ``[q*Cv, (q+1)*Cv)`` of
    copy ``c`` of expert ``e`` with ``Cv = C*r/Sh``: one virtual expert per GPU, ``r*k`` virtual choices per token."""
    C, k, S = plan.C, plan.k, plan.S
    per = Sh // r
    Cv = C * r // Sh
    slot = plan.slot_src.view(E, 1, per, Cv).expand(E, r, per, Cv).reshape(-1).contiguous()
    idx, loc = plan.idx_ks.to(torch.int64), plan.loc_ks.to(torch.int64)
    valid = (loc < C) & (idx >= 0)
    q = torch.where(valid, loc // Cv, torch.zeros_like(loc))
    base = idx * Sh + q                                                       # [k, S]
    copies = torch.arange(r, device=idx.device, dtype=torch.int64).view(r, 1, 1) * per
    idx_v = (base.unsqueeze(0) + copies).reshape(r * k, S).to(torch.int32)
    loc_v = torch.where(valid, loc % Cv, torch.full_like(loc, 0x3fffffff)).unsqueeze(0).expand(r, k, S).reshape(r * k, S)
    return _Plan(idx_v.contiguous(), loc_v.to(torch.int32).contiguous(), slot)


# ----------------------------------------------------------------------------------------------------------------
# buffer ring (shared by all layers with the same geometry)
# ----------------------------------------------------------------------------------------------------------------
class _BufferSet:
    """One (IN, OUT) pair + flag areas at identical offsets on every rank."""

    def __init__(self, t: 'p2p.P2PTransport', tag: str, geo: _Geometry):
        half = geo.E * geo.rows_quantum() * geo.width * geo.es
        self.off_in = t.alloc(tag + '/in', half)
        self.off_out = t.alloc(tag + '/out', half)
        self.f_in = t.ctrl_alloc(tag + '/f_in', geo.G * _FLAGS_PER_SEG * 4)
        self.f_out = t.ctrl_alloc(tag + '/f_out', geo.E * 4)
        self.epoch = 0                 # published by the encode kernels on f_in (one writer per flag)
        self.out_total = 0             # cumulative tile count expected on f_out
        self.holder = None             # weakref to the _Lease of a forward whose backward is pending
        self.tables: Dict[Any, torch.Tensor] = {}


class _Lease:
    """What a forward leaves behind for its backward: the received rows (IN) and the combined rows (OUT).  They stay in
    the arena until the ring needs the set again (then they are copied out) or the backward has run."""

    def __init__(self, bufs: _BufferSet, x_recv: Optional[torch.Tensor], y_comb: Optional[torch.Tensor], own_x: bool = False):
        self.bufs, self.x_recv, self.y_comb = bufs, x_recv, y_comb
        self.own_x = own_x             # x_recv is already an ordinary tensor (fp8 path: the de-quantised copy of the rows)
        self.spill_event = None

    def spill(self, stream: torch.cuda.Stream):
        stream.wait_stream(torch.cuda.current_stream())      # the rows were completed by work queued on the main stream
        with torch.cuda.stream(stream):
            if self.x_recv is not None and not self.own_x:
                self.x_recv = self.x_recv.clone()
            if self.y_comb is not None:
                self.y_comb = self.y_comb.clone()
            self.spill_event = torch.cuda.Event()
            self.spill_event.record(stream)
        self.bufs.holder = None

    def ready(self):
        """Make the current stream wait for a spill that may still be in flight on the communication stream."""
        if self.spill_event is not None:
            cur = torch.cuda.current_stream()
            cur.wait_event(self.spill_event)
            for t in (self.x_recv, self.y_comb):
                if t is not None:
                    t.record_stream(cur)

    def release(self):
        if self.bufs.holder is not None and self.bufs.holder() is self:
            self.bufs.holder = None


class _Ring:
    def __init__(self, t: 'p2p.P2PTransport', geo: _Geometry, serial: int):
        self.sets: List[_BufferSet] = []
        for i in range(_ring_size()):
            if not t.can_alloc(geo.set_bytes() + 4096):
                break
            self.sets.append(_BufferSet(t, 'fused%d/set%d' % (serial, i), geo))
        self.cursor = 0

    def usable(self) -> bool:
        return len(self.sets) >= 2

    def next(self, side: torch.cuda.Stream) -> _BufferSet:
        """The set of this transaction; spills the lease (if any) on the set the NEXT transaction will use."""
        n = len(self.sets)
        s = self.sets[self.cursor % n]
        self.cursor += 1
        for cand in (s, self.sets[self.cursor % n]):     # `s` itself was normally spilled one transaction ago
            if cand.holder is not None:
                lease = cand.holder()
                if lease is not None:
                    lease.spill(side)
                cand.holder = None
        return s


class FusedEngine:
    """Per-transport state: rings keyed by geometry, the communication stream, election counters of the push kernel."""

    def __init__(self, transport: 'p2p.P2PTransport'):
        self.t = transport
        self.W, self.rank = transport.world, transport.rank
        self.rings: Dict[tuple, Optional[_Ring]] = {}
        self.side = torch.cuda.Stream()
        self.counters: Dict[int, torch.Tensor] = {}
        self.warned = False

    def ring_for(self, geo: _Geometry) -> Optional[_Ring]:
        key = geo.key()
        if key not in self.rings:
            ring = None
            try:
                ring = _Ring(self.t, geo, len(self.rings) + 1)
            except RuntimeError:
                ring = None
            self.rings[key] = ring if ring is not None and ring.usable() else None
        return self.rings[key]

    def chunk_counters(self, E: int) -> torch.Tensor:
        c = self.counters.get(E)
        if c is None:
            c = torch.zeros([E * _FLAGS_PER_SEG], dtype=torch.int32, device='cuda')
            self.counters[E] = c
        return c

    @staticmethod
    def chunk_rows(C: int, d: int) -> int:
        """Rows per arrival flag.  One MMA tile (256 rows) is the finest useful granularity; `d` (the layer's
        a2a_ffn_overlap_degree) can only make it finer than the default C/8, never coarser than C."""
        rows = -(-C // max(d, 8))
        rows = max(256, rows, -(-C // _FLAGS_PER_SEG))
        return (rows + 255) // 256 * 256

    @staticmethod
    def tile_counts(C: int, N: int):
        """(cta_group, block_n, completion signals per group) of a combine GEMM over [C, N] outputs.  A CTA signals once
        per 128 x 128 tile it finishes, so a group of ceil(C / 128) * ceil(N / 128) tiles raises its counter by that number."""
        return 1, 128, (-(-C // 128)) * (-(-N // 128))


def _engine(transport) -> FusedEngine:
    eng = getattr(transport, '_fused_engine', None)
    if eng is None:
        eng = FusedEngine(transport)
        transport._fused_engine = eng
    return eng


# ----------------------------------------------------------------------------------------------------------------
# one transaction (forward or backward of one layer call)
# ----------------------------------------------------------------------------------------------------------------
class _Txn:
    def __init__(self, eng: FusedEngine, geo: _Geometry, plan: _Plan, bufs: _BufferSet, d: int, dtype: torch.dtype):
        self.eng, self.geo, self.plan, self.bufs, self.dtype = eng, geo, plan, bufs, dtype
        self.chunk = eng.chunk_rows(geo.C, d)
        self.base = eng.t.base_ptr(geo.rank)
        bufs.epoch += 1
        self.epoch = bufs.epoch
        self.out_target = bufs.out_total

    # ---- pointer tables (device int64 arrays, cached per buffer set) ----
    def _table(self, key, values: List[int]) -> int:
        tab = self.bufs.tables.get(key)
        if tab is None:
            tab = torch.tensor(values, dtype=torch.int64, device='cuda')
            if len(self.bufs.tables) < 512:
                self.bufs.tables[key] = tab
            else:       # a capacity that keeps changing: stop caching, keep the last few alive for the kernels still queued
                recent = self.bufs.tables.setdefault('__recent__', [])
                recent.append(tab)
                del recent[:-64]
        return tab.data_ptr()

    def _push_tables(self, width: int):
        """Encode side: expert e's rows go to rank e // El, segment (e % El, my rank) of its IN buffer."""
        g, t, b = self.geo, self.eng.t, self.bufs
        hit = b.tables.get(('pd', width, g.C)), b.tables.get(('ps',))
        if hit[0] is not None and hit[1] is not None:
            return hit[0].data_ptr(), hit[1].data_ptr()
        dst = [t.base_ptr(e // g.El) + b.off_in + ((e % g.El) * g.W + g.rank) * g.C * width * g.es for e in range(g.E)]
        sig = [t.base_ptr(e // g.El) + b.f_in + ((e % g.El) * g.W + g.rank) * _FLAGS_PER_SEG * 4 for e in range(g.E)]
        return self._table(('pd', width, g.C), dst), self._table(('ps',), sig)

    def _combine_tables(self, width: int):
        """GEMM epilogue side: group (local expert, source rank) is written into the source rank's OUT buffer."""
        g, t, b = self.geo, self.eng.t, self.bufs
        hit = b.tables.get(('cd', width, g.C)), b.tables.get(('cs',))
        if hit[0] is not None and hit[1] is not None:
            return hit[0].data_ptr(), hit[1].data_ptr()
        dst, sig = [], []
        for grp in range(g.G):
            el, src = divmod(grp, g.W)
            e = g.rank * g.El + el
            dst.append(t.base_ptr(src) + b.off_out + e * g.C * width * g.es)
            sig.append(t.base_ptr(src) + b.f_out + e * 4)
        return self._table(('cd', width, g.C), dst), self._table(('cs',), sig)

    # ---- the primitives ----
    def push(self, src: torch.Tensor, gates_f32: Optional[torch.Tensor], width: int) -> torch.cuda.Event:
        """Scatter-and-send on the communication stream: rows of `src` -> the expert GPUs' IN buffers (+ arrival flags)."""
        g, eng = self.geo, self.eng
        dst_tab, sig_tab = self._push_tables(width)
        cur = torch.cuda.current_stream()
        eng.side.wait_stream(cur)
        chunks_per_expert = -(-g.C // self.chunk)
        with torch.cuda.stream(eng.side):
            backend.count_launch()
            backend.require_ext().encode_rows(src, gates_f32, self.plan.slot_src, src, g.real_k, g.E, g.C, dst_tab, sig_tab,
                                              self.chunk, g.rank * g.El * chunks_per_expert, self.epoch,
                                              eng.chunk_counters(g.E).data_ptr(), None)
            ev = torch.cuda.Event()
            ev.record(eng.side)
        for tns in (src, self.plan.slot_src, gates_f32):
            if tns is not None:
                tns.record_stream(eng.side)
        return ev

    def push_fp8(self, src: torch.Tensor, gates_f32: Optional[torch.Tensor], width: int) -> torch.cuda.Event:
        """The same scatter-and-send with per-row e4m3 quantisation: rows of `width` bytes + one fp32 scale per row (half the
        NVLink bytes of the 16-bit push)."""
        g, eng, t, b = self.geo, self.eng, self.eng.t, self.bufs
        soff = self._scale_off(width)
        if ('pd8', width, g.C) in b.tables:
            dst_tab, scl_tab = b.tables[('pd8', width, g.C)].data_ptr(), b.tables[('psc8', width, g.C)].data_ptr()
        else:
            dst = [t.base_ptr(e // g.El) + b.off_in + ((e % g.El) * g.W + g.rank) * g.C * width for e in range(g.E)]
            scl = [t.base_ptr(e // g.El) + b.off_in + soff + ((e % g.El) * g.W + g.rank) * g.C * 4 for e in range(g.E)]
            dst_tab, scl_tab = self._table(('pd8', width, g.C), dst), self._table(('psc8', width, g.C), scl)
        _, sig_tab = self._push_tables(width)
        cur = torch.cuda.current_stream()
        eng.side.wait_stream(cur)
        chunks_per_expert = -(-g.C // self.chunk)
        with torch.cuda.stream(eng.side):
            backend.count_launch()
            backend.require_ext().encode_rows_fp8(src, gates_f32, self.plan.slot_src, g.real_k, g.E, g.C, dst_tab, scl_tab, sig_tab,
                                                  self.chunk, g.rank * g.El * chunks_per_expert, self.epoch,
                                                  eng.chunk_counters(g.E).data_ptr())
            ev = torch.cuda.Event()
            ev.record(eng.side)
        for tns in (src, self.plan.slot_src, gates_f32):
            if tns is not None:
                tns.record_stream(eng.side)
        return ev

    def _scale_off(self, width: int) -> int:
        g = self.geo
        return (g.G * g.C * width + 1023) // 1024 * 1024

    def recv_view_fp8(self, width: int):
        """(e4m3 rows [G, C, width], fp32 row scales [G, C]) of the IN buffer."""
        g, t = self.geo, self.eng.t
        q = t.view(self.bufs.off_in, [g.G, g.C, width], torch.float8_e4m3fn)
        sc = t.view(self.bufs.off_in + self._scale_off(width), [g.G, g.C], torch.float32)
        return q, sc

    def recv_view(self, width: int) -> torch.Tensor:
        g = self.geo
        return self.eng.t.view(self.bufs.off_in, [g.G, g.C, width], self.dtype)

    def wait_kwargs(self) -> dict:
        g = self.geo
        return dict(wait_flags=self.base + self.bufs.f_in, wait_rows_per_flag=self.chunk, wait_flags_per_group=_FLAGS_PER_SEG,
                    wait_target=self.epoch, group_rot=g.rank, group_mod=-g.W, b_group_div=g.W)

    def combine_kwargs(self, width: int) -> dict:
        g = self.geo
        cg, bn, tiles = self.eng.tile_counts(g.C, width)
        d_tab, s_tab = self._combine_tables(width)
        self.bufs.out_total += tiles
        self.out_target = self.bufs.out_total
        return dict(out=self.eng.t.view(self.bufs.off_out, [g.E, g.C, width], self.dtype), cta_group=cg, block_n=bn,
                    d_ptr_table=d_tab, signal_ptr_table=s_tab, group_rot=g.rank, group_mod=-g.W, b_group_div=g.W)

    def comb_view(self, width: int) -> torch.Tensor:
        g = self.geo
        return self.eng.t.view(self.bufs.off_out, [g.E * g.C, width], self.dtype)

    def decode(self, gates_v: Optional[torch.Tensor], width: int, shared: Optional[tuple] = None) -> torch.Tensor:
        """Weighted sum of each token's (virtual) choices once their experts have delivered (+ the shared experts' term
        ``shared = (base, fp32 logits or None)`` in the same launch, ops/dispatch.py: raw_decode)."""
        g = self.geo
        backend.count_launch()
        if shared is None:
            return backend.require_ext().decode_rows(self.comb_view(width), gates_v, self.plan.idx_ks, self.plan.loc_ks, g.E,
                                                     g.C, self.base + self.bufs.f_out, self.out_target)
        return backend.require_ext().decode_rows(self.comb_view(width), gates_v, self.plan.idx_ks, self.plan.loc_ks, g.E, g.C,
                                                 self.base + self.bufs.f_out, self.out_target, None, shared[0], shared[1])


def _gate_grad(a: torch.Tensor, buf: torch.Tensor, plan: _Plan, geo: _Geometry) -> torch.Tensor:
    """[k, S] fp32 gate gradients <a[s], buf[slot_j(s)]>, summed over the copies of a sharded expert."""
    backend.count_launch()
    dg = backend.require_ext().gate_grad(a, buf, plan.idx_ks, plan.loc_ks, geo.E, geo.C)
    if geo.copies > 1:
        dg = dg.view(geo.copies, geo.real_k, -1).sum(dim=0)
    return dg


def _virtual_gates(gates_f32: torch.Tensor, geo: _Geometry) -> torch.Tensor:
    return gates_f32 if geo.copies == 1 else gates_f32.repeat(geo.copies, 1)


def _shared_in(base: Optional[torch.Tensor], shared_logit: Optional[torch.Tensor]) -> Optional[tuple]:
    """The shared experts' terms as decode_rows takes them, or None."""
    if base is None:
        return None
    return base.contiguous(), (None if shared_logit is None else shared_logit.detach().to(torch.float32).contiguous().view(-1))


def _shared_grads(ctx: Any, dout: torch.Tensor):
    """(d_base, d_shared_logit) of the shared experts' term: dout itself without the shared gate; with it, the
    gate-gradient kernel with zero routed choices (csrc/moe_kernels.cu: gate_grad_kernel)."""
    if not ctx.has_shared:
        return ()
    if not ctx.shared_gated:
        return dout, None
    base, shared_logit = ctx.shared_saved
    idx = torch.empty([0, dout.size(0)], dtype=torch.int32, device=dout.device)
    backend.count_launch()
    _, d_base, d_logit = backend.require_ext().gate_grad(dout, None, idx, idx, 1, 1, None, base.contiguous(),
                                                         shared_logit.detach().to(torch.float32).contiguous().view(-1))
    return d_base, d_logit.to(shared_logit.dtype).view_as(shared_logit)


def _save_shared(ctx: Any, base: Optional[torch.Tensor], shared_logit: Optional[torch.Tensor]) -> None:
    ctx.has_shared, ctx.shared_gated = base is not None, shared_logit is not None
    ctx.shared_saved = (base.detach(), shared_logit.detach()) if ctx.shared_gated else None


# ----------------------------------------------------------------------------------------------------------------
# eligibility + entry point
# ----------------------------------------------------------------------------------------------------------------
def engine_for(layer, x: torch.Tensor, crit, d: int):
    """Return a runnable fused call for this forward, or None when the generic path must be used."""
    if not _enabled() or not backend.use_wgmma(x):
        return None
    ex = layer.experts
    from ..models.experts.ffn import FusedExpertsNetwork
    from ..models.experts.llama_ffn import LlamaFFNNetwork
    if layer.adaptive_degree == 0 or layer.megablocks_size > 0:
        return None
    t = p2p.transport_for(layer.group)
    if t is None:
        return None
    Sh, r = layer.sharded_count, layer.adaptive_degree
    if Sh > 1 and 1 < t.world < C_.get_world_size():
        r = Sh              # experts sharded inside a sub-group are always model-parallel (models/experts/ffn.py: materialize)
    if isinstance(ex, FusedExpertsNetwork):
        if ex._act_kind not in G.FWD_EPILOGUE or ex.skip_expert or (ex.fp8 and ex._act_kind != 'relu'):
            return None
        if getattr(ex, 'mx', False) or getattr(ex, 'block', False):
            return None     # MX and block-fp8 experts run on the unfused path (ops/mx.py, ops/block_fp8.py)
        if ex.fp8 and (layer.model_dim % 16 or ex.hidden_size % 16 or ex.output_dim % 16):
            return None
        if ex.batched_fc1_w.dtype != x.dtype or (layer.model_dim % 8) or (ex.hidden_size % 8) or (ex.output_dim % 8):
            return None
        M, H, Mo = layer.model_dim, ex.hidden_size * (Sh // r if Sh > 1 else 1), ex.output_dim
    elif isinstance(ex, LlamaFFNNetwork):
        if getattr(ex, 'block', False) or getattr(ex, 'weight_format', None) is not None:
            return None     # block-fp8 and stored experts (no W_fc1) run on the unfused path (ops/block_fp8.py, ops/int4.py)
        if G.classify_activation(ex.activation_fn) not in G.ACT_CODES or ex.W_fc1.dtype != x.dtype:
            return None
        align = 16 if ex.fp8 else 8
        if any(int(v) % align for v in ex.full_shapes['W_fc1'][1:]) or int(ex.full_shapes['W_fc3'][2]) % align:
            return None
        M, H, Mo = layer.model_dim, int(ex.full_shapes['W_fc1'][2]), int(ex.full_shapes['W_fc3'][2])
    else:
        return None
    eng = _engine(t)
    plan = DispatchPlan.from_critical(crit)
    W, E, k, C = t.world, layer.num_global_experts, plan.k, plan.C
    es = x.element_size()
    if Sh > 1:
        if r < 1 or Sh % r or (C * r) % Sh or k * r > 16 or C * r // Sh < 1:
            return None
        geo = _Geometry(W, t.rank, W, 1, C * r // Sh, k * r, M, H, Mo, es, copies=r, real_k=k)
    else:
        geo = _Geometry(W, t.rank, E, layer.num_local_experts, C, k, M, H, Mo, es)
    ring = eng.ring_for(geo)
    if ring is None:
        if not eng.warned:
            logging.warning('tutel_b200: symmetric heap too small for the fused MoE buffers of this layer (C=%d); using the '
                            'generic all-to-all path. Raise TUTEL_B200_HEAP_MB to enable the fused engine.', plan.C)
            eng.warned = True
        return None
    return _Runner(eng, ring, geo, d, plan)


class _Runner:
    def __init__(self, eng: FusedEngine, ring: _Ring, geo: _Geometry, d: int, plan: DispatchPlan):
        self.eng, self.ring, self.geo, self.d, self.plan = eng, ring, geo, d, plan

    def run(self, layer, x: torch.Tensor, crit, base: Optional[torch.Tensor] = None,
            shared_logit: Optional[torch.Tensor] = None) -> torch.Tensor:
        """The fused MoE call; ``base`` / ``shared_logit``: the shared experts' output and gate logits, added in the
        combine launch.  (Multi-GPU only: not exercised on a single-GPU machine.)"""
        geo, plan = self.geo, self.plan
        ex = layer.experts
        gates = crit.gates_ks if hasattr(crit, 'gates_ks') else torch.stack([g.view(-1) for g in crit[3]])
        if geo.copies > 1 or layer.sharded_count > 1:
            kplan = _virtual_plan(plan, layer.num_global_experts, layer.sharded_count, geo.copies)
        else:
            kplan = _Plan(plan.idx_ks, plan.loc_ks, plan.slot_src)
        call = (self.eng, self.ring, geo, kplan, self.d, layer.is_postscore, bool(getattr(ex, 'fp8', False)))
        if hasattr(ex, 'full_shapes'):
            w1, w2, w3 = (ex._full(n, layer.group) for n in ('W_fc1', 'W_fc2', 'W_fc3'))
            if base is None:
                return _FusedGLUMoE.apply(call, G.classify_activation(ex.activation_fn), x, gates, w1, w2, w3)
            return _FusedGLUMoE.apply(call, G.classify_activation(ex.activation_fn), x, gates, w1, w2, w3, base, shared_logit)
        w1, b1, w2, b2 = ex.materialize(layer)
        if base is None:
            return _FusedMoE.apply(call, ex._act_kind, x, gates, w1, b1, w2, b2)
        return _FusedMoE.apply(call, ex._act_kind, x, gates, w1, b1, w2, b2, base, shared_logit)


def _begin(call, dtype) -> _Txn:
    eng, ring, geo, kplan, d = call[:5]
    return _Txn(eng, geo, kplan, ring.next(eng.side), d, dtype)


class _FusedMoE(torch.autograd.Function):
    """``ffn`` experts: y = act(x W1^T + b1) W2 + b2 between a fused dispatch and a fused combine."""

    @staticmethod
    def forward(ctx: Any, call, act_kind: str, x, gates, w1, b1, w2, b2, base=None, shared_logit=None):
        eng, ring, geo, kplan, d, is_postscore, fp8 = call
        M, H, Mo = geo.M, geo.H, geo.Mo
        need_grad = any(ctx.needs_input_grad[2:])
        _save_shared(ctx, base, shared_logit)
        gates_f32 = gates.detach().to(torch.float32).contiguous()
        tx = _begin(call, x.dtype)

        b1v = None if b1 is None else b1.reshape(w1.size(0), -1)
        b2v = None if b2 is None else b2.reshape(w2.size(0), -1)
        cg, bn1, _ = eng.tile_counts(geo.C, H)
        pre, x16_event = None, None
        if fp8:
            # e4m3 end to end: rows are quantised in the push (half the NVLink bytes), both GEMMs run at the fp8 rate on
            # weight copies quantised once per optimizer step; scales are applied in the epilogues
            ev = tx.push_fp8(x, None if is_postscore else gates_f32, M)
            xq, sx = tx.recv_view_fp8(M)
            w1q, s1 = G.fp8_operand(w1, transpose=False)
            act = G.raw_gemm(xq, w1q, epilogue=G.EPI_BIAS_RELU, bias=b1v, out_dtype=x.dtype, scale_a=sx, scale_b=s1, cta_group=cg,
                             block_n=bn1, **tx.wait_kwargs())
            x_recv = None
            if need_grad:       # the 16-bit weight-gradient GEMM needs the rows back in 16 bit: de-quantise next to GEMM2
                eng.side.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(eng.side):
                    backend.count_launch()
                    x_recv = backend.require_ext().dequant_rows(xq, sx, x.dtype)
                    x16_event = torch.cuda.Event()
                    x16_event.record(eng.side)
            aq, sa = G.quantize_rows(act)
            w2q, s2 = G.fp8_operand(w2, transpose=True)
            G.raw_gemm(aq, w2q, epilogue=G.EPI_BIAS if b2 is not None else G.EPI_NONE, bias=b2v, scale_a=sa, scale_b=s2,
                       **tx.combine_kwargs(Mo))
        else:
            # (1) dispatch: tokens -> expert GPUs' IN buffers (communication stream, overlaps GEMM1)
            ev = tx.push(x, None if is_postscore else gates_f32, M)

            # (2) GEMM1 + bias + activation on rows as they arrive
            x_recv = tx.recv_view(M)
            if act_kind != 'relu' and need_grad:
                pre = torch.empty([geo.G, geo.C, H], dtype=x.dtype, device=x.device)
            act = G.raw_gemm(x_recv, w1, epilogue=G.FWD_EPILOGUE[act_kind], bias=b1v, cta_group=cg, block_n=bn1, d2=pre,
                             **tx.wait_kwargs())

            # (3) GEMM2 + bias, epilogue writes into the source GPUs' OUT buffers and signals per expert
            G.raw_gemm(act, w2, b_mn=True, epilogue=G.EPI_BIAS if b2 is not None else G.EPI_NONE, bias=b2v,
                       **tx.combine_kwargs(Mo))

        # (4) combine: weighted sum of each token's k rows once their experts have delivered (+ the shared experts)
        out = tx.decode(_virtual_gates(gates_f32, geo) if is_postscore else None, Mo, _shared_in(base, shared_logit))
        torch.cuda.current_stream().wait_event(ev)

        ctx.call, ctx.act_kind = call, act_kind
        ctx.has_b1, ctx.has_b2 = b1 is not None, b2 is not None
        if need_grad:
            lease = _Lease(tx.bufs, x_recv, tx.comb_view(Mo) if is_postscore else None, own_x=fp8)
            lease.spill_event = x16_event
            tx.bufs.holder = weakref.ref(lease)
            ctx.lease = lease
            ctx.save_for_backward(x, gates, w1, w2, act, pre)
        return out

    @staticmethod
    def backward(ctx: Any, dout: torch.Tensor):
        call, act_kind, lease = ctx.call, ctx.act_kind, ctx.lease
        eng, ring, geo, kplan, d, is_postscore, fp8 = call
        x, gates, w1, w2, act, pre = ctx.saved_tensors
        M, H, Mo, W, El, C = geo.M, geo.H, geo.Mo, geo.W, geo.El, geo.C
        dout = dout.contiguous()
        gates_f32 = gates.detach().to(torch.float32).contiguous()
        lease.ready()
        x_recv, y_comb = lease.x_recv, lease.y_comb

        # (a) gate gradients of the combine:  <dout[s], y[slot_j(s)]>
        dgates = None
        if is_postscore and ctx.needs_input_grad[3]:
            dgates = _gate_grad(dout, y_comb, kplan, geo).to(gates.dtype)

        # (b) dispatch the output gradients to the expert GPUs (decode.bwd == encode of dout)
        tx = _begin(call, dout.dtype)
        cg, bnh, _ = eng.tile_counts(C, H)
        want_db1 = ctx.has_b1 and ctx.needs_input_grad[5]
        db1_acc = torch.zeros([w1.size(0), H], dtype=torch.float32, device=dout.device) if want_db1 else None
        need_dx = ctx.needs_input_grad[2] or (not is_postscore and ctx.needs_input_grad[3])
        if fp8:
            ev = tx.push_fp8(dout, gates_f32 if is_postscore else None, Mo)
            dyq, sdy = tx.recv_view_fp8(Mo)
            w2q, s2 = G.fp8_operand(w2, transpose=False)        # dh = dy @ W2^T: W2 [H, Mout] is K-major for this product
            dh = G.raw_gemm(dyq, w2q, epilogue=G.EPI_RELU_BWD, aux=act, out_dtype=dout.dtype, scale_a=sdy, scale_b=s2,
                            cta_group=cg, block_n=bnh, colsum=db1_acc, **tx.wait_kwargs())
            if need_dx:
                dhq, sdh = G.quantize_rows(dh)
                w1q, s1 = G.fp8_operand(w1, transpose=True)     # dx = dh @ W1: W1^T [M, H] K-major
                G.raw_gemm(dhq, w1q, scale_a=sdh, scale_b=s1, **tx.combine_kwargs(M))
            backend.count_launch()
            dy_recv = backend.require_ext().dequant_rows(dyq, sdy, dout.dtype)     # all rows have arrived (dh GEMM is queued before)
        else:
            ev = tx.push(dout, gates_f32 if is_postscore else None, Mo)
            dy_recv = tx.recv_view(Mo)

            # (c) dh = (dy @ W2^T) * act'(.)   as rows arrive
            if act_kind == 'relu':
                dh = G.raw_gemm(dy_recv, w2, epilogue=G.EPI_RELU_BWD, aux=act, cta_group=cg, block_n=bnh, colsum=db1_acc,
                                **tx.wait_kwargs())
            else:
                dh = G.raw_gemm(dy_recv, w2, epilogue=G.EPI_ACT_BWD, aux=pre, act=G.ACT_CODES[act_kind], cta_group=cg, block_n=bnh,
                                colsum=db1_acc, **tx.wait_kwargs())

            # (e) dX_e = dh @ W1, epilogue pushes into the source GPUs' OUT buffers.  Collective decision: every rank
            #     must run it if any rank needs input gradients - the flag is part of the saved context (same program).
            if need_dx:
                G.raw_gemm(dh, w1, b_mn=True, **tx.combine_kwargs(M))

        # (d, f) weight gradients over all W*C received rows of each local expert
        act_e, dh_e = act.view(El, W * C, H), dh.view(El, W * C, H)
        dw2 = G.raw_gemm(act_e, dy_recv.view(El, W * C, Mo), a_mn=True, b_mn=True) if ctx.needs_input_grad[6] else None
        dw1 = G.raw_gemm(dh_e, x_recv.reshape(El, W * C, M), a_mn=True, b_mn=True) if ctx.needs_input_grad[4] else None
        db1 = db1_acc.to(dh.dtype) if want_db1 else None
        db2 = G.column_sums(dy_recv.view(El, W * C, Mo)) if ctx.has_b2 and ctx.needs_input_grad[7] else None

        # (g) combine the input gradients (encode.bwd == decode of the gradient buffer)
        dx = None
        if need_dx:
            dx = tx.decode(None if is_postscore else _virtual_gates(gates_f32, geo), M)
            if not is_postscore and ctx.needs_input_grad[3]:
                dgates = _gate_grad(x, tx.comb_view(M), kplan, geo).to(gates.dtype)
        torch.cuda.current_stream().wait_event(ev)
        lease.release()
        return (None, None, dx, dgates, dw1, db1, dw2, db2) + _shared_grads(ctx, dout)


class _FusedGLUMoE(torch.autograd.Function):
    """The same engine for gated (SwiGLU / "LLaMA") experts: dispatch feeds the dual-B GLU GEMM tile by tile, the down
    projection writes into the source GPUs' combine buffers; backward mirrors it with the fused GLU-gradient epilogue.
    (reference: tutel/experts/llama_ffn.py:38-41 between the two all-to-alls of tutel/impls/moe_layer.py:349-351)"""

    @staticmethod
    def forward(ctx: Any, call, act: str, x, gates, w1, w2, w3, base=None, shared_logit=None):
        eng, ring, geo, kplan, d, is_postscore, fp8 = call
        M, H, Mo = geo.M, geo.H, geo.Mo
        need_grad = any(ctx.needs_input_grad[2:])
        _save_shared(ctx, base, shared_logit)
        gates_f32 = gates.detach().to(torch.float32).contiguous()
        tx = _begin(call, x.dtype)
        cg, _, _ = eng.tile_counts(geo.C, H)
        x16_event = None
        if fp8:
            ev = tx.push_fp8(x, None if is_postscore else gates_f32, M)
            xq, sx = tx.recv_view_fp8(M)
            (q1, s1), (q2, s2) = G.fp8_operand(w1, transpose=True), G.fp8_operand(w2, transpose=True)      # [El, H, M] K-major
            h, g, u = G.glu_gemm(xq, q1, q2, b_mn=False, act=act, save_pre=need_grad, scale_a=sx, scale_b=s1, scale_b2=s2,
                                 out_dtype=x.dtype, cta_group=cg, **tx.wait_kwargs())
            x_recv = None
            if need_grad:
                eng.side.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(eng.side):
                    backend.count_launch()
                    x_recv = backend.require_ext().dequant_rows(xq, sx, x.dtype)
                    x16_event = torch.cuda.Event()
                    x16_event.record(eng.side)
            hq, sh = G.quantize_rows(h)
            q3, s3 = G.fp8_operand(w3, transpose=True)                                                        # [El, Mo, H]
            G.raw_gemm(hq, q3, scale_a=sh, scale_b=s3, **tx.combine_kwargs(Mo))
        else:
            ev = tx.push(x, None if is_postscore else gates_f32, M)
            x_recv = tx.recv_view(M)
            h, g, u = G.glu_gemm(x_recv, w1, w2, b_mn=True, act=act, save_pre=need_grad, cta_group=cg, **tx.wait_kwargs())
            G.raw_gemm(h, w3, b_mn=True, **tx.combine_kwargs(Mo))
        out = tx.decode(_virtual_gates(gates_f32, geo) if is_postscore else None, Mo, _shared_in(base, shared_logit))
        torch.cuda.current_stream().wait_event(ev)
        ctx.call, ctx.act = call, act
        if need_grad:
            lease = _Lease(tx.bufs, x_recv, tx.comb_view(Mo) if is_postscore else None, own_x=fp8)
            lease.spill_event = x16_event
            tx.bufs.holder = weakref.ref(lease)
            ctx.lease = lease
            ctx.save_for_backward(x, gates, w1, w2, w3, g, u, h)
        return out

    @staticmethod
    def backward(ctx: Any, dout: torch.Tensor):
        call, act, lease = ctx.call, ctx.act, ctx.lease
        eng, ring, geo, kplan, d, is_postscore, fp8 = call
        x, gates, w1, w2, w3, g, u, h = ctx.saved_tensors
        M, H, Mo, W, El, C = geo.M, geo.H, geo.Mo, geo.W, geo.El, geo.C
        dout = dout.contiguous()
        gates_f32 = gates.detach().to(torch.float32).contiguous()
        lease.ready()
        x_recv, y_comb = lease.x_recv, lease.y_comb
        dgates = None
        if is_postscore and ctx.needs_input_grad[3]:
            dgates = _gate_grad(dout, y_comb, kplan, geo).to(gates.dtype)
        tx = _begin(call, dout.dtype)
        cg, _, _ = eng.tile_counts(C, H)
        need_dx = ctx.needs_input_grad[2] or (not is_postscore and ctx.needs_input_grad[3])
        if fp8:
            ev = tx.push_fp8(dout, gates_f32 if is_postscore else None, Mo)
            dyq, sdy = tx.recv_view_fp8(Mo)
            q3, s3 = G.fp8_operand(w3, transpose=False)          # dh = dy @ W3^T: W3 [H, Mo] is K-major for this product
            dg, du = G.glu_gemm_bwd(dyq, q3, g, u, b_mn=False, act=act, scale_a=sdy, scale_b=s3, cta_group=cg, **tx.wait_kwargs())
            if need_dx:
                ck = tx.combine_kwargs(M)
                (dgq, sg), (duq, su) = G.quantize_rows(dg), G.quantize_rows(du)
                (q1, s1), (q2, s2) = G.fp8_operand(w1, transpose=False), G.fp8_operand(w2, transpose=False)   # [El, M, H]
                part = G.raw_gemm(dgq, q1, out_dtype=dout.dtype, scale_a=sg, scale_b=s1, b_group_div=W, cta_group=ck['cta_group'],
                                  block_n=ck['block_n'])
                G.raw_gemm(duq, q2, epilogue=G.EPI_ADD, aux=part, scale_a=su, scale_b=s2, **ck)
            backend.count_launch()
            dy_recv = backend.require_ext().dequant_rows(dyq, sdy, dout.dtype)
        else:
            ev = tx.push(dout, gates_f32 if is_postscore else None, Mo)
            dy_recv = tx.recv_view(Mo)
            # dh = dy @ W3^T stays in registers; the epilogue emits dg and du as the gradient rows arrive
            dg, du = G.glu_gemm_bwd(dy_recv, w3, g, u, b_mn=False, act=act, cta_group=cg, **tx.wait_kwargs())
            if need_dx:
                ck = tx.combine_kwargs(M)
                part = G.raw_gemm(dg, w1, b_group_div=W, cta_group=ck['cta_group'], block_n=ck['block_n'])   # dg @ W1^T (local)
                G.raw_gemm(du, w2, epilogue=G.EPI_ADD, aux=part, **ck)
        x_e, dy_e = x_recv.reshape(El, W * C, M), dy_recv.view(El, W * C, Mo)
        dw3 = G.raw_gemm(h.view(El, W * C, H), dy_e, a_mn=True, b_mn=True) if ctx.needs_input_grad[6] else None
        dw1 = G.raw_gemm(x_e, dg.view(El, W * C, H), a_mn=True, b_mn=True) if ctx.needs_input_grad[4] else None
        dw2 = G.raw_gemm(x_e, du.view(El, W * C, H), a_mn=True, b_mn=True) if ctx.needs_input_grad[5] else None
        dx = None
        if need_dx:
            dx = tx.decode(None if is_postscore else _virtual_gates(gates_f32, geo), M)
            if not is_postscore and ctx.needs_input_grad[3]:
                dgates = _gate_grad(x, tx.comb_view(M), kplan, geo).to(gates.dtype)
        torch.cuda.current_stream().wait_event(ev)
        lease.release()
        return (None, None, dx, dgates, dw1, dw2, dw3) + _shared_grads(ctx, dout)
