"""fp64 reference of one training step of ``MOELayer`` on one GPU, conditioned on the layer's own routing decision.

Routing is discontinuous: a 16-bit run and an fp64 run may choose differently at near-ties.  The reference therefore
takes the decision the layer made (ids, queue locations, counts, capacity), checks that it is a valid decision for the
layer's inputs, and computes everything else in fp64 from those inputs (x and the parameters) and from the gradients
that reached the layer's outputs (``dy``, and the coefficient ``dl`` of ``l_aux`` in the loss).  The user's loss is
then outside the bound and any loss can be used.

What one step computes (written from the documented semantics, not from the kernels):

    logits z = x Wg^T                                    (in Wg's dtype; fp32 with ``fp32_gate``)
    softmax: p = softmax(z), r_j = p[id_j]               l_aux = E / S^2 sum_e ce_e sum_s p_se  (ce: first choices)
    sigmoid: p = sigmoid(z), r_j = p[id_j]               l_aux = E / (k S^2) sum_e n_e sum_s p_se / T_s
    gates    g_j = scale r_j / max(sum_j r_j, eps)       (normalize_gate and k > 1; eps = finfo(logits dtype).eps)
    queue    j-th choices queue behind all (j-1)-th ones; capacity C from ops/routing._capacity; dropped: loc >= C
    experts  ffn: act(x W1^T + b1) W2 + b2        llama_ffn: (act(x W1) * (x W2)) W3
    combine  y_s = sum_{kept j} g_j f_{id_j}(x_s) + w_s base_s        (postscore)
             y_s = sum_{kept j} f_{id_j}(g_j x_s) + w_s base_s        (prescore)
    shared   base = f_shared(x), w_s = 1 or sigmoid(x_s . w)

Backward is the same graph differentiated by hand with the ids held fixed; :func:`autograd_check` verifies those
formulas against fp64 autograd of the forward.

Bounds: a first-order "magnitude graph".  Every value is carried as ``B(v, e)``: its fp64 value ``v`` and a bound
``e`` on |layer - v| elementwise.  Each operation propagates its operands' bounds exactly to first order
(``|a| e_b + e_a |b| + e_a e_b`` for a product, ``L e`` through a function of slope at most L) and adds its own
evaluation error:

* every fp32 operation of a kernel: one rounding, u |result| (u = 2^-24); a reduction over n terms n u sum|terms|;
* a GEMM: ``C_ACC[dtype] u S`` with S = (|A| + e_A) (|B| + e_B) (``gemm_reference.C_ACC``; the wgmma and cuBLAS
  tensor-core accumulators are not round-to-nearest fp32 sums), ``K u S`` for fp32 operands;
* e4m3 operands (fp8 ``row`` and ``mx`` experts): each element is off by at most 2^-4 |a| (half an e4m3 ulp) plus
  2^-16 max|row| (e4m3 subnormals: the scale is at most 2 max|row| / 448), and the accumulation is ``C_ACC[e4m3]``;
* an activation: ``ACT_LIPSCHITZ`` times the input bound plus ``gemm_reference.FN_REL``; act' moves by at most 0.8 times
  the input bound (|GELU''| <= 0.8, |SiLU''| <= 0.5), and ReLU' is charged in full where the sign is uncertain;
* each rounding point of the layer adds half an ulp of its dtype at |v| + e: the 16-bit logits, the scores of the
  torch softmax path, the gates of the op-by-op gate, the stored hidden activations (and pre-activations), the expert
  output, the combine output, the encoded gradient rows, dh, the expert dx, the parameter gradients, ``dlogits``, the
  shared-gate logit and its gradient, and the 16-bit sum of the input-gradient terms (one rounding per added term).

A check passes where |layer - v| <= SLACK e + TINY (``dispatch_reference``).  The normalised error |layer - v| / bound
is recorded per output in ``OBSERVED``.

The gate path is checked on its own as well: the input gradient's gate term ``dlogits Wg`` is far smaller than the
expert term's bound, so :func:`check_step` is also run on steps whose loss is ``l_aux`` alone (dy = 0), where
``dlogits``, ``wg.grad`` and ``dx`` are the gate path alone.

The decision check (:func:`check_decision`): logits against fp64 ``x Wg^T`` under the GEMM bound; the chosen ids
are a top-k of the fp64 scores in descending order, with ties allowed up to the sum of the two scores' bounds
(the sigmoid gate: keys and expert groups likewise); locations, counts and slot map exactly (``ref_locations``; with
batch-prioritised routing each expert's queue must be in order of non-increasing confidence); the capacity by the rule
of ops/routing._capacity; the packed layout exactly (``packed_reference.layout``).

Out of scope: gate noise and ``is_gshard_loss=False`` (the load-importance loss needs noise), custom gates and
experts, ``reserve_dims > 1``, sharded experts and the multi-GPU fused engine.
"""
from __future__ import annotations

import math
from contextlib import contextmanager
from dataclasses import dataclass
from typing import Dict, Optional

import torch

from dispatch_reference import SLACK, TINY, U, ref_locations
from expert_ffn_reference import ACT_LIPSCHITZ
from gemm_reference import C_ACC, FN_REL, half_ulp

Q_REL = 2.0 ** -4            # e4m3: half an ulp, relative
Q_ABS = 2.0 ** -16           # e4m3 subnormal spacing / 2 times the largest scale (2 max|row| / 448), relative to max|row|
ACT2 = 0.8                   # largest |act''| of GELU (0.798) and SiLU (0.5)
OBSERVED: Dict[str, float] = {}


# ------------------------------------------------------------------------------------------------------------------
# bounded values
# ------------------------------------------------------------------------------------------------------------------
class B:
    """fp64 value ``v`` and elementwise bound ``e`` on the layer's deviation from it (None: exact)."""
    __slots__ = ('v', 'e')

    def __init__(self, v: torch.Tensor, e: Optional[torch.Tensor] = None):
        self.v, self.e = v, e

    @property
    def err(self):
        return torch.zeros_like(self.v) if self.e is None else self.e

    @property
    def mag(self):
        return self.v.abs() if self.e is None else self.v.abs() + self.e

    def __getitem__(self, i):
        return B(self.v[i], None if self.e is None else self.e[i])

    def t(self):
        return B(self.v.transpose(-1, -2), None if self.e is None else self.e.transpose(-1, -2))

    def view(self, *shape):
        return B(self.v.reshape(*shape), None if self.e is None else self.e.reshape(*shape))


def exact(t: torch.Tensor) -> B:
    return B(t.double())


def _as(t: torch.Tensor, dtype) -> torch.Tensor:
    """t in the dtype the layer reads it in (a no-op for the fp64 leaves of autograd_check: its values are the same)."""
    return t if t.dtype == torch.float64 else t.to(dtype)


def rnd(a: B, dtype) -> B:
    """A store in ``dtype``: half an ulp at |v| + e."""
    if dtype == torch.float64:
        return a
    return B(a.v, a.err + half_ulp(a.mag, dtype))


def _op(v, e):
    return B(v, e + U * v.abs().detach())


def add(a: B, b: B) -> B:
    return _op(a.v + b.v, a.err + b.err)


def sub(a: B, b: B) -> B:
    return _op(a.v - b.v, a.err + b.err)


def mul(a: B, b: B) -> B:
    return _op(a.v * b.v, a.v.abs().detach() * b.err + a.err * b.mag)


def div(a: B, b: B) -> B:
    v = a.v / b.v
    lo = (b.v.abs() - b.err).clamp_min(1e-300)
    return _op(v, (a.err + v.abs().detach() * b.err) / lo)


def rsum(a: B, dim) -> B:
    """An fp32 reduction in any order: n u sum|terms| on top of the propagated bounds."""
    n = a.v.size(dim)
    return B(a.v.sum(dim), a.err.sum(dim) + n * U * a.mag.sum(dim))


def mm(a: B, b: B, kind) -> B:
    """a [.., T, K] @ b [.., K, N] on a GEMM: ``kind`` is the operand dtype (16 bit or fp32), or 'fp8'."""
    K = a.v.size(-1)
    am, bm = a.v.abs().detach(), b.v.abs().detach()
    ea, eb = a.e, b.e
    if kind == 'fp8':
        qa = Q_REL * am + Q_ABS * am.amax(-1, keepdim=True)
        qb = Q_REL * bm + Q_ABS * bm.amax(-2, keepdim=True)
        ea = qa if ea is None else ea + qa
        eb = qb if eb is None else eb + qb
    c = K * U if kind in (torch.float32, torch.float64) else C_ACC[torch.float8_e4m3fn if kind == 'fp8' else kind] * U
    Am = am if ea is None else am + ea
    Bm = bm if eb is None else bm + eb
    e = c * (Am @ Bm)
    if eb is not None:
        e = e + Am @ eb
    if ea is not None:
        e = e + ea @ bm
    return B(a.v @ b.v, e)


def act(a: B, kind: str) -> B:
    v = a.v
    if kind == 'relu':
        return B(v.clamp_min(0), a.e)
    out = 0.5 * v * (1 + torch.erf(v / math.sqrt(2))) if kind == 'gelu' else v * torch.sigmoid(v)
    return B(out, ACT_LIPSCHITZ * a.err + FN_REL * (out.abs() + v.abs()).detach())


def dact(a: B, kind: str) -> B:
    """act'(a): ReLU's step is charged in full where the sign of a is uncertain."""
    v = a.v.detach()
    if kind == 'relu':
        return B((v > 0).double(), (v.abs() <= a.err).double())
    if kind == 'gelu':
        d = 0.5 * (1 + torch.erf(v / math.sqrt(2))) + v * torch.exp(-0.5 * v * v) / math.sqrt(2 * math.pi)
    else:
        s = torch.sigmoid(v)
        d = s * (1 + v * (1 - s))
    return B(d, ACT2 * a.err + FN_REL * (d.abs() + 1))


def sigmoid(a: B) -> B:
    p = torch.sigmoid(a.v)
    pd = p.detach()
    return B(p, pd * (1 - pd) * a.err + 6 * U * pd + 2.0 ** -126)


def softmax(z: B) -> B:
    """softmax over the last dim; the fp32 evaluation bound of dispatch_reference.ref_softmax, widened to any E."""
    p = torch.softmax(z.v, -1)
    pd = p.detach()
    E = z.v.size(-1)
    prop = pd * (z.err + (pd * z.err).sum(-1, keepdim=True))
    rel = (4 + (z.v - z.v.amax(-1, keepdim=True)).abs().detach()) * U            # exp(z - max): its argument and expf
    rel = rel + (pd * rel).sum(-1, keepdim=True) + (-(-E // 32) + 4 + 2) * U      # the sum, the reciprocal, the product
    return B(p, prop + pd * rel + TINY)


def scatter_rows(shape, index: torch.Tensor, src: B, device) -> B:
    """zeros(shape).scatter_add_(1, index, src) for B values."""
    v = torch.zeros(shape, dtype=torch.float64, device=device).scatter_add(1, index, src.v)
    e = torch.zeros(shape, dtype=torch.float64, device=device).scatter_add(1, index, src.err)
    return B(v, e)


# ------------------------------------------------------------------------------------------------------------------
# what one step computed
# ------------------------------------------------------------------------------------------------------------------
@dataclass
class Config:
    """The layer options the reference needs.  ``gate_path``: 'fused' (the CUDA gate+routing kernels), 'op' (the same
    formulas op by op in torch: 16-bit gates and gate gradients) or 'torch' (F.softmax in the logits dtype and the
    torch GShard loss: 16-bit scores as well)."""
    E: int
    k: int
    dtype: torch.dtype
    logit_dtype: torch.dtype
    expert: str = 'ffn'                  # 'ffn' | 'llama_ffn'
    act: str = 'relu'
    fp8: Optional[str] = None            # None | 'row' | 'mx'
    normalize: bool = True
    postscore: bool = True
    scoring: str = 'softmax'
    n_group: int = 1
    topk_group: int = 1
    scale: float = 1.0
    gate_path: str = 'fused'
    bpr: bool = False
    cf: float = 1.0
    alignment: int = 1
    shared: bool = False
    shared_gated: bool = False


@dataclass
class Step:
    """Inputs and results of one step: the values the parameters had in it (``params``, by state-dict name), the
    routing decision, what the layer returned and the gradients it produced (None where nothing reached them)."""
    x: torch.Tensor
    params: Dict[str, torch.Tensor]
    logits: torch.Tensor
    idx: torch.Tensor
    loc: torch.Tensor
    counts: torch.Tensor
    capacity: Optional[int]              # None: packed (dropless, no capacity)
    y: torch.Tensor
    l_aux: torch.Tensor
    dy: Optional[torch.Tensor]
    dl: float
    dlogits: Optional[torch.Tensor]
    dx: Optional[torch.Tensor]
    grads: Dict[str, Optional[torch.Tensor]]
    slot: Optional[torch.Tensor] = None
    layout: object = None
    bias: Optional[torch.Tensor] = None  # sigmoid gate's selection bias


def capacity_rule(S, E, k, cf, counts, alignment) -> int:
    """ops/routing._capacity on one GPU: cf > 0: k int(cf ceil(S/E)); cf <= 0: the fullest expert, capped at
    k int(-cf ceil(S/E)) for cf < 0; rounded up to the alignment."""
    spe = (S + E - 1) // E
    if cf > 0:
        cap = k * int(cf * spe)
    else:
        cap = int(counts.max())
        if cf < 0:
            cap = min(cap, k * int(-cf * spe))
    return (cap + alignment - 1) // alignment * alignment


def layer_alignment(sharded_count: int, overlap_degree: int) -> int:
    a = sharded_count * overlap_degree
    return (a + 127) // 128 * 128 if a > 256 else a


# ------------------------------------------------------------------------------------------------------------------
# experts
# ------------------------------------------------------------------------------------------------------------------
def expert_params(cfg: Config, params, prefix, e, M, H, dev):
    """fp64 weights of expert e: ffn (W1 [H, M], b1, W2 [H, Mo], b2) or llama_ffn (W1, W2 [M, H], W3 [H, M])."""
    if cfg.expert == 'ffn':
        w = [params[prefix + 'batched_fc1_w'][e], params.get(prefix + 'batched_fc1_bias'),
             params[prefix + 'batched_fc2_w'][e], params.get(prefix + 'batched_fc2_bias')]
        w[1] = None if w[1] is None else w[1][e]
        w[3] = None if w[3] is None else w[3][e]
    else:
        w = [params[prefix + n].view(-1, *s)[e] for n, s in (('W_fc1', (M, H)), ('W_fc2', (M, H)), ('W_fc3', (H, M)))]
    return [None if t is None else exact(t.to(dev)).v for t in w]


def expert_forward(cfg: Config, w, x: B, dtype, fp8: bool):
    """(output, saved) of one expert on its rows x [T, M]; every stored tensor rounded to dtype."""
    kind = 'fp8' if fp8 else dtype
    if cfg.expert == 'ffn':
        w1, b1, w2, b2 = w
        pre = mm(x, B(w1.t()), kind)
        if b1 is not None:
            pre = add(pre, B(b1))
        h = rnd(act(pre, cfg.act), dtype)
        out = mm(h, B(w2), kind)
        if b2 is not None:
            out = add(out, B(b2))
        return rnd(out, dtype), (x, rnd(pre, dtype), h)
    w1, w2, w3 = w
    g, u = mm(x, B(w1), kind), mm(x, B(w2), kind)
    h = rnd(mul(act(g, cfg.act), u), dtype)
    return rnd(mm(h, B(w3), kind), dtype), (x, rnd(g, dtype), rnd(u, dtype), h)


def expert_backward(cfg: Config, w, saved, dout: B, dtype, fp8: bool, pdtype):
    """(dx, [weight gradients in the order of expert_params]) of one expert; 16-bit weight-gradient GEMMs."""
    kind = 'fp8' if fp8 else dtype
    if cfg.expert == 'ffn':
        w1, b1, w2, b2 = w
        x, pre, h = saved
        dh = rnd(mul(mm(dout, B(w2.t()), kind), dact(pre, cfg.act)), dtype)
        dw2 = rnd(mm(h.t(), dout, dtype), pdtype)
        db2 = rnd(rsum(dout, 0), pdtype) if b2 is not None else None
        dx = rnd(mm(dh, B(w1), kind), dtype)
        dw1 = rnd(mm(dh.t(), x, dtype), pdtype)
        db1 = rnd(rsum(dh, 0), pdtype) if b1 is not None else None
        return dx, [dw1, db1, dw2, db2]
    w1, w2, w3 = w
    x, g, u, h = saved
    dh = rnd(mm(dout, B(w3.t()), kind), dtype)
    dg = rnd(mul(mul(dh, u), dact(g, cfg.act)), dtype)
    du = rnd(mul(dh, act(g, cfg.act)), dtype)
    dx = rnd(add(rnd(mm(dg, B(w1.t()), kind), dtype), mm(du, B(w2.t()), kind)), dtype)
    return dx, [rnd(mm(x.t(), dg, dtype), pdtype), rnd(mm(x.t(), du, dtype), pdtype), rnd(mm(h.t(), dout, dtype), pdtype)]


def _expert_names(cfg: Config):
    if cfg.expert == 'ffn':
        return ['batched_fc1_w', 'batched_fc1_bias', 'batched_fc2_w', 'batched_fc2_bias']
    return ['W_fc1', 'W_fc2', 'W_fc3']


# ------------------------------------------------------------------------------------------------------------------
# the reference step
# ------------------------------------------------------------------------------------------------------------------
def _gate_weights(cfg: Config, step: Step, z: B):
    """(scores p, gates g [k, S], l_aux, chosen ids [k, S] long with E for 'nowhere', valid [k, S])."""
    S, E = z.v.shape
    k = step.idx.size(0)
    idx = step.idx.long()
    valid = (idx >= 0) & (idx < E)
    safe = torch.where(valid, idx, torch.zeros_like(idx))
    eps = float(torch.finfo(cfg.logit_dtype).eps)
    if cfg.scoring == 'softmax':
        p = softmax(z)
        if cfg.gate_path == 'torch':
            p = rnd(p, cfg.logit_dtype)
        ce = torch.bincount(safe[0][valid[0]], minlength=E).double()
        colsum = rsum(p, 0)
        l_aux = B((colsum.v * ce).sum() * E / (S * S), (colsum.err * ce).sum() * E / (S * S))
        l_aux = B(l_aux.v, l_aux.err + (-(-E // 256) + 5 + 8 + 4) * U * l_aux.v.abs().detach())
        if cfg.gate_path == 'torch':        # the torch GShard loss: 16-bit ce * E / S, product, sum, division
            for _ in range(4):
                l_aux = rnd(l_aux, cfg.logit_dtype)
    else:
        p = sigmoid(z)
        n = torch.zeros(E + 1, dtype=torch.float64, device=z.v.device).scatter_add(
            0, torch.where(valid, idx, torch.full_like(idx, E)).reshape(-1),
            torch.ones(idx.numel(), dtype=torch.float64, device=z.v.device))[:E]
        T = rsum(p, 1)
        q = div(p, B(T.v[:, None], T.err[:, None]))
        qs = rsum(q, 0)
        l_aux = B((qs.v * n).sum() * E / (k * S * S), (qs.err * n).sum() * E / (k * S * S))
        l_aux = B(l_aux.v, l_aux.err + (-(-E // 256) + 5 + 8 + 4) * U * l_aux.v.abs().detach())
    l_aux = rnd(l_aux, cfg.logit_dtype)
    r = p.t()[safe, torch.arange(S, device=z.v.device)[None, :].expand(k, S)]          # [k, S]
    zero = torch.zeros((), dtype=torch.float64, device=z.v.device)
    r = B(torch.where(valid, r.v, zero), torch.where(valid, r.err, zero))
    if cfg.normalize and k > 1:
        D = rsum(r, 0)
        if cfg.gate_path == 'torch':
            D = rnd(D, cfg.logit_dtype)
        g = div(r, B(D.v.clamp_min(eps)[None], D.e[None]))
    else:
        g = r
    if cfg.scoring == 'sigmoid' and cfg.scale != 1.0:
        g = mul(g, B(torch.full_like(g.v, float(torch.tensor(cfg.scale, dtype=torch.float32)))))
    if cfg.gate_path != 'fused':
        g = rnd(g, cfg.logit_dtype)
    return p, r, g, l_aux, safe, valid


def reference(cfg: Config, step: Step) -> Dict[str, B]:
    """fp64 values and bounds of every output of the step: 'logits', 'scores', 'y', 'l_aux', and with gradients
    'dlogits', 'dx' and one entry per parameter gradient (state-dict names)."""
    dev = step.logits.device
    dt, ldt = cfg.dtype, cfg.logit_dtype
    P = step.params
    x = exact(step.x.to(dev))
    S, M = x.v.shape
    k = step.idx.size(0)
    E = cfg.E
    Wg = P['gates.0.wg.weight'].to(dev)
    wdt = Wg.dtype
    xg = exact(_as(step.x.to(dev), wdt))
    z = rnd(mm(xg, exact(Wg).t(), wdt), ldt)
    p, r, g, l_aux, ids, valid = _gate_weights(cfg, step, z)
    C = step.capacity
    kept = valid & ((step.loc.long() < C) if C is not None else torch.ones_like(valid))
    out = {'logits': z, 'scores': p, 'l_aux': l_aux}

    # ---- experts, one at a time ----
    if cfg.expert == 'ffn':
        H = P['experts.batched_fc1_w'].size(1)
        Mo = P['experts.batched_fc2_w'].size(2)
    else:
        H = P['experts.W_fc1'].numel() // (E * M)
        Mo = M
    pdt = P['experts.' + _expert_names(cfg)[0]].dtype
    fp8 = cfg.fp8 is not None
    zeros = lambda *s: torch.zeros(*s, dtype=torch.float64, device=dev)   # noqa: E731
    O = B(zeros(k, S, Mo), zeros(k, S, Mo))
    saved = {}
    for e in range(E):
        sel = kept & (ids == e)
        if not bool(sel.any()):
            continue
        jj, ss = sel.nonzero(as_tuple=True)
        xin = x[ss]
        if not cfg.postscore:
            gj = g[jj, ss]
            xin = rnd(mul(xin, B(gj.v[:, None], gj.err[:, None])), dt)
        w = expert_params(cfg, P, 'experts.', e, M, H, dev)
        o, sv = expert_forward(cfg, w, xin, dt, fp8)
        O.v[jj, ss], O.e[jj, ss] = o.v, o.err
        saved[e] = (jj, ss, sv)
    if cfg.postscore:
        terms = mul(B(g.v[..., None], g.err[..., None]), O)
    else:
        terms = O
    base = ws = sl = None
    if cfg.shared:
        Hs = P['shared_experts.' + _expert_names(cfg)[0]].numel() // M
        wsh = expert_params(cfg, P, 'shared_experts.', 0, M, Hs, dev)
        base, sh_saved = expert_forward(cfg, wsh, x, dt, fp8)
        bterm = base
        if cfg.shared_gated:
            wv = P['shared_expert_gate.weight'].to(dev)
            sl = rnd(mm(exact(_as(step.x.to(dev), wv.dtype)), exact(wv).t(), wv.dtype), wv.dtype)     # [S, 1]
            ws = sigmoid(sl)
            bterm = mul(base, ws)
        terms = B(torch.cat([terms.v, bterm.v[None]]), torch.cat([terms.err, bterm.err[None]]))
    y = rnd(rsum(terms, 0), dt)
    out['y'] = y
    if step.dy is None and step.dl == 0:
        return out

    # ---- backward ----
    dy = exact(step.dy.to(dev).reshape(S, Mo)) if step.dy is not None else B(zeros(S, Mo))
    grads: Dict[str, list] = {}
    dX = B(zeros(k, S, M), zeros(k, S, M))
    dgate = B(zeros(k, S), zeros(k, S))
    for e, (jj, ss, sv) in saved.items():
        dye = dy[ss]
        if cfg.postscore:
            gj = g[jj, ss]
            dout = rnd(mul(dye, B(gj.v[:, None], gj.err[:, None])), dt)
            oe = O[jj, ss]
            d = rsum(mul(dye, oe), 1)
            dgate.v[jj, ss], dgate.e[jj, ss] = d.v, d.err
        else:
            dout = dye
        w = expert_params(cfg, P, 'experts.', e, M, H, dev)
        dxe, dws = expert_backward(cfg, w, sv, dout, dt, fp8, pdt)
        dX.v[jj, ss], dX.e[jj, ss] = dxe.v, dxe.err
        if not cfg.postscore:
            d = rsum(mul(x[ss], dxe), 1)
            dgate.v[jj, ss], dgate.e[jj, ss] = d.v, d.err
        for name, dw in zip(_expert_names(cfg), dws):
            if dw is not None:
                grads.setdefault(name, [None] * E)[e] = dw
    if cfg.postscore:
        dx_terms = [rnd(rsum(dX, 0), dt)]
    else:
        dx_terms = [rnd(rsum(mul(B(g.v[..., None], g.err[..., None]), dX), 0), dt)]

    # ---- gate backward ----
    if cfg.gate_path != 'fused':
        dgate = rnd(dgate, ldt)
    eps = float(torch.finfo(ldt).eps)
    if cfg.normalize and k > 1:
        D = rsum(r, 0)
        Dc = B(D.v.clamp_min(eps)[None], D.err[None])
        dot = rsum(mul(dgate, r), 0)
        dr = sub(div(dgate, Dc), div(B(dot.v[None], dot.err[None]), mul(Dc, Dc)))
    else:
        dr = dgate
    if cfg.scoring == 'sigmoid':
        dr = mul(dr, B(torch.full_like(dr.v, float(torch.tensor(cfg.scale, dtype=torch.float32)))))
    if cfg.gate_path != 'fused':
        dr = rnd(dr, ldt)
    if cfg.gate_path == 'torch':        # autograd of the 16-bit division: two 16-bit terms and their sum
        dr = rnd(rnd(dr, ldt), ldt)
    zk = torch.zeros_like(dr.v)
    dr = B(torch.where(valid, dr.v, zk), torch.where(valid, dr.err, zk))
    dp = scatter_rows((S, E), ids.t(), dr.t(), dev)
    dl = float(step.dl)
    if cfg.scoring == 'softmax':
        ce = torch.bincount(ids[0][valid[0]], minlength=E).double()
        aux = dl * E / (S * S) * ce
        dp = B(dp.v + aux[None], dp.err + 4 * U * abs(aux)[None] + U * (dp.v + aux[None]).abs())
        if cfg.gate_path == 'torch':
            dp = rnd(dp, ldt)
        dot = rsum(mul(dp, p), 1)
        dz = mul(p, sub(dp, B(dot.v[:, None], dot.err[:, None])))
    else:
        n = torch.zeros(E + 1, dtype=torch.float64, device=dev).scatter_add(
            0, torch.where(valid, step.idx.long(), torch.full_like(step.idx.long(), E)).reshape(-1),
            torch.ones(step.idx.numel(), dtype=torch.float64, device=dev))[:E]
        T = rsum(p, 1)
        c = div(B(torch.full_like(T.v, dl * E / (k * S * S))), T)
        m = div(rsum(mul(B(n[None].expand(S, E)), p), 1), T)
        diff = sub(B(n[None].expand(S, E)), B(m.v[:, None], m.err[:, None]))
        dp = add(dp, mul(B(c.v[:, None], c.err[:, None]), diff))
        dz = mul(mul(p, sub(B(torch.ones_like(p.v)), p)), dp)
    dz = rnd(dz, ldt)
    out['dlogits'] = dz
    grads_out = {'gates.0.wg.weight': rnd(mm(dz.t(), xg, wdt), wdt)}
    dxg = rnd(mm(dz, exact(Wg), wdt), wdt)
    dx_terms.append(rnd(dxg, dt) if wdt != dt else dxg)

    # ---- shared experts ----
    if cfg.shared:
        if cfg.shared_gated:
            dbase = rnd(mul(dy, ws), dt)
            yb = rsum(mul(dy, base), 1)
            dsl = rnd(mul(mul(ws, sub(B(torch.ones_like(ws.v)), ws)), B(yb.v[:, None], yb.err[:, None])), wv.dtype)
            grads_out['shared_expert_gate.weight'] = rnd(mm(dsl.t(), exact(_as(step.x.to(dev), wv.dtype)), wv.dtype),
                                                         wv.dtype)
            dx_terms.append(rnd(mm(dsl, exact(wv), wv.dtype), dt))
        else:
            dbase = dy
        dxs, dws = expert_backward(cfg, wsh, sh_saved, dbase, dt, fp8, pdt)
        dx_terms.append(dxs)
        for name, dw in zip(_expert_names(cfg), dws):
            if dw is not None:
                grads_out['shared_experts.' + name] = dw
    # autograd adds the input-gradient terms in the input's dtype: one rounding per added term
    tot = B(sum(t.v for t in dx_terms), sum(t.err for t in dx_terms))
    extra = (len(dx_terms) - 1) * half_ulp(tot.mag, dt) if dt != torch.float64 else 0
    out['dx'] = B(tot.v, tot.err + extra)

    for name, per in grads.items():
        shape = P['experts.' + name].shape
        one = next(t for t in per if t is not None).v.shape
        v, ev = zeros(E, *one), zeros(E, *one)
        for e, t in enumerate(per):
            if t is not None:
                v[e], ev[e] = t.v, t.err
        grads_out['experts.' + name] = B(v.reshape(shape), ev.reshape(shape))
    for name in _expert_names(cfg):          # experts that received no token: zero gradient
        if 'experts.' + name not in grads_out and P.get('experts.' + name) is not None:
            grads_out['experts.' + name] = B(zeros(*P['experts.' + name].shape))
    out.update(grads_out)
    return out


# ------------------------------------------------------------------------------------------------------------------
# checks
# ------------------------------------------------------------------------------------------------------------------
def compare(name: str, got: torch.Tensor, ref: B) -> float:
    """Largest |got - ref| / (SLACK e + TINY); recorded in OBSERVED.  Raises AssertionError above 1."""
    want = ref.v.detach()
    bound = SLACK * ref.err.detach() + TINY
    g = got.detach().to(want.device).double().reshape(want.shape)
    err = (g - want).abs()
    err = torch.where(torch.isnan(g) | torch.isnan(want), torch.full_like(err, math.inf), err)
    ratio = err / bound
    worst = float(ratio.max()) if ratio.numel() else 0.0
    OBSERVED[name] = max(OBSERVED.get(name, 0.0), worst)
    if worst > 1.0:
        i = tuple(int(v) for v in (ratio == ratio.max()).nonzero()[0])
        raise AssertionError('%s: %d of %d elements outside the bound; worst err/bound %.3g at %s: layer=%r reference=%r '
                             'bound=%.3g' % (name, int((ratio > 1).sum()), ratio.numel(), worst, i, float(g[i]),
                                             float(want[i]), float(bound[i])))
    return worst


def _check_softmax_ids(p: B, ids: torch.Tensor, valid: torch.Tensor):
    """Chosen ids beat every unchosen expert, and each choice beats the next, up to the sum of the two bounds."""
    S, E = p.v.shape
    k = ids.size(0)
    assert bool(valid.all()), 'a softmax gate routed a choice nowhere'
    sel = ids.t()                                                    # [S, k]
    hi_c = p.v.gather(1, sel) + p.err.gather(1, sel)
    lo_c = p.v.gather(1, sel) - p.err.gather(1, sel)
    for j in range(k - 1):
        bad = hi_c[:, j] < lo_c[:, j + 1]
        assert not bool(bad.any()), 'ids: choice %d of token %d scores below choice %d beyond the bound' % (
            j, int(bad.nonzero()[0]), j + 1)
    if k < E:
        chosen = torch.zeros_like(p.v, dtype=torch.bool).scatter_(1, sel, True)
        lo = torch.where(chosen, p.v + p.err, torch.full_like(p.v, math.inf)).amin(1)
        hi = torch.where(chosen, torch.full_like(p.v, -math.inf), p.v - p.err).amax(1)
        bad = lo < hi
        assert not bool(bad.any()), 'ids: token %d chose an expert that loses to an unchosen one beyond the bound (%r < %r)' % (
            int(bad.nonzero()[0]), float(lo[bad][0]), float(hi[bad][0]))


def _check_sigmoid_ids(cfg: Config, p: B, bias: torch.Tensor, ids: torch.Tensor, valid: torch.Tensor):
    """Keys p + bias: chosen groups are among the topk_group best (sum of a group's two best keys) and, within the
    groups that must have been kept, chosen keys beat unchosen ones, each up to the sum of the bounds."""
    S, E = p.v.shape
    key = p.v + bias.double().to(p.v.device)[None]
    ke = p.err
    assert bool(valid.all()), 'a sigmoid gate with finite logits routed a choice nowhere'
    sel = ids.t()
    allowed = torch.ones_like(key, dtype=torch.bool)
    if cfg.n_group > 1:
        G, gsz = cfg.n_group, E // cfg.n_group
        top = key.view(S, G, gsz).topk(min(2, gsz), dim=2)
        gs = top.values.sum(2)
        ge = ke.view(S, G, gsz).amax(2) * min(2, gsz)
        cg = torch.zeros(S, G, dtype=torch.bool, device=key.device).scatter_(1, sel // gsz, True)
        thr = (gs - ge).topk(cfg.topk_group, dim=1).values[:, -1:]
        bad = cg & (gs + ge < thr)
        assert not bool(bad.any()), 'ids: token %d chose an expert of a group outside the best topk_group' % int(
            bad.any(1).nonzero()[0])
        low = torch.where(cg, gs + ge, torch.full_like(gs, math.inf)).amin(1, keepdim=True)
        kept = cg | (gs - ge > low)
        allowed = kept.repeat_interleave(gsz, dim=1)
    chosen = torch.zeros_like(key, dtype=torch.bool).scatter_(1, sel, True)
    lo = torch.where(chosen, key + ke, torch.full_like(key, math.inf)).amin(1)
    hi = torch.where(chosen | ~allowed, torch.full_like(key, -math.inf), key - ke).amax(1)
    bad = lo < hi
    assert not bool(bad.any()), 'ids: token %d chose a key that loses to an unchosen one beyond the bound' % int(
        bad.nonzero()[0])


def _check_bpr_locations(idx, loc, counts, conf: B, E):
    """Batch-prioritised routing: per expert, locations 0..count-1, all j-th choices before (j+1)-th ones, and within
    one choice tokens in order of non-increasing confidence (ties up to the bounds)."""
    k, S = idx.shape
    idx, loc = idx.long().cpu(), loc.long().cpu()
    cv, ce = conf.v.detach().cpu(), conf.err.cpu()
    want = torch.bincount(idx.reshape(-1), minlength=E)[:E].to(torch.int32)
    assert torch.equal(counts.cpu().to(torch.int32), want), 'counts differ from the ids'
    jj = torch.arange(k)[:, None].expand(k, S)
    ss = torch.arange(S)[None, :].expand(k, S)
    for e in range(E):
        m = idx == e
        order = loc[m].argsort()
        assert torch.equal(loc[m][order], torch.arange(int(m.sum()))), 'expert %d: locations are not 0..count-1' % e
        j, s = jj[m][order], ss[m][order]
        assert bool((j[1:] >= j[:-1]).all()), 'expert %d: a choice queued before an earlier choice' % e
        same = j[1:] == j[:-1]
        up = cv[s[1:]] - ce[s[1:]] > cv[s[:-1]] + ce[s[:-1]]
        assert not bool((same & up).any()), 'expert %d: a token queued behind a less confident one' % e


def check_decision(cfg: Config, step: Step, ref: Dict[str, B]):
    """The routing decision is valid for the layer's inputs (see the module docstring)."""
    S, E = step.logits.shape[0], cfg.E
    k = step.idx.size(0)
    compare('logits', step.logits, ref['logits'])
    idx = step.idx.long()
    valid = (idx >= 0) & (idx < E)
    p = ref['scores']
    if cfg.scoring == 'softmax':
        _check_softmax_ids(p, idx, valid)
    else:
        _check_sigmoid_ids(cfg, p, step.bias, idx, valid)
    if cfg.bpr:
        conf = p[torch.arange(S, device=p.v.device), idx[0]]
        if cfg.gate_path == 'op':          # the op-by-op gate returns its first-choice score in the logits dtype
            conf = rnd(conf, cfg.logit_dtype)
        _check_bpr_locations(step.idx, step.loc, step.counts, conf, E)
    else:
        C = step.capacity or 0
        rl, rc, _, rs = ref_locations(step.idx.cpu(), E, C)
        assert torch.equal(step.loc.cpu().to(torch.int32), rl), 'locations are not the stable choice-major queue order'
        assert torch.equal(step.counts.cpu().to(torch.int32), rc), 'counts differ from the ids'
        if step.slot is not None and C > 0:
            assert torch.equal(step.slot.cpu().to(torch.int32), rs), 'slot map differs from the ids and locations'
    if step.capacity is not None:
        want = capacity_rule(S, E, k, cfg.cf, step.counts.cpu(), cfg.alignment)
        assert step.capacity == want, 'capacity %d, the rule gives %d' % (step.capacity, want)
    else:
        assert cfg.cf == 0, 'a packed (capacity-free) routing for capacity_factor %r' % cfg.cf
    if step.layout is not None:
        import packed_reference
        lay = step.layout
        want = packed_reference.layout(step.idx, step.loc, step.counts, lay.R)
        for name, got, w in zip(('seg_off', 'block_expert', 'block_rows', 'slot_src'),
                                (lay.seg_off, lay.block_expert, lay.block_rows, lay.slot_src), want):
            assert torch.equal(got.cpu().to(torch.int32), w), 'packed layout: %s differs' % name


def check_step(cfg: Config, step: Step, ref: Optional[Dict[str, B]] = None) -> Dict[str, float]:
    """Decision check, then every output against the reference.  Returns {output: largest err / bound}; raises one
    AssertionError naming every output outside its bound.  Every gradient the step produced must have a reference, and
    an output the layer left without a gradient must have a zero reference."""
    ref = reference(cfg, step) if ref is None else ref
    check_decision(cfg, step, ref)
    got = {'y': step.y, 'l_aux': step.l_aux, 'dlogits': step.dlogits, 'dx': step.dx}
    got.update(step.grads)
    worst, failed = {}, []
    backward = 'dlogits' in ref
    for name, g in got.items():
        if name not in ref:
            if backward and g is not None:
                failed.append('%s: a gradient the reference does not model' % name)
            continue
        if g is None:
            if bool((ref[name].v != 0).any()):
                failed.append('%s: no gradient, the reference has one' % name)
            continue
        try:
            worst[name] = compare(name, g, ref[name])
        except AssertionError as ex:
            failed.append(str(ex))
    if failed:
        raise AssertionError('\n'.join(failed))
    return worst


def autograd_check(cfg: Config, step: Step, ref: Dict[str, B]):
    """The hand-written backward of :func:`reference` equals fp64 autograd of its forward (to 1e-6 of the bound)."""
    leaves = {n: t.detach().double().requires_grad_(True) for n, t in step.params.items()}
    x = step.x.detach().double().requires_grad_(True)
    st = Step(**{**step.__dict__, 'x': x, 'params': leaves})
    fwd = reference(cfg, Step(**{**st.__dict__, 'dy': None, 'dl': 0.0}))
    dev = fwd['y'].v.device
    loss = fwd['l_aux'].v * float(step.dl)
    if step.dy is not None:
        loss = loss + (fwd['y'].v * step.dy.to(dev).double().reshape(fwd['y'].v.shape)).sum()
    names = [n for n in leaves if n in ref]
    grads = torch.autograd.grad(loss, [fwd['logits'].v, x] + [leaves[n] for n in names], allow_unused=True)
    for name, g in zip(['dlogits', 'dx'] + names, grads):
        r = ref[name]
        g = torch.zeros_like(r.v) if g is None else g.to(r.v.device).reshape(r.v.shape)
        d = (g - r.v).abs()
        tol = 1e-6 * (SLACK * r.err + TINY)
        assert bool((d <= tol).all()), 'autograd and the hand-written backward differ: %s (max %r)' % (name, float(d.max()))


# ------------------------------------------------------------------------------------------------------------------
# capture
# ------------------------------------------------------------------------------------------------------------------
@contextmanager
def recording(layer):
    """Record every forward of ``layer`` (one dict per call): the gate's logits (with ``retain_grad``, so that their
    gradient lands in ``logits.grad``), the selection bias of a sigmoid gate, the ``CriticalData`` the layer routed
    with, ``y``, ``l_aux`` and the gradients reaching them.  The tensors are referenced, not copied: in a step captured
    into a CUDA graph they are the graph's buffers and hold each replay's values."""
    import tutel_b200.models.moe_layer as ML
    records = []

    def wrap(fn):
        def routed(*a, **kw):
            crit, l_aux = fn(*a, **kw)
            records[-1]['crit'] = crit
            return crit, l_aux
        return routed

    def on_logits(mod, inp, out):
        if out.requires_grad:
            out.retain_grad()
        records[-1]['logits'] = out
        bias = getattr(mod, 'e_score_correction_bias', None)
        records[-1]['bias'] = None if bias is None else bias.detach().clone()

    def before(mod, inp):
        records.append({'dy': None, 'dl': None})

    def after(mod, inp, y):
        rec = records[-1]
        rec['y'], rec['l_aux'] = y, y.l_aux
        if y.requires_grad:
            y.register_hook(lambda g: rec.__setitem__('dy', g))
        if y.l_aux is not None and y.l_aux.requires_grad:
            y.l_aux.register_hook(lambda g: rec.__setitem__('dl', g))

    saved = ML.extract_critical, ML.fused_extract_critical
    ML.extract_critical, ML.fused_extract_critical = wrap(saved[0]), wrap(saved[1])
    hooks = [layer.register_forward_pre_hook(before), layer.register_forward_hook(after)]
    hooks += [g.register_forward_hook(on_logits) for g in layer.gates]
    try:
        yield records
    finally:
        ML.extract_critical, ML.fused_extract_critical = saved
        for h in hooks:
            h.remove()


def snapshot(layer) -> Dict[str, torch.Tensor]:
    return {n: p.detach().clone() for n, p in layer.named_parameters()}


def make_step(layer, rec, x, params, x_grad=None) -> Step:
    """A :class:`Step` from one record of :func:`recording`, the input, the parameter values of that step and (after
    its backward) the gradients now in ``x.grad`` / ``.grad``."""
    crit = rec['crit']
    plan = getattr(crit, '_plan', None)
    slot = crit._slot_src if crit._slot_src is not None else (plan._slot_src if plan is not None else None)
    layout = getattr(crit, 'layout', None)
    if layout is not None:             # a copy: in a CUDA graph the next replay rewrites the layout's buffers
        from types import SimpleNamespace
        layout = SimpleNamespace(R=layout.R, **{n: getattr(layout, n).clone() for n in
                                                ('seg_off', 'block_expert', 'block_rows', 'slot_src')})
    y = rec['y']
    logits = rec['logits']
    grads = {n: (None if p.grad is None else p.grad.detach().clone()) for n, p in layer.named_parameters()}
    return Step(x=x.detach().reshape(-1, x.size(-1)).clone(), params=params, logits=logits.detach().clone(),
                idx=crit.idx_ks.clone(), loc=crit.loc_ks.clone(), counts=crit[5].clone(),
                capacity=None if layout is not None else int(crit[4]), y=y.detach().reshape(-1, y.size(-1)).clone(),
                l_aux=rec['l_aux'].detach().clone(), dy=None if rec['dy'] is None else rec['dy'].detach().clone(),
                dl=0.0 if rec['dl'] is None else float(rec['dl']),
                dlogits=None if logits.grad is None else logits.grad.detach().clone(),
                dx=None if x_grad is None else x_grad.detach().reshape(-1, x.size(-1)).clone(), grads=grads,
                slot=None if slot is None else slot.clone(), layout=layout, bias=rec['bias'])


def config_of(layer, x, capacity_factor=None, top_k=None, overlap_degree=None) -> Config:
    """The reference's view of a layer (and of the gate path ``MOELayer._route`` takes for it)."""
    from tutel_b200.ops.gating import fused_gate_mode
    from tutel_b200.ops import gemm as G
    gate = layer.gates[0]
    E = layer.num_global_experts
    k = min(top_k or gate.top_k, E)
    ex = layer.experts
    if type(ex).__name__ == 'LlamaFFNNetwork':
        expert, act_kind, fp8 = 'llama_ffn', G.classify_activation(ex.activation_fn), ('row' if ex.fp8 else None)
    else:
        expert, act_kind = 'ffn', ex._act_kind
        fp8 = 'row' if ex.fp8 else ('mx' if ex.mx else None)
    scoring = getattr(gate, 'scoring_func', 'softmax')
    mode = fused_gate_mode()
    # The sigmoid gate's torch path (sigmoid_topk_gate: batch-prioritised routing, TUTEL_B200_FUSED_GATE=0, CPU) keeps
    # its scores, gates, gate gradients and first-choice confidence in fp32 and returns l_aux in the logits dtype, like
    # the fused kernels: both take the 'fused' rounding model.
    if scoring == 'sigmoid' or (x.is_cuda and mode != 'off' and not layer.batch_prioritized_routing):
        path = 'fused'
    elif mode == 'force':
        path = 'op'
    else:
        path = 'torch'
    cfg = Config(E=E, k=k, dtype=x.dtype, logit_dtype=gate.wg.weight.dtype, expert=expert, act=act_kind, fp8=fp8,
                 normalize=layer.normalize_gate, postscore=layer.is_postscore, scoring=scoring,
                 gate_path=path, bpr=layer.batch_prioritized_routing,
                 cf=capacity_factor if capacity_factor else gate.capacity_factor,
                 alignment=layer_alignment(layer.sharded_count, overlap_degree or layer.a2a_ffn_overlap_degree),
                 shared=layer.shared_experts is not None, shared_gated=layer.shared_expert_gate is not None)
    if scoring == 'sigmoid':
        cfg.n_group, cfg.topk_group, cfg.scale = gate.n_group, gate.topk_group, gate.routed_scaling_factor
    return cfg
