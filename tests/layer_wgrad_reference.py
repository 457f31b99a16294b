"""tests/layer_reference.py for layers whose expert weight gradients run on e4m3 operands too (``fp8_wgrad``).

``expert_backward`` below is that of layer_reference with the weight-gradient products charged as ``'fp8'`` operands.
The e4m3 operand bound there uses each operand's row and column maxima over the whole token dimension, which are never
below the maximum of a 128 x 1 token block, so it covers the column-wise block scales.  ``check_step`` runs
``layer_reference.check_step`` with this expert backward in place of the 16-bit one.
"""
from contextlib import contextmanager

import layer_reference as LR


def expert_backward(cfg: LR.Config, w, saved, dout: LR.B, dtype, fp8: bool, pdtype):
    """(dx, [weight gradients in the order of expert_params]) of one expert, every GEMM on e4m3 operands when fp8."""
    kind = 'fp8' if fp8 else dtype
    if cfg.expert == 'ffn':
        w1, b1, w2, b2 = w
        x, pre, h = saved
        dh = LR.rnd(LR.mul(LR.mm(dout, LR.B(w2.t()), kind), LR.dact(pre, cfg.act)), dtype)
        dw2 = LR.rnd(LR.mm(h.t(), dout, kind), pdtype)
        db2 = LR.rnd(LR.rsum(dout, 0), pdtype) if b2 is not None else None
        dx = LR.rnd(LR.mm(dh, LR.B(w1), kind), dtype)
        dw1 = LR.rnd(LR.mm(dh.t(), x, kind), pdtype)
        db1 = LR.rnd(LR.rsum(dh, 0), pdtype) if b1 is not None else None
        return dx, [dw1, db1, dw2, db2]
    w1, w2, w3 = w
    x, g, u, h = saved
    dh = LR.rnd(LR.mm(dout, LR.B(w3.t()), kind), dtype)
    dg = LR.rnd(LR.mul(LR.mul(dh, u), LR.dact(g, cfg.act)), dtype)
    du = LR.rnd(LR.mul(dh, LR.act(g, cfg.act)), dtype)
    dx = LR.rnd(LR.add(LR.rnd(LR.mm(dg, LR.B(w1.t()), kind), dtype), LR.mm(du, LR.B(w2.t()), kind)), dtype)
    return dx, [LR.rnd(LR.mm(x.t(), dg, kind), pdtype), LR.rnd(LR.mm(x.t(), du, kind), pdtype),
                LR.rnd(LR.mm(h.t(), dout, kind), pdtype)]


@contextmanager
def _fp8_weight_gradients():
    # layer_reference.reference looks expert_backward up in its module at call time
    orig = LR.expert_backward
    LR.expert_backward = expert_backward
    try:
        yield
    finally:
        LR.expert_backward = orig


def check_step(cfg: LR.Config, step: LR.Step):
    """``layer_reference.check_step`` with e4m3 weight-gradient operands (cfg.fp8 must be set)."""
    assert cfg.fp8 is not None, 'fp8 weight gradients come with an fp8 recipe'
    with _fp8_weight_gradients():
        return LR.check_step(cfg, step)
