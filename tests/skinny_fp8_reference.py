"""float64 references with per-element error bounds for the weight-only fp8 skinny expert kernels
(csrc/skinny_gemm.cu: skinny_ffn_fp8_kernel, skinny_glu_ffn_fp8_kernel).  Plain torch: runs on the CPU or the GPU.

The reference is built from exactly what the kernel reads: the 16-bit x, the e4m3 weights and their fp32 row scales,
dequantised as ``q.double() * s``.  The kernel's arithmetic is exact up to fp32 rounding: e4m3 and 16-bit values are
exact in fp32, and so is each product of the two (at most 4 + 11 significant bits).  What remains is

* the fp32 sums over K (layer 1) and over the hidden units H (layer 2, inside a block and across the blocks' atomics):
  at most n * 2^-24 * sum|terms| each to first order, so ``C * (K + H) * 2^-24 * T`` with the magnitudes T below;
* one rounding per applied scale (s1 for the FFN; s1, s2 for the gate / up of the SwiGLU; s2 / s3 on the output),
  ``2^-24 * T`` each;
* the rounding of the output itself, ``2^-24 * |y|``.

C = 2, derived as ``C_GLU`` in tests/test_gpu_glu_dropless.py: c = 1 covers the first-order terms of both sums, the factor
2 the second-order terms and the few ulps of erff / __expf, the bias add and the act(g) * u product, which
(K + H) * |h| dominates.  It is not calibrated on a GPU.
"""
import torch
import torch.nn.functional as F

U32 = 2.0 ** -24
C_FP8 = 2.0
# Largest |act'(v)|: 1 for ReLU, 1.0998 for SiLU, 1.1289 for erf-GELU.  Bounds a layer-1 error's effect on act(.).
ACT_LIPSCHITZ = 1.13
ACTS = {'relu': 1, 'gelu': 2, 'silu': 3}
_FN = {'relu': torch.relu, 'gelu': F.gelu, 'silu': F.silu}


def quantize(w: torch.Tensor):
    """Per-row e4m3 copy of ``w [G, R, C]`` with fp32 scales max|row| / 448, the form ops/gemm.py: fp8_weight caches."""
    s = (w.float().abs().amax(-1) / 448.0).clamp(min=1e-12)
    return (w.float() / s.unsqueeze(-1)).to(torch.float8_e4m3fn).contiguous(), s.contiguous()


def dequant(q: torch.Tensor, s: torch.Tensor) -> torch.Tensor:
    """fp64 values of per-row-scaled e4m3 weights: ``q [G, R, C]`` times ``s [G, R]`` along the rows."""
    return q.double() * s.double().unsqueeze(-1)


def ffn_reference(x, q1, s1, b1, q2t, s2, b2, act):
    """y = act(x @ W1^T + b1) @ W2^T + b2 with W1 = s1 * Q1 [G, H, K] and W2 = s2 * Q2t [G, N, H]; returns (y, bound)."""
    xd, w1, w2 = x.double(), dequant(q1, s1), dequant(q2t, s2)
    pre = xd @ w1.transpose(1, 2)
    bias1 = torch.zeros((), dtype=torch.float64, device=x.device) if b1 is None else b1.double().reshape(w1.size(0), 1, -1)
    pre = pre + bias1
    h = _FN[act](pre)
    y = h @ w2.transpose(1, 2)
    if b2 is not None:
        y = y + b2.double().reshape(w2.size(0), 1, -1)
    a = xd.abs() @ w1.abs().transpose(1, 2) + bias1.abs()          # magnitude of layer 1's sum, bias included
    terms = (ACT_LIPSCHITZ * a + h.abs()) @ w2.abs().transpose(1, 2)
    if b2 is not None:
        terms = terms + b2.double().abs().reshape(w2.size(0), 1, -1)
    K, H = q1.size(2), q1.size(1)
    return y, U32 * y.abs() + (C_FP8 * (K + H) + 2) * U32 * terms     # + s1, s2


def glu_reference(x, q1t, s1, q2t, s2, q3t, s3, act):
    """y = (act(x @ W1^T) * (x @ W2^T)) @ W3^T with W1 / W2 = s1 / s2 * Q [G, H, M] and W3 = s3 * Q3t [G, N, H];
    returns (y, bound)."""
    xd, w1, w2, w3 = x.double(), dequant(q1t, s1), dequant(q2t, s2), dequant(q3t, s3)
    g, u = xd @ w1.transpose(1, 2), xd @ w2.transpose(1, 2)
    a = _FN[act](g)
    h = a * u
    y = h @ w3.transpose(1, 2)
    sg, su = xd.abs() @ w1.abs().transpose(1, 2), xd.abs() @ w2.abs().transpose(1, 2)
    terms = (ACT_LIPSCHITZ * sg * u.abs() + a.abs() * su + h.abs()) @ w3.abs().transpose(1, 2)
    M, H = q1t.size(2), q1t.size(1)
    return y, U32 * y.abs() + (C_FP8 * (M + H) + 3) * U32 * terms     # + s1, s2, s3


def check(y, ref, bound, counts):
    """Rows below each group's count within their bound, every other row exactly zero.  Returns the largest
    (|err| - output rounding) / rest of the bound (<= 1 when it passes); raises AssertionError otherwise."""
    R = y.size(1)
    worst = 0.0
    for g, c in enumerate(counts.clamp(max=R).tolist()):
        if c > 0:
            err = (y[g, :c].double() - ref[g, :c]).abs()
            out = U32 * ref[g, :c].abs()
            ratio = float(((err - out).clamp(min=0) / (bound[g, :c] - out)).max())
            assert bool((err <= bound[g, :c]).all()), 'group %d: error %.3g x its bound' % (g, float((err / bound[g, :c]).max()))
            worst = max(worst, ratio)
        assert torch.count_nonzero(y[g, c:]) == 0, 'group %d: rows at or past the count %d are not zero' % (g, c)
    return worst
