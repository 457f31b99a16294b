"""float64 reference with per-element error bounds for the block-scaled fp8 skinny SwiGLU kernel
(csrc/skinny_gemm.cu: skinny_glu_ffn_block_fp8_kernel).  Plain torch: runs on the CPU or the GPU.

The reference is built from exactly what the kernel reads: the bf16 x, the stored e4m3 bytes (``qglu`` with gate / up
rows interleaved every 64, ``q3t``) and their fp32 block scales, dequantised as ``q.double() * s`` per block.  It follows
the error model of tests/skinny_fp8_reference.py.  Products of a bf16 and an e4m3 value (8 + 4 significant bits) are
exact in fp32, so what remains is fp32 rounding:

* layer 1, per lane: a 16-term partial sum of one 128-deep K block (16 roundings), one fma with that block's scale (one
  rounding of the sum), the lane's sum over its M / 512 chunks, and a 5-step shuffle tree: at most 16 + M / 16 + 5 <= M
  roundings of sums bounded by ``sum |x| |w|`` (M >= 128);
* layer 2, per output: a 16-term partial, a 3-step 8-lane tree, one scaling, and H / 128 fp32 atomics across the
  blocks: at most 16 + 3 + 1 + H / 128 <= H roundings of sums bounded by ``sum |h| |w3|``;
* act(g) * u (the Lipschitz constant of act on a layer-1 error, a few ulps of __expf / erff) and the output rounding.

So ``C_FP8 * (M + H) * 2^-24 * T`` with the first-order magnitudes T of tests/skinny_fp8_reference.py bounds every
element, with C_FP8 = 2 covering second-order terms and the special-function ulps.  The scale of a 128-element block is
applied to a finished partial sum, never to a weight element: a per-element dequantisation would round each weight
(error up to 2^-24 |w| per element), which the bound also covers, but the promotion order is what makes the M-term small.
"""
import torch

from skinny_fp8_reference import ACT_LIPSCHITZ, C_FP8, U32, _FN, check  # noqa: F401  (check is re-exported)


def dequant_block(q: torch.Tensor, s: torch.Tensor) -> torch.Tensor:
    """fp64 values of ``q [G, N, K]`` e4m3 with one fp32 scale per ``N / s.size(1)`` rows and 128 columns."""
    G, N, K = q.shape
    rows = N // s.size(1)
    return (q.double().view(G, s.size(1), rows, K // 128, 128) * s.double()[:, :, None, :, None]).view(G, N, K)


def split_glu(w: torch.Tensor):
    """[G, 2H, M] rows interleaved every 64 (gate, up) -> gate [G, H, M], up [G, H, M]."""
    G, H2, M = w.shape
    t = w.view(G, H2 // 128, 2, 64, M)
    return t[:, :, 0].reshape(G, H2 // 2, M), t[:, :, 1].reshape(G, H2 // 2, M)


def glu_reference(x, qglu, sglu, q3t, s3t, act, groups=None):
    """y = (act(x @ W1^T) * (x @ W2^T)) @ W3^T on the dequantised stored weights; returns (y, bound), fp64 [G, R, N].
    ``groups``: compute only these groups (others stay zero), to keep large cases cheap."""
    G, R, M = x.shape
    H, N = qglu.size(1) // 2, q3t.size(1)
    y = torch.zeros(G, R, N, dtype=torch.float64, device=x.device)
    bound = torch.zeros_like(y)
    for g in (range(G) if groups is None else groups):
        w1, w2 = split_glu(dequant_block(qglu[g:g + 1], sglu[g:g + 1]))
        w3 = dequant_block(q3t[g:g + 1], s3t[g:g + 1])
        xd = x[g:g + 1].double()
        gt, u = xd @ w1.transpose(1, 2), xd @ w2.transpose(1, 2)
        a = _FN[act](gt)
        h = a * u
        yg = h @ w3.transpose(1, 2)
        sg, su = xd.abs() @ w1.abs().transpose(1, 2), xd.abs() @ w2.abs().transpose(1, 2)
        terms = (ACT_LIPSCHITZ * sg * u.abs() + a.abs() * su + h.abs()) @ w3.abs().transpose(1, 2)
        y[g] = yg[0]
        bound[g] = (U32 * yg.abs() + (C_FP8 * (M + H) + 3) * U32 * terms)[0]
    return y, bound
