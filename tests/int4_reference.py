"""Exact definitions of the group-32 int4 weight format (ops/int4.py) and float64 references with per-element error
bounds for its two kernels.  Plain torch, written element by element and independently of ops/int4.py, so that the
module's packing, unpacking and quantiser are checked against a second statement of the format.

Definitions:
* a weight is ``w = q * s``: ``q`` an int4 in [-8, 7], ``s`` a bf16 scale per 32 consecutive input (K) elements of a row;
* nibble packing: byte ``j`` of a row = ``(q[2j] + 8) | (q[2j + 1] + 8) << 4``;
* compressed-tensors int32 packing: word ``i`` of a row holds elements ``8i .. 8i + 7``, element ``8i + e`` in bits
  ``4e .. 4e + 3`` as ``q + 8``;
* quantiser: ``amax`` = the largest non-NaN magnitude of the group, ``s = max(bf16_rn(amax / 7), 2^-126)``, ``s = 1``
  when ``amax == 0``; ``q = clamp(round_half_even(w / s), -8, 7)``, NaN -> 0.

Error models (u32 = 2^-24, fp32 unit roundoff; u16 = 2^-8, bf16 unit roundoff).  A product ``q * x`` of an int4 and a bf16
value (4 + 8 significant bits) and ``q * s`` are exact in fp32, so only sums and the listed roundings contribute:

* decode (``skinny_glu_ffn_int4_kernel``): layer 1 per lane is a 32-term fp32 partial sum of one group (31 roundings),
  one fma with the group's scale (one rounding), the lane's sum over M / 1024 groups and a 5-step shuffle tree: at most
  32 + M / 1024 + 5 <= M roundings (M >= 128) of sums bounded by ``sum |x| |q s|``.  Layer 2 per output: a 32-term
  partial, one scale multiply, a 2-step 4-lane tree and H / 128 fp32 atomics: at most 35 + H / 128 <= H roundings of sums
  bounded by ``sum |h| |q3 s3|``.  With act(g) * u, the special functions and the output rounding this is the model of
  tests/skinny_fp8_reference.py: ``u32 |y| + (C (M + H) + 3) u32 T`` with the first-order magnitudes T below, C = 2.
* prefill (``w4a16_gemm_kernel``, GLU then down): every weight is expanded on chip and rounded once to bf16, ``bf16_rn(q s)``
  (relative error <= u16), so layer 1 carries ``u16 sum |x| |q s|`` on top of the fp32 accumulation ``C M u32 sum |x| |q s|``
  of the bf16 GEMM bound (tests/gemm_reference.py), h is stored in bf16 (u16 |h|), layer 2 carries ``u16`` for its rounded
  weights plus ``C H u32`` for its sums, and the bf16 output rounds once more (u16 |y|).  C = 2 also covers the
  second-order terms and the few ulps of the epilogue's activation.
"""
import torch
import torch.nn.functional as F

U32 = 2.0 ** -24
U16 = 2.0 ** -8
C_ACC = 2.0
ACT_LIPSCHITZ = 1.13          # largest |act'|: 1 ReLU, 1.0998 SiLU, 1.1289 erf-GELU
GROUP = 32
_FN = {'relu': torch.relu, 'gelu': F.gelu, 'silu': F.silu, 'none': lambda t: t}


# ---------------------------------------------------------------------------------------------------------------------
# definitions
# ---------------------------------------------------------------------------------------------------------------------
def pack(q: torch.Tensor) -> torch.Tensor:
    """int8 [..., K] -> uint8 [..., K / 2], element by element."""
    flat = q.reshape(-1, q.size(-1)).tolist()
    out = [[(row[2 * j] + 8) | ((row[2 * j + 1] + 8) << 4) for j in range(len(row) // 2)] for row in flat]
    return torch.tensor(out, dtype=torch.uint8).reshape(*q.shape[:-1], q.size(-1) // 2)


def unpack(packed: torch.Tensor) -> torch.Tensor:
    """uint8 [..., K / 2] -> int8 [..., K], element by element."""
    flat = packed.reshape(-1, packed.size(-1)).tolist()
    out = [[v for b in row for v in ((b & 15) - 8, (b >> 4) - 8)] for row in flat]
    return torch.tensor(out, dtype=torch.int8).reshape(*packed.shape[:-1], packed.size(-1) * 2)


def pack_int32(q: torch.Tensor) -> torch.Tensor:
    """int8 [..., K] -> the compressed-tensors int32 words [..., K / 8], element by element."""
    flat = q.reshape(-1, q.size(-1)).tolist()
    out = []
    for row in flat:
        words = []
        for i in range(len(row) // 8):
            v = sum((row[8 * i + e] + 8) << (4 * e) for e in range(8))
            words.append(v - (1 << 32) if v >= (1 << 31) else v)
        out.append(words)
    return torch.tensor(out, dtype=torch.int32).reshape(*q.shape[:-1], q.size(-1) // 8)


def quantize(w: torch.Tensor):
    """bf16 [..., K] -> (q int8 [..., K], s bf16 [..., K / 32]) by the quantiser rule, group by group."""
    rows = w.reshape(-1, w.size(-1)).double()
    qs, ss = [], []
    for row in rows:
        qrow, srow = [], []
        for g in range(row.numel() // GROUP):
            grp = row[g * GROUP:(g + 1) * GROUP]
            mags = grp.abs()[~torch.isnan(grp)]
            amax = float(mags.max()) if mags.numel() else 0.0
            s = 1.0 if amax == 0 else max(float(torch.tensor(amax / 7, dtype=torch.float64).to(torch.bfloat16)), 2.0 ** -126)
            srow.append(s)
            for v in grp.tolist():
                qrow.append(0 if v != v else int(min(7, max(-8, torch.round(torch.tensor(v / s, dtype=torch.float64))))))
        qs.append(qrow)
        ss.append(srow)
    return (torch.tensor(qs, dtype=torch.int8).reshape(w.shape),
            torch.tensor(ss, dtype=torch.float64).to(torch.bfloat16).reshape(*w.shape[:-1], w.size(-1) // GROUP))


def values(q: torch.Tensor, s: torch.Tensor) -> torch.Tensor:
    """fp64 q * s of int8 q [..., K] with bf16 scales [..., K / 32] (exact)."""
    return (q.double().reshape(*q.shape[:-1], -1, GROUP) * s.double().unsqueeze(-1)).reshape(q.shape)


def split_glu(w: torch.Tensor):
    """[G, 2H, *] rows interleaved every 64 (gate, up) -> gate [G, H, *], up [G, H, *]."""
    G, H2 = w.shape[:2]
    t = w.reshape(G, H2 // 128, 2, 64, *w.shape[2:])
    return t[:, :, 0].reshape(G, H2 // 2, *w.shape[2:]), t[:, :, 1].reshape(G, H2 // 2, *w.shape[2:])


def stored_values(packed: torch.Tensor, s: torch.Tensor) -> torch.Tensor:
    """fp64 q * s of a stored operand (nibbles [G, R, K / 2], bf16 scales [G, R, K / 32]); vectorised unpack."""
    lo = (packed & 15).to(torch.int16) - 8
    hi = (packed >> 4).to(torch.int16) - 8
    q = torch.stack([lo, hi], dim=-1).reshape(*packed.shape[:-1], packed.size(-1) * 2)
    return values(q, s)


# ---------------------------------------------------------------------------------------------------------------------
# fp64 references and bounds of the two kernels
# ---------------------------------------------------------------------------------------------------------------------
def reference(x, wg, wu, w3, act, kernel, groups=None):
    """y = (act(x @ Wg^T) * (x @ Wu^T)) @ W3^T in fp64 from the exact weights (wg, wu [G, H, M], w3 [G, N, H], fp64) and
    the bound of ``kernel`` ('decode' or 'prefill') for every element; returns (y, bound), fp64 [G, R, N].  ``groups``:
    compute only these groups (others stay zero)."""
    G, R, M = x.shape
    H, N = wg.size(1), w3.size(1)
    y = torch.zeros(G, R, N, dtype=torch.float64, device=x.device)
    bound = torch.zeros_like(y)
    for g in (range(G) if groups is None else groups):
        xd = x[g].double()
        gt, u = xd @ wg[g].T, xd @ wu[g].T
        a = _FN[act](gt)
        h = a * u
        yg = h @ w3[g].T
        sg, su = xd.abs() @ wg[g].abs().T, xd.abs() @ wu[g].abs().T
        terms1 = (ACT_LIPSCHITZ * sg * u.abs() + a.abs() * su) @ w3[g].abs().T
        terms2 = h.abs() @ w3[g].abs().T
        if kernel == 'decode':
            bound[g] = U32 * yg.abs() + (C_ACC * (M + H) + 3) * U32 * (terms1 + terms2)
        else:
            bound[g] = U16 * yg.abs() + C_ACC * ((U16 + M * U32) * terms1 + (2 * U16 + H * U32) * terms2)
        y[g] = yg
    return y, bound


def stored_reference(x, qglu, sglu, q3t, s3t, act, kernel, groups=None):
    """``reference`` on the stored operands of LlamaFFNNetwork(weight_format='int4')."""
    wg, wu = split_glu(stored_values(qglu, sglu))
    return reference(x, wg, wu, stored_values(q3t, s3t), act, kernel, groups)


def check(y, ref, bound, counts=None):
    """Rows below each group's count within their bound, every other row exactly zero.  Returns the largest error / bound
    (<= 1 when it passes); raises AssertionError otherwise."""
    G, R = y.shape[:2]
    counts = [R] * G if counts is None else [min(int(c), R) for c in counts]
    worst = 0.0
    for g, c in enumerate(counts):
        if c > 0:
            err = (y[g, :c].double() - ref[g, :c]).abs()
            ratio = float(torch.where(err > 0, err / bound[g, :c], torch.zeros_like(err)).max())
            assert bool((err <= bound[g, :c]).all()), 'group %d: error %.3g x its bound' % (g, ratio)
            worst = max(worst, ratio)
        assert torch.count_nonzero(y[g, c:]) == 0, 'group %d: rows at or past the count %d are not zero' % (g, c)
    return worst
