#!/usr/bin/env python3
"""Group-32 int4 expert weights (``weight_format='int4'``) against bf16 and block-scaled fp8 at the flagship expert
shapes: 8 experts, 2048 rows each, model 4096, hidden 14336.

    python bench/int4_bench.py --iters 30

Prints one JSON line per arm with CUDA-event times (median of ``--iters`` launches after a warm-up), TFLOP/s from shapes
(2 * rows * N * K per expert; the GLU arm counts both halves) and the card name and power limit:

* ``glu``:  h = act(x W1) * (x W2), [8, 2048, 4096] -> [8, 2048, 14336];
* ``down``: y = h W3, [8, 2048, 14336] -> [8, 2048, 4096];

each as ``bf16`` (the dual-B / plain wgmma GEMMs on bf16 weights), ``block_fp8`` (the stored block-fp8 GEMMs, the
activation quantisation included) and ``int4`` (``w4a16_gemm_kernel``, the mixed-input GEMM that expands the nibbles in
shared memory).  Arms alternate over ``--rounds`` rounds; each line is one round.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from tutel_b200.ops import block_fp8 as BF8  # noqa: E402
from tutel_b200.ops import gemm as G  # noqa: E402
from tutel_b200.ops import int4 as I4  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument('--iters', type=int, default=30)
ap.add_argument('--rounds', type=int, default=3)
ap.add_argument('--experts', type=int, default=8)
ap.add_argument('--rows', type=int, default=2048)
ap.add_argument('--dim', type=int, default=4096)
ap.add_argument('--hidden', type=int, default=14336)
args = ap.parse_args()


def card():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i',
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:  # noqa
        out = 'unknown'
    return {'gpu': torch.cuda.get_device_name(), 'power_limit': out}


def timed(fn, iters):
    for _ in range(3):
        fn()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = []
    for _ in range(iters):
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        times.append(s.elapsed_time(e))
    return sorted(times)[len(times) // 2]


def main():
    assert torch.cuda.is_available(), 'int4_bench needs a GPU'
    info = card()
    E, Rw, M, H = args.experts, args.rows, args.dim, args.hidden
    torch.manual_seed(0)
    x = torch.randn(E, Rw, M, device='cuda').bfloat16()
    h = torch.randn(E, Rw, H, device='cuda').bfloat16()
    w1, w2 = ((torch.randn(E, M, H, device='cuda') * 0.02).bfloat16() for _ in range(2))
    w3 = (torch.randn(E, H, M, device='cuda') * 0.02).bfloat16()
    qglu, sglu, q3t, s3t = I4.load_glu_weights(*I4.export_glu_weights(w1, w2, w3))
    wg, wu = (w.bfloat16().contiguous() for w in I4._split_glu(I4.stored_values(qglu, sglu)))
    down = I4.stored_values(q3t, s3t).bfloat16().contiguous()
    gate, up = wg, wu
    del w1, w2, w3
    torch.cuda.empty_cache()
    bq = BF8.load_glu_weights(*BF8.export_glu_weights(gate.transpose(1, 2).contiguous(), up.transpose(1, 2).contiguous(),
                                                      down.transpose(1, 2).contiguous()))
    flops = {'glu': 2.0 * E * Rw * 2 * H * M, 'down': 2.0 * E * Rw * M * H}
    arms = {
        ('glu', 'bf16'): lambda: G.glu_gemm(x, gate, up, b_mn=False, act='silu'),
        ('glu', 'block_fp8'): lambda: BF8.block_fp8_gemm(*BF8.quantize_act(x), bq[0], bq[1], epilogue=BF8.EPI_GLU, act='silu'),
        ('glu', 'int4'): lambda: I4.w4a16_gemm(x, qglu, sglu, 'silu'),
        ('down', 'bf16'): lambda: G.raw_gemm(h, down),
        ('down', 'block_fp8'): lambda: BF8.block_fp8_gemm(*BF8.quantize_act(h), bq[2], bq[3]),
        ('down', 'int4'): lambda: I4.w4a16_gemm(h, q3t, s3t),
    }
    with torch.no_grad():
        for rnd in range(args.rounds):
            for (gemm, mode), fn in arms.items():
                ms = timed(fn, args.iters)
                print(json.dumps(dict(info, round=rnd, gemm=gemm, mode=mode, experts=E, rows=Rw, dim=M, hidden=H, ms=ms,
                                      tflops=flops[gemm] / (ms * 1e-3) / 1e12)), flush=True)


if __name__ == '__main__':
    main()
