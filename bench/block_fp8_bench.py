#!/usr/bin/env python3
"""Block-scaled fp8 (``fp8='block'``, DeepSeek-V3 recipe) against the other expert GEMM recipes on one GPU.

    python bench/block_fp8_bench.py                       # everything below
    python bench/block_fp8_bench.py --parts gemm --iters 50

Three parts, each printing JSON lines with the card name and power limit:

* ``gemm``: kernel time and TFLOP/s at the flagship expert shapes (8 experts, 2048 rows each; fc1 4096 -> 14336 and
  fc2 14336 -> 4096) for the bf16 grouped GEMM, row-scaled e4m3, MX and block-scaled e4m3, CUDA events over ``--iters``
  launches after a warm-up.  Operand quantisation is not timed.  The weight-gradient shapes (``wgrad``: 14336 x 4096,
  the ``ffn`` dW1 and dW2; ``wgrad_glu``: 4096 x 28672, the ``llama_ffn`` [dW1 | dW2] in one split launch) over K = 2048
  tokens per expert time the bf16 GEMM on the 16-bit activations against ``block_wgrad``, the block-scaled GEMM on
  column-wise e4m3 copies; ``dual_quant`` is the dual quantiser on one [8, 2048, 14336] activation.
* ``accuracy``: max |err| / max |ref| against an fp64 product of the same bf16 operands, row-scaled and block-scaled,
  at K = 4096 and 14336 (1024 x 1024 outputs), quantisation included; and of the weight-gradient GEMM ``a^T b`` over
  K = 2048 and 16384 tokens, bf16 and block-scaled.
* ``train``: whole training steps (forward, backward, SGD) of the flagship ``ffn`` (ReLU) and ``llama_ffn`` layers
  (top-2 of 8, 4096 / 14336, 8192 tokens, capacity factor 1) in bf16, row, MX (ffn only), block and block with
  ``fp8_wgrad``, alternated in ``--rounds`` rounds of ``--steps`` steps; median step time and peak memory
  (``torch.cuda.max_memory_allocated`` over the mode's steps) per mode.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument('--parts', default='gemm,accuracy,train')
ap.add_argument('--iters', type=int, default=30)
ap.add_argument('--steps', type=int, default=5)
ap.add_argument('--warmup', type=int, default=2)
ap.add_argument('--rounds', type=int, default=3)
ap.add_argument('--tokens', type=int, default=8192)
args = ap.parse_args()


def card():
    name = torch.cuda.get_device_name()
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i',
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:  # noqa
        out = 'unknown'
    return {'gpu': name, 'power_limit': out}


def emit(**kw):
    print(json.dumps(dict(kw, **CARD)), flush=True)


def timed(fn, iters):
    for _ in range(3):
        fn()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / iters


def gemm_part():
    from tutel_b200.ops import block_fp8 as BF
    from tutel_b200.ops import gemm as G
    from tutel_b200.ops import mx as MX
    E, T = 8, 2048
    for name, K, N in (('fc1', 4096, 14336), ('fc2', 14336, 4096)):
        torch.manual_seed(0)
        x = torch.randn(E, T, K, device='cuda').bfloat16()
        w = (torch.randn(E, N, K, device='cuda') * K ** -0.5).bfloat16()
        xq, sx = G.quantize_rows(x)
        wq, sw = G.quantize_rows(w)
        xm, sxm = MX.mx_quantize(x)
        wm, swm = MX.mx_quantize(w)
        xb, sxb = BF.quantize_act(x)
        wb, swb, _, _ = BF.quantize_weight(w)
        flops = 2.0 * E * T * N * K
        runs = {
            'bf16': lambda: G.raw_gemm(x, w),
            'row': lambda: G.raw_gemm(xq, wq, out_dtype=torch.bfloat16, scale_a=sx, scale_b=sw),
            'mx': lambda: MX.mx_gemm(xm, sxm, wm, swm),
            'block': lambda: BF.block_fp8_gemm(xb, sxb, wb, swb),
        }
        for mode, fn in runs.items():
            ms = timed(fn, args.iters)
            emit(part='gemm', shape=name, experts=E, rows=T, K=K, N=N, mode=mode, ms=round(ms, 4),
                 tflops=round(flops / ms / 1e9, 1))
        del x, w, xq, wq, xm, wm, xb, wb
    # weight gradients: D [E, Ma, N] = a^T b over the T tokens of each expert
    for name, Ma, N in (('wgrad', 14336, 4096), ('wgrad_glu', 4096, 2 * 14336)):
        torch.manual_seed(0)
        a = torch.randn(E, T, Ma, device='cuda').bfloat16()
        b = (torch.randn(E, T, N, device='cuda') * 1e-3).bfloat16()
        _, _, aT, saT = BF.quantize_act_dual(a, rowwise=False)
        _, _, bT, sbT = BF.quantize_act_dual(b, rowwise=False)
        split = N // 2 if name == 'wgrad_glu' else None
        flops = 2.0 * E * Ma * N * T
        runs = {
            'bf16': lambda: G.raw_gemm(a, b, a_mn=True, b_mn=True),
            'block_wgrad': lambda: BF.wgrad_gemm(aT, saT, bT, sbT, split=split),
        }
        for mode, fn in runs.items():
            ms = timed(fn, args.iters)
            emit(part='gemm', shape=name, experts=E, rows=Ma, K=T, N=N, mode=mode, ms=round(ms, 4),
                 tflops=round(flops / ms / 1e9, 1))
        if name == 'wgrad':
            ms = timed(lambda: BF.quantize_act_dual(a), args.iters)
            emit(part='gemm', shape='dual_quant', experts=E, rows=T, K=Ma, mode='block', ms=round(ms, 4),
                 gbps=round(E * T * Ma * (2 + 2 + 8 / 128) / ms / 1e6, 1))
        del a, b, aT, bT


def accuracy_part():
    from tutel_b200.ops import block_fp8 as BF
    from tutel_b200.ops import gemm as G
    M = N = 1024
    for K in (4096, 14336):
        gen = torch.Generator(device='cuda').manual_seed(K)
        x = torch.randn(1, M, K, device='cuda', generator=gen).bfloat16()
        w = (torch.randn(1, N, K, device='cuda', generator=gen) * K ** -0.5).bfloat16()
        ref = x.double() @ w.double().transpose(1, 2)
        scale = float(ref.abs().max())
        xq, sx = G.quantize_rows(x)
        wq, sw = G.quantize_rows(w)
        row = G.raw_gemm(xq, wq, out_dtype=torch.float32, scale_a=sx, scale_b=sw)
        xb, sxb = BF.quantize_act(x)
        wb, swb, _, _ = BF.quantize_weight(w)
        blk = BF.block_fp8_gemm(xb, sxb, wb, swb)[0]
        for mode, out in (('row', row), ('block', blk)):
            emit(part='accuracy', K=K, M=M, N=N, mode=mode, output=str(out.dtype).replace('torch.', ''),
                 max_err_over_max_ref=float((out.double() - ref).abs().max()) / scale)
    for T in (2048, 16384):
        gen = torch.Generator(device='cuda').manual_seed(T)
        a = torch.randn(1, T, M, device='cuda', generator=gen).bfloat16()
        b = (torch.randn(1, T, N, device='cuda', generator=gen) * 1e-3).bfloat16()
        ref = a.double().transpose(1, 2) @ b.double()
        scale = float(ref.abs().max())
        bf = G.raw_gemm(a, b, a_mn=True, b_mn=True)
        blk = BF.wgrad_gemm(*BF.quantize_act_dual(a, rowwise=False)[2:], *BF.quantize_act_dual(b, rowwise=False)[2:])[0]
        for mode, out in (('bf16', bf), ('block_wgrad', blk)):
            emit(part='accuracy', shape='wgrad', K=T, M=M, N=N, mode=mode, output=str(out.dtype).replace('torch.', ''),
                 max_err_over_max_ref=float((out.double() - ref).abs().max()) / scale)


def train_part():
    from tutel_b200 import moe
    from tutel_b200.ops import gemm as G
    M, H, E = 4096, 14336, 8
    for kind in ('ffn', 'llama_ffn'):
        modes = ['bf16', 'row', 'mx', 'block', 'block+wgrad'] if kind == 'ffn' else ['bf16', 'row', 'block', 'block+wgrad']
        layers = {}
        for mode in modes:
            torch.manual_seed(0)
            experts = {'type': kind, 'num_experts_per_device': E, 'hidden_size_per_expert': H}
            if kind == 'ffn':
                experts['activation_fn'] = lambda t: F.relu(t)
            if mode == 'block+wgrad':
                experts.update(fp8='block', fp8_wgrad=True)
            elif mode != 'bf16':
                experts['fp8'] = mode
            layer = moe.moe_layer(gate_type={'type': 'top', 'k': 2, 'capacity_factor': 1.0}, model_dim=M,
                                  experts=experts, seeds=(1, 2, 3)).cuda().bfloat16()
            layers[mode] = (layer, torch.optim.SGD(layer.parameters(), lr=1e-5))
        x = torch.randn(2, args.tokens // 2, M, device='cuda').bfloat16().requires_grad_(True)

        def step(mode):
            layer, opt = layers[mode]
            opt.zero_grad(set_to_none=True)
            x.grad = None
            y = layer(x)
            (y.float().pow(2).mean() + 0.01 * y.l_aux.float()).backward()
            opt.step()

        times = {m: [] for m in modes}
        peak = {m: 0 for m in modes}
        for m in modes:
            for _ in range(args.warmup):
                step(m)
        for _ in range(args.rounds):
            for m in modes:
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                ms = timed(lambda: step(m), args.steps)
                times[m].append(ms)
                peak[m] = max(peak[m], torch.cuda.max_memory_allocated())
                G.invalidate_fp8_cache()
        for m in modes:
            emit(part='train', expert=kind, mode=m, model_dim=M, hidden=H, experts=E, tokens=args.tokens,
                 median_step_ms=round(statistics.median(times[m]), 3), rounds=[round(t, 3) for t in times[m]],
                 peak_mem_gib=round(peak[m] / 2 ** 30, 3))
        del layers


if __name__ == '__main__':
    assert torch.cuda.is_available(), 'block_fp8_bench.py needs a GPU'
    CARD = card()
    parts = args.parts.split(',')
    if 'gemm' in parts:
        gemm_part()
    if 'accuracy' in parts:
        accuracy_part()
    if 'train' in parts:
        train_part()
