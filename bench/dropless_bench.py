#!/usr/bin/env python3
"""BASELINE config #4: dropless (capacity_factor=0) decoder-style inference, 128 local experts on one GPU,
32 tokens, top-1, model_dim = hidden = 2048, fp32 - the reference's "Megablocks" demo (README.md:52-58).

    python bench/dropless_bench.py --impl ours      --megablocks_size 1
    python bench/dropless_bench.py --impl reference --megablocks_size 1
    python bench/dropless_bench.py --expert_type llama_ffn --experts 8 --dim 4096 --hidden 14336 --top_k 2 \\
        --tokens 1 --dtype bfloat16                                   # Mixtral-like SwiGLU decode step

`--megablocks_size 0` times the padded path (the capacity is read back to the host, every expert computes the whole
buffer).  With `--megablocks_size 1` only the experts that received tokens cost anything: up to 64 rows per expert the
whole expert is one weight-streaming launch (`ffn`: skinny_ffn_kernel, `llama_ffn`: skinny_glu_ffn_kernel), above that
the wgmma kernels skip rows past the device-side counts.
Device-timed forward latency (CUDA events, L2 flushed between iterations), one JSON line with the number of active
experts (experts that received at least one token), the weight bytes those experts hold, and those bytes over the median
time (`active_weight_GBps`: the weight bandwidth the dropless path needs, whatever the path actually read).  The expert
module alone is timed the same way on the dispatch buffer of one call (`experts_median_ms`,
`experts_active_weight_GBps`), and the output is compared with the padded path (`rel_err_vs_padded`).

`--fp8` builds fp8 experts (`fp8=True`: e4m3 weight copies with one fp32 scale per row; in dropless decoding the skinny
kernels `skinny_ffn_fp8_kernel` / `skinny_glu_ffn_fp8_kernel` stream those copies, x stays 16 bit).  With it,
`active_weight_bytes` and both `*_GBps` count the bytes that path needs - the e4m3 copies, their fp32 scales and any
biases - not the bytes of the 16-bit master parameters.  `rel_err_vs_padded` then compares with the padded fp8 path.

`--fp8_weights` (`llama_ffn`, bfloat16) builds the experts with `weight_format='fp8_block'`: block-scaled e4m3 weights
(DeepSeek-V3 checkpoint format, one fp32 scale per 128 x 128 block) and no 16-bit copy, loaded from the export of a bf16
`fp8='block'` layer.  Dropless decoding streams them with `skinny_glu_ffn_block_fp8_kernel`; larger steps run the block
GEMMs with device row counts.  `active_weight_bytes` counts the e4m3 bytes and their scales.  `expert_memory_bytes` is
what the expert module holds; with `--fp8_weights`, `bf16_block_expert_memory_bytes` is what the source bf16
`fp8='block'` layer held after one forward (its parameters and the cached e4m3 copies).
`--int4_weights` (`llama_ffn`, bfloat16) builds the experts with `weight_format='int4'` (group-32 int4, one bf16 scale
per 32 input elements, doc/INT4.md), loaded from `export_int4_weights()` of a bf16 layer.  Dropless decoding streams them
with `skinny_glu_ffn_int4_kernel`; larger steps run the mixed-input GEMM `w4a16_gemm_kernel` with device row counts.
`active_weight_bytes` counts the nibbles and their scales.  `--shared_int4 0` keeps the shared experts 16-bit
(`shared_experts={'weight_format': None}`, as Kimi-K2-Thinking ships them); the JSON records `shared_format`.
`--shared_experts N` adds N shared experts (DeepSeek-V3: 1).
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ap = argparse.ArgumentParser()
ap.add_argument('--impl', default='ours', choices=['ours', 'reference'])
ap.add_argument('--megablocks_size', type=int, default=1)
ap.add_argument('--expert_type', default='ffn', choices=['ffn', 'llama_ffn'])
ap.add_argument('--experts', type=int, default=128)
ap.add_argument('--tokens', type=int, default=32)
ap.add_argument('--top_k', type=int, default=1)
ap.add_argument('--dim', type=int, default=2048)
ap.add_argument('--hidden', type=int, default=0, help='hidden size per expert (default: --dim)')
ap.add_argument('--dtype', default='float32')
ap.add_argument('--iters', type=int, default=50)
ap.add_argument('--fp8', action='store_true', help='fp8 experts (e4m3 weights with per-row scales); 16-bit --dtype only')
ap.add_argument('--fp8_weights', action='store_true',
                help="llama_ffn, bfloat16: stored block-fp8 experts (weight_format='fp8_block') with no 16-bit copy")
ap.add_argument('--int4_weights', action='store_true',
                help="llama_ffn, bfloat16: group-32 int4 experts (weight_format='int4') exported from a bf16 layer")
ap.add_argument('--shared_int4', type=int, default=1, help='with --int4_weights: 1 int4 shared experts, 0 16-bit ones')
ap.add_argument('--shared_experts', type=int, default=0, help='shared experts of the routed type (0: none)')
ap.add_argument('--graph', action='store_true', help='ours only: replay the forward as one CUDA graph (tutel_b200.utils.graph)')
args = ap.parse_args()
hidden = args.hidden or args.dim
assert not args.fp8 or (args.impl == 'ours' and args.dtype in ('bfloat16', 'float16')), '--fp8: ours, with a 16-bit --dtype'
assert not args.fp8_weights or (args.impl == 'ours' and args.dtype == 'bfloat16' and args.expert_type == 'llama_ffn' and
                                not args.fp8), '--fp8_weights: ours, llama_ffn, bfloat16, without --fp8'
assert not args.int4_weights or (args.impl == 'ours' and args.dtype == 'bfloat16' and args.expert_type == 'llama_ffn' and
                                 not args.fp8 and not args.fp8_weights), '--int4_weights: ours, llama_ffn, bfloat16, alone'
if args.impl == 'reference':
    sys.path.insert(0, os.path.join(ROOT, 'baseline', '_ref'))
    from tutel import moe, system
else:
    sys.path.insert(0, ROOT)
    from tutel_b200 import moe, system
import torch
import torch.nn.functional as F

env = system.init_data_model_parallel(backend='nccl')
dev = env.local_device
torch.set_default_dtype(getattr(torch, args.dtype))
torch.manual_seed(0)
experts = {'type': args.expert_type, 'num_experts_per_device': args.experts, 'hidden_size_per_expert': hidden}
if args.expert_type == 'ffn':
    experts['activation_fn'] = lambda x: F.relu(x)
if args.fp8:
    experts['fp8'] = True
shared = {'shared_experts': {'num_experts': args.shared_experts}} if args.shared_experts else {}


def build(spec):
    with torch.device(dev):        # initialise the (multi-GB) weights on the GPU
        return moe.moe_layer(gate_type={'type': 'top', 'k': args.top_k, 'capacity_factor': 0.0}, model_dim=args.dim,
                             experts=spec, seeds=(1, 1, 1), **shared).eval()


def module_bytes(m):
    return sum(t.numel() * t.element_size() for t in list(m.parameters()) + list(m.buffers()))


bf16_block_bytes = None
if args.fp8_weights:
    from tutel_b200.ops import block_fp8 as BF8
    src = build(dict(experts, fp8='block'))
    with torch.no_grad():
        src(torch.randn(1, 256, args.dim, device=dev))        # one padded forward: the block path caches its e4m3 copies
    cached = sum(t.numel() * t.element_size() for v in BF8._WEIGHT_CACHE.values() for t in v[1])
    bf16_block_bytes = module_bytes(src.experts) + cached
    layer = build(dict(experts, weight_format='fp8_block'))
    layer.load_state_dict({k: v for k, v in src.state_dict().items() if not k.startswith(('experts.', 'shared_experts.'))},
                          strict=False)
    layer.experts.load_fp8_block_weights(*src.experts.export_fp8_block_weights())
    if args.shared_experts:
        layer.shared_experts.load_fp8_block_weights(*src.shared_experts.export_fp8_block_weights())
    del src
    BF8._WEIGHT_CACHE.clear()
    torch.cuda.empty_cache()
elif args.int4_weights:
    src = build(experts)
    if args.shared_experts and not args.shared_int4:
        shared['shared_experts'] = dict(shared['shared_experts'], weight_format=None)
    layer = build(dict(experts, weight_format='int4'))
    layer.load_state_dict({k: v for k, v in src.state_dict().items() if not k.startswith(('experts.', 'shared_experts.'))},
                          strict=False)
    layer.experts.load_int4_weights(*src.experts.export_int4_weights())
    if args.shared_experts and args.shared_int4:
        layer.shared_experts.load_int4_weights(*src.shared_experts.export_int4_weights())
    elif args.shared_experts:
        layer.shared_experts.load_state_dict(src.shared_experts.state_dict())
    del src
    torch.cuda.empty_cache()
else:
    layer = build(experts)
x = torch.randn(1, args.tokens, args.dim, device=dev)
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
eager = (lambda t: layer(t, megablocks_size=args.megablocks_size)) if args.megablocks_size > 0 else (lambda t: layer(t))
call = eager
if args.graph and args.impl == 'ours':
    from tutel_b200.utils.graph import GraphedForward
    call = GraphedForward(eager, x)


def timed(fn, iters):
    times = []
    for i in range(iters + 5):
        flush.zero_()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        out = fn()
        e.record()
        torch.cuda.synchronize()
        if i >= 5:
            times.append(s.elapsed_time(e))
    return out, sorted(times)


with torch.no_grad():
    y, times = timed(lambda: call(x), args.iters)
    y = y.clone()
    active = int((layer.dispatch_count > 0).sum())       # counts of the timed call (a graph replay refreshes them too)
    # the experts alone (no gate, routing, encode, decode), on the dispatch buffer of one eager call of the same mode
    bufs = []
    hook = layer.experts.register_forward_pre_hook(lambda m, a: bufs.append(a[0]))
    eager(x)
    hook.remove()
    _, expert_times = timed(lambda: layer.experts(bufs[-1], layer), args.iters)
    padded = layer(x)


def expert_bytes():
    """Weight bytes one expert's forward reads: the parameters, or with --fp8 the e4m3 copies (1 byte per weight), one
    fp32 scale per quantised row (ops/gemm.py: fp8_weight) and the 16-bit biases."""
    e = layer.experts
    if args.fp8_weights or args.int4_weights:   # stored W_gate_up [2H, M] + W_down [M, H] bytes and their scales
        return module_bytes(e) // args.experts
    if not args.fp8:
        return sum(p.numel() * p.element_size() for p in e.parameters()) // args.experts
    M, H, N = args.dim, hidden, args.dim
    if args.expert_type == 'ffn':          # Q1 [H, M] + s1 [H], Q2^T [N, H] + s2 [N], biases
        biases = sum(p.numel() * p.element_size() for p in (e.batched_fc1_bias, e.batched_fc2_bias) if p is not None)
        return H * M + N * H + 4 * (H + N) + biases // args.experts
    return 2 * H * M + N * H + 4 * (2 * H + N)   # Q1^T, Q2^T [H, M] + s1, s2 [H], Q3^T [N, H] + s3 [N]


bytes_per_expert = expert_bytes()
median, expert_median = times[len(times) // 2], expert_times[len(expert_times) // 2]
config = 'dropless cf=0 top-%d E=%d tokens=%d dim=%d hidden=%d %s %s megablocks_size=%d%s%s' % (
    args.top_k, args.experts, args.tokens, args.dim, hidden, args.expert_type, args.dtype, args.megablocks_size,
    ' fp8' if args.fp8 else '', ' cuda-graph' if args.graph and args.impl == 'ours' else '')
config += ' fp8_weights' if args.fp8_weights else ''
config += ' int4_weights' if args.int4_weights else ''
config += ' shared=%d' % args.shared_experts if args.shared_experts else ''
shared_format = None
if args.shared_experts:
    shared_format = getattr(layer.shared_experts, 'weight_format', None) or args.dtype
print(json.dumps({'impl': args.impl, 'config': config, 'median_ms': median, 'min_ms': times[0], 'max_ms': times[-1],
    'experts_median_ms': expert_median, 'active_experts': active, 'active_weight_bytes': active * bytes_per_expert,
    'active_weight_GBps': active * bytes_per_expert / (median * 1e-3) / 1e9,
    'experts_active_weight_GBps': active * bytes_per_expert / (expert_median * 1e-3) / 1e9,
    'rel_err_vs_padded': float((y.float() - padded.float()).norm() / padded.float().norm()),
    'checksum': float(y.float().abs().sum()), 'expert_memory_bytes': module_bytes(layer.experts),
    'bf16_block_expert_memory_bytes': bf16_block_bytes, 'shared_format': shared_format}))
