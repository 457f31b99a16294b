#!/usr/bin/env python3
"""Dropless training on one GPU: whole training steps (forward, backward, SGD step) of one MoE layer on the
expert-packed layout (a gate with capacity_factor=0) against the padded layout (the same layer with the non-binding
cap capacity_factor=-E, which pads every expert to the fullest one and reads that count back to the host).

    python bench/dropless_train_bench.py                                   # flagship ffn + llama_ffn, fine-grained ffn
    python bench/dropless_train_bench.py --shapes flagship --experts_types llama_ffn --repeats 5
    python bench/dropless_train_bench.py --fp8 block [--fp8_wgrad]       # block-fp8 experts (fp8_packed=True)

For each shape, expert type and routing (``skewed``: the gate weight favours a few experts; ``balanced``: a random
gate), the two layouts are timed alternately, ``--repeats`` rounds of ``--steps`` steps each after ``--warmup`` steps,
with CUDA events.  Prints one JSON line per configuration with the per-expert row counts, the work ratio
``E * max(count) / sum(roundup128(count))`` (expert-GEMM rows of the padded layout over those of the packed one), the
median step time of each layout, and the card name and power limit.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

SHAPES = {  # name -> (experts, top_k, model_dim, hidden, tokens)
    'flagship': (8, 2, 4096, 14336, 8192),
    'fine': (64, 6, 2048, 1408, 8192),
}

ap = argparse.ArgumentParser()
ap.add_argument('--shapes', default='flagship,fine')
ap.add_argument('--experts_types', default='ffn,llama_ffn', help='for the flagship shape; the fine-grained one runs ffn')
ap.add_argument('--routings', default='skewed,balanced')
ap.add_argument('--steps', type=int, default=5)
ap.add_argument('--warmup', type=int, default=2)
ap.add_argument('--repeats', type=int, default=3)
ap.add_argument('--fp8', default=None, choices=['block'],
                help="block: experts with fp8='block' and fp8_packed=True (block-scaled e4m3 GEMMs on both layouts)")
ap.add_argument('--fp8_wgrad', action='store_true', help='with --fp8 block: block-scaled e4m3 weight gradients too')
ap.add_argument('--profile', default=None, metavar='DIR',
                help='also write a torch.profiler table of --steps steps of each layout per configuration into DIR')
args = ap.parse_args()


def card():
    name = torch.cuda.get_device_name()
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i',
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:  # noqa
        out = 'unknown'
    return name, out


def build(kind, E, k, M, H, routing):
    from tutel_b200 import moe
    torch.manual_seed(0)
    experts = {'type': kind, 'num_experts_per_device': E, 'hidden_size_per_expert': H}
    if args.fp8 == 'block':
        experts.update(fp8='block', fp8_packed=True, fp8_wgrad=args.fp8_wgrad)
    if kind == 'ffn':
        experts['activation_fn'] = F.relu
    layer = moe.moe_layer(gate_type={'type': 'top', 'k': k, 'capacity_factor': 0}, model_dim=M, experts=experts,
                          seeds=(1, 2, 3)).cuda().bfloat16()
    if routing == 'skewed':
        with torch.no_grad():
            w = layer.gates[0].wg.weight
            w.mul_(2.0)
            w[: max(E // 8, 1)] += 0.02
    return layer


def time_steps(layer, opt, x, cf, n):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(n):
        opt.zero_grad(set_to_none=True)
        y = layer(x, capacity_factor=cf)
        (y.float().pow(2).mean() + 0.01 * y.l_aux.float()).backward()
        opt.step()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / n


def profile_steps(layer, opt, x, cf, name):
    """Device time per kernel over --steps steps (a separate run from the timed rounds: tracing slows the host)."""
    from torch.profiler import ProfilerActivity, profile
    os.makedirs(args.profile, exist_ok=True)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        time_steps(layer, opt, x, cf, args.steps)
    with open(os.path.join(args.profile, name + '.txt'), 'w') as f:
        f.write(prof.key_averages().table(sort_by='cuda_time_total', row_limit=40, max_name_column_width=90))


def main():
    if args.fp8_wgrad and args.fp8 != 'block':
        raise SystemExit('--fp8_wgrad needs --fp8 block')
    name, power = card()
    precision = 'bf16' if args.fp8 is None else 'block_fp8' + ('+fp8_wgrad' if args.fp8_wgrad else '')
    for shape in args.shapes.split(','):
        E, k, M, H, S = SHAPES[shape]
        kinds = args.experts_types.split(',') if shape == 'flagship' else ['ffn']
        for kind in kinds:
            for routing in args.routings.split(','):
                layer = build(kind, E, k, M, H, routing)
                opt = torch.optim.SGD(layer.parameters(), lr=1e-6)
                x = torch.randn(S, M, device='cuda', dtype=torch.bfloat16)
                with torch.no_grad():
                    layer(x, capacity_factor=-E)
                counts = [int(c) for c in layer.dispatch_count.cpu()]
                packed_rows = sum((c + 127) // 128 * 128 for c in counts)
                modes = {'packed': None, 'padded': -E}
                for cf in modes.values():
                    time_steps(layer, opt, x, cf, args.warmup)
                times = {m: [] for m in modes}
                for _ in range(args.repeats):
                    for m, cf in modes.items():
                        times[m].append(time_steps(layer, opt, x, cf, args.steps))
                med = {m: sorted(v)[len(v) // 2] for m, v in times.items()}
                if args.profile:
                    for m, cf in modes.items():
                        profile_steps(layer, opt, x, cf, '%s_%s_%s_%s_%s' % (precision, shape, kind, routing, m))
                print(json.dumps({
                    'shape': shape, 'experts': kind, 'routing': routing, 'E': E, 'top_k': k, 'model_dim': M, 'hidden': H,
                    'tokens': S, 'dtype': 'bfloat16', 'experts_precision': precision, 'counts': counts,
                    'work_ratio': round(E * max(counts) / max(packed_rows, 1), 3),
                    'packed_step_ms': [round(t, 3) for t in times['packed']],
                    'padded_step_ms': [round(t, 3) for t in times['padded']],
                    'median_ms': {m: round(t, 3) for m, t in med.items()},
                    'speedup': round(med['padded'] / med['packed'], 3), 'card': name, 'power_limit': power}), flush=True)
                del layer, opt, x
                torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
