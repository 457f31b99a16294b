#!/usr/bin/env python3
"""Per-kernel device time of the flagship training step (torch.profiler / CUPTI), rank 0 only.
    torchrun --nproc-per-node=2 bench/profile_step.py --out bench_out/step_profile_2gpu.txt"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch
import torch.nn.functional as F
from torch.profiler import ProfilerActivity, profile

ap = argparse.ArgumentParser()
ap.add_argument('--out', type=str, default=os.path.join(ROOT, 'bench_out', 'step_profile.txt'))
ap.add_argument('--steps', type=int, default=5)
ap.add_argument('--experts', type=int, default=8)
ap.add_argument('--expert_type', type=str, default='ffn')
ap.add_argument('--overlap', type=int, default=1)
ap.add_argument('--fp8', action='store_true')
ap.add_argument('--reference', action='store_true', help='profile the unmodified reference (baseline/_ref) instead')
args = ap.parse_args()
if args.reference:
    sys.path.insert(0, os.path.join(ROOT, 'baseline', '_ref'))
    from tutel import moe, net, system
else:
    from tutel_b200 import moe, net, system

env = system.init_data_model_parallel(backend='nccl')
rank, world, dev = env.global_rank, env.global_size, env.local_device
torch.set_default_dtype(torch.bfloat16)
layer = moe.moe_layer(gate_type={'type': 'top', 'k': 2, 'capacity_factor': 1.0}, model_dim=4096,
                      experts={'type': args.expert_type, 'num_experts_per_device': args.experts // world, 'hidden_size_per_expert': 14336,
                               'activation_fn': lambda x: F.relu(x), **({'fp8': True} if args.fp8 else {})},
                      scan_expert_func=lambda n, p: setattr(p, 'skip_allreduce', True), seeds=(1, rank + 1, 1), a2a_ffn_overlap_degree=args.overlap).to(dev)
opt = torch.optim.SGD(layer.parameters(), lr=1e-5)
shared = [p for p in layer.parameters() if not hasattr(p, 'skip_allreduce')]
torch.manual_seed(rank)
x = torch.randn(16, 512, 4096, device=dev).requires_grad_(True)      # as in bench.py: the input gradient is part of the step
y = torch.zeros(16, dtype=torch.int64, device=dev)


def step():
    opt.zero_grad()
    x.grad = None
    loss = F.nll_loss(F.log_softmax(torch.sum(layer(x), dim=2), dim=1), y)
    loss.backward()
    if world > 1:
        for p in shared:
            p.grad /= world
            p.grad = net.simple_all_reduce(p.grad)
    opt.step()


for _ in range(4):
    step()
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
    for _ in range(args.steps):
        step()
    torch.cuda.synchronize()
if rank == 0:
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    rows = []
    for e in prof.key_averages():
        t = getattr(e, 'device_time_total', 0) or getattr(e, 'cuda_time_total', 0)
        if t > 0 and e.device_type.name == 'CUDA':
            rows.append((t / args.steps, e.count / args.steps, e.key))
    rows.sort(reverse=True)
    with open(args.out, 'w') as f:
        f.write('# per-step device time (us), launches per step, kernel  [world=%d fused=%s]\n' % (world, os.environ.get('TUTEL_B200_FUSED', '1')))
        f.write('# total kernel time per step: %.1f us\n' % sum(r[0] for r in rows))
        for t, c, k in rows:
            f.write('%10.1f %6.1f  %s\n' % (t, c, k[:160]))
    # timeline of the last profiled step: start offset (us), duration (us), stream, kernel
    evs = [e for e in prof.events() if e.device_type.name == 'CUDA' and e.time_range.end > e.time_range.start]
    evs.sort(key=lambda e: e.time_range.start)
    if evs:
        t_end = evs[-1].time_range.end
        span = (t_end - evs[0].time_range.start) / args.steps
        last = [e for e in evs if e.time_range.start >= t_end - span * 1.02 and not e.name.startswith('Optimizer')]
        t0 = last[0].time_range.start
        with open(args.out.replace('.txt', '_timeline.txt'), 'w') as f:
            f.write('# start_us dur_us stream kernel (last profiled step, rank 0)\n')
            for e in last:
                f.write('%9.1f %8.1f %3s  %s\n' % (e.time_range.start - t0, e.time_range.end - e.time_range.start,
                                                   getattr(e, 'device_index', ''), e.name[:110]))
    print(open(args.out).read()[:3000])
