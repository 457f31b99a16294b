"""Gate + routing kernels and a one-layer training step, softmax against sigmoid scoring (models/gates/top.py).

    python bench/gate_bench.py [--rounds 5] [--iters 50] [--out bench_out/gate_bench.json]

Kernel times: CUDA events around `iters` launches of gate_route_forward / sigmoid_gate_route_forward (two launches
each) and of the backward kernels, bf16 logits, S = 8192, at three router shapes:

    moonlight  E = 64,  k = 6, no groups
    deepseek   E = 256, k = 8, n_group = 8, topk_group = 4
    kimi       E = 384, k = 8, no groups

Step time: one MoE layer at a Moonlight-like shape (64 llama_ffn experts, top-6, model_dim 2048, hidden 1408, bf16,
8192 tokens), forward + backward + SGD step.  The two scoring modes alternate round by round in one process; every
number is the median over rounds.  The card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SHAPES = {'moonlight': (64, 6, 1, 1), 'deepseek': (256, 8, 8, 4), 'kimi': (384, 8, 1, 1)}
S = 8192


def _card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def _time(fn, iters):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / iters * 1e3          # microseconds per call


def kernel_calls(C, mode, E, k, G, TG):
    gen = torch.Generator('cuda').manual_seed(E)
    logits = torch.randn(S, E, device='cuda', generator=gen).to(torch.bfloat16)
    bias = torch.randn(E, device='cuda', generator=gen) * 0.1
    load = torch.zeros(E, device='cuda')
    cap = S * k // E * 2
    dl = torch.ones((), device='cuda', dtype=torch.bfloat16)
    dg = torch.randn(k, S, device='cuda', generator=gen)
    if mode == 'softmax':
        def fwd():
            return C.gate_route_forward(logits, k, cap, True, 0.0078125)
        out = fwd()

        def bwd():
            return C.gate_route_backward(out[0], out[1], out[2], dg, out[6], dl, logits, True, 0.0078125)
    else:
        def fwd():
            return C.sigmoid_gate_route_forward(logits, bias, k, cap, True, 0.0078125, G, TG, 2.5, load)
        out = fwd()

        def bwd():
            return C.sigmoid_gate_route_backward(out[0], out[1], out[2], dg, out[6], dl, logits, True, 0.0078125, 2.5)
    return fwd, bwd


def step_fn(mode):
    import torch.nn.functional as F  # noqa: F401
    from tutel_b200 import moe
    gate = {'type': 'top', 'k': 6}
    if mode == 'sigmoid':
        gate.update(scoring_func='sigmoid', routed_scaling_factor=2.5, bias_update_speed=1e-3)
    layer = moe.moe_layer(gate_type=gate, model_dim=2048,
                          experts={'type': 'llama_ffn', 'num_experts_per_device': 64, 'hidden_size_per_expert': 1408},
                          seeds=(1, 1, 1)).cuda().to(torch.bfloat16)
    opt = torch.optim.SGD(layer.parameters(), lr=1e-4)
    x = torch.randn(S, 2048, device='cuda', dtype=torch.bfloat16, generator=torch.Generator('cuda').manual_seed(0))

    def step():
        opt.zero_grad(set_to_none=True)
        y = layer(x)
        (y.float().pow(2).mean() + 1e-4 * y.l_aux.float()).backward()
        opt.step()
    return step


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--iters', type=int, default=50)
    ap.add_argument('--step-iters', type=int, default=10)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'gate_bench needs a GPU'
    from tutel_b200.ops import backend
    C = backend.require_ext()
    card = _card()
    calls = {(name, mode): kernel_calls(C, mode, *shape) for name, shape in SHAPES.items()
             for mode in ('softmax', 'sigmoid')}
    steps = {mode: step_fn(mode) for mode in ('softmax', 'sigmoid')}
    for f, b in calls.values():                  # warm-up: module loads, smem attributes, allocator
        for _ in range(5):
            f()
            b()
    for s in steps.values():
        for _ in range(3):
            s()
    torch.cuda.synchronize()
    samples = {}
    for _ in range(a.rounds):
        for (name, mode), (f, b) in calls.items():
            samples.setdefault((name, mode, 'fwd_us'), []).append(_time(f, a.iters))
            samples.setdefault((name, mode, 'bwd_us'), []).append(_time(b, a.iters))
        for mode, s in steps.items():
            samples.setdefault(('step', mode, 'ms'), []).append(_time(s, a.step_iters) / 1e3)
    result = {'card': card, 'S': S, 'rounds': a.rounds}
    for key, v in samples.items():
        result['/'.join(key)] = {'median': round(statistics.median(v), 3), 'min': round(min(v), 3),
                                 'max': round(max(v), 3)}
    line = json.dumps(result)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or '.', exist_ok=True)
        with open(a.out, 'w') as fh:
            fh.write(line + '\n')


if __name__ == '__main__':
    main()
