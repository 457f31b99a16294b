#!/usr/bin/env python3
"""Shared experts on one GPU: what the shared term in the combine kernel costs and saves, on a Moonlight-like layer
(64 experts, top-6, model_dim 2048, hidden 1408 per expert, 2 shared experts, bf16, 8192 tokens, sigmoid gate with
8 groups of which 4 are kept).

    python bench/shared_expert_bench.py
    python bench/shared_expert_bench.py --experts_type ffn --repeats 7

Configurations, run in one process and alternated, ``--repeats`` rounds each, median reported:

* ``shared``: the layer with ``shared_experts={'num_experts': 2}`` (the shared output is added inside the combine);
* ``routed``: the same layer without shared experts;
* ``workaround``: the layer without shared experts plus a separate identical expert module of hidden size 2H, added
  with ``y + shared(x)`` outside the layer.

Training steps (forward, backward, SGD step) run on the packed dropless path (``capacity_factor=0``).  Decoding steps
are no-grad forwards of 1 and 4 tokens on the bound-based dropless path (``megablocks_size=1``).  Times come from CUDA
events around ``--steps`` steps (training) or ``--decode_steps`` forwards (decoding).  One JSON line per step kind,
with the card name and power limit.
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

ap = argparse.ArgumentParser()
ap.add_argument('--experts_type', default='llama_ffn', choices=['llama_ffn', 'ffn'])
ap.add_argument('--experts', type=int, default=64)
ap.add_argument('--top_k', type=int, default=6)
ap.add_argument('--model_dim', type=int, default=2048)
ap.add_argument('--hidden', type=int, default=1408)
ap.add_argument('--num_shared', type=int, default=2)
ap.add_argument('--tokens', type=int, default=8192)
ap.add_argument('--steps', type=int, default=5)
ap.add_argument('--decode_steps', type=int, default=50)
ap.add_argument('--warmup', type=int, default=2)
ap.add_argument('--repeats', type=int, default=5)
args = ap.parse_args()


def card():
    name = torch.cuda.get_device_name()
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i',
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:  # noqa
        out = 'unknown'
    return name, out


def experts_spec():
    spec = {'type': args.experts_type, 'num_experts_per_device': args.experts, 'hidden_size_per_expert': args.hidden}
    if args.experts_type == 'ffn':
        spec['activation_fn'] = F.relu
    return spec


def build_layer(shared: bool):
    from tutel_b200 import moe
    gate = {'type': 'top', 'k': args.top_k, 'capacity_factor': 0, 'scoring_func': 'sigmoid', 'n_group': 8,
            'topk_group': 4, 'bias_update_speed': 0.001}
    return moe.moe_layer(gate_type=gate, model_dim=args.model_dim, experts=experts_spec(), seeds=(1, 2, 3),
                         shared_experts={'num_experts': args.num_shared} if shared else None).cuda().bfloat16()


class Workaround(torch.nn.Module):
    """The routed layer plus a separate dense expert module of the same type, added outside the layer."""

    def __init__(self):
        super().__init__()
        from tutel_b200.models.moe_layer import _SharedExpertContext
        self.layer = build_layer(False)
        spec = experts_spec()
        kind = spec.pop('type')
        spec.update(model_dim=args.model_dim, num_experts_per_device=1, sharded_count=1,
                    hidden_size_per_expert=args.hidden * args.num_shared)
        if kind == 'llama_ffn':
            from tutel_b200.models.experts.llama_ffn import LlamaFFNNetwork as Expert
        else:
            from tutel_b200.models.experts.ffn import FusedExpertsNetwork as Expert
        self.shared = Expert(**spec).cuda().bfloat16()
        self._ctx = _SharedExpertContext

    def forward(self, x, **kw):
        y = self.layer(x, **kw)
        S = x.size(0)
        rows = None
        if not torch.is_grad_enabled() and S <= 64:
            from tutel_b200.models.moe_layer import _shared_rows
            rows = _shared_rows(S, x.device)
        out = y + self.shared(x.view(1, S, -1), self._ctx(self.layer, rows)).view(S, -1)
        out.l_aux = y.l_aux
        return out


def time_train(model, opt, x, n):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(n):
        opt.zero_grad(set_to_none=True)
        y = model(x)
        (y.float().pow(2).mean() + 0.01 * y.l_aux.float()).backward()
        opt.step()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / n


def time_decode(model, x, n):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.no_grad():
        start.record()
        for _ in range(n):
            model(x, megablocks_size=1)
        end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / n


def report(kind, tokens, times, name, power):
    med = {m: sorted(v)[len(v) // 2] for m, v in times.items()}
    print(json.dumps({
        'step': kind, 'tokens': tokens, 'experts_type': args.experts_type, 'E': args.experts, 'top_k': args.top_k,
        'model_dim': args.model_dim, 'hidden': args.hidden, 'num_shared': args.num_shared, 'dtype': 'bfloat16',
        'ms': {m: [round(t, 4) for t in v] for m, v in times.items()},
        'median_ms': {m: round(t, 4) for m, t in med.items()},
        'shared_over_routed': round(med['shared'] / med['routed'], 3),
        'workaround_over_shared': round(med['workaround'] / med['shared'], 3),
        'card': name, 'power_limit': power}), flush=True)


def main():
    assert torch.cuda.is_available(), 'this benchmark needs a GPU'
    name, power = card()
    models = {'shared': build_layer(True), 'routed': build_layer(False), 'workaround': Workaround()}
    opts = {m: torch.optim.SGD(model.parameters(), lr=1e-6) for m, model in models.items()}
    x = torch.randn(args.tokens, args.model_dim, device='cuda', dtype=torch.bfloat16)
    for m in models:
        time_train(models[m], opts[m], x, args.warmup)
    times = {m: [] for m in models}
    for _ in range(args.repeats):
        for m in models:
            times[m].append(time_train(models[m], opts[m], x, args.steps))
    report('train', args.tokens, times, name, power)
    for tokens in (1, 4):
        xd = x[:tokens].contiguous()
        for m in models:
            time_decode(models[m], xd, args.warmup * 5)
        times = {m: [] for m in models}
        for _ in range(args.repeats):
            for m in models:
                times[m].append(time_decode(models[m], xd, args.decode_steps))
        report('decode', tokens, times, name, power)


if __name__ == '__main__':
    main()
