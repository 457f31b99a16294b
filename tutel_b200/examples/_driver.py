"""Shared scaffolding of the hello-world style examples: argument parsing, session setup, synthetic data and the
timed training loop with the reference's log format (``STEP-i: loss = ..., step_time = ... sec, perf = ... tflops.``)."""
import argparse

import torch
import torch.nn.functional as F

from tutel_b200 import moe as tutel_moe
from tutel_b200 import net, system

DTYPES = {'float32': torch.float32, 'float64': torch.float64, 'float16': torch.float16, 'bfloat16': torch.bfloat16}


def base_parser(**defaults):
    p = argparse.ArgumentParser()
    p.add_argument('--local_rank', type=int, default=-1)
    p.add_argument('--batch_size', type=int, default=16)
    p.add_argument('--num_tokens', type=int, default=512)
    p.add_argument('--model_dim', type=int, default=2048)
    p.add_argument('--hidden_size', type=int, default=2048)
    p.add_argument('--num_local_experts', type=int, default=2)
    p.add_argument('--dtype', type=str, default='float32')
    p.add_argument('--fp32_gate', default=False, action='store_true')
    p.add_argument('--top', type=int, default=2)
    p.add_argument('--l_aux_wt', type=float, default=0.0)
    p.add_argument('--a2a_ffn_overlap_degree', type=int, default=1)
    p.add_argument('--allreduce_degree', type=int, default=1)
    p.add_argument('--num_steps', type=int, default=100)
    p.add_argument('--parallel_type', type=str, default='adaptive:1')
    p.add_argument('--checkpoint_path', type=str, default='')
    p.add_argument('--device', type=str, default='cuda' if torch.cuda.is_available() else 'cpu')
    p.add_argument('--use_2dh', default=False, action='store_true')
    p.add_argument('--eval', default=False, action='store_true')
    p.add_argument('--capacity_factor', type=float, default=1.0)
    p.add_argument('--cap_factor', type=float, default=1.0)
    p.add_argument('--num_shared_experts', type=int, default=0)    # > 0: shared experts (n x hidden_size), weight 1
    p.set_defaults(**defaults)
    return p


class Session:
    def __init__(self, args):
        self.args = args
        self.env = system.init_data_model_parallel(backend='nccl' if args.device == 'cuda' else 'gloo')
        self.rank, self.world, self.print = self.env.global_rank, self.env.global_size, self.env.dist_print
        self.device = self.env.local_device
        args.local_rank = self.device.index
        if args.dtype not in DTYPES:
            raise Exception('Unrecognized data type specified: %s' % args.dtype)
        torch.set_default_dtype(DTYPES[args.dtype])

    def synthetic_batch(self):
        a = self.args
        torch.manual_seed(0)
        x = torch.randn([a.batch_size, a.num_tokens, a.model_dim], dtype=torch.float32, device='cpu')
        x = x.to(dtype=torch.get_default_dtype(), device=self.device)
        y = torch.LongTensor(a.batch_size).random_(1).to(self.device)
        return x, y

    def report_params(self, layer):
        local = sum(p.numel() for _, p in layer.get_parameter_iterator(param_type='local_experts'))
        shared = sum(p.numel() for _, p in layer.get_parameter_iterator(param_type='gate'))
        self.print('[Statistics] param count for MoE local_experts = %s, param count for MoE gate = %s.\n' % (local, shared))

    def banner(self, extra=''):
        a = self.args
        self.print('[Benchmark] world_size = %s, dtype = %s, model_dim = %s, hidden_size = %s, samples = %s, num_local_experts = %s, topK = %s, a2a_ffn_overlap_degree = %s%s, device = `%s`' % (
            self.world, a.dtype, a.model_dim, a.hidden_size, a.batch_size * a.num_tokens, a.num_local_experts, a.top,
            a.a2a_ffn_overlap_degree, extra, self.device))

    def train(self, model, optimizer, x, y, sync_grads=None, forward=None, suffix=None, scaler=None):
        """The timed loop.  ``sync_grads(model)`` runs after backward, ``forward(model, x)`` customises the forward."""
        a = self.args
        E = tutel_moe.moe_layer.global_expert_count(a.num_local_experts, group=system.get_local_session().model_group)
        total = 0.0
        for i in range(a.num_steps):
            t0 = system.record_time()
            if not a.eval:
                optimizer.zero_grad()
                out = forward(model, x) if forward else model(x)
                loss = F.nll_loss(out, y)
                if a.l_aux_wt and getattr(model, '_moe_layer', None) is not None:
                    loss = loss + a.l_aux_wt * model._moe_layer.l_aux
                if scaler is not None:
                    scaler.scale(loss).backward()
                else:
                    loss.backward()
                if sync_grads is not None:
                    sync_grads(model)
                if scaler is not None:
                    scaler.step(optimizer)
                    scaler.update()
                else:
                    optimizer.step()
            else:
                with torch.no_grad():
                    out = forward(model, x) if forward else model(x)
                    loss = F.nll_loss(out, y)
            t1 = system.record_time()
            mm, cap = (1 if a.eval else 3), min(a.top, E)
            tflops = (a.batch_size * a.num_tokens * a.model_dim * a.hidden_size) * 4 * mm * cap * 1e-12 / (t1 - t0)
            tail = (' ' + suffix(model)) if suffix else ''
            self.print('STEP-%s: loss = %.5f, step_time = %.6f sec, perf = %.2f tflops.%s' % (i, float(loss.data), t1 - t0, tflops, tail))
            if i + 10 >= a.num_steps:
                total += t1 - t0
        self.print('\n[Summary] Average synchronized step_time = %s sec.' % (total / 10))


def manual_allreduce(session, model):
    """Average the gradients of parameters that are replicated on every rank (everything not tagged skip_allreduce)."""
    if session.world <= 1 or session.args.allreduce_degree == -1:
        return None
    shared = [p for p in model.parameters() if not hasattr(p, 'skip_allreduce') and getattr(p, 'requires_grad', False)]

    def sync(_):
        for p in shared:
            p.grad /= session.world
            p.grad = net.simple_all_reduce(p.grad)
    return sync


class MoEClassifier(torch.nn.Module):
    """MoE layer followed by sum-pool + log-softmax, the toy model of every hello-world example."""

    def __init__(self, layer, call=None):
        super().__init__()
        self._moe_layer = layer
        self._call = call

    def forward(self, x):
        y = self._call(self._moe_layer, x) if self._call else self._moe_layer(x)
        return F.log_softmax(torch.sum(y, dim=2), dim=1)


def default_layer(session, **overrides):
    a = session.args
    kw = dict(
        gate_type={'type': 'top', 'k': a.top, 'fp32_gate': a.fp32_gate, 'capacity_factor': a.capacity_factor},
        experts={'type': 'ffn', 'num_experts_per_device': a.num_local_experts, 'hidden_size_per_expert': a.hidden_size,
                 'activation_fn': lambda x: F.relu(x)},
        model_dim=a.model_dim,
        scan_expert_func=lambda name, param: setattr(param, 'skip_allreduce', True),
        seeds=(1, session.rank + 1, 1),
        a2a_ffn_overlap_degree=a.a2a_ffn_overlap_degree,
        parallel_type=a.parallel_type,
        use_2dh=a.use_2dh,
    )
    if getattr(a, 'num_shared_experts', 0) > 0:
        kw['shared_experts'] = {'num_experts': a.num_shared_experts}
    kw.update(overrides)
    return tutel_moe.moe_layer(**kw)
