#!/usr/bin/env python3
"""On-GPU numerics + timing sweep of the native kernels (needs a GPU).

Every case runs in its own subprocess with a timeout, so a trapping / hanging kernel variant cannot take the
rest of the sweep with it.  Results: bench_out/kernel_check.json (+ a readable .txt).

    python bench/kernel_check.py            # full sweep
    python bench/kernel_check.py --case N   # (internal) run one case in-process
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gemm_cases():
    cases = []
    for cg in (1, 2):
        for bn in (256, 128):
            for a_mn in (False, True):
                for b_mn in (False, True):
                    cases.append(dict(kind='gemm', M=256, N=256, K=128, G=1, a_mn=a_mn, b_mn=b_mn, cg=cg, bn=bn))
    for cg in (1, 2):
        cases.append(dict(kind='gemm', M=200, N=136, K=72, G=3, a_mn=False, b_mn=False, cg=cg, bn=256))
        cases.append(dict(kind='gemm', M=200, N=136, K=72, G=3, a_mn=True, b_mn=True, cg=cg, bn=256))
        cases.append(dict(kind='gemm', M=1000, N=520, K=1096, G=2, a_mn=False, b_mn=True, cg=cg, bn=256, epi=2, bias=True))
        cases.append(dict(kind='gemm', M=1000, N=520, K=1096, G=2, a_mn=False, b_mn=False, cg=cg, bn=256, epi=5))
        cases.append(dict(kind='gemm', M=512, N=512, K=512, G=4, a_mn=False, b_mn=False, cg=cg, bn=256, dtype='float16'))
        cases.append(dict(kind='gemm', M=512, N=512, K=512, G=2, a_mn=True, b_mn=True, cg=cg, bn=256, out='float32'))
        cases.append(dict(kind='gemm', M=512, N=512, K=512, G=4, a_mn=False, b_mn=False, cg=cg, bn=256, counts=[512, 0, 130, 257]))
    # performance shapes (flagship: 16384 x 14336 x 4096)
    for cg in (1, 2):
        for (a_mn, b_mn) in ((False, False), (False, True), (True, True)):
            cases.append(dict(kind='gemm', M=16384, N=14336, K=4096, G=1, a_mn=a_mn, b_mn=b_mn, cg=cg, bn=256, perf=True))
    cases.append(dict(kind='gemm', M=2048, N=14336, K=4096, G=8, a_mn=False, b_mn=False, cg=2, bn=256, perf=True))
    cases.append(dict(kind='gemm', M=16384, N=4096, K=14336, G=1, a_mn=False, b_mn=True, cg=2, bn=256, perf=True))
    cases.append(dict(kind='gemm', M=14336, N=4096, K=16384, G=1, a_mn=True, b_mn=True, cg=2, bn=256, perf=True))
    cases.append(dict(kind='gemm', M=8192, N=8192, K=8192, G=1, a_mn=False, b_mn=False, cg=2, bn=256, perf=True))
    cases.append(dict(kind='gemm', M=4096, N=14336, K=2048, G=8, a_mn=True, b_mn=True, cg=2, bn=256, perf=True))   # per-expert wgrad, short K
    cases.append(dict(kind='gemm', M=8192, N=8192, K=8192, G=1, a_mn=False, b_mn=False, cg=1, bn=256, perf=True))
    cases.append(dict(kind='fp8', M=16384, N=14336, K=4096, G=1, cg=2))
    cases.append(dict(kind='fp8', M=16384, N=4096, K=14336, G=1, cg=2))
    # the six GEMMs of one flagship training step, issued as FusedReluFFN issues them
    cases.append(dict(kind='flagship', G=8, T=2048, D=4096, H=14336, perf=True))
    return cases


def other_cases():
    return [
        dict(kind='route', S=8192, E=8, k=2),
        dict(kind='route', S=5000, E=130, k=3),
        dict(kind='route', S=32, E=128, k=1),
        dict(kind='dispatch', S=8192, E=8, k=2, M=4096, dtype='bfloat16', C=2048),
        dict(kind='dispatch', S=1000, E=6, k=2, M=264, dtype='float16', C=300),
        dict(kind='dispatch', S=1000, E=6, k=2, M=257, dtype='float32', C=200),
        dict(kind='gate', S=8192, E=8, k=2),
        dict(kind='gate', S=777, E=130, k=4),
        dict(kind='jit'),
    ]


ALL = gemm_cases() + other_cases()


def run_gemm(c):
    import torch
    from tutel_b200 import _C
    dt = getattr(torch, c.get('dtype', 'bfloat16'))
    odt = getattr(torch, c.get('out', c.get('dtype', 'bfloat16')))
    M, N, K, G = c['M'], c['N'], c['K'], c['G']
    dev = 'cuda'
    g = torch.Generator(device=dev).manual_seed(1234)
    a = (torch.randn(G, M, K, device=dev, generator=g) * 0.5).to(dt)
    b = (torch.randn(G, N, K, device=dev, generator=g) * 0.5).to(dt)
    a_op = a.transpose(1, 2).contiguous() if c['a_mn'] else a   # [G,K,M] storage for MN-major
    b_op = b.transpose(1, 2).contiguous() if c['b_mn'] else b   # [G,K,N]
    d = torch.full((G, M, N), float('nan'), device=dev, dtype=odt)
    bias = (torch.randn(G, N, device=dev, generator=g)).to(dt) if c.get('bias') else None
    epi = c.get('epi', 0)
    aux = None
    if epi == 5:
        aux = (torch.randn(G, M, N, device=dev, generator=g)).to(odt)
    counts = None
    if c.get('counts'):
        counts = torch.tensor(c['counts'], device=dev, dtype=torch.int32)

    def call():
        _C.gemm(a_op, b_op, d, c['a_mn'], c['b_mn'], epi, bias, aux, counts, 1.0, 1, c['cg'], c['bn'], 0, 0, 0, 0, 0, 0, 0, 0, 1, None, None, None)

    call()
    torch.cuda.synchronize()
    res = {}
    if not c.get('perf') or True:
        # reference on a subset of rows for the huge shapes
        rows = slice(0, M) if M * N * G <= (1 << 24) else slice(0, 512)
        ref = torch.matmul(a[:, rows].float(), b.float().transpose(1, 2))
        if bias is not None:
            ref = ref + bias.float().unsqueeze(1)
        if epi == 2:
            ref = torch.relu(ref)
        if epi == 5:
            ref = torch.where(aux[:, rows].float() > 0, ref, torch.zeros_like(ref))
        got = d[:, rows].float()
        if counts is not None:
            for gi, cnt in enumerate(c['counts']):
                ref[gi, cnt:] = 0
                got[gi, cnt:] = 0  # rows past the count are unspecified (never written)
        err = (got - ref).abs().max().item()
        scale = ref.abs().max().item() + 1e-6
        res['max_abs_err'] = err
        res['rel_err'] = err / scale
        res['nan'] = bool(torch.isnan(got).any().item())
        if rows.stop != M:
            # also check the last rows of the big problem
            ref2 = torch.matmul(a[:, -256:].float(), b.float().transpose(1, 2))
            err2 = (d[:, -256:].float() - ref2).abs().max().item()
            res['rel_err_tail'] = err2 / (ref2.abs().max().item() + 1e-6)
        tol = 2e-2 if odt != torch.float32 else 1e-3
        res['ok'] = (not res['nan']) and res['rel_err'] < tol and res.get('rel_err_tail', 0) < tol
    if c.get('perf'):
        flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
        def timeit(fn, iters=10):
            for _ in range(3):
                fn()
            ts = []
            for _ in range(iters):
                flush.zero_()
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record(); fn(); e.record(); torch.cuda.synchronize()
                ts.append(s.elapsed_time(e))
            ts.sort()
            return ts[len(ts) // 2], ts[0]
        med, best = timeit(call)
        flops = 2.0 * M * N * K * G
        res['ms_median'] = med
        res['tflops_median'] = flops / med * 1e-9
        res['tflops_best'] = flops / best * 1e-9
        bt = b.transpose(1, 2)
        at_ = a_op.transpose(1, 2) if c['a_mn'] else a
        bt_ = b_op if c['b_mn'] else bt
        out = torch.empty(G, M, N, device=dev, dtype=dt)
        med2, best2 = timeit(lambda: torch.matmul(at_, bt_, out=out))
        res['cublas_ms_median'] = med2
        res['cublas_tflops_median'] = flops / med2 * 1e-9
        res['cublas_tflops_best'] = flops / best2 * 1e-9
    return res


def run_route(c):
    import torch
    from tutel_b200 import _C
    S, E, k = c['S'], c['E'], c['k']
    g = torch.Generator().manual_seed(7)
    scores = torch.rand(S, E, generator=g)
    idx = torch.topk(scores, k, dim=1).indices.t().contiguous().to(torch.int32)
    loc_ref, cnt_ref = _C.cpu_route_locations(idx, E)
    C = max(1, (S * k // E) // 2)
    out = _C.route_locations(idx.cuda(), E, C)
    loc, cnt, slot = out
    ok = bool((loc.cpu() == loc_ref).all() and (cnt.cpu() == cnt_ref).all())
    # slot map check
    slot_ref = torch.full((E * C,), -1, dtype=torch.int32)
    for j in range(k):
        m = loc_ref[j] < C
        s_ids = torch.nonzero(m).view(-1)
        slot_ref[(idx[j][m].long() * C + loc_ref[j][m].long())] = (s_ids * k + j).to(torch.int32)
    ok = ok and bool((slot.cpu() == slot_ref).all())
    return dict(ok=ok)


def run_dispatch(c):
    import torch
    from tutel_b200 import _C
    S, E, k, M, C = c['S'], c['E'], c['k'], c['M'], c['C']
    dt = getattr(torch, c['dtype'])
    g = torch.Generator().manual_seed(11)
    scores = torch.rand(S, E, generator=g)
    idx = torch.topk(scores, k, dim=1).indices.t().contiguous().to(torch.int32)
    loc, cnt = _C.cpu_route_locations(idx, E)
    gates = torch.rand(k, S, generator=g)
    x = torch.randn(S, M, generator=g).to(dt)
    xr = x.float()
    ref_enc = _C.cpu_encode(xr, gates, idx, loc, E, C)
    ref_enc1 = _C.cpu_encode(xr, None, idx, loc, E, C)
    idx_d, loc_d, gates_d, x_d = idx.cuda(), loc.cuda(), gates.cuda(), x.cuda()
    slot = _C.build_slot_map(idx_d, loc_d, E, C)
    out = torch.full((E * C, M), float('nan'), dtype=dt, device='cuda')
    _C.encode_rows(x_d, gates_d, slot, out, k, E, C, 0, 0, 0, 0, 0, 0, None)
    out1 = torch.full((E * C, M), float('nan'), dtype=dt, device='cuda')
    _C.encode_rows(x_d, None, slot, out1, k, E, C, 0, 0, 0, 3, 0, 0, None)
    tol = 1e-5 if dt == torch.float32 else 2e-2
    e1 = (out.float().cpu() - ref_enc).abs().max().item()
    e2 = (out1.float().cpu() - ref_enc1).abs().max().item()
    y = torch.randn(E * C, M, generator=g).to(dt)
    ref_dec = _C.cpu_decode(y.float(), gates, idx, loc, E, C)
    dec = _C.decode_rows(y.cuda(), gates_d, idx_d, loc_d, E, C, 0, 0)
    e3 = (dec.float().cpu() - ref_dec).abs().max().item() / (ref_dec.abs().max().item() + 1e-6)
    ref_gg = _C.cpu_gate_grad(xr, y.float(), idx, loc, E, C)
    gg = _C.gate_grad(x_d, y.cuda(), idx_d, loc_d, E, C)
    e4 = (gg.cpu() - ref_gg).abs().max().item() / (ref_gg.abs().max().item() + 1e-6)
    res = dict(enc_err=e1, enc1_err=e2, dec_rel=e3, gg_rel=e4)
    res['ok'] = e1 < tol and e2 < tol and e3 < tol and e4 < tol
    # timing of the flagship shape
    if S >= 4096:
        ev = lambda: torch.cuda.Event(enable_timing=True)
        for name, fn in (('encode_ms', lambda: _C.encode_rows(x_d, None, slot, out1, k, E, C, 0, 0, 0, 0, 0, 0, None)),
                         ('decode_ms', lambda: _C.decode_rows(out1, gates_d, idx_d, loc_d, E, C, 0, 0)),
                         ('gate_grad_ms', lambda: _C.gate_grad(x_d, out1, idx_d, loc_d, E, C))):
            for _ in range(3):
                fn()
            s, e = ev(), ev()
            s.record()
            for _ in range(10):
                fn()
            e.record(); torch.cuda.synchronize()
            res[name] = s.elapsed_time(e) / 10
    return res


def run_gate(c):
    """Fused gate + routing (2 launches) and its one-launch backward, plus the small kernels that have no other case:
    column sums, the public column scan, the one-launch skinny FFN, fp8 encode / dequant."""
    import torch
    import torch.nn.functional as F
    from tutel_b200 import _C
    S, E, k = c['S'], c['E'], c['k']
    g = torch.Generator().manual_seed(5)
    logits = torch.randn(S, E, generator=g).cuda()
    cap = k * ((S + E - 1) // E)
    scores, idx, top, gates, loc, counts, ce, l_aux, slot = _C.gate_route_forward(logits, k, cap, True, 1e-7)
    ref = torch.softmax(logits, dim=1)
    tv, ti = torch.topk(ref, k, dim=1)
    ok = bool(torch.allclose(scores, ref, atol=1e-6, rtol=1e-5))
    ok = ok and bool((idx.t().long() == ti).float().mean() > 0.999) and bool(torch.allclose(top.t(), tv, atol=1e-6, rtol=1e-5))
    onehot = F.one_hot(idx.reshape(-1).long(), E)
    pos = (torch.cumsum(onehot, 0) - 1).gather(1, idx.reshape(-1, 1).long()).view(k, S)
    ok = ok and bool((loc.long() == pos).all()) and bool((counts.long() == onehot.sum(0)).all())
    dl = torch.ones((), device='cuda')
    dlog = _C.gate_route_backward(scores, idx, top, torch.randn(k, S, device='cuda'), ce, dl, logits, True, 1e-7)
    ok = ok and bool(torch.isfinite(dlog).all())
    x = torch.randn(3, 700, 264, device='cuda').bfloat16()
    ok = ok and bool(torch.allclose(_C.grouped_colsum(x).float(), x.float().sum(1), atol=1.0, rtol=2e-2))
    mask = (torch.rand(S, E, device='cuda') < 0.3).int()
    ok = ok and bool((_C.cumsum_sub_one(mask).long() == torch.cumsum(mask.long(), 0) - 1).all())
    xs = torch.randn(4, 8, 128, device='cuda')
    w1, w2 = torch.randn(4, 96, 128, device='cuda') * 0.1, torch.randn(4, 96, 64, device='cuda') * 0.1
    cnt = torch.tensor([8, 0, 3, 5], device='cuda', dtype=torch.int32)
    y = _C.skinny_ffn(xs, w1, None, w2, None, cnt, 1)
    yr = torch.relu(xs @ w1.transpose(1, 2)) @ w2
    yr = yr * (torch.arange(8, device='cuda').view(1, 8, 1) < cnt.view(4, 1, 1))
    ok = ok and bool(torch.allclose(y, yr, atol=1e-3, rtol=1e-3))
    tok = torch.randn(300, 256, device='cuda').bfloat16()
    q, sc = _C.encode_rows_fp8(tok, None, slot[: E * cap].contiguous() % 300, 1, E, cap, 0, 0, 0, 0, 0, 0, 0)
    back = _C.dequant_rows(q, sc, torch.bfloat16)
    ok = ok and bool(torch.isfinite(back.float()).all())
    return dict(ok=ok)


def run_jit(c):
    import torch
    from tutel_b200 import _C
    src = r'''
    extern "C" __global__ void scale_add(float* x, float* y, int n, int mul) {
      // [thread_extent] blockIdx.x = 64
      // [thread_extent] threadIdx.x = 256
      for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) y[i] = x[i] * mul + 1.0f;
    }'''
    h = _C.jit_inject_source(src)
    x = torch.randn(100000, device='cuda')
    y = torch.empty_like(x)
    _C.jit_invoke([x, y], [x.numel(), 3], [], h)
    torch.cuda.synchronize()
    return dict(ok=bool(torch.allclose(y, x * 3 + 1, rtol=1e-5, atol=1e-5)), y=y[:4].tolist(), x=x[:4].tolist())


def run_fp8(c):
    import torch
    from tutel_b200.ops import gemm as G
    M, N, K, Gn = c['M'], c['N'], c['K'], c['G']
    a = (torch.randn(Gn, M, K, device='cuda') * 0.5).bfloat16()
    b = (torch.randn(Gn, N, K, device='cuda') * 0.5).bfloat16()
    aq, sa = G.quantize_rows(a)
    bq, sb = G.quantize_rows(b)
    d = torch.empty(Gn, M, N, device='cuda', dtype=torch.bfloat16)
    call = lambda: G.raw_gemm(aq, bq, out=d, scale_a=sa, scale_b=sb, cta_group=c['cg'])
    call()
    ref = torch.matmul(a[:, :512].float(), b.float().transpose(1, 2))
    rel = ((d[:, :512].float() - ref).norm() / ref.norm()).item()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device='cuda')
    def timeit(fn):
        for _ in range(3):
            fn()
        ts = []
        for _ in range(10):
            flush.zero_()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record(); fn(); e.record(); torch.cuda.synchronize()
            ts.append(s.elapsed_time(e))
        return sorted(ts)[5]
    t = timeit(call)
    tq = timeit(lambda: G.quantize_rows(a))
    return dict(ok=rel < 0.06, rel_err=rel, ms_median=t, tflops_median=2.0 * M * N * K * Gn / t * 1e-9, quantize_rows_ms=tq,
                quantize_GBps=(a.numel() * 3) / tq * 1e-6)


def run_flagship(c):
    """The six expert GEMMs of the flagship step (G experts, T = capacity rows, D = model_dim, H = hidden) with the
    layouts, epilogues and fused bias gradient of FusedReluFFN.  Each is timed three ways, interleaved round by round:
    block_n=128 (the 128 x 128 configuration of the fused multi-GPU engine), block_n=0 (the launcher's choice) and
    torch.matmul on the same operands (matmul only, no epilogue)."""
    import torch
    from tutel_b200.ops import gemm as GM
    Gn, T, D, H = c['G'], c['T'], c['D'], c['H']
    dev = 'cuda'
    g = torch.Generator(device=dev).manual_seed(4321)
    rnd = lambda *s, sc=1.0: (torch.randn(*s, device=dev, generator=g) * sc).bfloat16()
    x, dy = rnd(Gn, T, D), rnd(Gn, T, D, sc=0.01)
    w1, w2 = rnd(Gn, H, D, sc=D ** -0.5), rnd(Gn, H, D, sc=H ** -0.5)
    b1, b2 = rnd(Gn, H, sc=0.1), rnd(Gn, D, sc=0.1)
    act = GM.raw_gemm(x, w1, epilogue=GM.EPI_BIAS_RELU, bias=b1)
    db1 = torch.zeros(Gn, H, device=dev)
    dh = GM.raw_gemm(dy, w2, epilogue=GM.EPI_RELU_BWD, aux=act, colsum=db1)
    tr = lambda t: t.transpose(1, 2)
    # name: (M, N, K, native call(block_n, out), torch call(out))
    calls = {
        'fc1 bias_relu': (T, H, D, lambda bn, o: GM.raw_gemm(x, w1, epilogue=GM.EPI_BIAS_RELU, bias=b1, out=o, block_n=bn),
                          lambda o: torch.matmul(x, tr(w1), out=o)),
        'fc2 bias': (T, D, H, lambda bn, o: GM.raw_gemm(act, w2, b_mn=True, epilogue=GM.EPI_BIAS, bias=b2, out=o, block_n=bn),
                     lambda o: torch.matmul(act, w2, out=o)),
        'dh relu_bwd+colsum': (T, H, D, lambda bn, o: GM.raw_gemm(dy, w2, epilogue=GM.EPI_RELU_BWD, aux=act, colsum=db1, out=o,
                                                                   block_n=bn),
                               lambda o: torch.matmul(dy, tr(w2), out=o)),
        'dw2 wgrad': (H, D, T, lambda bn, o: GM.raw_gemm(act, dy, a_mn=True, b_mn=True, out=o, block_n=bn),
                      lambda o: torch.matmul(tr(act), dy, out=o)),
        'dx dgrad': (T, D, H, lambda bn, o: GM.raw_gemm(dh, w1, b_mn=True, out=o, block_n=bn),
                     lambda o: torch.matmul(dh, w1, out=o)),
        'dw1 wgrad': (H, D, T, lambda bn, o: GM.raw_gemm(dh, x, a_mn=True, b_mn=True, out=o, block_n=bn),
                      lambda o: torch.matmul(tr(dh), x, out=o)),
    }
    ev = lambda: torch.cuda.Event(enable_timing=True)
    res, ok = {}, True
    for name, (M, N, K, native, ref) in calls.items():
        outs = {v: torch.empty(Gn, M, N, device=dev, dtype=torch.bfloat16) for v in ('narrow', 'auto', 'torch')}
        fns = {'narrow': lambda: native(128, outs['narrow']), 'auto': lambda: native(0, outs['auto']),
               'torch': lambda: ref(outs['torch'])}
        for fn in fns.values():
            fn(); fn()
        times = {v: [] for v in fns}
        for _ in range(5):
            for v, fn in fns.items():
                s, e = ev(), ev()
                s.record()
                for _ in range(4):
                    fn()
                e.record()
                torch.cuda.synchronize()
                times[v].append(s.elapsed_time(e) / 4)
        flops = 2.0 * Gn * M * N * K
        r = {'M': M, 'N': N, 'K': K}
        for v, ts in times.items():
            ms = sorted(ts)[len(ts) // 2]
            r[v + '_ms'] = round(ms, 4)
            r[v + '_tflops'] = round(flops / ms * 1e-9, 1)
        # narrow and automatic configurations against each other: same epilogue math, same K order per element
        na, au = outs['narrow'].float(), outs['auto'].float()
        r['auto_vs_narrow_rel'] = ((na - au).abs().max() / (na.abs().max() + 1e-6)).item()
        ok = ok and r['auto_vs_narrow_rel'] < 1e-2 and bool(torch.isfinite(au).all())
        res[name] = r
    res['ok'] = ok
    return res


RUNNERS = dict(flagship=run_flagship, fp8=run_fp8, gemm=run_gemm, route=run_route, dispatch=run_dispatch, gate=run_gate, jit=run_jit)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--case', type=int, default=-1)
    ap.add_argument('--filter', type=str, default='')
    ap.add_argument('--no_perf', action='store_true', help='skip the large performance shapes (sanitizer runs)')
    ap.add_argument('--inline', action='store_true', help='run the cases in this process (no subprocess per case)')
    ap.add_argument('--out', type=str, default=os.path.join(ROOT, 'bench_out', 'kernel_check.json'))
    args = ap.parse_args()
    if args.case >= 0:
        c = ALL[args.case]
        try:
            r = RUNNERS[c['kind']](c)
        except Exception as ex:  # noqa
            r = dict(ok=False, error=repr(ex)[:500])
        print('RESULT ' + json.dumps(r))
        return
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    results = []
    for i, c in enumerate(ALL):
        if args.filter and args.filter not in json.dumps(c):
            continue
        if args.no_perf and (c.get('perf') or c.get('kind') == 'fp8'):
            continue
        t0 = time.time()
        if args.inline:
            try:
                r = RUNNERS[c['kind']](c)
            except Exception as ex:  # noqa
                r = dict(ok=False, error=repr(ex)[:500])
            r['case'] = c
            r['wall_s'] = round(time.time() - t0, 1)
            results.append(r)
            print(json.dumps(r), flush=True)
            continue
        try:
            p = subprocess.run([sys.executable, os.path.abspath(__file__), '--case', str(i)], capture_output=True,
                               text=True, timeout=180)
            r = None
            for line in p.stdout.splitlines():
                if line.startswith('RESULT '):
                    r = json.loads(line[7:])
            if r is None:
                r = dict(ok=False, error='no result', rc=p.returncode, tail=(p.stdout + p.stderr)[-600:])
        except subprocess.TimeoutExpired:
            r = dict(ok=False, error='timeout')
        r['case'] = c
        r['wall_s'] = round(time.time() - t0, 1)
        results.append(r)
        print(json.dumps(r), flush=True)
        with open(args.out, 'w') as f:
            json.dump(results, f, indent=1)
    nfail = sum(1 for r in results if not r.get('ok'))
    print('kernel_check: %d cases, %d failed' % (len(results), nfail))


if __name__ == '__main__':
    main()
