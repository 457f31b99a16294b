"""H100 check of the MX block-scaled GEMM (csrc/gemm_mx.cu): exactness on crafted operands (full grid and 5 persistent CTAs), agreement with the PyTorch
definition on random data, throughput next to the row-scaled fp8 and bf16 GEMMs.

    python bench/mx_check.py [--out bench_out/mx] [--no_perf]

Each group of cases runs in its own process under a timeout (a wrong descriptor traps or hangs the context).
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def crafted(mode, G, M, N, K, dev, seed=0):
    """Small-integer e4m3 operands and small exponents: every product and partial sum is exact in fp32."""
    import torch
    g = torch.Generator(device='cpu').manual_seed(seed)
    a = torch.randint(-3, 4, (G, M, K), generator=g).float()
    b = torch.randint(-3, 4, (G, N, K), generator=g).float()

    def exps(R):
        if mode == 'ones':
            return torch.zeros(G, R, K // 32, dtype=torch.int32)
        if mode == 'rows':
            return (torch.arange(R, dtype=torch.int32) % 5 - 2).view(1, R, 1).expand(G, R, K // 32).contiguous()
        if mode == 'kblocks':
            return (torch.arange(K // 32, dtype=torch.int32) % 4 - 1).view(1, 1, K // 32).expand(G, R, K // 32).contiguous()
        return torch.randint(-2, 3, (G, R, K // 32), generator=g, dtype=torch.int32)
    ea, eb = exps(M), exps(N)
    return a.to(dev), ea.to(dev), b.to(dev), eb.to(dev)


def run_exact(tag, mode, G, M, N, K, block_n, small_grid, cg=1):
    import torch
    from tutel_b200.ops import mx
    dev = torch.device('cuda')
    a, ea, b, eb = crafted(mode, G, M, N, K, dev)
    aq, bq = a.to(torch.float8_e4m3fn), b.to(torch.float8_e4m3fn)
    sa, sb = mx.pack_scales(ea), mx.pack_scales(eb)
    ref = torch.matmul(mx.mx_dequantize(aq, sa), mx.mx_dequantize(bq, sb).transpose(1, 2))
    y = mx.mx_gemm(aq, sa, bq, sb, block_n=block_n, cta_group=cg, max_ctas=((4 if cg == 2 else 5) if small_grid else 0))
    torch.cuda.synchronize()
    want = ref.to(torch.bfloat16).float()
    bad = (y.float() != want)
    rec = {'case': tag, 'mode': mode, 'shape': [G, M, N, K], 'block_n': block_n, 'cta_group': cg, 'small_grid': bool(small_grid),
           'mismatch': int(bad.sum()), 'of': bad.numel(), 'max_abs': float((y.float() - want).abs().max())}
    if rec['mismatch']:
        idx = bad.nonzero()[:6].tolist()
        rec['first_bad'] = [(i, float(y[tuple(i)]), float(want[tuple(i)])) for i in idx]
        ok = want != 0
        ratio = torch.where(ok, y.float() / torch.where(ok, want, torch.ones_like(want)), torch.ones_like(want))
        rec['ratio_rows'] = [round(float(ratio[0, r].abs().median()), 4) for r in (0, 1, 31, 32, 33, 64, 96, min(127, M - 1))]
        rec['ratio_cols'] = [round(float(ratio[0, :, c].abs().median()), 4) for c in (0, 1, 31, 32, 33, 64, 96, 127)]
        rec['bad_rows'] = int(bad.any(-1).sum())
        rec['bad_cols'] = int(bad.any(-2).sum())
    print(json.dumps(rec), flush=True)
    return rec['mismatch'] == 0


def group_exact_cg2(small_grid):
    """CTA pairs (cta_group::2, 256 x 256 tiles): scales of A per CTA, scales of B in both."""
    import torch
    from tutel_b200.ops import backend
    backend.require_ext().set_spin_timeout(5.0)
    ok = True
    cases = [('cg2_ones', 'ones', 1, 256, 256, 128), ('cg2_rows', 'rows', 1, 256, 256, 128), ('cg2_kblk', 'kblocks', 1, 256, 256, 128),
             ('cg2_rand', 'random', 1, 256, 256, 128), ('cg2_tail', 'random', 1, 100, 256, 256), ('cg2_wrap', 'random', 2, 300, 512, 1024),
             ('cg2_big', 'random', 2, 1000, 1024, 2048)]
    for tag, mode, G, M, N, K in cases:
        ok = run_exact(tag, mode, G, M, N, K, 256, small_grid, cg=2) and ok
    print(json.dumps({'group': 'exact_cg2', 'small_grid': bool(small_grid), 'ok': ok}), flush=True)


def group_exact(small_grid, quick):
    import torch
    from tutel_b200.ops import backend
    backend.require_ext().set_spin_timeout(5.0)
    ok = True
    cases = [('ones128', 'ones', 1, 128, 128, 128, 128), ('rows128', 'rows', 1, 128, 128, 128, 128),
             ('kblk128', 'kblocks', 1, 128, 128, 128, 128), ('rand128', 'random', 1, 128, 128, 128, 128)]
    if not quick:
        cases += [('wrap', 'random', 2, 200, 384, 512, 128), ('bn256', 'random', 1, 256, 512, 1024, 256),
                  ('bn256rows', 'rows', 1, 128, 256, 128, 256), ('big', 'random', 2, 1000, 1024, 2048, 0)]
    for tag, mode, G, M, N, K, bn in cases:
        ok = run_exact(tag, mode, G, M, N, K, bn, small_grid) and ok
    print(json.dumps({'group': 'exact', 'max_ctas': 5 if small_grid else 0, 'ok': ok}), flush=True)


def group_random():
    """Kernel quantiser == PyTorch definition (bytes), GEMM vs fp32 matmul of the dequantised operands."""
    import torch
    from tutel_b200.ops import backend, mx
    backend.require_ext().set_spin_timeout(5.0)
    torch.manual_seed(0)
    ok = True
    for (G, M, N, K) in [(1, 128, 128, 128), (2, 300, 768, 1024), (1, 4096, 2048, 4096)]:
        x = (torch.randn(G, M, K, device='cuda') * torch.exp(torch.randn(G, M, 1, device='cuda'))).to(torch.bfloat16)
        w = (torch.randn(G, N, K, device='cuda') * 0.05).to(torch.bfloat16)
        x[0, 0, :4] = 0
        xq, xs = mx.mx_quantize(x)
        wq, ws = mx.mx_quantize(w)
        rq, rs = mx.mx_quantize_reference(x)
        same_q = bool((xq.view(torch.uint8) == rq.view(torch.uint8)).all())
        same_s = bool((xs == rs).all())
        y = mx.mx_gemm(xq, xs, wq, ws).float()
        ref = torch.matmul(mx.mx_dequantize(xq, xs), mx.mx_dequantize(wq, ws).transpose(1, 2))
        full = torch.matmul(x.float(), w.float().transpose(1, 2))
        err_def = float((y - ref).abs().max() / ref.abs().max())
        err_full = float((y - full).norm() / full.norm())
        yr = mx.mx_gemm(xq, xs, wq, ws, epilogue=mx.EPI_RELU).float()
        relu_ok = bool((yr == torch.relu(y)).all())
        good = same_q and same_s and err_def < 8e-3 and err_full < 0.06 and relu_ok
        ok = ok and good
        print(json.dumps({'case': 'random', 'shape': [G, M, N, K], 'quantiser_bytes_equal': same_q, 'scales_equal': same_s,
                          'rel_err_vs_definition': err_def, 'rel_fro_err_vs_bf16_matmul': err_full, 'relu_ok': relu_ok,
                          'ok': good}), flush=True)
    print(json.dumps({'group': 'random', 'ok': ok}), flush=True)


def group_perf(cg=1):
    import torch
    from tutel_b200.ops import backend, gemm, mx
    backend.require_ext().set_spin_timeout(20.0)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device='cuda')

    def timeit(fn, iters=20):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        ts = []
        for _ in range(iters):
            flush.zero_()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record(); fn(); e.record()
            torch.cuda.synchronize()
            ts.append(s.elapsed_time(e))
        ts.sort()
        return ts[len(ts) // 2]

    out = []
    for (G, M, N, K) in [(2, 8192, 4096, 4096), (1, 8192, 14336, 4096), (1, 8192, 4096, 14336), (8, 2048, 2048, 2048)]:
        x = torch.randn(G, M, K, device='cuda', dtype=torch.bfloat16)
        w = (torch.randn(G, N, K, device='cuda') * 0.05).to(torch.bfloat16)
        xq, xs = mx.mx_quantize(x)
        wq, ws = mx.mx_quantize(w)
        flops = 2.0 * G * M * N * K
        rec = {'shape': [G, M, N, K]}
        for tag, bn, g2 in (('mx_cg2', 256, 2), ('mx_cg1_bn256', 256, 1), ('mx_cg1_bn128', 128, 1)):
            if N % bn:
                continue
            ms = timeit(lambda: mx.mx_gemm(xq, xs, wq, ws, block_n=bn, cta_group=g2))
            rec[tag + '_ms'] = round(ms, 4)
            rec[tag + '_tflops'] = round(flops / ms / 1e9, 1)
        if cg == 2:
            print(json.dumps(rec), flush=True)
            continue
        rq, rscale = gemm.quantize_rows(x)
        wq8, wscale = gemm.quantize_rows(w)
        d = torch.empty(G, M, N, device='cuda', dtype=torch.bfloat16)
        ms = timeit(lambda: gemm.raw_gemm(rq, wq8, out=d, scale_a=rscale, scale_b=wscale))
        rec['rowscaled_fp8_ms'] = round(ms, 4); rec['rowscaled_fp8_tflops'] = round(flops / ms / 1e9, 1)
        ms = timeit(lambda: gemm.raw_gemm(x, w, out=d))
        rec['bf16_ms'] = round(ms, 4); rec['bf16_tflops'] = round(flops / ms / 1e9, 1)
        ms = timeit(lambda: mx.mx_quantize(x))
        rec['mx_quantize_ms'] = round(ms, 4)
        rec['mx_quantize_gbps'] = round((x.numel() * 3 + xs.numel()) / ms / 1e6, 1)
        ms = timeit(lambda: gemm.quantize_rows(x))
        rec['row_quantize_ms'] = round(ms, 4)
        ms = timeit(lambda: mx.mx_quantize_transpose(w))
        rec['mx_quantize_transpose_ms'] = round(ms, 4)
        rec['mx_quantize_transpose_gbps'] = round(w.numel() * 3 / ms / 1e6, 1)
        bias = torch.randn(G, N, device='cuda', dtype=torch.bfloat16)
        ms = timeit(lambda: mx.mx_gemm(xq, xs, wq, ws, bias=bias, epilogue=mx.EPI_RELU))
        rec['mx_bias_relu_ms'] = round(ms, 4)
        print(json.dumps(rec), flush=True)
        out.append(rec)
    if cg == 2:
        print(json.dumps({'group': 'perf_cg2', 'ok': True}), flush=True)
        return
    # expert FFN of the flagship layer on one GPU (8 experts x 1024 rows, 4096 -> 14336 -> 4096), forward + backward
    E, C, M, H = 8, 1024, 4096, 14336
    x = torch.randn(E, C, M, device='cuda', dtype=torch.bfloat16, requires_grad=True)
    w1 = (torch.randn(E, H, M, device='cuda') * M ** -0.5).to(torch.bfloat16).requires_grad_()
    w2 = (torch.randn(E, H, M, device='cuda') * H ** -0.5).to(torch.bfloat16).requires_grad_()
    b1 = torch.zeros(E, H, device='cuda', dtype=torch.bfloat16, requires_grad=True)
    b2 = torch.zeros(E, M, device='cuda', dtype=torch.bfloat16, requires_grad=True)
    dy = torch.randn(E, C, M, device='cuda', dtype=torch.bfloat16)
    rec = {'ffn_shape': [E, C, M, H]}
    modes = {'bf16': lambda: gemm.fused_act_ffn(x, w1, b1, w2, b2, None, 'relu'),
             'fp8_row': lambda: gemm.fused_relu_ffn_fp8(x, w1, b1, w2, b2),
             'fp8_mx': lambda: mx.fused_relu_ffn_mx(x, w1, b1, w2, b2)}
    ref = None
    for name, fn in modes.items():
        def step():
            for t in (x, w1, w2, b1, b2):
                t.grad = None
            y = fn()
            y.backward(dy)
            return y
        ms = timeit(step, iters=10)               # weights unchanged between iterations: quantised copies are cached
        y = step()
        if ref is None:
            ref = (y.detach().float(), x.grad.float().clone())
        rec[name + '_fwd_bwd_ms'] = round(ms, 3)
        rec[name + '_y_rel_err'] = round(float((y.detach().float() - ref[0]).norm() / ref[0].norm()), 4)
        rec[name + '_dx_rel_err'] = round(float((x.grad.float() - ref[1]).norm() / ref[1].norm()), 4)

        def requant():
            gemm.invalidate_fp8_cache()
            return fn()
        if name != 'bf16':
            rec[name + '_fwd_with_weight_quantisation_ms'] = round(timeit(requant, iters=5), 3)
            rec[name + '_fwd_ms'] = round(timeit(fn, iters=10), 3)
    print(json.dumps(rec), flush=True)
    print(json.dumps({'group': 'perf', 'ok': True}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default='bench_out/mx')
    ap.add_argument('--group', default=None)
    ap.add_argument('--small_grid', type=int, default=0)     # 5 persistent CTAs: every CTA walks several tiles
    ap.add_argument('--quick', type=int, default=0)
    ap.add_argument('--no_perf', action='store_true')
    ap.add_argument('--only', default='')               # comma-separated group names of the plan
    args = ap.parse_args()
    if args.group == 'exact':
        return group_exact(bool(args.small_grid), bool(args.quick))
    if args.group == 'random':
        return group_random()
    if args.group == 'perf':
        return group_perf()
    if args.group == 'perf_cg2':
        return group_perf(2)
    if args.group == 'exact_cg2':
        return group_exact_cg2(bool(args.small_grid))
    os.makedirs(args.out, exist_ok=True)
    plan = [('exact_sub', ['--group', 'exact'], 240),
            ('exact_small_grid', ['--group', 'exact', '--small_grid', '1'], 100),
            ('random', ['--group', 'random'], 150),
            ('exact_cg2', ['--group', 'exact_cg2'], 120),
            ('exact_cg2_small_grid', ['--group', 'exact_cg2', '--small_grid', '1'], 120)]
    if args.only:
        plan = [p for p in plan if p[0] in args.only.split(',')]
    if not args.no_perf:
        plan.append(('perf_cg2', ['--group', 'perf_cg2'], 200))
        if not args.only:
            plan.append(('perf', ['--group', 'perf'], 200))
    summary = {}
    for name, extra, tmo in plan:
        t0 = time.time()
        try:
            r = subprocess.run([sys.executable, os.path.abspath(__file__)] + extra, capture_output=True, text=True, timeout=tmo)
            text, rc = r.stdout + '\n--- stderr ---\n' + r.stderr[-4000:], r.returncode
        except subprocess.TimeoutExpired as ex:
            text = ((ex.stdout or b'').decode() if isinstance(ex.stdout, bytes) else (ex.stdout or '')) + '\nTIMEOUT'
            rc = -9
        with open(os.path.join(args.out, name + '.log'), 'w') as f:
            f.write(text)
        oks = [json.loads(l).get('ok') for l in text.splitlines() if l.startswith('{"group"')]
        summary[name] = {'rc': rc, 'ok': bool(oks and all(oks)), 'sec': round(time.time() - t0, 1)}
        print(name, summary[name], flush=True)
        for l in text.splitlines():
            if l.startswith('{'):
                print('   ', l[:600], flush=True)
        if rc != 0:
            print(text[-1500:], flush=True)
    with open(os.path.join(args.out, 'summary.json'), 'w') as f:
        json.dump(summary, f, indent=1)


if __name__ == '__main__':
    main()
