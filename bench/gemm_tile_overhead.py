#!/usr/bin/env python3
"""Fixed cost per output tile of the 128 x 256 grouped GEMM, per epilogue (needs a GPU).

The fc1 / dh geometry of the flagship step (G=8 experts, M=2048 rows, N=14336 columns, K-major bf16 operands) is timed
at several K.  The tile count does not depend on K, so for each epilogue

    time = tiles_per_SM x (t_tile + t_kb x K / 64)

is fitted by least squares: t_kb is the cost of one 64-deep K block of a tile's main loop and t_tile the cost of
everything around it (epilogue, output store, side inputs, pipeline fill).  tiles_per_SM is the busiest SM's count.
All variants are interleaved round by round, so clock drift hits them alike.

    python bench/gemm_tile_overhead.py [--ks 1024,2048,4096,8192] [--rounds 5] [--json out.json]
"""
import argparse
import json
import math
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

G, M, N = 8, 2048, 14336
BM, BN = 128, 256


def gpu_info(index):
    q = 'name,power.limit,clocks.sm,clocks.max.sm'
    try:
        out = subprocess.run(['nvidia-smi', '-i', str(index), '--query-gpu=' + q, '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return dict(zip(q.split(','), [s.strip() for s in out.split(',')]))
    except Exception as ex:  # noqa
        return {'error': repr(ex)}


def fit(ks, ms, tiles_per_sm):
    """Least-squares line through (K / 64, ms); returns t_tile, t_kb in microseconds per tile."""
    xs = [k / 64 for k in ks]
    n = len(xs)
    mx, my = sum(xs) / n, sum(ms) / n
    slope = sum((x - mx) * (y - my) for x, y in zip(xs, ms)) / sum((x - mx) ** 2 for x in xs)
    icpt = my - slope * mx
    resid = max(abs(icpt + slope * x - y) for x, y in zip(xs, ms))
    return icpt * 1e3 / tiles_per_sm, slope * 1e3 / tiles_per_sm, resid * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--ks', default='1024,2048,4096,8192')
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--reps', type=int, default=4, help='launches per timed sample')
    ap.add_argument('--json', default=None)
    args = ap.parse_args()

    import torch
    from tutel_b200.ops import gemm as GM
    if not torch.cuda.is_available():
        raise SystemExit('gemm_tile_overhead: needs a CUDA GPU')
    dev = torch.device('cuda', torch.cuda.current_device())
    ks = [int(k) for k in args.ks.split(',')]
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    tiles = G * math.ceil(M / BM) * math.ceil(N / BN)
    tiles_per_sm = math.ceil(tiles / sms)

    g = torch.Generator(device=dev).manual_seed(2024)
    rnd = lambda *s, sc=1.0: (torch.randn(*s, device=dev, generator=g) * sc).bfloat16()
    bias = rnd(G, N, sc=0.1)
    aux = rnd(G, M, N)
    colsum = torch.zeros(G, N, device=dev)
    out = torch.empty(G, M, N, device=dev, dtype=torch.bfloat16)
    ops = {}
    for k in ks:
        a, b = rnd(G, M, k), rnd(G, N, k, sc=k ** -0.5)
        bt = b.transpose(1, 2)
        ops[k] = {
            'none': lambda a=a, b=b: GM.raw_gemm(a, b, out=out),
            'bias_relu': lambda a=a, b=b: GM.raw_gemm(a, b, epilogue=GM.EPI_BIAS_RELU, bias=bias, out=out),
            'relu_bwd': lambda a=a, b=b: GM.raw_gemm(a, b, epilogue=GM.EPI_RELU_BWD, aux=aux, out=out),
            'relu_bwd+colsum': lambda a=a, b=b: GM.raw_gemm(a, b, epilogue=GM.EPI_RELU_BWD, aux=aux, colsum=colsum, out=out),
            'add': lambda a=a, b=b: GM.raw_gemm(a, b, epilogue=GM.EPI_ADD, aux=aux, out=out),
            'torch.matmul': lambda a=a, bt=bt: torch.matmul(a, bt, out=out),
        }
    variants = list(ops[ks[0]])
    for k in ks:
        for fn in ops[k].values():
            fn(); fn()
    torch.cuda.synchronize()

    times = {(v, k): [] for v in variants for k in ks}
    ev = lambda: torch.cuda.Event(enable_timing=True)
    for _ in range(args.rounds):
        for k in ks:
            for v in variants:
                s, e = ev(), ev()
                s.record()
                for _ in range(args.reps):
                    ops[k][v]()
                e.record()
                torch.cuda.synchronize()
                times[(v, k)].append(s.elapsed_time(e) / args.reps)
    info = gpu_info(dev.index or 0)   # right after the timed rounds: the SM clock under this load

    med = {key: sorted(ts)[len(ts) // 2] for key, ts in times.items()}
    res = {'gpu': info, 'G': G, 'M': M, 'N': N, 'ks': ks, 'tiles': tiles, 'sms': sms, 'tiles_per_sm': tiles_per_sm,
           'variants': {}}
    print('%s, power limit %s, SM clock %s (max %s)' % (info.get('name'), info.get('power.limit'),
                                                       info.get('clocks.sm'), info.get('clocks.max.sm')))
    print('G=%d M=%d N=%d bf16, %d tiles of %dx%d, %d per SM' % (G, M, N, tiles, BM, BN, tiles_per_sm))
    hdr = '%-16s' % 'epilogue' + ''.join('%12s' % ('K=%d ms' % k) for k in ks) + '%12s%12s%12s' % (
        't_tile us', 't_kb us', 'resid us')
    print(hdr)
    for v in variants:
        ms = [med[(v, k)] for k in ks]
        t_tile, t_kb, resid = fit(ks, ms, tiles_per_sm)
        tf = [2.0 * G * M * N * k / (m * 1e-3) * 1e-12 for k, m in zip(ks, ms)]
        res['variants'][v] = {'ms': ms, 'tflops': tf, 't_tile_us': t_tile, 't_kb_us': t_kb, 'max_resid_us': resid,
                              'spread_ms': [max(times[(v, k)]) - min(times[(v, k)]) for k in ks]}
        print('%-16s' % v + ''.join('%12.3f' % m for m in ms) + '%12.2f%12.3f%12.1f' % (t_tile, t_kb, resid))
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
