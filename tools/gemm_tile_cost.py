"""Per-tile fixed cost of the K-major bf16x3 GEMM with the planes epilogue (EPI_PLANES_FWD).

    python tools/gemm_tile_cost.py [--M 32000] [--N 512] [--ks 64,128,256,512,1024] [--p 0.5] [--iters 50]

Times the first layer of a [K, N, 1] MLP forward (gantts_mlp_fwd: one K-major launch that writes the bf16 hi/lo planes
and the derivative codes of an M x N hidden layer; the 1-wide last layer is a GEMV and is not counted) with the library's
per-launch CUDA events, for each K.  Every persistent CTA takes the same number of 128 x BN tiles, so a launch is
`waves` rounds of one tile per CTA, and a tile is K / 64 ring stages followed by one epilogue:

    time = waves * (a + b * K / 64)

The least-squares intercept `a` is the per-tile fixed cost (epilogue arithmetic, plane and code stores, mainloop ramp)
and `b` the cost of one 64-deep stage.  The card's name, power limit and max SM clock are read in the same run.
"""
import argparse
import ctypes
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__  # noqa: E402

TC_BM = 128


def pick_bn(n):
    bn = (n + 63) // 64 * 64
    if bn <= 128:
        return bn
    tiles = (n + 127) // 128
    return ((n + tiles - 1) // tiles + 63) // 64 * 64


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                              "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return out.stdout.strip() or out.stderr.strip()
    except Exception as e:
        return "nvidia-smi unavailable (%s): %s" % (e, torch.cuda.get_device_name(0))


def time_launch(lib, ops, M, N, K, p, iters, dev):
    """Mean microseconds of the K-major planes launch of one forward."""
    torch.manual_seed(K)
    Ws = [torch.randn(N, K, device=dev) / K ** 0.5, torch.randn(1, N, device=dev) / N ** 0.5]
    bs = [torch.randn(N, device=dev) * 0.1, torch.zeros(1, device=dev)]
    x = torch.rand(M, K, device=dev)
    with torch.no_grad():
        for _ in range(10):
            ops.mlp_stack(x, Ws, bs, p=p, training=p > 0, seed=7)
        torch.cuda.synchronize()
        lib.gantts_profile_enable(1)
        for _ in range(iters):
            ops.mlp_stack(x, Ws, bs, p=p, training=p > 0, seed=7)
        torch.cuda.synchronize()
    ms, wk, cnt = (ctypes.c_double * 8)(), (ctypes.c_double * 8)(), (ctypes.c_longlong * 8)()
    lib.gantts_profile_collect(ms, wk, cnt)
    lib.gantts_profile_enable(0)
    if cnt[0] != iters:
        raise RuntimeError("expected one K-major launch per forward, counted %d over %d" % (cnt[0], iters))
    return ms[0] / cnt[0] * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--M", type=int, default=32000)
    ap.add_argument("--N", type=int, default=512)
    ap.add_argument("--ks", default="64,128,256,512,1024")
    ap.add_argument("--p", type=float, default=0.5, help="dropout probability of the hidden layer (0 = off)")
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--tag", default="", help="label printed with the results")
    args = ap.parse_args()
    __graft_entry__.build()
    from gantts_b200 import _lib, ops
    lib = _lib.load()
    dev = torch.device("cuda:0")
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    ks = [int(k) for k in args.ks.split(",")]
    bn = pick_bn(args.N)
    tiles = -(-args.M // TC_BM) * -(-args.N // bn)
    waves = -(-tiles // sms)
    print("Card (name, power limit, max SM clock): %s.  %d SMs.  %s" % (card(), sms, args.tag))
    print("M %d, N %d (BN %d), dropout p %.2f: %d tiles, %d per CTA" % (args.M, args.N, bn, args.p, tiles, waves))
    rows = []
    for k in ks:
        us = time_launch(lib, ops, args.M, args.N, k, args.p, args.iters, dev)
        rows.append((k, us))
    xs = [k / 64.0 for k, _ in rows]
    ys = [us / waves for _, us in rows]
    n = len(rows)
    mx, my = sum(xs) / n, sum(ys) / n
    sxx = sum((x - mx) ** 2 for x in xs)
    b = sum((x - mx) * (y - my) for x, y in zip(xs, ys)) / sxx if sxx else 0.0
    a = my - b * mx
    print("| K | us / launch | us / tile round | fit | stage MMA TFLOP/s executed |")
    print("|---|---|---|---|---|")
    for (k, us), y in zip(rows, ys):
        fl = 3.0 * 2.0 * args.M * args.N * k
        print("| %d | %.1f | %.2f | %.2f | %.0f |" % (k, us, y, a + b * k / 64.0, fl / (us * 1e-6) / 1e12))
    print("fit: a = %.2f us per tile (fixed), b = %.3f us per 64-deep stage  %s" % (a, b, args.tag))


if __name__ == "__main__":
    main()
