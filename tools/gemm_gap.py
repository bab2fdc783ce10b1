"""Per-launch gap table of one fused GAN step: each bf16x3 GEMM launch against its floor.

    python tools/gemm_gap.py [--workload cfg2] [--warmup 10] [--steps 5] [--out FILE.md]

Captures --steps fused steps under torch.profiler (tools/trace_step.py: same labels, same capture) and takes each
launch's median kernel time over them.  For every GEMM launch it writes the executed TFLOP/s (bf16x3: 3 x 2MNK), the
algorithmic HBM bytes (operand planes read once, output planes + derivative code plane or fp32 written, split-K partials
of the weight gradients), the floor max(executed flops / tensor peak, bytes / HBM bandwidth) and time over floor.  The
non-GEMM kernels follow with their times.  The card's name, power limit and max SM clock are read in the same run.

The peaks are the H100 SXM data-sheet figures (dense BF16 989 TFLOP/s, HBM3 3.35 TB/s at 700 W): the floor is a bound
no launch reaches, and "x floor" says how far each launch sits from it, not what is attainable.
"""
import argparse
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import trace_step  # noqa: E402

PEAK_TFLOPS = 989.0     # H100 SXM, dense BF16
PEAK_TBS = 3.35         # H100 SXM, HBM3
TC_BM, TC_MN_BK = 128, 32


def pitch(cols):
    return (cols + 15) // 16 * 16


def pick_bn(n):
    bn = (n + 63) // 64 * 64
    if bn <= 128:
        return bn
    tiles = (n + 127) // 128
    return ((n + tiles - 1) // tiles + 63) // 64 * 64


def mn_splits(red, rows_a, cols_b, sms):
    """Split count of a weight-gradient launch (gemm_tc.cu mn_partial_bytes)."""
    bn = pick_bn(cols_b)
    tiles = ((rows_a + TC_BM - 1) // TC_BM) * ((cols_b + bn - 1) // bn)
    blocks = (red + TC_MN_BK - 1) // TC_MN_BK
    splits = max(1, sms // tiles)
    splits = min(splits, blocks)
    chunk = (blocks + splits - 1) // splits * TC_MN_BK
    return (red + chunk - 1) // chunk


def kk_bytes(label, rows, n, k, kind):
    b = 2 * 2 * (rows * pitch(k) + n * pitch(k))          # hi + lo planes of both operands
    if kind == "planes":
        b += 2 * 2 * rows * pitch(n)                        # hi + lo output planes
        b += 4 * rows * ((n + 15) // 16)                    # derivative code: written (fwd) or read (bwd)
    else:
        b += 4 * rows * n * (2 if "+=" in label else 1)     # fp32 out (read + write when accumulating)
    return b


def mn_bytes(rows, n, k, sms):
    # gW[n][k] = sum_m gz[m][n] x[m][k]: planes of gz and x read, one fp32 partial per split written (+ bias column sums)
    splits = mn_splits(rows, n, k, sms)
    return 2 * 2 * rows * (pitch(n) + pitch(k)) + 4 * splits * (n * k + n), splits


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                              "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return out.stdout.strip() or out.stderr.strip()
    except Exception as e:   # the table is still worth having without the query
        return "nvidia-smi unavailable (%s): %s" % (e, torch.cuda.get_device_name(0))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="cfg2",
                    choices=[k for k, v in trace_step.bench.WORKLOADS.items() if v["kind"] == "mlp"])
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--out", default=None, help="markdown file for the table (default: stdout only)")
    ap.add_argument("--pdl", action="store_true",
                    help="keep programmatic dependent launch on: a kernel's traced span then includes its wait for the "
                         "previous one, so per-launch times overlap (default: off, one kernel at a time)")
    args = ap.parse_args()
    if not args.pdl:
        os.environ["GANTTS_B200_PDL"] = "0"     # read once, at the library's first launch
    steps, w, _ = trace_step.capture(args)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    kernels = [(steps[0][i][0], statistics.median(s[i][1] for s in steps)) for i in range(len(steps[0]))]
    scale = w["B"] * w["T"] // 32000
    kk, mn = list(trace_step.KK), list(trace_step.MN)
    gemm, other = [], []
    for name, us in kernels:
        n = trace_step.short(name)
        if not n.startswith("gemm_bf16x3_kernel<"):
            other.append((n, us))
            continue
        is_mn = n.startswith("gemm_bf16x3_kernel<true") or n.startswith("gemm_bf16x3_kernel<1")
        queue = mn if is_mn else kk
        if not queue:
            gemm.append(("(unlabelled GEMM)", us, None, None, ""))
            continue
        ent = queue.pop(0)
        rows, N, K = ent[1] * scale, ent[2], ent[3]
        flops = 3.0 * 2.0 * rows * N * K
        if is_mn:
            b, splits = mn_bytes(rows, N, K, sms)
            note = "MN, %d splits" % splits
        else:
            b = kk_bytes(ent[0], rows, N, K, ent[4])
            note = "KK, BN %d, %s out" % (pick_bn(N), ent[4])
        gemm.append(("%s [%d x %d x %d]" % (ent[0], rows, N, K), us, flops, b, note))

    lines = ["# GEMM gap table of one fused %s step (torch.profiler; median of %d steps after %d warm-up; PDL %s)"
             % (args.workload, args.steps, args.warmup, "on" if args.pdl else "off"), "",
             "Card (name, power limit, max SM clock): %s.  %d SMs." % (card(), sms),
             "Floor = max(executed flops / %.0f TFLOP/s, bytes / %.2f TB/s) (H100 SXM data sheet, not measured)."
             % (PEAK_TFLOPS, PEAK_TBS), "",
             "| # | GEMM launch | layout | us | executed TFLOP/s | HBM MB | floor us | bound | x floor |",
             "|---|---|---|---|---|---|---|---|---|"]
    g_us = g_fl = g_floor = 0.0
    for i, (label, us, fl, b, note) in enumerate(gemm):
        if fl is None:
            lines.append("| %d | %s | | %.1f | | | | | |" % (i, label, us))
            continue
        t_fl, t_b = fl / (PEAK_TFLOPS * 1e12) * 1e6, b / (PEAK_TBS * 1e12) * 1e6
        floor = max(t_fl, t_b)
        g_us += us
        g_fl += fl
        g_floor += floor
        lines.append("| %d | %s | %s | %.1f | %.0f | %.1f | %.1f | %s | %.2f |"
                     % (i, label, note, us, fl / (us * 1e-6) / 1e12, b / 1e6, floor,
                        "tensor" if t_fl >= t_b else "HBM", us / floor))
    o_us = sum(us for _, us in other)
    lines += ["", "GEMM launches: %d, %.1f us, %.0f executed TFLOP/s, floor %.1f us (%.2f x floor)."
              % (len(gemm), g_us, g_fl / (g_us * 1e-6) / 1e12 if g_us else 0.0, g_floor,
                 g_us / g_floor if g_floor else 0.0)]
    if kk or mn:
        lines.append("%d GEMM labels unused: the launch structure differs from trace_step.py's lists." % (len(kk) + len(mn)))
    lines += ["", "## Other kernels (%d launches, %.1f us)" % (len(other), o_us), "", "| kernel | us |", "|---|---|"]
    lines += ["| `%s` | %.1f |" % (n[:70], us) for n, us in other]
    text = "\n".join(lines) + "\n"
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
