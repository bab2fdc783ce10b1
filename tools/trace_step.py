"""Per-launch view of one fused GAN step under torch.profiler (CUDA activities).

    python tools/trace_step.py [--workload cfg2] [--warmup 10] [--steps 3] [--out FILE.md]

Runs `--warmup` fused steps, then `--steps` more under the profiler with a synchronise after each, and splits the
kernel list into steps (every step launches the same kernels).  Writes the launch list of the middle step in launch
order with each kernel's duration.  The tensor-core GEMM launches are labelled with their shapes (the per-kind launch
order in KK and MN below) and get their executed TFLOP/s (3 x 2MNK for the bf16x3 split) and share of the step.
Tracing adds host overhead between launches, so the step span here is not a bench value; compare kernel times and
shares, and take step times from bench.py.
"""
import argparse
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402

M = 32000
# K-major launches (y = x W^T or gx = gz W) and MN-major launches (gW = gz^T x) of one step, in launch order per kind:
# (label, rows, N, K, output kind)
KK = [("G fwd 425->512 (+act, planes)", M, 512, 425, "planes"), ("G fwd 512->512", M, 512, 512, "planes"),
      ("G fwd 512->512", M, 512, 512, "planes"), ("G fwd 512->187 (fp32 y_hat, ld 187)", M, 187, 512, "f32"),
      ("D fwd 58->256, real|fake 2M rows", 2 * M, 256, 58, "planes"), ("D fwd 256->256, 2M rows", 2 * M, 256, 256, "planes"),
      ("D fwd 256->256, 2M rows", 2 * M, 256, 256, "planes"),
      ("D bwd gx3 = gz W", 2 * M, 256, 256, "planes"), ("D bwd gx2", 2 * M, 256, 256, "planes"),
      ("D bwd gx1 (fake half, fp32, ld 58)", M, 58, 256, "f32"),
      ("D(adv) fwd 58->256, M rows", M, 256, 58, "planes"), ("D(adv) fwd 256->256", M, 256, 256, "planes"),
      ("D(adv) fwd 256->256", M, 256, 256, "planes"),
      ("D(adv) bwd gx3", M, 256, 256, "planes"), ("D(adv) bwd gx2", M, 256, 256, "planes"),
      ("D(adv) bwd gx1 -> += g_static window (fp32)", M, 58, 256, "f32"),
      ("G bwd gx4 = gz W (512 wide)", M, 512, 187, "planes"), ("G bwd gx3", M, 512, 512, "planes"),
      ("G bwd gx2", M, 512, 512, "planes")]
MN = [("D bwd gW3 = gz^T h (256x256)", 2 * M, 256, 256), ("D bwd gW2", 2 * M, 256, 256), ("D bwd gW1 (256x58)", 2 * M, 256, 58),
      ("G bwd gW4 (187x512)", M, 187, 512), ("G bwd gW3 (512x512)", M, 512, 512), ("G bwd gW2 (512x512)", M, 512, 512),
      ("G bwd gW1 (512x425)", M, 512, 425)]


def short(name):
    n = name.replace("gantts::", "").replace("void ", "")
    cut = n.find("(")
    return n[:cut] if cut > 0 else n


def label_gemms(kernels, scale):
    """kernels: [(name, us)] of one step -> [(name, us, label, executed flops or None)]."""
    kk = list(KK)
    mn = list(MN)
    out = []
    for name, us in kernels:
        n = short(name)
        label, flops = "", None
        if n.startswith("gemm_bf16x3_kernel<"):
            is_mn = n.startswith("gemm_bf16x3_kernel<true") or n.startswith("gemm_bf16x3_kernel<1")
            queue = mn if is_mn else kk
            if queue:
                ent = queue.pop(0)
                label, rows, N, K = ent[0], ent[1] * scale, ent[2], ent[3]
                flops = 3.0 * 2.0 * rows * N * K
                label = "%s [%d x %d x %d]" % (label, rows, N, K)
            else:
                label = "(unlabelled GEMM)"
        out.append((n, us, label, flops))
    return out, len(kk) + len(mn)


def capture(args):
    """Runs args.warmup fused steps, then args.steps under the profiler.  Returns (per-step kernel lists [[(name, us)]],
    workload dict, us from first start to last end of the middle step)."""
    if not torch.cuda.is_available():
        raise SystemExit("%s: no CUDA device" % os.path.basename(sys.argv[0]))
    import __graft_entry__
    __graft_entry__.build()
    from gantts_b200 import fused, step as gstep
    from torch.profiler import ProfilerActivity, profile

    dev = torch.device("cuda", 0)
    w = bench.WORKLOADS[args.workload]
    torch.manual_seed(1234)
    mg, md = bench.build_models(w, dev)
    hpd = w["hp"]
    hp = gstep.HParams(windows=bench.WINDOWS, stream_sizes=hpd["stream_sizes"],
                       has_dynamic_features=hpd["has_dynamic_features"], adversarial_streams=hpd["adversarial_streams"],
                       mask_nth_mgc_for_adv_loss=hpd["mask_nth_mgc_for_adv_loss"],
                       discriminator_linguistic_condition=False)
    fs = fused.FusedGanStep(mg, md, hp, w["B"], w["T"], w_d=1.0, mse_w=0.0, mge_w=1.0)
    lengths = torch.full((w["B"],), w["T"], dtype=torch.int64, device=dev)
    batches = [(x.to(dev), y.to(dev)) for x, y in bench.make_batches(w, 1234, bench.NUM_BATCHES, pinned=False)]
    frames = w["B"] * w["T"]
    for i in range(args.warmup):
        fs.step(*batches[i % len(batches)], lengths, frames=frames)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(args.steps):
            fs.step(*batches[i % len(batches)], lengths, frames=frames)
            torch.cuda.synchronize()
    evs = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
           and not e.name.startswith(("Memcpy", "Memset", "[memory]"))]
    evs.sort(key=lambda e: e.time_range.start)
    if not evs or len(evs) % args.steps:
        raise SystemExit("%s: %d kernels over %d steps do not split into equal steps"
                         % (os.path.basename(sys.argv[0]), len(evs), args.steps))
    per = len(evs) // args.steps
    steps = [[(e.name, e.time_range.end - e.time_range.start) for e in evs[per * i: per * (i + 1)]]
             for i in range(args.steps)]
    mid = evs[per * (args.steps // 2): per * (args.steps // 2 + 1)]
    return steps, w, mid[-1].time_range.end - mid[0].time_range.start


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="cfg2", choices=[k for k, v in bench.WORKLOADS.items() if v["kind"] == "mlp"])
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--out", default=None, help="markdown file for the launch list (default: stdout only)")
    args = ap.parse_args()
    steps, w, span = capture(args)
    kernels = steps[args.steps // 2]
    per = len(kernels)
    rows, unmatched = label_gemms(kernels, w["B"] * w["T"] // 32000)
    tot = sum(us for _, us, _, _ in rows)
    gemm_us = sum(us for _, us, _, f in rows if f is not None)
    gemm_fl = sum(f for _, _, _, f in rows if f is not None)
    lines = ["# Launch list of one fused %s step (torch.profiler, CUDA activities; step %d of %d after %d warm-up)"
             % (args.workload, args.steps // 2 + 1, args.steps, args.warmup), "",
             "Device: %s.  %d launches, %.1f us of kernel time, %.1f us from first start to last end (traced: host "
             "overhead between launches is not a bench value)." % (torch.cuda.get_device_name(0), per, tot, span), "",
             "| # | kernel | GEMM | us | executed TFLOP/s | share of kernel time |", "|---|---|---|---|---|---|"]
    for i, (n, us, label, fl) in enumerate(rows):
        tf = "%.0f" % (fl / (us * 1e-6) / 1e12) if fl and us else ""
        lines.append("| %d | `%s` | %s | %.1f | %s | %.3f |" % (i, n[:60], label, us, tf, us / tot if tot else 0.0))
    lines += ["", "GEMM launches: %d, %.1f us = %.3f of kernel time, %.0f TFLOP/s executed (bf16x3 = 3 x 2MNK)."
              % (sum(1 for r in rows if r[3] is not None), gemm_us, gemm_us / tot if tot else 0.0,
                 gemm_fl / (gemm_us * 1e-6) / 1e12 if gemm_us else 0.0)]
    if unmatched:
        lines.append("%d GEMM labels unused: the launch structure differs from the KK and MN lists." % unmatched)
    text = "\n".join(lines) + "\n"
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
