"""The objective measures of 100 ragged utterances (200..1000 frames, 60 columns, the utterances of time_generate.py) at
the notebooks' n = 4096: device FeatureStats, host to host (pad, copy each batch to the device, gantts_global_variance and
gantts_modspec, copy the variances and the summed spectra back), against the per-utterance numpy loop of the notebooks
(np.var and np.log(modspec) in float64, then np.mean).  The two alternate within each round, timed with CUDA events
around a device synchronise; "device_kernels" times the kernels alone on batches already on the device.  The outputs
are checked against each other within the test tolerances.

    python tools/time_objective.py [--json OUT]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(1, os.path.join(ROOT, "tests"))
import __graft_entry__  # noqa: E402

__graft_entry__.build()
from gantts_b200 import generate, objective  # noqa: E402
import objective_oracle as ref  # noqa: E402

dev = torch.device("cuda:0")
N, D, NFFT, ROUNDS, BATCH = 100, 60, 4096, 5, 20


def utterances():
    rng = np.random.RandomState(0)
    lens = rng.randint(200, 1001, N)
    return [(rng.randn(n, D) * rng.uniform(0.1, 2.0, D) + rng.randn(D)).astype(np.float32) for n in lens]


def numpy_loop(arrays):
    gvs = [np.var(a.astype(np.float64), axis=0) for a in arrays]
    mss = [np.log(ref.modspec(a, NFFT)) for a in arrays]
    return np.array(gvs), np.mean(np.array(gvs), axis=0), np.mean(np.array(mss), axis=0)


def device(arrays):
    stats = objective.FeatureStats(D, NFFT, dev)
    plan = generate.plan_batches([len(a) for a in arrays], BATCH)
    for idx in plan:
        stats.add(objective.pad_batch([arrays[i] for i in idx], dev),
                  torch.tensor([len(arrays[i]) for i in idx], dtype=torch.int64).to(dev))
    gv, gv_mean, ms_mean = stats.result()
    order = np.array([i for idx in plan for i in idx])
    gv_in = np.empty_like(gv)
    gv_in[order] = gv
    return gv_in, gv_mean, ms_mean


def device_kernels(batches):
    stats = objective.FeatureStats(D, NFFT, dev)
    for x, lengths in batches:
        stats.add(x, lengths)
    return stats


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    res = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), res


def disagreement(a, b, arrays):
    """The largest errors of a against the float64 loop b, each over its test tolerance (<= 1 passes)."""
    gv_err = max(float(np.max(np.abs(a[0] - b[0]) / np.abs(b[0]))), float(np.max(np.abs(a[1] - b[1]) / b[1]))) / 1e-12
    powers = [ref.modspec(x, NFFT) for x in arrays]
    big = np.all([p > 1e-3 * p.max(axis=0, keepdims=True) for p in powers], axis=0)
    ms_err = float(np.max(np.abs(a[2] - b[2])[big])) / 1e-6
    return {"gv_over_tol": gv_err, "ms_mean_over_tol": ms_err, "ms_bins_compared": float(big.mean()),
            "ms_mean_max_abs_diff_all_bins": float(np.max(np.abs(a[2] - b[2])))}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--json", default=None, help="also write the results to this file")
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    arrays = utterances()
    batches = [(objective.pad_batch([arrays[i] for i in idx], dev),
                torch.tensor([len(arrays[i]) for i in idx], dtype=torch.int64).to(dev))
               for idx in generate.plan_batches([len(a) for a in arrays], BATCH)]
    runs = [("device", lambda: device(arrays)), ("numpy_loop", lambda: numpy_loop(arrays)),
            ("device_kernels", lambda: device_kernels(batches))]
    for _, fn in runs:                                            # warm every shape once
        fn()
    ms = {name: [] for name, _ in runs}
    agree = None
    for _ in range(ROUNDS):
        results = {}
        for name, fn in runs:
            t, results[name] = timed(fn)
            ms[name].append(t)
        err = disagreement(results["device"], results["numpy_loop"], arrays)
        agree = err if agree is None else {k: max(agree[k], v) for k, v in err.items()}
    report = {"gpu": gpu, "utterances": N, "frames": int(sum(len(a) for a in arrays)), "columns": D, "n": NFFT,
              "batch_size": BATCH, "rounds": ROUNDS, "max_error_over_tolerance": agree}
    for name, v in ms.items():
        report["%s_ms" % name] = {"median": float(np.median(v)), "min": float(min(v)), "max": float(max(v))}
    report["speedup"] = report["numpy_loop_ms"]["median"] / report["device_ms"]["median"]
    print(json.dumps(report, indent=1))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(report, f, indent=1)
    if agree["gv_over_tol"] > 1 or agree["ms_mean_over_tol"] > 1:
        raise SystemExit("time_objective: the device and the numpy loop disagree beyond the test tolerances")


if __name__ == "__main__":
    main()
