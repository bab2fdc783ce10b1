"""Time the fused GAN step (FusedGanStep: one C call per mini-batch) against the modular GanTrainer (Python autograd
over the native ops) on the In2OutRNNHighwayNet generator (the RNN VC model, bench.py cfg3) and the same MLP discriminator.

Workload:
  cfg3  In2OutRNNHighwayNet 177 -> 177 (static 59, 3 x 512 bidirectional LSTM, LSTM dropout 0.5), D 59 -> 256 -> 256 -> 1
        with dropout 0.5, Adagrad lr 0.01 wd 0, B = 16 x T = 2000 full-length, w_d = 1, mse_w = 0, mge_w = 1

The two paths alternate in one process, round by round, each round timed with CUDA events after a warm-up; the GPU's
name, power limit and maximum SM clock are queried in the same run (nvidia-smi, read-only).  Needs a CUDA device.

    python tools/time_rnn_highway_step.py [--rounds 5] [--steps 5] [--warmup 3] [--json OUT]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

WINDOWS = [(0, 0, np.array([1.0])), (1, 1, np.array([-0.5, 0.0, 0.5])), (1, 1, np.array([1.0, -2.0, 1.0]))]
WORKLOADS = {
    "cfg3": dict(B=16, T=2000, w_d=1.0, mse_w=0.0, mge_w=1.0),
}


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    line = q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else ""
    parts = [s.strip() for s in line.split(",")] if line else []
    return {"name": parts[0] if parts else torch.cuda.get_device_name(0),
            "power_limit": parts[1] if len(parts) > 1 else None,
            "sm_clock_max": parts[2] if len(parts) > 2 else None}


def run(name, w, rounds, steps, warmup, dev):
    import gantts_b200
    from gantts_b200 import fused, step as gstep
    from oracle import nnmnkwii_port as nnp
    B, T = w["B"], w["T"]
    hp = gstep.HParams(windows=WINDOWS, stream_sizes=[177], has_dynamic_features=[True], adversarial_streams=[True],
                       mask_nth_mgc_for_adv_loss=0, discriminator_linguistic_condition=False)
    kw = dict(w_d=w["w_d"], mse_w=w["mse_w"], mge_w=w["mge_w"], lr=0.01, weight_decay=0.0)

    def models():
        torch.manual_seed(1234)
        mg = gantts_b200.models.In2OutRNNHighwayNet(in_dim=177, out_dim=177, static_dim=59, num_hidden=3,
                                                    hidden_dim=512, bidirectional=True, dropout=0.5)
        md = gantts_b200.models.MLP(59, 1, 2, 256, dropout=0.5, last_sigmoid=True)
        return mg.to(dev).train(), md.to(dev).train()
    g = torch.Generator().manual_seed(7)
    x = torch.randn(B, T, 177, generator=g).to(dev)
    y = torch.randn(B, T, 177, generator=g).to(dev)
    lengths = torch.full((B,), T, dtype=torch.int64, device=dev)
    adv_w = 1.0 if w["w_d"] > 0 else 0.0
    fs = fused.FusedGanStep(*models(), hp, B, T, seed=1, **kw)
    tr = gstep.GanTrainer(*models(), hp, **kw)
    R = torch.from_numpy(nnp.unit_variance_mlpg_matrix(WINDOWS, T)).to(dev)
    steps_of = {"fused": lambda: fs.step(x, y, lengths, adv_w=adv_w),
                "modular": lambda: tr.step(x, y, lengths, R, adv_w=adv_w)}
    for fn in steps_of.values():
        for _ in range(warmup):
            fn()
    torch.cuda.synchronize()
    ms = {k: [] for k in steps_of}
    for _ in range(rounds):
        for k, fn in steps_of.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(steps):
                fn()
            b.record()
            b.synchronize()
            ms[k].append(a.elapsed_time(b) / steps)
    out = {"workload": name, "B": B, "T": T, "rounds": rounds, "steps_per_round": steps}
    for k, v in ms.items():
        med = float(np.median(v))
        out[k] = {"ms_per_step_median": round(med, 4), "ms_per_step_min": round(min(v), 4),
                  "ms_per_step_max": round(max(v), 4), "frames_per_s": round(B * T / med * 1e3, 1)}
    out["speedup_fused_vs_modular"] = round(out["modular"]["ms_per_step_median"] / out["fused"]["ms_per_step_median"], 3)
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--workload", choices=sorted(WORKLOADS) + ["all"], default="all")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--json", default=None, help="also write the results to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_rnn_highway_step.py: needs a CUDA device (there is no CPU path to time)")
    import __graft_entry__
    __graft_entry__.build()
    dev = torch.device("cuda:0")
    res = {"gpu": gpu_info(), "results": []}
    for name in (sorted(WORKLOADS) if args.workload == "all" else [args.workload]):
        r = run(name, WORKLOADS[name], args.rounds, args.steps, args.warmup, dev)
        print(json.dumps(r), flush=True)
        res["results"].append(r)
    print(json.dumps({"gpu": res["gpu"]}))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
