"""Time one epoch of train.py-style ragged mini-batches through the fused GAN step and through GanTrainer.

The epoch is built like train.py's DataLoader with collate_fn (train.py:145-155): utterance lengths drawn from a seed,
sorted descending, cut into batches of B, each batch padded to its OWN max_len, the last batch short (no drop_last).  It
runs at the widths of the `vc` and `tts_acoustic` workloads of tools/time_fused_step.py (same models and optimisers;
capacity B x T = 20 x 1000) through
  fused_ragged   FusedGanStep with per-batch shapes (each call its own (b, t); device-built MLPG tables, cached)
  fused_padded   FusedGanStep with every batch padded to the capacity T (what a fixed-shape step needs; MLPG then solves
                 over T frames, so the results differ from the reference's, see DESIGN section 5)
  modular        GanTrainer with R = unit_variance_mlpg_matrix(windows, max_len) per batch (built before timing)
One warm-up epoch per path (every shape and table), then rounds of one epoch per path, alternating, each timed with CUDA
events.  Reported: ms per epoch (median, min, max) and valid frames per second (sum of the lengths over the epoch time).
The device MLPG table builder (ops.mlpg_table_device) is timed once at T = 2000.  The GPU's name and power limit are
queried in the same run (nvidia-smi, read-only).  Needs a CUDA device.

    python tools/time_ragged_epoch.py [--workload vc|tts_acoustic|all] [--utterances N] [--rounds R] [--json OUT]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

import time_fused_step as tfs  # noqa: E402


def epoch(n_utt, B, T, d_in, d_out, seed):
    """[(x, y, lengths list)] on the host: collate_fn batches of a seeded epoch, lengths in [T / 4, T]."""
    rng = np.random.RandomState(seed)
    lens_all = sorted((int(v) for v in rng.randint(T // 4, T + 1, n_utt)), reverse=True)
    g = torch.Generator().manual_seed(seed)
    out = []
    for i in range(0, n_utt, B):
        lens = lens_all[i:i + B]
        t = lens[0]
        x = torch.randn(len(lens), t, d_in, generator=g)
        y = torch.randn(len(lens), t, d_out, generator=g)
        for b, n in enumerate(lens):
            x[b, n:] = 0
            y[b, n:] = 0
        out.append((x, y, lens))
    return out


def run(name, n_utt, rounds, dev):
    from gantts_b200 import fused, step as gstep
    from oracle import nnmnkwii_port as nnp
    w = tfs.WORKLOADS[name]
    B, T = w["B"], w["T"]
    hp = tfs.hparams(name)
    d_in, d_out = w.get("in_dim", 177), w.get("out_dim", 177)
    host = epoch(n_utt, B, T, d_in, d_out, 11)
    batches = []
    for x, y, lens in host:
        t = x.shape[1]
        pad = (0, 0, 0, T - t)
        batches.append(dict(x=x.to(dev), y=y.to(dev), lengths=torch.LongTensor(lens).to(dev),
                            xp=torch.nn.functional.pad(x, pad).to(dev), yp=torch.nn.functional.pad(y, pad).to(dev),
                            R=torch.from_numpy(nnp.unit_variance_mlpg_matrix(hp.windows, t)).to(dev)))
    frames = sum(sum(lens) for _, _, lens in host)
    adv_w = 1.0 if w["w_d"] > 0 else 0.0
    kw = dict(w_d=w["w_d"], mse_w=w["mse_w"], mge_w=w["mge_w"], optimizer=w["optimizer"], optimizer_params=w["okw"])
    fs_r = fused.FusedGanStep(*tfs.models(w, dev), hp, B, T, seed=1, **kw)
    fs_p = fused.FusedGanStep(*tfs.models(w, dev), hp, B, T, seed=1, **kw)
    tr = gstep.GanTrainer(*tfs.models(w, dev), hp, **kw)
    paths = {
        "fused_ragged": lambda bt: fs_r.step(bt["x"], bt["y"], bt["lengths"], adv_w=adv_w),
        "fused_padded": lambda bt: fs_p.step(bt["xp"], bt["yp"], bt["lengths"], adv_w=adv_w),
        "modular": lambda bt: tr.step(bt["x"], bt["y"], bt["lengths"], bt["R"], adv_w=adv_w),
    }
    for fn in paths.values():
        for bt in batches:
            fn(bt)
    torch.cuda.synchronize()
    ms = {k: [] for k in paths}
    for _ in range(rounds):
        for k, fn in paths.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for bt in batches:
                fn(bt)
            b.record()
            b.synchronize()
            ms[k].append(a.elapsed_time(b))
    out = {"workload": name, "capacity_B": B, "capacity_T": T, "utterances": n_utt, "batches": len(batches),
           "last_batch": len(host[-1][2]), "valid_frames": frames,
           "padded_frames_ragged": sum(x.shape[0] * x.shape[1] for x, _, _ in host),
           "padded_frames_to_T": sum(x.shape[0] for x, _, _ in host) * T, "rounds": rounds}
    for k, v in ms.items():
        med = float(np.median(v))
        out[k] = {"ms_per_epoch_median": round(med, 2), "ms_per_epoch_min": round(min(v), 2),
                  "ms_per_epoch_max": round(max(v), 2), "valid_frames_per_s": round(frames / med * 1e3, 1)}
    for k in ("fused_padded", "modular"):
        out["speedup_ragged_vs_%s" % k] = round(out[k]["ms_per_epoch_median"] / out["fused_ragged"]["ms_per_epoch_median"], 3)
    return out


def time_table_builder(dev, T=2000, reps=10):
    from gantts_b200 import ops
    windows = tfs.WINDOWS
    ops.mlpg_table_device(windows, T, dev)
    torch.cuda.synchronize()
    v = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        ops.mlpg_table_device(windows, T, dev)
        b.record()
        b.synchronize()
        v.append(a.elapsed_time(b))
    return {"mlpg_table_device_T": T, "ms_median": round(float(np.median(v)), 3), "ms_min": round(min(v), 3),
            "ms_max": round(max(v), 3), "reps": reps}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--workload", choices=("vc", "tts_acoustic", "all"), default="all")
    ap.add_argument("--utterances", type=int, default=110, help="utterances per epoch (default 110: 5 batches of 20 and one of 10)")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--json", default=None, help="also write the results to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_ragged_epoch.py: needs a CUDA device (there is no CPU path to time)")
    import __graft_entry__
    __graft_entry__.build()
    dev = torch.device("cuda:0")
    res = {"gpu": tfs.gpu_info(), "results": []}
    for name in (("vc", "tts_acoustic") if args.workload == "all" else (args.workload,)):
        r = run(name, args.utterances, args.rounds, dev)
        print(json.dumps(r), flush=True)
        res["results"].append(r)
    res["table_builder"] = time_table_builder(dev)
    print(json.dumps({"table_builder": res["table_builder"], "gpu": res["gpu"]}))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
