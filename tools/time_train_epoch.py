"""Time one epoch of the training command's loop with its device-side epoch log against the same loop with train.py's
per-batch reads.

The epochs are the seeded ragged epochs of tools/time_ragged_epoch.py (vc and tts_acoustic widths, capacity B x T =
20 x 1000, FusedGanStep with the models and optimisers of tools/time_fused_step.py).  Per epoch, one train phase:
  device_log   gantts_b200.train.run_phase's batch body: FusedGanStep.step, then EpochLog.add; one EpochLog.read at the end
  per_batch    FusedGanStep.step, then loss_dict() and metrics.compute_distortions(get_static_features(y), ...) per
               batch, as a loop over the fused step written after train.py:562-595 does
Batches are on the device before timing (the loader is not timed).  One warm-up epoch per path, then rounds of one
epoch per path, alternating, each timed with CUDA events and ended by a synchronise.  The GPU's name and power limit
are queried in the same run (nvidia-smi, read-only).  Needs a CUDA device.

    python tools/time_train_epoch.py [--workload vc|tts_acoustic|all] [--utterances N] [--rounds R] [--json OUT]
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
import time_ragged_epoch as tre  # noqa: E402


def run(name, n_utt, rounds, dev):
    from gantts_b200 import fused, metrics, multistream
    from gantts_b200.epochlog import EpochLog
    w = tfs.WORKLOADS[name]
    B, T = w["B"], w["T"]
    hp = tfs.hparams(name)
    hp.update(name="vc", order=59) if name == "vc" else hp.update(name="acoustic")
    d_in, d_out = w.get("in_dim", 177), w.get("out_dim", 177)
    batches = [(x.to(dev), y.to(dev), torch.LongTensor(lens).to(dev)) for x, y, lens in tre.epoch(n_utt, B, T, d_in,
                                                                                                     d_out, 11)]
    rng = np.random.RandomState(0)
    Ym, Ys = rng.randn(d_out) * 0.1, rng.rand(d_out) + 0.5
    kw = dict(w_d=w["w_d"], mse_w=w["mse_w"], mge_w=w["mge_w"], optimizer=w["optimizer"], optimizer_params=w["okw"])
    fs = fused.FusedGanStep(*tfs.models(w, dev), hp, B, T, seed=1, **kw)
    log = EpochLog(hp, Ym, Ys, dev)
    nw = len(hp.windows)

    def device_log():
        log.reset()
        for x, y, lens in batches:
            fs.step(x, y, lens, adv_w=1.0)
            log.add(fs.losses, y, fs.y_hat_static, lens, True, True)
        return log.read("train")

    def per_batch():
        out = []
        for x, y, lens in batches:
            fs.step(x, y, lens, adv_w=1.0)
            v = fs.loss_dict()
            ys = multistream.get_static_features(y, nw, hp.stream_sizes, hp.has_dynamic_features)
            v.update(metrics.compute_distortions(ys, fs.y_hat_static, Ym, Ys, lens, hp=hp))
            out.append(v)
        return out

    paths = {"device_log": device_log, "per_batch": per_batch}
    for fn in paths.values():
        fn()
    torch.cuda.synchronize()
    ms = {k: [] for k in paths}
    for _ in range(rounds):
        for k, fn in paths.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            torch.cuda.synchronize()
            ms[k].append(a.elapsed_time(b))
    out = {"workload": name, "capacity_B": B, "capacity_T": T, "utterances": n_utt, "batches": len(batches),
           "rounds": rounds}
    for k, v in ms.items():
        out[k] = {"ms_per_epoch_median": round(float(np.median(v)), 2), "ms_per_epoch_min": round(min(v), 2),
                  "ms_per_epoch_max": round(max(v), 2)}
    out["speedup_device_log_vs_per_batch"] = round(out["per_batch"]["ms_per_epoch_median"] /
                                                   out["device_log"]["ms_per_epoch_median"], 3)
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--workload", choices=("vc", "tts_acoustic", "all"), default="all")
    ap.add_argument("--utterances", type=int, default=110, help="utterances per epoch (default 110: 5 batches of 20 and one of 10)")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--json", default=None, help="also write the results to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_train_epoch.py: needs a CUDA device (there is no CPU path to time)")
    import __graft_entry__
    __graft_entry__.build()
    dev = torch.device("cuda:0")
    res = {"gpu": tfs.gpu_info(), "results": []}
    for name in (("vc", "tts_acoustic") if args.workload == "all" else (args.workload,)):
        r = run(name, args.utterances, args.rounds, dev)
        print(json.dumps(r), flush=True)
        res["results"].append(r)
    print(json.dumps({"gpu": res["gpu"]}))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
