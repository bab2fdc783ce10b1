"""Time the training command's loop with each of its loaders: the host DataLoader of train.py (per batch: collate_fn in
float32, sort_batch, a copy to the device) against DeviceBatches (the normalised corpus resident on the device, one
gantts_corpus_gather launch per batch).

The corpus is seeded .npy files written to a temporary directory: 129 time-aligned utterances of 200-1000 frames, so
that train.load_data's split gives 110 train utterances (5 batches of 20 and one of 10) and 14 test ones (one batch).
Widths: vc 177 -> 177 (In2OutHighwayNet and MLP D of tools/time_fused_step.py) and tts_acoustic 425 -> 187 (SRURNN and
the conditioned MLP D), both FusedGanStep, Adagrad, w_d = 1, MGE.  The host loader runs with the reference hparams'
num_workers = 1 and pin_memory = True.

What is timed: one epoch of train.run_phase, the train phase then the test phase, each on the host clock from its
start to the end of its EpochLog.read (which synchronises).  Each loader drives its own FusedGanStep built from the same
seed; the warm-up epoch of both starts from the same torch seed, and the tool checks that the two logged exactly the same
values.  Then the loaders alternate for --rounds rounds; the median is reported.  Also: train.load_data's time with
each loader (the device one normalises and uploads the corpus once per command), and the gather kernel alone over the
train epoch's batches with CUDA events (microseconds per batch, GB/s written), and each loader alone, without the step,
in ms per train batch (the host DataLoader with num_workers 0 and 1, and the device corpus).  The GPU's name and power limit are
queried in the same run (nvidia-smi, read-only).  Needs a CUDA device.

    python tools/time_train_loader.py [--workload vc|tts_acoustic|all] [--rounds R] [--json OUT]
"""
import argparse
import copy
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

import time_fused_step as tfs  # noqa: E402

N_FILES = 129       # 124 after the five held-out files: 110 train, 14 test


def hparams(name):
    from compat.tensorflow.contrib.training import HParams
    w = tfs.WORKLOADS[name]
    kw = dict(windows=tfs.WINDOWS, generator_add_noise=False, generator_noise_dim=200, optimizer_g="Adagrad",
              optimizer_g_params=dict(w["okw"]), optimizer_d="Adagrad", optimizer_d_params=dict(w["okw"]),
              discriminator="MLP", nepoch=1, lr_decay_schedule=False, lr_decay_epoch=10, batch_size=w["B"],
              num_workers=1, pin_memory=True, cache_size=1200)
    if name == "vc":
        kw.update(name="vc", order=59, stream_sizes=[177], has_dynamic_features=[True], adversarial_streams=[True],
                  mask_nth_mgc_for_adv_loss=0, discriminator_linguistic_condition=False, generator="In2OutHighwayNet",
                  generator_params=dict(in_dim=177, out_dim=177, static_dim=59, num_hidden=3, hidden_dim=512,
                                        dropout=0.5),
                  discriminator_params=dict(in_dim=59, out_dim=1, num_hidden=2, hidden_dim=256, dropout=0.5,
                                            last_sigmoid=True))
    else:
        kw.update(name="acoustic", order=59, recompute_delta_features=False, stream_sizes=[180, 3, 1, 3],
                  has_dynamic_features=[True, True, False, True], adversarial_streams=[True, False, False, False],
                  mask_nth_mgc_for_adv_loss=2, discriminator_linguistic_condition=True, generator="SRURNN",
                  generator_params=dict(in_dim=425, out_dim=187, num_hidden=6, hidden_dim=512, bidirectional=True,
                                        dropout=0.2, use_relu=1, rnn_dropout=0.2),
                  discriminator_params=dict(in_dim=483, out_dim=1, num_hidden=3, hidden_dim=256, dropout=0.5,
                                            last_sigmoid=True))
    return HParams(**copy.deepcopy(kw))


def write_corpus(root, dx, dy, seed=0):
    rng = np.random.RandomState(seed)
    xd, yd = os.path.join(root, "X"), os.path.join(root, "Y")
    os.makedirs(xd), os.makedirs(yd)
    for i in range(N_FILES):
        n = int(rng.randint(200, 1001))
        x = rng.rand(n, dx).astype(np.float32)
        y = (0.5 * rng.randn(n, dy)).astype(np.float32)
        if dy == 187:
            y[:, 183] = rng.rand(n) > 0.4
        np.save(os.path.join(xd, "utt%03d.npy" % i), x)
        np.save(os.path.join(yd, "utt%03d.npy" % i), y)
    return xd, yd


def load(name, xd, yd, on_device, num_workers=1):
    """train.load_data with the device corpus or, its budget patched to 0, the host DataLoader; seconds included."""
    from gantts_b200 import train
    budget = train.device_corpus_budget
    if not on_device:
        train.device_corpus_budget = lambda: 0
    try:
        hp = hparams(name)
        hp.num_workers = num_workers
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        loaders, Ym, Ys, longest = train.load_data(hp, xd, yd, -1)
        torch.cuda.synchronize()
        seconds = time.perf_counter() - t0
    finally:
        train.device_corpus_budget = budget
    assert isinstance(loaders["train"], train.DeviceBatches) == on_device
    return hp, loaders, Ym, Ys, longest, seconds


def time_kernel(batches, dev, loops=50):
    """gantts_corpus_gather alone over the train epoch's batches: (us per batch, GB/s written, GB/s read + written)."""
    from gantts_b200 import ops
    plan, bounds = batches.plan.epoch()
    pd = torch.from_numpy(plan).to(dev)
    args, written, read = [], 0, 0
    D = batches.X.shape[1] + batches.Y.shape[1]
    for j in range(len(bounds) - 1):
        s, e = bounds[j], bounds[j + 1]
        t = int(plan[1, s])
        outs = (torch.empty(e - s, t, batches.X.shape[1], device=dev), torch.empty(e - s, t, batches.Y.shape[1], device=dev))
        args.append((pd[0, s:e], pd[1, s:e], t, outs))
        written += (e - s) * t * D * 4
        read += int(plan[1, s:e].sum()) * D * 4
    run = lambda: [ops.corpus_gather(batches.X, batches.Y, o, n, t, x_out=a, y_out=b) for o, n, t, (a, b) in args]
    run()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(loops):
        run()
    b.record()
    torch.cuda.synchronize()
    sec = a.elapsed_time(b) / 1e3 / loops
    return {"us_per_batch": round(sec / len(args) * 1e6, 2), "batches": len(args),
            "GB_per_s_written": round(written / sec / 1e9, 1), "GB_per_s_read_and_written": round((written + read) / sec / 1e9, 1),
            "MB_written_per_epoch": round(written / 1e6, 1)}


def time_loaders_alone(name, xd, yd, rounds, dev):
    """The train split's batches alone, no step: ms per batch from the start of the epoch until its last batch is on the
    device (a synchronise), for the host DataLoader with num_workers 0 and 1 and for the device corpus; median of
    `rounds` alternated epochs after a warm-up one."""
    from gantts_b200 import train
    legs = {"host_workers0": load(name, xd, yd, False, 0)[1]["train"],
            "host_workers1": load(name, xd, yd, False, 1)[1]["train"],
            "device": load(name, xd, yd, True)[1]["train"]}

    def epoch(loader):
        batches = loader if isinstance(loader, train.DeviceBatches) else train.host_batches(loader, dev)
        n = 0
        t0 = time.perf_counter()
        for _ in batches:
            n += 1
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3 / n

    ms = {k: [] for k in legs}
    for r in range(rounds + 1):
        for k, loader in legs.items():
            v = epoch(loader)
            if r:
                ms[k].append(v)
    return {k: round(float(np.median(v)), 3) for k, v in ms.items()}


def run(name, rounds, dev, tmp):
    from gantts_b200 import fused, train
    from gantts_b200.epochlog import EpochLog
    w = tfs.WORKLOADS[name]
    xd, yd = write_corpus(os.path.join(tmp, name), w.get("in_dim", 177), w.get("out_dim", 177))
    legs = {}
    for kind, on_device in (("host", False), ("device", True)):
        hp, loaders, Ym, Ys, longest, seconds = load(name, xd, yd, on_device)
        mg, md = tfs.models(w, dev)
        # the same dropout seed stream for both legs (make_path would draw a new one for each)
        path = train.FusedPath(fused.FusedGanStep(mg, md, hp, hp.batch_size, longest, w_d=w["w_d"], mse_w=w["mse_w"],
                                                  mge_w=w["mge_w"], optimizer="Adagrad", optimizer_params=w["okw"],
                                                  optimizer_d="Adagrad", optimizer_d_params=w["okw"], seed=1))
        logs = {p: EpochLog(hp, Ym, Ys, dev) for p in ("train", "test")}
        legs[kind] = dict(loaders=loaders, models=(mg, md), path=path, logs=logs, load_s=seconds)

    def epoch(leg):
        ms, values = {}, {}
        for phase in ("train", "test"):
            for m in leg["models"]:
                m.train() if phase == "train" else m.eval()
            t0 = time.perf_counter()
            train.run_phase(leg["path"], leg["loaders"][phase], leg["logs"][phase], phase, 1.0, True, True, dev)
            values.update(leg["logs"][phase].read(phase))
            ms[phase] = (time.perf_counter() - t0) * 1e3
        return ms, values

    warm = {}
    for kind, leg in legs.items():
        torch.manual_seed(7)
        warm[kind] = epoch(leg)[1]
    same = lambda a, b: a == b or (a != a and b != b)         # a NaN metric (no frame voiced in both) is logged as NaN
    identical = (warm["host"].keys() == warm["device"].keys()
                 and all(same(v, warm["device"][k]) for k, v in warm["host"].items()))
    times = {k: {"train": [], "test": [], "epoch": []} for k in legs}
    for _ in range(rounds):
        for kind, leg in legs.items():
            ms, _ = epoch(leg)
            for phase in ("train", "test"):
                times[kind][phase].append(ms[phase])
            times[kind]["epoch"].append(ms["train"] + ms["test"])
    out = {"workload": name, "utterances": {p: len(legs["device"]["loaders"][p].plan.lengths) for p in ("train", "test")},
           "batches": {p: len(legs["device"]["loaders"][p]) for p in ("train", "test")}, "rounds": rounds,
           "identical_logged_values": identical}
    for kind in legs:
        r = {k: round(float(np.median(v)), 2) for k, v in times[kind].items()}
        r["epoch_min"], r["epoch_max"] = round(min(times[kind]["epoch"]), 2), round(max(times[kind]["epoch"]), 2)
        r["load_data_s"] = round(legs[kind]["load_s"], 3)
        out[kind + "_ms"] = r
    out["speedup_epoch"] = round(out["host_ms"]["epoch"] / out["device_ms"]["epoch"], 2)
    dev_batches = legs["device"]["loaders"]["train"]
    out["corpus_MB_on_device"] = round(sum((v.X.numel() + v.Y.numel()) * 4 for v in legs["device"]["loaders"].values())
                                       / 2**20, 1)
    out["gather_kernel"] = time_kernel(dev_batches, dev)
    out["loader_alone_ms_per_batch"] = time_loaders_alone(name, xd, yd, rounds, dev)
    if not identical:
        out["differing_values"] = {k: (warm["host"].get(k), warm["device"].get(k)) for k in
                                   set(warm["host"]) | set(warm["device"])
                                   if not same(warm["host"].get(k), warm["device"].get(k))}
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--workload", choices=("vc", "tts_acoustic", "all"), default="all")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--json", default=None, help="also write the results to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_train_loader.py: needs a CUDA device (there is no CPU path to time)")
    import __graft_entry__
    __graft_entry__.build()
    dev = torch.device("cuda:0")
    res = {"gpu": tfs.gpu_info(), "results": []}
    with tempfile.TemporaryDirectory() as tmp:
        for name in (("vc", "tts_acoustic") if args.workload == "all" else (args.workload,)):
            r = run(name, args.rounds, dev, tmp)
            print(json.dumps(r), flush=True)
            res["results"].append(r)
    print(json.dumps({"gpu": res["gpu"]}))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)
    if not all(r["identical_logged_values"] for r in res["results"]):
        sys.exit("time_train_loader.py: the two loaders logged different values")


if __name__ == "__main__":
    main()
