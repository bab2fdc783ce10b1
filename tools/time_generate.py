"""Batched generation (ParameterGenerator.generate_utterances) against the per-utterance loop a user would otherwise write
(forward at B = 1, then the compat nnmnkwii.paramgen.mlpg, numpy in and out, one call per stream), on 100 ragged
utterances (200..1000 frames) at the vc shape (In2OutHighwayNet 177 -> 3 x 512 -> 177) and the tts_acoustic shape
(SRURNN 425 -> 6 x 512 bidirectional -> 187).  Both end with every feature on the host; the four runs alternate within
each round, timed with CUDA events around a device synchronise.

    python tools/time_generate.py [--json OUT]
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
sys.path.insert(1, os.path.join(ROOT, "compat"))
sys.path.insert(2, os.path.join(ROOT, "tests"))
import __graft_entry__  # noqa: E402

__graft_entry__.build()
from gantts_b200 import generate, models  # noqa: E402
import evaltts_mirror  # noqa: E402
import train_cli_helpers as H  # noqa: E402
from nnmnkwii import paramgen, preprocessing  # noqa: E402

dev = torch.device("cuda:0")
N, ROUNDS, BATCH = 100, 3, 20


def setup(kind):
    rng = np.random.RandomState(0)
    lens = rng.randint(200, 1001, N)
    if kind == "vc":
        hp = H.vc_hp(order=59, generator_params={"in_dim": 177, "out_dim": 177, "num_hidden": 3, "hidden_dim": 512,
                                                 "static_dim": 59, "dropout": 0.5})
        model = models.In2OutHighwayNet(**hp.generator_params)
        stats = {"data_mean": rng.randn(177), "data_std": 0.5 + rng.rand(177)}
        arrays = [rng.randn(n, 177).astype(np.float32) for n in lens]
    else:
        hp = H.tts_acoustic_hp(generator="SRURNN", generator_params={
            "in_dim": 425, "out_dim": 187, "num_hidden": 6, "hidden_dim": 512, "bidirectional": True, "dropout": 0.2,
            "use_relu": 1, "rnn_dropout": 0.2, "last_sigmoid": False})
        model = models.SRURNN(**hp.generator_params)
        stats = {"X_min": np.zeros(425), "X_max": np.ones(425), "Y_mean": rng.randn(187), "Y_std": 0.5 + rng.rand(187)}
        arrays = [rng.rand(n, 425).astype(np.float32) for n in lens]
    model = model.to(dev).eval()
    return hp, model, stats, arrays, generate.ParameterGenerator(model, hp, stats)


def per_utterance(kind, hp, model, stats, arrays):
    out = []
    with torch.no_grad():
        for a in arrays:
            x = torch.from_numpy(generate.normalize_input(a, hp, stats)).to(dev)[None]
            T = x.shape[1]
            if kind == "vc":
                R = torch.from_numpy(paramgen.unit_variance_mlpg_matrix(hp.windows, T)).to(dev)
                _, y = model(x, R, lengths=[T])
                y = y[0].cpu().numpy()
                out.append(preprocessing.inv_scale(y, stats["data_mean"][:59], stats["data_std"][:59]))
            else:
                y = model(x, [T])[0].cpu().numpy()
                out.append(evaltts_mirror.gen_parameters(y, stats["Y_mean"], stats["Y_std"], True, hp.stream_sizes,
                                                         hp.windows, paramgen, preprocessing))
    return out


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    res = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), res


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--json", default=None, help="also write the results to this file")
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    setups = {k: setup(k) for k in ("vc", "tts_acoustic")}
    frames = {k: int(sum(len(a) for a in s[3])) for k, s in setups.items()}
    runs = []
    for k, (hp, model, stats, arrays, pg) in setups.items():        # warm every shape once
        runs += [(k, "batched", lambda pg=pg, arrays=arrays: pg.generate_utterances(arrays, BATCH)),
                 (k, "per_utterance", lambda k=k, hp=hp, model=model, stats=stats, arrays=arrays:
                  per_utterance(k, hp, model, stats, arrays))]
    for _, _, fn in runs:
        fn()
    ms = {(k, how): [] for k, how, _ in runs}
    agree = {}
    for _ in range(ROUNDS):
        results = {}
        for k, how, fn in runs:
            t, results[(k, how)] = timed(fn)
            ms[(k, how)].append(t)
        for k in setups:
            b, p = results[(k, "batched")], results[(k, "per_utterance")]
            if k == "vc":
                err = max(float(np.abs(r["mc"] - q).max() / np.abs(q).max()) for r, q in zip(b, p))
            else:
                err = max(float(np.abs(r[n] - np.asarray(q[i]).reshape(r[n].shape)).max() / np.abs(q[i]).max())
                          for r, q in zip(b, p) for i, n in enumerate(("mgc", "lf0", "vuv", "bap")))
            agree[k] = max(agree.get(k, 0.0), err)
    report = {"gpu": gpu, "utterances": N, "batch_size": BATCH, "rounds": ROUNDS, "frames": frames,
              "max_rel_diff_batched_vs_loop": agree}
    for (k, how), v in ms.items():
        report["%s_%s_ms" % (k, how)] = {"median": float(np.median(v)), "min": float(min(v)), "max": float(max(v))}
    for k in setups:
        report["%s_speedup" % k] = report["%s_per_utterance_ms" % k]["median"] / report["%s_batched_ms" % k]["median"]
    print(json.dumps(report, indent=1))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
