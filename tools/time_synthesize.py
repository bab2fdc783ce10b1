"""Synthesis with predicted durations (Synthesizer.synthesize_utterances, batch size 20) against the per-utterance chain a
user would otherwise write (duration generate at B = 1, durations to the host, the frame expansion and
generate.normalize_input in numpy, acoustic generate at B = 1), on 100 ragged synthetic utterances of 20..120 phones
at the shipped shapes (duration SRURNN 416 -> 6 x 512 bidirectional -> 5, acoustic SRURNN 425 -> 6 x 512
bidirectional -> 187), state durations near 2 frames so that utterances have about 200..1000 frames.  Both legs end with
every feature on the host; they alternate within each round, timed with CUDA events around a device synchronise.  Also
times gantts_state_frame_offsets and gantts_expand_state_frames alone on the first batch of 20.

    python tools/time_synthesize.py [--json OUT]
"""
import argparse
import ctypes
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
from gantts_b200 import _lib, generate, models, ops, synthesize  # noqa: E402
from oracle import merlin_port  # noqa: E402
import tts_data_helpers as TH  # noqa: E402

dev = torch.device("cuda:0")
N, ROUNDS, BATCH, L, S = 100, 5, 20, 416, 5
KERNEL_REPS = 200


def setup():
    rng = np.random.RandomState(0)
    gp = lambda: {"in_dim": None, "out_dim": None, "num_hidden": 6, "hidden_dim": 512, "bidirectional": True,
                  "dropout": 0.0, "use_relu": 1, "rnn_dropout": 0.2, "last_sigmoid": False}
    hp_a = TH.acoustic_hp(generator="SRURNN", generator_params=gp())
    hp_d = TH.duration_hp(generator="SRURNN", generator_params=gp())
    sd = {"X_min": np.zeros(L, np.float32), "X_max": np.full(L, 10.0, np.float32),
          "Y_mean": np.full(S, 2.0), "Y_std": np.full(S, 0.5)}
    sa = {"X_min": np.zeros(L + 9, np.float32), "X_max": np.full(L + 9, 100.0, np.float32),
          "Y_mean": rng.randn(187), "Y_std": 0.5 + rng.rand(187)}
    generate.derive_dims(hp_a, sa), generate.derive_dims(hp_d, sd)
    torch.manual_seed(0)
    md = models.SRURNN(**hp_d.generator_params).to(dev).eval()
    ma = models.SRURNN(**hp_a.generator_params).to(dev).eval()
    syn = synthesize.Synthesizer(md, ma, hp_d, hp_a, sd, sa)
    phones = []
    for n in rng.randint(20, 121, N):
        x = (rng.rand(n, L) < 0.1).astype(np.float32)
        x[:, -8:] = rng.randint(0, 10, size=(n, 8))
        phones.append(x)
    return syn, phones


def per_utterance(syn, phones):
    out = []
    for x in phones:
        d = syn.gen_duration.generate_utterances([x], 1)[0]["duration"]
        r = {"duration": d}
        r.update(syn.gen_acoustic.generate_utterances([merlin_port.expand(x, d)], 1)[0])
        out.append(r)
    return out


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    res = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), res


def kernels_alone(syn, phones):
    """Per-call device time of the two kernels on the first batch of plan_batches, launched through the C ABI."""
    idx = generate.plan_batches([len(p) for p in phones], BATCH)[0]
    lens = [len(phones[i]) for i in idx]
    B, P = len(idx), max(lens)
    xb = np.zeros((B, P, L), np.float32)
    for j, i in enumerate(idx):
        xb[j, :lens[j]] = phones[i]
    x = torch.from_numpy(xb).to(dev)
    pl = torch.tensor(lens, dtype=torch.int64, device=dev)
    with torch.no_grad():
        d = syn.gen_duration.generate(syn.duration_inputs(x, pl), pl)["duration"]
    offsets, fl, host = ops.state_frame_offsets(d, pl)
    T = int(host.max())
    out = ops.expand_state_frames(x, d, offsets, fl, syn.scale_a, syn.min_a, T)
    lib, st = _lib.load(), ops._stream()
    status = torch.empty(1, dtype=torch.int64, device=dev)
    calls = {
        "state_frame_offsets": lambda: lib.gantts_state_frame_offsets(
            d.data_ptr(), d.stride(0), d.stride(1), pl.data_ptr(), B, P, S, offsets.data_ptr(), fl.data_ptr(),
            status.data_ptr(), st),
        "expand_state_frames": lambda: lib.gantts_expand_state_frames(
            x.data_ptr(), x.stride(0), x.stride(1), d.data_ptr(), d.stride(0), d.stride(1), offsets.data_ptr(),
            fl.data_ptr(), syn.scale_a.data_ptr(), syn.min_a.data_ptr(), B, P, L, S, T, out.data_ptr(), st),
    }
    res = {"batch": B, "phones_max": P, "frames_max": T, "frames": int(host.sum())}
    for name, call in calls.items():
        for _ in range(10):
            _lib.check(call())
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(KERNEL_REPS):
            call()
        e1.record()
        torch.cuda.synchronize()
        res[name + "_us"] = 1000.0 * e0.elapsed_time(e1) / KERNEL_REPS
    stored = B * T * (L + 9) * 4
    res["expand_bytes_stored"] = stored
    res["expand_store_GBps"] = stored / (res["expand_state_frames_us"] * 1e-6) / 1e9
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--json", default=None, help="also write the results to this file")
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    syn, phones = setup()
    runs = [("batched", lambda: syn.synthesize_utterances(phones, BATCH)),
            ("per_utterance", lambda: per_utterance(syn, phones))]
    for _, fn in runs:                                               # warm every shape once
        fn()
    ms = {how: [] for how, _ in runs}
    dur_equal, max_rel, frames = 1.0, 0.0, 0
    for _ in range(ROUNDS):
        results = {}
        for how, fn in runs:
            t, results[how] = timed(fn)
            ms[how].append(t)
        b, p = results["batched"], results["per_utterance"]
        same = [np.array_equal(r["duration"], q["duration"]) for r, q in zip(b, p)]
        dur_equal = min(dur_equal, float(np.mean(same)))
        frames = int(sum(len(r["mgc"]) for r in b))
        for r, q, s in zip(b, p, same):
            if s:
                for k in ("mgc", "lf0", "vuv", "bap"):
                    max_rel = max(max_rel, float(np.abs(r[k] - q[k]).max() / max(np.abs(q[k]).max(), 1e-30)))
    report = {"gpu": gpu, "utterances": N, "batch_size": BATCH, "rounds": ROUNDS, "frames": frames,
              "phones": int(sum(len(x) for x in phones)), "utterances_with_equal_durations": dur_equal,
              "max_rel_diff_batched_vs_loop": max_rel}
    for how, v in ms.items():
        report["%s_ms" % how] = {"median": float(np.median(v)), "min": float(min(v)), "max": float(max(v))}
    report["speedup"] = report["per_utterance_ms"]["median"] / report["batched_ms"]["median"]
    report["kernels"] = kernels_alone(syn, phones)
    print(json.dumps(report, indent=1))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
