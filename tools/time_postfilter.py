"""Merlin's post filter and mc2sp on the device (ops.mcep_postfilter, ops.mc2sp: padded batches of 20) against the same
operator form in numpy fp64 run per utterance on the host (w*mc with c0 shifted by the two r0 sums of exp(op_r . mc), then
exp(op_s . mc)), on 100 ragged tts_acoustic mgc utterances (200..1000 frames, order 59).  Both legs start and end with
every utterance on the host.  pysptk / nnmnkwii cannot be installed offline, so their per-frame C loop is not timed.
Also reports what post_filter=True, spectrogram=True add to ParameterGenerator.generate_utterances at the tts_acoustic
shape of tools/time_generate.py (SRURNN 425 -> 6 x 512 bidirectional -> 187).  The legs alternate within each round,
timed with CUDA events around a device synchronise.

    python tools/time_postfilter.py [--fs 16000,48000] [--json OUT]
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
from gantts_b200 import _lib, generate, models, ops  # noqa: E402
import train_cli_helpers as H  # noqa: E402

dev = torch.device("cuda:0")
N, ROUNDS, BATCH, M1 = 100, 3, 20, 60


def device_leg(mgcs, alpha, fftlen):
    out = []
    for i in range(0, len(mgcs), BATCH):
        chunk = mgcs[i:i + BATCH]
        lens = [len(m) for m in chunk]
        x = np.zeros((len(chunk), max(lens), M1), np.float32)
        for j, m in enumerate(chunk):
            x[j, :len(m)] = m
        lengths = torch.tensor(lens, dtype=torch.int64).to(dev)
        mgc = ops.mcep_postfilter(torch.from_numpy(x).to(dev), lengths, alpha)
        sp = ops.mc2sp(mgc, lengths, alpha, fftlen)
        mgc, sp = mgc.cpu().numpy(), sp.cpu().numpy()
        out += [(mgc[j, :L], sp[j, :L]) for j, L in enumerate(lens)]
    return out


def host_leg(mgcs, op_r, op_s):
    bins = np.full(op_r.shape[0], 2.0)
    bins[[0, -1]] = 1.0
    w = np.full(M1, generate.POSTFILTER_COEF)
    w[:2] = 1.0
    out = []
    for m in mgcs:
        m = m.astype(np.float64)
        f = w * m
        f[:, 0] += 0.5 * np.log((np.exp(m @ op_r.T) @ bins) / (np.exp(f @ op_r.T) @ bins))
        out.append((f, np.exp(f @ op_s.T)))
    return out


def kernels_only(xs, alpha, fftlen):
    """The two kernels over the same batches, inputs already on the device."""
    for x, lengths in xs:
        ops.mc2sp(ops.mcep_postfilter(x, lengths, alpha), lengths, alpha, fftlen)


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    res = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), res


def stats_ms(v):
    return {"median": float(np.median(v)), "min": float(min(v)), "max": float(max(v))}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--fs", default="16000,48000", help="comma-separated sampling frequencies")
    ap.add_argument("--json", default=None, help="also write the results to this file")
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    rng = np.random.RandomState(0)
    lens = rng.randint(200, 1001, N)
    mgcs = []
    for n in lens:
        m = rng.randn(n, M1) * np.exp(-0.1 * np.arange(M1))
        m[:, 0] = rng.uniform(-2.0, 2.0, n)
        mgcs.append(m.astype(np.float32))
    report = {"gpu": gpu, "utterances": N, "frames": int(lens.sum()), "batch_size": BATCH, "rounds": ROUNDS}

    for fs in (int(f) for f in args.fs.split(",")):
        alpha, fftlen = generate.mcep_alpha(fs), generate.cheaptrick_fft_size(fs)
        op_r = ops.mcep_operator_host(alpha, M1 - 1, ops.POSTFILTER_FFTLEN, _lib.MCEP_R0)
        op_s = ops.mcep_operator_host(alpha, M1 - 1, fftlen, _lib.MCEP_SP)
        resident = []
        for i in range(0, N, BATCH):
            chunk = mgcs[i:i + BATCH]
            x = np.zeros((len(chunk), max(len(m) for m in chunk), M1), np.float32)
            for j, m in enumerate(chunk):
                x[j, :len(m)] = m
            resident.append((torch.from_numpy(x).to(dev), torch.tensor([len(m) for m in chunk], device=dev)))
        legs = [("device", lambda: device_leg(mgcs, alpha, fftlen)), ("host_numpy", lambda: host_leg(mgcs, op_r, op_s)),
                ("kernels_only", lambda: kernels_only(resident, alpha, fftlen))]
        for _, fn in legs:                                       # warm every shape once
            fn()
        ms = {name: [] for name, _ in legs}
        err = {"mgc": 0.0, "sp": 0.0}
        for _ in range(ROUNDS):
            res = {}
            for name, fn in legs:
                t, res[name] = timed(fn)
                ms[name].append(t)
            for (dm, ds), (hm, hs) in zip(res["device"], res["host_numpy"]):
                err["mgc"] = max(err["mgc"], float(np.abs(dm - hm).max() / np.abs(hm).max()))
                err["sp"] = max(err["sp"], float(np.abs(ds / hs - 1).max()))
        r = {"alpha": alpha, "fftlen": fftlen, "max_rel_diff_device_vs_host": err}
        for name, v in ms.items():
            r[name + "_ms"] = stats_ms(v)
        r["speedup_device_vs_host"] = r["host_numpy_ms"]["median"] / r["device_ms"]["median"]
        report["fs%d" % fs] = r

    # what the two flags add to batched generation at the tts_acoustic shape
    hp = H.tts_acoustic_hp(generator="SRURNN", generator_params={
        "in_dim": 425, "out_dim": 187, "num_hidden": 6, "hidden_dim": 512, "bidirectional": True, "dropout": 0.2,
        "use_relu": 1, "rnn_dropout": 0.2, "last_sigmoid": False})
    model = models.SRURNN(**hp.generator_params).to(dev).eval()
    st = {"X_min": np.zeros(425), "X_max": np.ones(425), "Y_mean": rng.randn(187), "Y_std": 0.5 + rng.rand(187)}
    arrays = [rng.rand(n, 425).astype(np.float32) for n in lens]
    fs0 = int(args.fs.split(",")[0])
    gens = [("plain", generate.ParameterGenerator(model, hp, st)),
            ("post_filter_spectrogram", generate.ParameterGenerator(model, hp, st, post_filter=True, spectrogram=True,
                                                                    fs=fs0))]
    for _, pg in gens:
        pg.generate_utterances(arrays, BATCH)
    ms = {name: [] for name, _ in gens}
    for _ in range(ROUNDS):
        for name, pg in gens:
            ms[name].append(timed(lambda: pg.generate_utterances(arrays, BATCH))[0])
    g = {"fs": fs0}
    for name, v in ms.items():
        g["generate_utterances_%s_ms" % name] = stats_ms(v)
    g["added_ms"] = g["generate_utterances_post_filter_spectrogram_ms"]["median"] - \
        g["generate_utterances_plain_ms"]["median"]
    report["generate_utterances"] = g
    print(json.dumps(report, indent=1))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
