"""Time voice conversion on the GPU: ragged utterances of harmonic waveforms (1-5 s) through
VoiceConverter.convert_utterances with a random In2OutHighwayNet at the vc shape (177 -> 3 x 512 -> 177, order 59),
host to host, with CUDA-event time per stage of the same batches, the MLSA filter's time per sample on single
utterances, and the numpy restatement's filter (a Python loop per sample, not pysptk) on a few short utterances.  Prints
one JSON line with the card's name and power limit read in the same run.

usage: python tools/time_convert.py [--utts 100] [--fs 16000] [--batch-size 20] [--oracle-utts 2] [--repeats 3]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--utts", type=int, default=100)
    ap.add_argument("--fs", type=int, default=16000)
    ap.add_argument("--batch-size", type=int, default=20)
    ap.add_argument("--oracle-utts", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_convert: needs a CUDA device")
    import __graft_entry__
    __graft_entry__.build()
    import train_cli_helpers as H
    from gantts_b200 import analysis, convert, generate, models, ops
    from oracle import mlsa_port, sptk_port
    from test_gpu_world_analysis import wave
    dev = torch.device("cuda")
    rng = np.random.RandomState(0)
    order = 59
    torch.manual_seed(0)
    model = models.In2OutHighwayNet(3 * order, 3 * order, order, num_hidden=3, hidden_dim=512, dropout=0.0)
    hp = H.vc_hp(order=order)
    stats = {"data_mean": rng.randn(3 * order) * 0.1, "data_std": rng.uniform(0.5, 1.5, 3 * order)}
    conv = convert.VoiceConverter(model.to(dev), hp, stats, a.fs)
    waves = [wave(rng, a.fs, rng.uniform(1.0, 5.0))[0].astype(np.int16) for _ in range(a.utts)]
    conv.convert_utterances(waves, a.batch_size)                       # warm-up: modules, operator caches
    torch.cuda.synchronize()
    host = []
    for _ in range(a.repeats):
        t0 = time.perf_counter()
        conv.convert_utterances(waves, a.batch_size)
        host.append(time.perf_counter() - t0)
    # per stage: CUDA events around each step of VoiceConverter.convert, summed over the same batches
    names = ["analysis", "inputs", "generation", "mc2b", "filter"]
    stages = dict.fromkeys(names, 0.0)
    for idx in generate.plan_batches([len(w) for w in waves], a.batch_size):
        x, L = analysis.pad_waves([waves[i].astype(np.float64) for i in idx], dev)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(6)]
        ev[0].record()
        src, _, frames = conv.analyse(x, L)
        ev[1].record()
        xin, static = ops.vc_inputs(src, frames, conv.windows, conv.mean, conv.std)
        ev[2].record()
        pred = conv.gen.generate(xin, frames)["mc"]
        ev[3].record()
        b = ops.mc2b(pred, static, frames, conv.alpha)
        ev[4].record()
        ops.mlsa_filter(x, L, b, frames, conv.alpha, conv.hop)
        ev[5].record()
        torch.cuda.synchronize()
        for i, k in enumerate(names):
            stages[k] += ev[i].elapsed_time(ev[i + 1])
    # the filter alone, one utterance per launch: its loop-carried time per sample
    per_sample = []
    for seconds in (1.0, 5.0):
        w = wave(rng, a.fs, seconds)[0]
        x, L = analysis.pad_waves([w], dev)
        src, _, frames = conv.analyse(x, L)
        xin, static = ops.vc_inputs(src, frames, conv.windows, conv.mean, conv.std)
        b = ops.mc2b(conv.gen.generate(xin, frames)["mc"], static, frames, conv.alpha)
        ops.mlsa_filter(x, L, b, frames, conv.alpha, conv.hop)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(5):
            ops.mlsa_filter(x, L, b, frames, conv.alpha, conv.hop)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 5
        per_sample.append({"samples": len(w), "ms": round(ms, 3), "ns_per_sample": round(ms * 1e6 / len(w), 1)})
    # the numpy restatement of the filter (a Python loop per sample), a few short utterances
    t0 = time.perf_counter()
    n_oracle = 0
    for _ in range(a.oracle_utts):
        w = wave(rng, a.fs, 0.25)[0]
        bs = sptk_port.mc2b(rng.randn(len(w) // conv.hop + 1, order + 1) * 0.01, conv.alpha)
        mlsa_port.mlsa_synthesis([w], [bs], conv.alpha, conv.hop)
        n_oracle += len(w)
    oracle_ns = (time.perf_counter() - t0) * 1e9 / max(n_oracle, 1)
    seconds = sum(len(w) for w in waves) / a.fs
    print(json.dumps({"card": card(), "fs": a.fs, "utterances": a.utts, "batch_size": a.batch_size,
                      "audio_s": round(seconds, 1), "host_to_host_s": [round(h, 4) for h in host],
                      "audio_s_per_s": round(seconds / min(host), 1),
                      "stage_ms": {k: round(v, 3) for k, v in stages.items()},
                      "filter_single_utterance": per_sample,
                      "numpy_restatement_filter_ns_per_sample": round(oracle_ns, 1)}))


if __name__ == "__main__":
    main()
