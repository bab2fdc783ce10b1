"""Time the WORLD analysis chain on the GPU against the numpy restatement: ragged utterances of harmonic waveforms (1-5 s),
the device path host to host (analysis.analyse, one batch) with CUDA-event time per stage, and the restatement per
utterance on a sample of them.  Prints one JSON line with the card's name and power limit read in the same run.

usage: python tools/time_analysis.py [--utts 100] [--fs 16000] [--kind vc] [--oracle-utts 5] [--repeats 3]"""
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
    ap.add_argument("--kind", default="vc")
    ap.add_argument("--oracle-utts", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_analysis: needs a CUDA device")
    import __graft_entry__
    __graft_entry__.build()
    from gantts_b200 import analysis, generate, ops
    from oracle import sptk_port
    from oracle import world_analysis_port as A
    from test_gpu_world_analysis import wave
    dev = torch.device("cuda")
    rng = np.random.RandomState(0)
    waves = [wave(rng, a.fs, rng.uniform(1.0, 5.0))[0] for _ in range(a.utts)]
    fp, order = 5.0, 59
    analysis.analyse(waves[:4], a.fs, fp, order, a.kind, dev)                 # warm-up: modules, operator cache
    analysis.analyse(waves, a.fs, fp, order, a.kind, dev)
    torch.cuda.synchronize()
    host = []
    for _ in range(a.repeats):
        t0 = time.perf_counter()
        analysis.analyse(waves, a.fs, fp, order, a.kind, dev)
        host.append(time.perf_counter() - t0)
    # per stage, CUDA events around each op of the same chain
    x, L = analysis.pad_waves(waves, dev)
    n = generate.cheaptrick_fft_size(a.fs)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(6)]
    ev[0].record()
    f0, info = ops.world_dio(x, L, a.fs, fp)
    ev[1].record()
    f0 = ops.world_stonemask(x, L, f0, info, a.fs, fp)
    ev[2].record()
    sp = ops.world_cheaptrick(x, L, f0, info, a.fs, fp, n)
    ev[3].record()
    mc = ops.sp2mc(sp, info[:-1], order, generate.mcep_alpha(a.fs))
    ev[4].record()
    ops.modspec_smoothing(mc, info[:-1], analysis.modulation_rate(a.fs, fp))
    ev[5].record()
    torch.cuda.synchronize()
    names = ["dio", "stonemask", "cheaptrick", "sp2mc", "modspec_smoothing"]
    stages = {k: ev[i].elapsed_time(ev[i + 1]) for i, k in enumerate(names)}
    t0 = time.perf_counter()
    alpha = sptk_port.mcepalpha(a.fs)
    for x1 in waves[:a.oracle_utts]:
        g, t = A.dio(x1, a.fs, fp)
        s = A.cheaptrick(x1, A.stonemask(x1, g, t, a.fs), t, a.fs, n)
        A.sp2mc(s, order, alpha)
    oracle = (time.perf_counter() - t0) / max(a.oracle_utts, 1)
    seconds = sum(len(w) for w in waves) / a.fs
    print(json.dumps({"card": card(), "fs": a.fs, "kind": a.kind, "utterances": a.utts, "audio_s": round(seconds, 1),
                      "device_host_to_host_s": [round(h, 4) for h in host],
                      "stage_ms": {k: round(v, 3) for k, v in stages.items()},
                      "numpy_per_utterance_s": round(oracle, 3)}))


if __name__ == "__main__":
    main()
