"""Time WORLD waveform synthesis on the device (ops.world_*): 100 ragged utterances of 200-1000 frames, in batches of 20,
at 16 and 48 kHz.  f0 tracks have voiced runs of 100-250 Hz and unvoiced gaps; sp is ops.mc2sp of smooth random
order-59 mgc.  Reports the median of 5 rounds of the host-to-host time (features on the device to waveforms on the
host) and seconds of audio per second, CUDA-event times of each stage (decode, time base, noise here; responses and
overlap-add from the library's events around those launches, gantts_profile_collect), the fp64 FFT rate from the pulse
counts, and the time --waveform adds to Synthesizer.synthesize_utterances.  Prints one JSON line per sample rate, with the card's name and power limit.

usage: python tools/time_world.py [--rounds 5] [--out DIR]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))

FP = 5.0
N_UTT, BATCH = 100, 20
PROF_WORLD_RESPONSE, PROF_WORLD_OLA = 6, 7      # gantts_profile_collect's kinds of the two synthesis kernels


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return out
    except Exception as e:                      # noqa: BLE001 - reported, not fatal
        return "unknown (%s)" % e


def inputs(fs, dev, seed=0):
    from gantts_b200 import generate, ops
    rng = np.random.RandomState(seed)
    lens = rng.randint(200, 1001, size=N_UTT)
    n = generate.cheaptrick_fft_size(fs)
    nb = ops.world_band_count(fs)
    batches = []
    for i in range(0, N_UTT, BATCH):
        ls = lens[i:i + BATCH]
        T = int(ls.max())
        B = len(ls)
        mc = np.zeros((B, T, 60), np.float32)
        f0 = np.zeros((B, T), np.float32)
        bap = np.zeros((B, T, nb), np.float32)
        for b, F in enumerate(ls):
            mc[b, :F] = rng.randn(60) * np.exp(-0.15 * np.arange(60)) + \
                np.cumsum(rng.randn(F, 60) * 0.02, 0) * np.exp(-0.2 * np.arange(60))
            t = 0
            while t < F:                        # voiced runs of 100-250 Hz, unvoiced gaps
                e = min(F, t + rng.randint(20, 80))
                if rng.rand() < 0.7:
                    f0[b, t:e] = 100 + 150 * rng.rand() + 10 * np.sin(np.arange(e - t) / 7.0)
                t = e
            bap[b, :F] = np.where(f0[b, :F, None] > 0, -25 + 5 * rng.randn(F, nb), 0.0)
        mc[:, :, 0] -= 2.0
        L = torch.tensor(ls, dtype=torch.int64, device=dev)
        sp = ops.mc2sp(torch.from_numpy(mc).to(dev), L, generate.mcep_alpha(fs), n)
        batches.append((torch.from_numpy(f0).to(dev), sp, torch.from_numpy(bap).to(dev), L, n))
    return batches, int(lens.sum())


def fft_flops(pulses_voiced, pulses_unvoiced, n):
    """Real n-point FFTs as n/2-point complex radix-2 FFTs (5 (n/2) log2(n/2) flops) plus the split (~10 n/2): seven
    per voiced pulse, four per unvoiced one."""
    per = 5 * (n // 2) * np.log2(n // 2) + 10 * (n // 2)
    return per * (7 * pulses_voiced + 4 * pulses_unvoiced)


def run_rate(fs, dev, rounds):
    from gantts_b200 import _lib, ops
    lib = _lib.load()
    batches, frames = inputs(fs, dev)
    stages = ("decode", "time_base", "noise", "responses", "overlap_add")

    def once(times=None):
        waves = []
        for f0, sp, bap, L, n in batches:
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
            ev[0].record()
            ap = ops.world_decode_aperiodicity(bap, L, fs, n)
            ev[1].record()
            tb = ops.world_time_base(f0, L, fs, FP, n)              # the kernel and its count read
            ev[2].record()
            noise = ops.world_randn(max(int(tb["y_lengths"].max()), 1), dev)
            ev[3].record()
            y, yl = ops.world_synthesize(f0, sp, ap, L, fs, FP, pulses=tb, noise=noise)
            host = y.cpu().numpy()
            waves.append([host[b, :yl[b]] for b in range(len(yl))])
            if times is not None:
                for k, (a, b) in zip(stages[:3], ((0, 1), (1, 2), (2, 3))):
                    times[k] += ev[a].elapsed_time(ev[b])
                vv = tb["vuv"].cpu().numpy()
                for b, P in enumerate(tb["counts"]):
                    v = int(vv[b, :P].sum())
                    times["voiced"] += v
                    times["unvoiced"] += int(P) - v
                times["samples"] += int(yl.sum())
        return waves

    once()
    torch.cuda.synchronize()
    walls, stats = [], []
    for _ in range(rounds):
        st = dict.fromkeys(stages + ("voiced", "unvoiced", "samples"), 0.0)
        ms, work = (ctypes.c_double * 8)(), (ctypes.c_double * 8)()
        cnt = (ctypes.c_longlong * 8)()
        lib.gantts_profile_enable(1)
        t0 = time.perf_counter()
        once(st)
        walls.append(time.perf_counter() - t0)
        lib.gantts_profile_enable(0)
        _lib.check(lib.gantts_profile_collect(ms, work, cnt))          # the library's events around each launch
        st["responses"], st["overlap_add"] = ms[PROF_WORLD_RESPONSE], ms[PROF_WORLD_OLA]
        stats.append(st)
    st = stats[int(np.argsort(walls)[len(walls) // 2])]
    wall = float(np.median(walls))
    n = batches[0][4]
    audio_s = st["samples"] / fs
    return {"fs": fs, "fftlen": n, "utterances": N_UTT, "batch": BATCH, "frames": frames, "audio_s": audio_s,
            "host_to_host_s": wall, "audio_s_per_s": audio_s / wall, "pulses_voiced": int(st["voiced"]),
            "pulses_unvoiced": int(st["unvoiced"]), "event_ms": {k: st[k] for k in stages},
            "fp64_fft_gflops_in_responses": fft_flops(st["voiced"], st["unvoiced"], n) / (st["responses"] * 1e-3)
            / 1e9}


def waveform_overhead(dev, rounds):
    """Synthesizer.synthesize_utterances with and without waveform=True on the test models (alternating, median)."""
    import tempfile
    import tts_data_helpers as TH
    from gantts_b200 import generate, models, synthesize
    data = TH.write_tts_data(os.path.join(tempfile.mkdtemp(), "data"), n_files=40)
    hp_a, hp_d = TH.srurnn_hps()
    sd, sa = generate.load_stats(TH.duration_hp(), data), generate.load_stats(TH.acoustic_hp(), data)
    generate.derive_dims(hp_a, sa), generate.derive_dims(hp_d, sd)
    torch.manual_seed(0)
    md, ma = models.SRURNN(**hp_d.generator_params).to(dev), models.SRURNN(**hp_a.generator_params).to(dev)
    X = [np.load(os.path.join(data, "X_duration", f)) for f in sorted(os.listdir(os.path.join(data, "X_duration")))]
    syn = {w: synthesize.Synthesizer(md, ma, hp_d, hp_a, sd, sa, waveform=w) for w in (False, True)}
    for w in (False, True):
        syn[w].synthesize_utterances(X, 20)
    t = {False: [], True: []}
    for _ in range(rounds):
        for w in (False, True):
            t0 = time.perf_counter()
            syn[w].synthesize_utterances(X, 20)
            t[w].append(time.perf_counter() - t0)
    frames = int(sum(x[:, 0].size for x in X))
    return {"utterances": len(X), "phones": frames, "without_s": float(np.median(t[False])),
            "with_waveform_s": float(np.median(t[True]))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import __graft_entry__
    __graft_entry__.build()
    if not torch.cuda.is_available():
        raise SystemExit("time_world.py needs a CUDA device")
    dev = torch.device("cuda:0")
    res = {"card": card(), "rates": [run_rate(fs, dev, a.rounds) for fs in (16000, 48000)],
           "synthesize_utterances": waveform_overhead(dev, a.rounds)}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "time_world.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
