"""Compare the device WORLD synthesis with pyworld where pyworld is installed: ops.world_decode_aperiodicity against
pyworld.decode_aperiodicity and ops.world_synthesize against pyworld.synthesize, utterance by utterance, on seeded
inputs (f0 tracks with voiced runs and gaps, sp from random order-59 mgc through pysptk.mc2sp's device counterpart) or
on a directory of generated features (<name>.npz files with "f0", "bap" and "sp", as synthesize --spectrogram writes
them).  Prints the largest relative differences; exits non-zero when they exceed the tolerances.

usage: python tools/check_world.py [--fs 16000] [--frame-period 5] [--features DIR] [--utterances 8]
"""
import argparse
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))


def seeded(fs, count, seed=0):
    from gantts_b200 import generate, ops
    rng = np.random.RandomState(seed)
    n, nb = generate.cheaptrick_fft_size(fs), ops.world_band_count(fs)
    out = []
    for _ in range(count):
        F = int(rng.randint(50, 600))
        f0 = np.where((np.arange(F) // 40) % 3 == 2, 0.0, 100 + 150 * rng.rand(F)).astype(np.float32)
        mc = (rng.randn(60) * np.exp(-0.15 * np.arange(60)) + np.cumsum(rng.randn(F, 60) * 0.02, 0) *
              np.exp(-0.2 * np.arange(60))).astype(np.float32)
        mc[:, 0] -= 2.0
        L = torch.tensor([F], dtype=torch.int64, device="cuda")
        sp = ops.mc2sp(torch.from_numpy(mc[None]).cuda(), L, generate.mcep_alpha(fs), n)[0].cpu().numpy()
        bap = np.where(f0[:, None] > 0, -25 + 5 * rng.randn(F, nb), 0.0).astype(np.float32)
        out.append(("seeded%d" % len(out), f0, sp, bap))
    return out


def from_dir(d):
    out = []
    for f in sorted(os.listdir(d)):
        if f.endswith(".npz"):
            z = np.load(os.path.join(d, f))
            out.append((f[:-4], z["f0"].reshape(-1).astype(np.float32), z["sp"], z["bap"]))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--fs", type=int, default=16000)
    ap.add_argument("--frame-period", type=float, default=5.0)
    ap.add_argument("--features", default=None)
    ap.add_argument("--utterances", type=int, default=8)
    a = ap.parse_args()
    import pyworld
    import __graft_entry__
    __graft_entry__.build()
    from gantts_b200 import ops
    utts = from_dir(a.features) if a.features else seeded(a.fs, a.utterances)
    worst_ap = worst_y = 0.0
    for name, f0, sp, bap in utts:
        n = 2 * (sp.shape[1] - 1)
        L = torch.tensor([len(f0)], dtype=torch.int64, device="cuda")
        ap_d = ops.world_decode_aperiodicity(torch.from_numpy(bap[None]).cuda(), L, a.fs, n)
        y_d, _ = ops.world_synthesize(torch.from_numpy(f0[None]).cuda(), torch.from_numpy(sp[None]).cuda(), ap_d, L,
                                      a.fs, a.frame_period)
        ap_w = pyworld.decode_aperiodicity(np.ascontiguousarray(bap, dtype=np.float64), a.fs, n)
        y_w = pyworld.synthesize(f0.astype(np.float64), sp.astype(np.float64), ap_w, a.fs, a.frame_period)
        e_ap = float(np.max(np.abs(ap_d[0].cpu().numpy() - ap_w) / ap_w))
        y = y_d[0, :len(y_w)].cpu().numpy()
        e_y = float(np.max(np.abs(y - y_w)) / max(np.max(np.abs(y_w)), 1e-300)) if len(y) == len(y_w) else float("inf")
        print("%s: ap %.3g, y %.3g of max|y| (%d samples)" % (name, e_ap, e_y, len(y_w)))
        worst_ap, worst_y = max(worst_ap, e_ap), max(worst_y, e_y)
    print("worst: ap %.3g, y %.3g" % (worst_ap, worst_y))
    return 0 if worst_ap <= 1e-12 and worst_y <= 1e-10 else 1


if __name__ == "__main__":
    sys.exit(main())
