"""Compare the device analysis chain (ops.world_dio / world_stonemask / world_cheaptrick / sp2mc / modspec_smoothing)
and its numpy restatement oracle.world_analysis_port with pyworld, pysptk and nnmnkwii where those packages are installed:
seeded harmonic waveforms at 16 and 48 kHz, or the wavs given on the command line.  Prints one line per utterance with
the largest differences.  Needs a CUDA device for the device column.

usage: python tools/check_world_analysis.py [wav ...]"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))


def main(paths):
    import pysptk
    import pyworld
    import torch
    from nnmnkwii import preprocessing as P
    from gantts_b200 import analysis
    from oracle import world_analysis_port as A
    if paths:
        from scipy.io import wavfile
        utts = [wavfile.read(p)[::-1] + (p,) for p in paths]
    else:
        from test_gpu_world_analysis import wave
        rng = np.random.RandomState(0)
        utts = [(wave(rng, fs, 2.0)[0], fs, "seeded %d Hz" % fs) for fs in (16000, 48000)]
    dev = torch.device("cuda")
    for x, fs, name in utts:
        x = np.asarray(x).astype(np.float64)
        f0, t = pyworld.dio(x, fs, frame_period=5.0)
        f0 = pyworld.stonemask(x, f0, t, fs)
        sp = pyworld.cheaptrick(x, f0, t, fs)
        alpha = pysptk.util.mcepalpha(fs)
        mc = pysptk.sp2mc(sp, order=59, alpha=alpha)
        sm = P.modspec_smoothing(mc, analysis.modulation_rate(fs, 5.0), cutoff=50)
        g0, gt = A.dio(x, fs, 5.0)
        g0 = A.stonemask(x, g0, gt, fs)
        gsp = A.cheaptrick(x, g0, gt, fs)
        gmc = A.sp2mc(gsp, 59, alpha)
        dmc, frames, _ = analysis.analyse([x], fs, 5.0, 59, "tts_acoustic", dev)
        dmc = dmc.cpu().numpy()[0, :frames[0]]
        print("%s: frames %d/%d/%d, V/UV differs on %d frames, max |f0 diff| %.3g Hz, max |log sp diff| %.3g, "
              "max |mc diff| %.3g, max |smoothed mc diff| restatement %.3g device %.3g"
              % (name, len(f0), len(g0), frames[0], int(np.sum((f0 > 0) != (g0 > 0))), np.max(np.abs(f0 - g0)),
                 np.max(np.abs(np.log(sp) - np.log(gsp))), np.max(np.abs(mc - gmc)),
                 np.max(np.abs(sm - A.modspec_smoothing(gmc, analysis.modulation_rate(fs, 5.0)))),
                 np.max(np.abs(sm - dmc))))


if __name__ == "__main__":
    main(sys.argv[1:])
