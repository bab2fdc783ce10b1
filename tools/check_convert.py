"""Compare the device conversion chain and its numpy restatements with pysptk, pyworld and nnmnkwii where those packages
are installed: evaluation_vc.py's test_vc_from_path(diffvc=True) with a small random In2OutHighwayNet on seeded harmonic
waveforms at 16 and 48 kHz.  This is where the MLSA filter's gain convention (no exp(b[0])) and its frame loop
(Synthesizer.synthesis) are confirmed against pysptk.  Prints one line per utterance with the largest differences.
Needs a CUDA device for the device column.

usage: python tools/check_convert.py"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))


def main():
    import pysptk
    import pyworld
    import torch
    from nnmnkwii import preprocessing as P
    from pysptk.synthesis import MLSADF, Synthesizer
    import train_cli_helpers as H
    from gantts_b200 import analysis, convert, models
    from oracle import mlsa_port, sptk_port
    from test_gpu_world_analysis import wave
    dev = torch.device("cuda")
    order, fp = 24, 5.0
    rng = np.random.RandomState(0)
    torch.manual_seed(0)
    model = models.In2OutHighwayNet(3 * order, 3 * order, order, num_hidden=2, hidden_dim=64, dropout=0.0).to(dev)
    stats = {"data_mean": rng.randn(3 * order) * 0.1, "data_std": rng.uniform(0.5, 1.5, 3 * order)}
    hp = H.vc_hp(order=order)
    for fs in (16000, 48000):
        conv = convert.VoiceConverter(model, hp, stats, fs)
        x = wave(rng, fs, 1.5)[0].astype(np.int16).astype(np.float64)
        hop = int(fs * (fp * 0.001))
        alpha = pysptk.util.mcepalpha(fs)
        f0, t = pyworld.dio(x, fs, frame_period=fp)
        f0 = pyworld.stonemask(x, f0, t, fs)
        mc = pysptk.sp2mc(pyworld.cheaptrick(x, f0, t, fs), order=order, alpha=alpha)
        src = P.modspec_smoothing(mc[:, 1:], fs / hop, cutoff=50)
        d = P.delta_features(src, hp.windows).astype(np.float32)
        got = conv.convert_utterances([x], 1)[0]
        diff = np.hstack([np.zeros((len(d), 1)), got["mc"].astype(np.float64) - d[:, :order]])
        b = pysptk.mc2b(diff, alpha=alpha)
        y = Synthesizer(MLSADF(order=order, alpha=alpha), hopsize=hop).synthesis(x, b)
        y_port = mlsa_port.mlsa_synthesis([x], [b], alpha, hop)[0]
        print("%d Hz: frames %d/%d, max |smoothed mc diff| %.3g, filter on pysptk's b: restatement %.3g, device "
              "%.3g (relative to the peak)"
              % (fs, len(d), len(got["mc"]), np.max(np.abs(src[:, :] - conv.analyse(*analysis.pad_waves([x], dev))[0]
                                                          .cpu().numpy()[0, :len(d)])),
                 np.max(np.abs(y_port - y)) / np.max(np.abs(y)),
                 np.max(np.abs(got["waveform"] - y)) / np.max(np.abs(y))))


if __name__ == "__main__":
    main()
