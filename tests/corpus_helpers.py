"""Helpers of the device-corpus tests (test_corpus_host.py, test_gpu_corpus.py): seeded feature directories at the
widths the training command meets, the hyper parameters that read them, and a numpy restatement of gantts_corpus_gather
over a packed corpus."""
import os

import numpy as np

import train_cli_helpers as H

# name -> (hp factory, input width, output width)
KINDS = {
    "vc": (H.vc_hp, 12, 12),
    "tts_acoustic": (H.tts_acoustic_hp, 425, 187),
    "tts_acoustic_delta": (lambda **k: H.tts_acoustic_hp(recompute_delta_features=True, **k), 425, 187),
    "tts_duration": (H.tts_duration_hp, 416, 5),
}


def write_pairs(root, dx, dy, n_files=30, seed=0):
    """root/X and root/Y: n_files time-aligned float32 utterances of 1..40 frames, every fifth one a single frame."""
    rng = np.random.RandomState(seed)
    xd, yd = os.path.join(root, "X"), os.path.join(root, "Y")
    os.makedirs(xd), os.makedirs(yd)
    for i in range(n_files):
        n = 1 if i % 5 == 0 else int(rng.randint(2, 41))
        x = rng.rand(n, dx).astype(np.float32) * 3
        y = (0.5 * rng.randn(n, dy) + 0.2).astype(np.float32)
        if dy == 187:
            y[:, 183] = rng.rand(n) > 0.4                            # V/UV
        if dy == 5:
            y = rng.randint(1, 9, size=(n, dy)).astype(np.float32)  # state durations
        np.save(os.path.join(xd, "utt%03d.npy" % i), x)
        np.save(os.path.join(yd, "utt%03d.npy" % i), y)
    return xd, yd


def write_kind(root, kind):
    _, dx, dy = KINDS[kind]
    return write_pairs(root, dx, dy)


def gather(X, Y, offsets, lengths, t):
    """gantts_corpus_gather in numpy: rows [offsets[r], offsets[r] + lengths[r]) of X and Y, zero-padded to t frames."""
    b = len(offsets)
    x = np.zeros((b, t, X.shape[1]), dtype=np.float32)
    y = np.zeros((b, t, Y.shape[1]), dtype=np.float32)
    for r, (o, n) in enumerate(zip(offsets, lengths)):
        x[r, :n], y[r, :n] = X[o:o + n], Y[o:o + n]
    return x, y
