"""Helpers of the synthesis tests (test_synthesize_host.py, test_gpu_synthesize.py): tiny TTS hyper parameters with the
acoustic frame-feature settings, and a seeded prepared TTS data directory whose X_acoustic is the frame expansion
(oracle.merlin_port) of X_duration with the natural durations Y_duration, with the statistics the training command
saves next to them."""
import os

import numpy as np

from oracle import merlin_port
import train_cli_helpers as H

L_PHONE = 20        # linguistic columns of a phone (416 in the shipped question set)
S_STATES = 5


def acoustic_hp(**over):
    kw = dict(subphone_features="full", add_frame_features=True, use_phone_alignment=False)
    kw.update(over)
    return H.tts_acoustic_hp(**kw)


def duration_hp(**over):
    kw = dict(subphone_features=None, add_frame_features=False, use_phone_alignment=False)
    kw.update(over)
    return H.tts_duration_hp(**kw)


def srurnn_hps():
    """(acoustic hp, duration hp) with small bidirectional SRURNN generators, as the shipped hparams use."""
    gp = lambda: {"in_dim": None, "out_dim": None, "num_hidden": 2, "hidden_dim": 16, "bidirectional": True,
                  "dropout": 0.0, "last_sigmoid": False, "use_relu": 1}
    return acoustic_hp(generator="SRURNN", generator_params=gp()), duration_hp(generator="SRURNN", generator_params=gp())


def random_durations(rng, P, S=S_STATES, lo=1, hi=8):
    return rng.randint(lo, hi + 1, size=(P, S)).astype(np.float32)


def write_tts_data(root, n_files=14, L=L_PHONE, S=S_STATES, seed=0):
    """root/{X,Y}_{duration,acoustic}: n_files utterances of 3..30 phones, and the eight statistics files of
    gantts_b200.train.load_data in root.  Returns root."""
    from gantts_b200 import train
    rng = np.random.RandomState(seed)
    dirs = {k: os.path.join(root, k) for k in ("X_duration", "Y_duration", "X_acoustic", "Y_acoustic")}
    for d in dirs.values():
        os.makedirs(d)
    for i in range(n_files):
        P = int(rng.randint(3, 31))
        x = (rng.rand(P, L) < 0.3).astype(np.float32)
        x[:, -3:] = rng.randint(0, 10, size=(P, 3))                   # a few numeric questions
        d = random_durations(rng, P, S)
        xa = merlin_port.expand(x, d)
        ya = (0.5 * rng.randn(len(xa), 187)).astype(np.float32)
        ya[:, 183] = rng.rand(len(xa)) > 0.4                        # V/UV
        name = "utt%03d.npy" % i
        for k, a in (("X_duration", x), ("Y_duration", d), ("X_acoustic", xa), ("Y_acoustic", ya)):
            np.save(os.path.join(dirs[k], name), a)
    train.load_data(duration_hp(), dirs["X_duration"], dirs["Y_duration"], -1)
    train.load_data(acoustic_hp(), dirs["X_acoustic"], dirs["Y_acoustic"], -1)
    return root
