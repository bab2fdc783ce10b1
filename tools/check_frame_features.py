"""Check the frame expansion of gantts_expand_state_frames against a prepared TTS corpus (prepare_features_tts.py's
output, which nnmnkwii computed): every utterance's X_duration rows expanded on the device with its Y_duration state
durations, raw (scale 1, min 0), must equal its X_acoustic bit for bit.  Prints each mismatching utterance with the
mismatching columns and the largest absolute difference; exits 1 when any utterance differs.

    python tools/check_frame_features.py DATA_DIR [--batch-size N]
"""
import argparse
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__  # noqa: E402

__graft_entry__.build()
from gantts_b200 import _lib, generate, ops  # noqa: E402


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("data_dir")
    ap.add_argument("--batch-size", type=int, default=32)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    xa_dir = os.path.join(args.data_dir, "X_acoustic")
    names = sorted(os.path.splitext(f)[0] for f in os.listdir(xa_dir) if f.endswith(".npy"))
    load = lambda sub, n: np.load(os.path.join(args.data_dir, sub, n + ".npy"))
    X, D = [load("X_duration", n) for n in names], [load("Y_duration", n) for n in names]
    L, S = X[0].shape[1], D[0].shape[1]
    W = L + _lib.SUBPHONE_FEATURES
    ones, zeros = torch.ones(W, device=dev), torch.zeros(W, device=dev)
    bad = 0
    for idx in generate.plan_batches([len(x) for x in X], args.batch_size):
        lens = [len(X[i]) for i in idx]
        B, P = len(idx), max(lens)
        xb, db = np.zeros((B, P, L), np.float32), np.ones((B, P, S), np.float32)
        for j, i in enumerate(idx):
            xb[j, :lens[j]], db[j, :lens[j]] = X[i], D[i]
        dt = torch.from_numpy(db).to(dev)
        offsets, fl, host = ops.state_frame_offsets(dt, torch.tensor(lens, dtype=torch.int64, device=dev))
        out = ops.expand_state_frames(torch.from_numpy(xb).to(dev), dt, offsets, fl, ones, zeros,
                                      int(host.max())).cpu().numpy()
        for j, i in enumerate(idx):
            want = load("X_acoustic", names[i])
            got = out[j, :host[j]]
            if got.shape != want.shape:
                print("%s: %d frames from the durations, %d in X_acoustic (%d columns vs %d)"
                      % (names[i], len(got), len(want), got.shape[1], want.shape[1]))
                bad += 1
                continue
            diff = got.view(np.int32) != want.view(np.int32)
            if diff.any():
                cols = np.nonzero(diff.any(axis=0))[0]
                err = float(np.abs(got.astype(np.float64) - want)[diff].max())
                print("%s: %d frames differ in columns %s; max abs difference %.3g"
                      % (names[i], int(diff.any(axis=1).sum()), ", ".join(str(c) for c in cols[:20]), err))
                bad += 1
    print("%d of %d utterances match X_acoustic bit for bit" % (len(names) - bad, len(names)))
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
