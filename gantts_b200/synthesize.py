# coding: utf-8
"""Synthesise TTS features with predicted durations: the duration model, then the acoustic model on its durations.

usage: synthesize.py [options] <acoustic_checkpoint> <duration_checkpoint> <data_dir> <dst_dir>

options:
    --fs=<fs>                   Sampling frequency [default: 16000].
    --disable-duraton-gen       Disable duration generation: use the natural durations of <data_dir>/Y_duration.
    --post-filter               Apply Merlin's post filter to spectral features.
    --spectrogram               Also write the power spectral envelope "sp" (mc2sp of mgc).
    --batch-size=<N>            Utterances per batch (default: the acoustic hp.batch_size).
    --no-mge                    The acoustic generator was trained without MGE (de-normalise, then MLPG with the
                                variances of the statistics).
    -h, --help                  Show this help message and exit

The utterances are the evaluation split and the five test files of <data_dir>/X_acoustic; each one's phones are its
prepared rows in <data_dir>/X_duration, silences already removed.  The duration model runs on those silence-trimmed
phones, the sequences it was trained on, where the reference runs it on the label file's whole phone sequence and
removes silence frames afterwards: an MLP duration model predicts the same durations either way, a recurrent one (such
as the bidirectional SRURNN) can differ on the phones next to a silence.  Writes <dst_dir>/{eval,test}/<name>.npz with
"duration" and the acoustic features, no audio: WORLD synthesis is not done here.
"""
# evaluation_tts.py:143-225 (gen_duration, tts_from_label) on padded device batches: the duration model's min-max scaling
# and generation (rounded, at least 1), each phone's first frame (gantts_state_frame_offsets), the frame-level acoustic
# inputs with Merlin's "full" subphone features, min-max scaled (gantts_expand_state_frames), and the acoustic
# generation.  The HTS label front end is not needed: the prepared X_duration row of a phone is the question-feature
# part of every frame of that phone in X_acoustic, and the subphone features depend only on its state durations.
import os
import sys
from os.path import basename, exists, join, splitext

import numpy as np
import torch

from . import _lib
from . import generate
from . import models
from . import ops
from . import train


def _hp_rule(hp, name, expected):
    if hp.name != expected:
        raise ValueError("the %s hyper parameters must have name %r (got %r)" % (name, expected, hp.name))


def check_tts_hparams(hp_acoustic, hp_duration, mge_training=True, post_filter=False, spectrogram=False, fs=16000):
    """The configurations this command can run; raises ValueError naming the rule otherwise."""
    _hp_rule(hp_acoustic, "acoustic", "acoustic")
    _hp_rule(hp_duration, "duration", "duration")
    generate.check_hparams(hp_acoustic, mge_training, post_filter, spectrogram, fs)
    generate.check_hparams(hp_duration)
    sub = getattr(hp_acoustic, "subphone_features", None)
    if sub != "full":
        raise ValueError("the acoustic hp.subphone_features must be \"full\" (got %r): only Merlin's full subphone "
                         "features are generated" % (sub,))
    if not getattr(hp_acoustic, "add_frame_features", False):
        raise ValueError("the acoustic hp.add_frame_features must be True: the acoustic model runs on frames")
    for hp, name in ((hp_acoustic, "acoustic"), (hp_duration, "duration")):
        if getattr(hp, "use_phone_alignment", False):
            raise ValueError("the %s hp.use_phone_alignment=True is not supported: the frames come from state "
                             "durations" % name)


def check_tts_stats(hp_duration, stats_duration, stats_acoustic):
    """S, the number of states per phone, from the statistics; ValueError naming the rule when the two models' shapes
    disagree."""
    S = int(np.shape(stats_duration["Y_mean"])[-1])
    total = int(sum(hp_duration.stream_sizes))
    if S != total:
        raise ValueError("the duration statistics have %d state columns but hp_duration.stream_sizes totals %d"
                         % (S, total))
    if not 1 <= S <= 16:
        raise ValueError("S = %d states per phone must be in [1, 16]" % S)
    L, La = int(np.shape(stats_duration["X_min"])[-1]), int(np.shape(stats_acoustic["X_min"])[-1])
    if La != L + _lib.SUBPHONE_FEATURES:
        raise ValueError("the acoustic input statistics have %d columns but the duration ones %d: the acoustic inputs "
                         "must be the %d phone columns and the %d subphone features"
                         % (La, L, L, _lib.SUBPHONE_FEATURES))
    return S


def _f32_params(stats, device):
    """train.minmax_scale_params of the statistics, as float32 device vectors (min_, scale_)."""
    min_, scale_ = train.minmax_scale_params(stats["X_min"], stats["X_max"])
    f32 = lambda a: torch.as_tensor(np.ascontiguousarray(a), dtype=torch.float32, device=device)
    return f32(min_), f32(scale_)


class Synthesizer(object):
    """A trained duration model and acoustic model chained on the device, as evaluation_tts.py's tts_from_label chains
    them.  ``stats_*`` as generate.load_stats returns them; ``mge_training``, ``post_filter``, ``spectrogram`` and ``fs``
    configure the acoustic generation as in generate.ParameterGenerator."""

    def __init__(self, model_duration, model_acoustic, hp_duration, hp_acoustic, stats_duration, stats_acoustic,
                 mge_training=True, post_filter=False, spectrogram=False, fs=16000):
        check_tts_hparams(hp_acoustic, hp_duration, mge_training, post_filter, spectrogram, fs)
        self.S = check_tts_stats(hp_duration, stats_duration, stats_acoustic)
        self.gen_duration = generate.ParameterGenerator(model_duration, hp_duration, stats_duration)
        self.gen_acoustic = generate.ParameterGenerator(model_acoustic, hp_acoustic, stats_acoustic, mge_training,
                                                        post_filter, spectrogram, fs)
        if self.gen_duration.ncols != self.S:
            raise ValueError("the duration model generates %d columns for S = %d states"
                             % (self.gen_duration.ncols, self.S))
        self.device = self.gen_acoustic.device
        self.L = int(np.shape(stats_duration["X_min"])[-1])
        self.min_d, self.scale_d = _f32_params(stats_duration, self.device)
        self.min_a, self.scale_a = _f32_params(stats_acoustic, self.device)

    def duration_inputs(self, phone_x_raw, phone_lengths):
        """The duration model's inputs: P.minmax_scale of the phone rows as generate.normalize_input computes it on
        float32 statistics, a float32 multiply and then a float32 add (not a fused addcmul), and 0 for padding
        phones."""
        P = phone_x_raw.shape[1]
        x = torch.add(torch.mul(phone_x_raw, self.scale_d), self.min_d)
        valid = (torch.arange(P, device=self.device)[None, :] < phone_lengths[:, None]).unsqueeze(-1)
        return torch.where(valid, x, torch.zeros_like(x))

    def synthesize(self, phone_x_raw, phone_lengths, durations=None):
        """phone_x_raw: (B, P, L) un-normalised phone rows (X_duration), CUDA float32; phone_lengths: int64 CUDA (B,);
        durations: None to predict them, or natural (B, P, S) CUDA float32 state durations.  Returns (out, frame
        lengths as a host int64 array): out holds "duration" (B, P, S) and the acoustic keys of
        generate.ParameterGenerator.generate (B, T, ...), T the longest frame length.  The durations never leave the
        device; the frame lengths are the one host read."""
        ops.require_cuda(phone_x_raw, durations)
        if phone_x_raw.dim() != 3 or phone_x_raw.shape[-1] != self.L:
            raise RuntimeError("gantts_b200: synthesize needs phone rows (B, P, %d)" % self.L)
        B, P, _ = phone_x_raw.shape
        with torch.no_grad():
            if durations is None:
                x = self.duration_inputs(phone_x_raw, phone_lengths)
                durations = self.gen_duration.generate(x, phone_lengths)["duration"]
            elif tuple(durations.shape) != (B, P, self.S):
                raise RuntimeError("gantts_b200: synthesize needs durations (B, P, S) = (%d, %d, %d)" % (B, P, self.S))
            offsets, frame_lengths, host_lengths = ops.state_frame_offsets(durations, phone_lengths)
            T = int(host_lengths.max())
            if T < 1:
                raise RuntimeError("gantts_b200: synthesize needs at least one phone per batch")
            x = ops.expand_state_frames(phone_x_raw, durations, offsets, frame_lengths, self.scale_a, self.min_a, T)
            out = {"duration": durations}
            out.update(self.gen_acoustic.generate(x, frame_lengths))
        return out, host_lengths

    def synthesize_utterances(self, phone_arrays, batch_size, durations=None):
        """Un-normalised phone rows (P_i, L) (and natural state durations (P_i, S), or None) -> one dict of float32
        numpy arrays per utterance, in input order: "duration" (P_i, S) and the acoustic features of its frames.  The
        utterances are batched by phone count (generate.plan_batches); each batch makes one host-to-device copy, the
        one frame-lengths read and one device-to-host copy."""
        for i, a in enumerate(phone_arrays):
            if len(a) < 1:
                raise ValueError("utterance %d has no phones" % i)
        results = [None] * len(phone_arrays)
        L, S = self.L, self.S
        for idx in generate.plan_batches([len(a) for a in phone_arrays], batch_size):
            B, lens = len(idx), [len(phone_arrays[i]) for i in idx]
            P = max(lens)
            nx, nd = B * P * L, (B * P * S if durations is not None else 0)
            host = np.zeros(nx + nd + B, dtype=np.float32)          # rows, durations, phone counts: one copy
            hx = host[:nx].reshape(B, P, L)
            hd = host[nx:nx + nd].reshape(B, P, S) if nd else None
            for j, i in enumerate(idx):
                hx[j, :lens[j]] = phone_arrays[i]
                if nd:
                    hd[j, :lens[j]] = durations[i]
            host[nx + nd:] = lens
            dev = torch.from_numpy(host).to(self.device)
            x = dev[:nx].view(B, P, L)
            d = dev[nx:nx + nd].view(B, P, S) if nd else None
            out, flen = self.synthesize(x, dev[nx + nd:].to(torch.int64), d)
            names = list(out)
            flat = torch.cat([out[k].reshape(-1) for k in names]).cpu().numpy()
            pos = 0
            per = {}
            for k in names:
                shape = tuple(out[k].shape)
                per[k] = flat[pos:pos + int(np.prod(shape))].reshape(shape)
                pos += int(np.prod(shape))
            for j, i in enumerate(idx):
                r = {"duration": np.ascontiguousarray(per["duration"][j, :lens[j]])}
                for k in names[1:]:
                    r[k] = np.ascontiguousarray(per[k][j, :flen[j]])
                results[i] = r
        return results


# ---- the command (evaluation_tts.py:228-300 without the vocoder) ----

def utterance_names(data_dir):
    """[("eval", names), ("test", names)]: get_lab_files' utterances (evaluation_tts.py:236-245), the evaluation split
    and the five test files of <data_dir>/X_acoustic."""
    return [(sub, [splitext(basename(f))[0] for f in files])
            for sub, files in generate.utterance_files(join(data_dir, "X_acoustic"))]


def check_files(data_dir, splits, natural_durations):
    """ValueError naming the first utterance whose X_duration (or, for natural durations, Y_duration) file is missing."""
    dirs = ["X_duration"] + (["Y_duration"] if natural_durations else [])
    for sub, names in splits:
        for n in names:
            for d in dirs:
                if not exists(join(data_dir, d, n + ".npy")):
                    raise ValueError("%s split: %s has no %s/%s.npy" % (sub, n, d, n))


def parse_args(argv=None):
    from compat.docopt import docopt
    return docopt(__doc__, argv=argv)


def main(argv=None, hp_acoustic=None, hp_duration=None):
    """``hp_acoustic`` / ``hp_duration``: the hyper-parameter objects to use instead of hparams.tts_acoustic and
    hparams.tts_duration (``import hparams`` from the caller's path otherwise)."""
    args = parse_args(argv)
    if hp_acoustic is None or hp_duration is None:
        import hparams
        hp_acoustic = hparams.tts_acoustic if hp_acoustic is None else hp_acoustic
        hp_duration = hparams.tts_duration if hp_duration is None else hp_duration
    mge_training = not args["--no-mge"]
    post_filter, spectrogram = bool(args["--post-filter"]), bool(args["--spectrogram"])
    natural = bool(args["--disable-duraton-gen"])
    data_dir, dst_dir = args["<data_dir>"], args["<dst_dir>"]
    try:
        try:
            fs = int(args["--fs"])
            batch_size = int(args["--batch-size"]) if args["--batch-size"] is not None else int(hp_acoustic.batch_size)
        except ValueError:
            raise ValueError("--fs and --batch-size must be integers (got %r, %r)" % (args["--fs"],
                                                                                      args["--batch-size"]))
        check_tts_hparams(hp_acoustic, hp_duration, mge_training, post_filter, spectrogram, fs)
        if batch_size < 1:
            raise ValueError("--batch-size must be >= 1 (got %d)" % batch_size)
        stats_d, stats_a = generate.load_stats(hp_duration, data_dir), generate.load_stats(hp_acoustic, data_dir)
        check_tts_stats(hp_duration, stats_d, stats_a)
        splits = utterance_names(data_dir)
        check_files(data_dir, splits, natural)
    except ValueError as e:
        raise SystemExit("gantts_b200.synthesize: %s" % e)
    if not torch.cuda.is_available():
        raise SystemExit("gantts_b200.synthesize: needs a CUDA device (there is no CPU path)")
    device = torch.device("cuda")

    loaded = []
    for hp, stats, ck in ((hp_duration, stats_d, args["<duration_checkpoint>"]),
                          (hp_acoustic, stats_a, args["<acoustic_checkpoint>"])):
        generate.derive_dims(hp, stats)
        model = getattr(models, hp.generator)(**hp.generator_params)
        train.load_checkpoint(model, ck)
        loaded.append(model.to(device))
    synth = Synthesizer(loaded[0], loaded[1], hp_duration, hp_acoustic, stats_d, stats_a, mge_training, post_filter,
                        spectrogram, fs)

    for sub, names in splits:
        out_dir = join(dst_dir, sub)
        os.makedirs(out_dir, exist_ok=True)
        phones = [np.load(join(data_dir, "X_duration", n + ".npy")) for n in names]
        durs = [np.load(join(data_dir, "Y_duration", n + ".npy")) for n in names] if natural else None
        for n, r in zip(names, synth.synthesize_utterances(phones, batch_size, durs)):
            path = join(out_dir, n + ".npz")
            np.savez(path, **r)
            print(path)
    return 0


if __name__ == "__main__":
    sys.exit(main())
