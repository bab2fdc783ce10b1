# coding: utf-8
"""Synthesise TTS features with predicted durations: the duration model, then the acoustic model on its durations.

usage: synthesize.py [options] <acoustic_checkpoint> <duration_checkpoint> <data_dir> <dst_dir>

options:
    --fs=<fs>                   Sampling frequency [default: 16000].
    --disable-duraton-gen       Disable duration generation: use the natural durations of <data_dir>/Y_duration.
    --post-filter               Apply Merlin's post filter to spectral features.
    --spectrogram               Also write the power spectral envelope "sp" (mc2sp of mgc).
    --waveform                  Also write <dst_dir>/{eval,test}/<name>.wav: WORLD synthesis of f0, sp and the decoded
                                aperiodicity, scaled to int16 as evaluation_tts.py writes it.
    --batch-size=<N>            Utterances per batch (default: the acoustic hp.batch_size).
    --no-mge                    The acoustic generator was trained without MGE (de-normalise, then MLPG with the
                                variances of the statistics).
    -h, --help                  Show this help message and exit

The utterances are the evaluation split and the five test files of <data_dir>/X_acoustic; each one's phones are its
prepared rows in <data_dir>/X_duration, silences already removed.  The duration model runs on those silence-trimmed
phones, the sequences it was trained on, where the reference runs it on the label file's whole phone sequence and
removes silence frames afterwards: an MLP duration model predicts the same durations either way, a recurrent one (such
as the bidirectional SRURNN) can differ on the phones next to a silence.  Writes <dst_dir>/{eval,test}/<name>.npz with
"duration" and the acoustic features, and with --waveform also <name>.wav, the WORLD synthesis of its f0, sp and
aperiodicity on the device.
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
from . import objective
from . import ops
from . import train

WAVEFORM_NAME = "waveform"  # the extra output of waveform=True: WORLD synthesis, float64 (B, Ymax)


class UtteranceError(ValueError):
    """A refusal about one utterance; ``index`` is its position in the input list."""

    def __init__(self, index, msg):
        ValueError.__init__(self, msg)
        self.index = index


def check_waveform(hp_acoustic, fs):
    """The rules of waveform=True, checked before any model is loaded; ValueError naming the rule otherwise."""
    if generate.cheaptrick_fft_size(fs) > generate.MAX_FFTLEN:
        raise ValueError("--fs=%d needs a %d-point FFT; at most %d points are supported"
                         % (fs, generate.cheaptrick_fft_size(fs), generate.MAX_FFTLEN))
    bap_width = int(hp_acoustic.stream_sizes[3]) // (len(hp_acoustic.windows) if hp_acoustic.has_dynamic_features[3]
                                                     else 1)
    nb = ops.world_band_count(fs)
    if bap_width != nb:
        raise ValueError("the bap stream has %d static columns, but WORLD codes %d aperiodicity bands at --fs=%d"
                         % (bap_width, nb, fs))


def _hp_rule(hp, name, expected):
    if hp.name != expected:
        raise ValueError("the %s hyper parameters must have name %r (got %r)" % (name, expected, hp.name))


def check_tts_hparams(hp_acoustic, hp_duration, mge_training=True, post_filter=False, spectrogram=False, fs=16000,
                      waveform=False):
    """The configurations this command can run; raises ValueError naming the rule otherwise."""
    _hp_rule(hp_acoustic, "acoustic", "acoustic")
    _hp_rule(hp_duration, "duration", "duration")
    generate.check_hparams(hp_acoustic, mge_training, post_filter, spectrogram, fs)
    if waveform:
        check_waveform(hp_acoustic, fs)
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
    configure the acoustic generation as in generate.ParameterGenerator.  ``waveform`` adds WORLD synthesis
    (evaluation_tts.py:116-122 gen_waveform: decode_aperiodicity, then synthesize at hp_acoustic.frame_period); it
    computes the envelope "sp" whether or not ``spectrogram`` asks to return it."""

    def __init__(self, model_duration, model_acoustic, hp_duration, hp_acoustic, stats_duration, stats_acoustic,
                 mge_training=True, post_filter=False, spectrogram=False, fs=16000, waveform=False):
        check_tts_hparams(hp_acoustic, hp_duration, mge_training, post_filter, spectrogram, fs, waveform)
        self.spectrogram, self.waveform, self.fs = bool(spectrogram), bool(waveform), int(fs)
        self.frame_period = float(getattr(hp_acoustic, "frame_period", objective.FRAME_PERIOD))
        self.S = check_tts_stats(hp_duration, stats_duration, stats_acoustic)
        self.gen_duration = generate.ParameterGenerator(model_duration, hp_duration, stats_duration)
        self.gen_acoustic = generate.ParameterGenerator(model_acoustic, hp_acoustic, stats_acoustic, mge_training,
                                                        post_filter, spectrogram or waveform, fs)
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
        generate.ParameterGenerator.generate (B, T, ...), T the longest frame length, and with waveform=True
        "waveform", WORLD's synthesis of each row, float64 (B, Ymax), 0 beyond the row's ops.world_y_length.  The
        durations never leave the device; the frame lengths are the one host read, and with waveform=True the pulse
        counts a second.  Raises UtteranceError for a row of fewer than 2 frames when waveform is set."""
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
            if self.waveform:
                short = np.nonzero(host_lengths < 2)[0]
                if len(short):
                    raise UtteranceError(int(short[0]), "row %d has %d frames: a waveform needs at least 2"
                                         % (short[0], host_lengths[short[0]]))
                sp = out[generate.SPECTROGRAM_NAME] if self.spectrogram else out.pop(generate.SPECTROGRAM_NAME)
                ap = ops.world_decode_aperiodicity(out["bap"], frame_lengths, self.fs, 2 * (sp.shape[-1] - 1))
                out[WAVEFORM_NAME], _ = ops.world_synthesize(out["f0"], sp, ap, frame_lengths, self.fs,
                                                             self.frame_period)
        return out, host_lengths

    def synthesize_utterances(self, phone_arrays, batch_size, durations=None):
        """Un-normalised phone rows (P_i, L) (and natural state durations (P_i, S), or None) -> one dict of float32
        numpy arrays per utterance, in input order: "duration" (P_i, S) and the acoustic features of its frames, and
        with waveform=True its float64 "waveform" of ops.world_y_length samples.  The utterances are batched by phone
        count (generate.plan_batches); each batch makes one host-to-device copy, the one frame-lengths read and one
        device-to-host copy (and with waveform=True the pulse-count read and a second copy, of the waveforms).  Raises
        UtteranceError, whose index is the utterance's, for one of fewer than 2 frames when waveform is set."""
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
            try:
                out, flen = self.synthesize(x, dev[nx + nd:].to(torch.int64), d)
            except UtteranceError as e:
                raise UtteranceError(idx[e.index], "utterance %d has fewer than 2 frames: a waveform needs at least 2"
                                     % idx[e.index])
            wave = out.pop(WAVEFORM_NAME).cpu().numpy() if self.waveform else None
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
                if wave is not None:
                    r[WAVEFORM_NAME] = wave[j, :ops.world_y_length(flen[j], self.fs, self.frame_period)].copy()
                results[i] = r
        return results


# ---- the command (evaluation_tts.py:228-320) ----

def write_wav(path, y, fs):
    """evaluation_tts.py:126-127,320: y / max|y| * 32767 as int16, written at fs by scipy.io.wavfile."""
    from scipy.io import wavfile
    wavfile.write(path, fs, (y / np.max(np.abs(y)) * 32767).astype(np.int16))
    print(path)


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
    waveform = bool(args["--waveform"])
    natural = bool(args["--disable-duraton-gen"])
    data_dir, dst_dir = args["<data_dir>"], args["<dst_dir>"]
    try:
        try:
            fs = int(args["--fs"])
            batch_size = int(args["--batch-size"]) if args["--batch-size"] is not None else int(hp_acoustic.batch_size)
        except ValueError:
            raise ValueError("--fs and --batch-size must be integers (got %r, %r)" % (args["--fs"],
                                                                                      args["--batch-size"]))
        check_tts_hparams(hp_acoustic, hp_duration, mge_training, post_filter, spectrogram, fs, waveform)
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
                        spectrogram, fs, waveform)

    for sub, names in splits:
        out_dir = join(dst_dir, sub)
        os.makedirs(out_dir, exist_ok=True)
        phones = [np.load(join(data_dir, "X_duration", n + ".npy")) for n in names]
        durs = [np.load(join(data_dir, "Y_duration", n + ".npy")) for n in names] if natural else None
        try:
            results = synth.synthesize_utterances(phones, batch_size, durs)
        except UtteranceError as e:
            raise SystemExit("gantts_b200.synthesize: %s split: %s: %s" % (sub, names[e.index], e))
        for n, r in zip(names, results):
            wave = r.pop(WAVEFORM_NAME, None)
            if wave is not None and not np.any(wave):
                raise SystemExit("gantts_b200.synthesize: %s split: %s: the waveform is all zero and cannot be scaled "
                                 "to int16" % (sub, n))
            path = join(out_dir, n + ".npz")
            np.savez(path, **r)
            print(path)
            if wave is not None:
                write_wav(join(out_dir, n + ".wav"), wave, fs)
    return 0


if __name__ == "__main__":
    sys.exit(main())
