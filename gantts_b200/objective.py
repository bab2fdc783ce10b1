# coding: utf-8
"""Compare the global variances and modulation spectra of generated and natural features.

usage: objective.py [options] <inputs_dir> <outputs_dir> <dst_dir> <checkpoint>...

options:
    --hparams_name=<name>       Name of hyper params: vc or tts_acoustic [default: vc].
    --hparams=<parmas>          Hyper parameters to be overrided [default: ].
    --labels=<a,b,...>          One label per checkpoint (default: each checkpoint's parent directory name).
    --batch-size=<N>            Utterances per batch (default: hp.batch_size).
    --no-mge                    tts_acoustic: the generator was trained without MGE.
    --ms-fftlen=<n>             FFT length of the modulation spectrum [default: 4096].
    --fs=<fs>                   Sampling frequency of ms_freq and of the --wav-dir wavs [default: 16000].
    --wav-dir=<dir>             Also analyse <dir>/<name>.wav of every utterance with WORLD, as the notebooks do, and
                                compare against those features too (label natural_wav).
    -h, --help                  Show this help message and exit

"Natural" features are the prepared targets of <outputs_dir> (Y, not normalised): the static mc columns for vc, the
static mgc columns for tts_acoustic.  The reference notebooks re-analyse the target wavs with WORLD instead; --wav-dir
adds those features beside the prepared ones (gantts_b200.analysis: DIO, StoneMask, CheapTrick, sp2mc, and for
tts_acoustic the modulation-spectrum smoothing), for vc from the target speaker's wavs.  tts_acoustic generates from the
prepared inputs, so with natural durations.
"""
# The measures of the reference notebooks (notebooks/Test VC.ipynb, Test RNN VC.ipynb, Test TTS.ipynb): vis_gv's
# np.var(mgc, axis=0) per utterance and mean_modspec's mean over utterances of np.log(P.modspec(mgc, n=4096)), for the
# natural features and for each checkpoint's generated ones.  Features stay on the device: the generator's output batch
# goes straight into the kernels (gantts_global_variance, gantts_modspec), and only the variances and the final sums of
# the spectra are copied back.  Writes <dst_dir>/{eval,test}.npz.
import os
import sys
from os.path import abspath, basename, dirname, join, splitext

import numpy as np
import torch

from . import analysis
from . import generate
from . import models
from . import multistream
from . import ops
from . import train

FEATURES = {"vc": "mc", "acoustic": "mgc"}      # the generated features compared, by hp.name
MIN_FFTLEN, MAX_FFTLEN = 64, 8192               # gantts_modspec's n
FRAME_PERIOD = 5                                # ms, hparams.py's frame_period, when hp does not say


class FeatureStats(object):
    """Per-utterance global variances and the summed log modulation spectrum of (B, T, D) device batches, on the
    device.  Spectra are folded one utterance at a time in the order ``add`` sees them, so with the utterances added in
    a fixed order (generate.plan_batches) the result has the same bits whatever the batch size."""

    def __init__(self, D, n, device):
        self.D, self.n = int(D), int(n)
        self.ms_sum = torch.zeros(self.n // 2 + 1, self.D, dtype=torch.float64, device=device)
        self.gv, self.count = [], 0

    def add(self, x, lengths):
        """x (B, T, D) CUDA float32, any batch and time strides; lengths int64 CUDA (B,).  No host sync."""
        if x.dim() != 3 or x.shape[-1] != self.D:
            raise RuntimeError("gantts_b200: FeatureStats of D = %d columns got x of shape %s"
                               % (self.D, tuple(x.shape)))
        self.gv.append(ops.global_variance(x, lengths))
        ops.modspec(x, lengths, self.n, out_sum=self.ms_sum)
        self.count += x.shape[0]

    def result(self):
        """(gv (U, D) in the order added, its mean over utterances (D,), the mean log modulation spectrum
        (n/2 + 1, D)), float64 numpy."""
        if self.count == 0:
            raise RuntimeError("gantts_b200: FeatureStats has no utterances")
        gv = torch.cat(self.gv).cpu().numpy()
        return gv, gv.mean(axis=0), self.ms_sum.cpu().numpy() / self.count


def check_fftlen(n):
    if not (MIN_FFTLEN <= n <= MAX_FFTLEN and n & (n - 1) == 0):
        raise ValueError("--ms-fftlen must be a power of two in [%d, %d] (got %d)" % (MIN_FFTLEN, MAX_FFTLEN, n))


def modulation_frequencies(n, fs, frame_period=FRAME_PERIOD):
    """ms_freq of the notebooks: arange(n//2 + 1) / n * modfs, modfs = fs / int(fs * frame_period * 0.001)."""
    hop = int(fs * (frame_period * 0.001))
    if hop < 1:
        raise ValueError("--fs=%d gives a hop of %d samples at a %g ms frame period; it must be >= 1"
                         % (fs, hop, frame_period))
    return np.arange(n // 2 + 1) / n * (fs / hop)


def natural_columns(hp):
    """The columns of the prepared targets compared: the static columns of the first stream."""
    streams = [True] + [False] * (len(hp.stream_sizes) - 1)
    cols = multistream.static_feature_columns(len(hp.windows), hp.stream_sizes, hp.has_dynamic_features, streams)
    return slice(cols[0], cols[-1] + 1)


def check_labels(labels, checkpoints, wavs=False):
    """The labels as given, or each checkpoint's parent directory name; ValueError naming the rule otherwise.  wavs:
    "natural_wav" is taken too."""
    if labels is None:
        labels = [basename(dirname(abspath(c))) for c in checkpoints]
        hint = " (the default labels are the checkpoints' directory names; pass --labels)"
    else:
        labels, hint = labels.split(","), ""
    if len(labels) != len(checkpoints):
        raise ValueError("--labels has %d labels for %d checkpoints: give one per checkpoint"
                         % (len(labels), len(checkpoints)))
    if any(not lab for lab in labels):
        raise ValueError("--labels: a label must not be empty")
    seen = ["natural"] + (["natural_wav"] if wavs else [])
    note = "\"natural\" is the prepared targets' label" + (", \"natural_wav\" the analysed wavs'" if wavs else "")
    for lab in labels:
        if lab in seen:
            raise ValueError("label %r is used twice (%s)%s" % (lab, note, hint))
        seen.append(lab)
    return labels


def paired_files(inputs_dir, outputs_dir):
    """[(split, X files, Y files)] for eval and test (generate.utterance_files); ValueError when the names differ."""
    out = []
    for (sub, xf), (_, yf) in zip(generate.utterance_files(inputs_dir), generate.utterance_files(outputs_dir)):
        xn, yn = [basename(f) for f in xf], [basename(f) for f in yf]
        if xn != yn:
            raise ValueError("%s split: the utterances of %s and %s differ (%s); X and Y must hold the same file names"
                             % (sub, inputs_dir, outputs_dir, ", ".join(sorted(set(xn) ^ set(yn))[:4])))
        if not xf:
            raise ValueError("%s split: %s has no utterances" % (sub, inputs_dir))
        out.append((sub, xf, yf))
    return out


def check_frames(files, X, Y):
    for f, x, y in zip(files, X, Y):
        if len(x) != len(y):
            raise ValueError("%s: %d input frames but %d target frames; X and Y must be time-aligned (train.load_data)"
                             % (basename(f), len(x), len(y)))


def read_wavs(wav_dir, files, fs=None):
    """The samples of <wav_dir>/<name>.wav for every utterance file, as the notebooks read them (scipy.io.wavfile,
    cast to float64 later); ValueError naming the wav when one is missing, is not at fs (None: at the first wav's rate)
    or is not mono."""
    from scipy.io import wavfile
    waves, first = [], None
    for f in files:
        path = join(wav_dir, splitext(basename(f))[0] + ".wav")
        if not os.path.isfile(path):
            raise ValueError("%s is missing (--wav-dir holds one <name>.wav per utterance)" % path)
        rate, data = wavfile.read(path)
        if fs is None and first is None:
            first = (path, rate)
        if first is not None and rate != first[1]:
            raise ValueError("%s is at %d Hz, but %s is at %d Hz: the wavs must share one rate"
                             % (path, rate, first[0], first[1]))
        if fs is not None and rate != fs:
            raise ValueError("%s is at %d Hz, but --fs=%d" % (path, rate, fs))
        if data.ndim != 1:
            raise ValueError("%s has %d channels; the analysis takes mono wavs" % (path, data.shape[1]))
        waves.append(data)
    return waves


def wav_stats(hp, waves, fs, batch_size, n, device):
    """FeatureStats.result() of the natural features analysed from the wavs (analysis.analyse), with gv in input order,
    and each utterance's DIO frame count.  The batches are generate.plan_batches' over the sample counts, so the means
    have the same bits for any batch size."""
    kind = "vc" if hp.name == "vc" else "tts_acoustic"
    fp = getattr(hp, "frame_period", FRAME_PERIOD)
    stats = FeatureStats(analysis.feature_width(kind, int(hp.order)), n, device)
    frames = np.zeros(len(waves), np.int64)
    plan = generate.plan_batches([len(w) for w in waves], batch_size)
    for idx in plan:
        mc, host, lengths = analysis.analyse([waves[i] for i in idx], fs, fp, int(hp.order), kind, device)
        stats.add(mc.float(), lengths)
        frames[idx] = host
    gv, gv_mean, ms_mean = stats.result()
    gv_in = np.empty_like(gv)
    gv_in[np.array([i for idx in plan for i in idx])] = gv
    return (gv_in, gv_mean, ms_mean), frames


def pad_batch(arrays, device):
    """(B, max length, D) float32 CUDA batch of (T_i, D) arrays, zero-padded."""
    xb = np.zeros((len(arrays), max(len(a) for a in arrays), arrays[0].shape[-1]), dtype=np.float32)
    for j, a in enumerate(arrays):
        xb[j, :len(a)] = a
    return torch.from_numpy(xb).to(device)


def split_stats(hp, generators, X, Y, batch_size, n, device):
    """[FeatureStats.result()] of the natural features (Y's static columns) and of each generator's (a
    generate.ParameterGenerator; X un-normalised inputs), with gv in input order.  Each batch of
    generate.plan_batches is copied to the device once, and the generated features never leave it."""
    cols, key = natural_columns(hp), FEATURES[hp.name]
    D = cols.stop - cols.start
    stats = [FeatureStats(D, n, device) for _ in range(1 + len(generators))]
    if generators:
        X = [generate.normalize_input(a, hp, generators[0].stats) for a in X]
    plan = generate.plan_batches([len(y) for y in Y], batch_size)
    for idx in plan:
        lengths = torch.tensor([len(Y[i]) for i in idx], dtype=torch.int64).to(device)
        stats[0].add(pad_batch([Y[i] for i in idx], device)[:, :, cols], lengths)
        if generators:
            x = pad_batch([X[i] for i in idx], device)
            for s, g in zip(stats[1:], generators):
                s.add(g.generate(x, lengths)[key], lengths)
    order = np.array([i for idx in plan for i in idx])
    out = []
    for s in stats:
        gv, gv_mean, ms_mean = s.result()
        gv_in = np.empty_like(gv)
        gv_in[order] = gv
        out.append((gv_in, gv_mean, ms_mean))
    return out


def split_arrays(labels, files, Y, ms_freq, results):
    """The arrays of <dst_dir>/<split>.npz: labels (natural first), names, lengths, ms_freq (K,), and per label
    (split_stats' results, in label order) gv (labels, U, D), gv_mean (labels, D), ms_mean (labels, K, D)."""
    return {"labels": np.array(labels), "names": np.array([splitext(basename(f))[0] for f in files]),
            "lengths": np.array([len(y) for y in Y], dtype=np.int64), "ms_freq": np.asarray(ms_freq, np.float64),
            "gv": np.stack([r[0] for r in results]), "gv_mean": np.stack([r[1] for r in results]),
            "ms_mean": np.stack([r[2] for r in results])}


def summary(labels, gv_mean, ms_mean, ref=0):
    """[(label, mean over columns of log10(gv_mean / the reference's), RMS over bins and columns of ms_mean - the
    reference's)] for every label after the reference labels[ref] (natural, or natural_wav at 1)."""
    rows = []
    for i in range(ref + 1, len(labels)):
        rows.append((labels[i], float(np.mean(np.log10(gv_mean[i] / gv_mean[ref]))),
                     float(np.sqrt(np.mean((ms_mean[i] - ms_mean[ref]) ** 2)))))
    return rows


def parse_args(argv=None):
    from compat.docopt import docopt
    return docopt(__doc__, argv=argv)


def main(argv=None, hp=None):
    """``hp``: the hyper-parameter object to use instead of ``getattr(hparams, --hparams_name)`` (``import hparams``
    from the caller's path otherwise); --hparams is parsed into it either way."""
    args = parse_args(argv)
    if hp is None:
        import hparams
        hp = getattr(hparams, args["--hparams_name"])
    hp.parse(args["--hparams"])
    mge_training = not args["--no-mge"]
    batch_size = int(args["--batch-size"]) if args["--batch-size"] is not None else int(hp.batch_size)
    checkpoints = args["<checkpoint>"]
    try:
        try:
            n, fs = int(args["--ms-fftlen"]), int(args["--fs"])
        except ValueError:
            raise ValueError("--ms-fftlen and --fs must be integers (got %r, %r)" % (args["--ms-fftlen"], args["--fs"]))
        if hp.name not in FEATURES:
            raise ValueError("hp.name %r: only vc and tts_acoustic generators are compared (the notebooks compute "
                             "neither global variances nor modulation spectra of durations)" % (hp.name,))
        generate.check_hparams(hp, mge_training)
        if batch_size < 1:
            raise ValueError("--batch-size must be >= 1 (got %d)" % batch_size)
        check_fftlen(n)
        if fs <= 0:
            raise ValueError("--fs must be > 0 (got %d)" % fs)
        ms_freq = modulation_frequencies(n, fs, getattr(hp, "frame_period", FRAME_PERIOD))
        wav_dir = args["--wav-dir"]
        labels = (["natural"] + (["natural_wav"] if wav_dir else [])
                  + check_labels(args["--labels"], checkpoints, wavs=bool(wav_dir)))
        inputs_dir, outputs_dir, dst_dir = args["<inputs_dir>"], args["<outputs_dir>"], args["<dst_dir>"]
        splits = []
        for sub, xf, yf in paired_files(inputs_dir, outputs_dir):
            X, Y = [np.load(f) for f in xf], [np.load(f) for f in yf]
            check_frames(xf, X, Y)
            splits.append((sub, xf, X, Y, read_wavs(wav_dir, xf, fs) if wav_dir else None))
        if wav_dir:
            kind = "vc" if hp.name == "vc" else "tts_acoustic"
            cols = natural_columns(hp)
            if analysis.feature_width(kind, int(hp.order)) != cols.stop - cols.start:
                raise ValueError("hp.order = %d gives %d analysed columns, but the prepared targets have %d"
                                 % (hp.order, analysis.feature_width(kind, int(hp.order)), cols.stop - cols.start))
    except ValueError as e:
        raise SystemExit("gantts_b200.objective: %s" % e)
    if not torch.cuda.is_available():
        raise SystemExit("gantts_b200.objective: needs a CUDA device (there is no CPU path)")
    device = torch.device("cuda")

    stats = generate.load_stats(hp, abspath(join(inputs_dir, os.pardir)))
    generate.derive_dims(hp, stats)
    generators = []
    for c in checkpoints:
        model_g = getattr(models, hp.generator)(**hp.generator_params)
        train.load_checkpoint(model_g, c)
        generators.append(generate.ParameterGenerator(model_g.to(device), hp, stats, mge_training))

    os.makedirs(dst_dir, exist_ok=True)
    for sub, xf, X, Y, waves in splits:
        results = split_stats(hp, generators, X, Y, batch_size, n, device)
        if waves is not None:
            wav_result, wav_frames = wav_stats(hp, waves, fs, batch_size, n, device)
            results.insert(1, wav_result)
        arrays = split_arrays(labels, xf, Y, ms_freq, results)
        if waves is not None:
            arrays["wav_lengths"] = wav_frames
        path = join(dst_dir, sub + ".npz")
        np.savez(path, **arrays)
        print(path)
        for ref in ((0, 1) if waves is not None else (0,)):
            for label, gv_ratio, ms_rms in summary(labels, arrays["gv_mean"], arrays["ms_mean"], ref):
                print("%s %s: mean log10 GV ratio to %s %+.4f, RMS log MS difference to %s %.4f"
                      % (sub, label, labels[ref], gv_ratio, labels[ref], ms_rms))
    return 0


if __name__ == "__main__":
    sys.exit(main())
