# coding: utf-8
"""Convert the source speaker's wavs with a trained VC generator and the difference MLSA filter.

usage: convert.py [options] <checkpoint> <data_dir> <wav_dir> <outputs_dir>

options:
    --hparams=<parmas>          Hyper parameters to be overrided [default: ].
    --batch-size=<N>            Utterances per batch (default: hp.batch_size).
    --diffvc                    Enable DIFF VC (required: the only mode converted here).
    -h, --help                  Show this help message and exit
"""
# evaluation_vc.py's test_vc_from_path(model, x, fs, data_mean, data_std, diffvc=True) (:40-110) for a padded batch of
# source wavs, on the device: WORLD analysis (analysis.analyse_batch), the delta features and their scaling
# (gantts_vc_inputs), the generator and its parameter generation (generate.ParameterGenerator), the difference filter's
# coefficients (gantts_mc2b) and the MLSA filtering of the source samples (gantts_mlsa_filter).  Each row gets what the
# script computes for that utterance alone.  The command writes <outputs_dir>/{eval,test}/<name>.wav as
# evaluation_vc.py --diffvc does (:132-177).
import os
import sys
from os.path import basename, join, splitext

import numpy as np
import torch

from . import analysis
from . import generate
from . import models
from . import objective
from . import ops
from . import train

FRAME_PERIOD = objective.FRAME_PERIOD
NO_DIFFVC = ("--diffvc is required: without it evaluation_vc.py resynthesises the converted features with WORLD, which "
             "needs D4C aperiodicity, and this package does not compute D4C")


class VoiceConverter(object):
    """A trained VC generator (``hparams.vc``) and the difference MLSA filter at sampling rate ``fs``; ``stats`` as
    generate.load_stats returns them."""

    def __init__(self, model_g, hp, stats, fs):
        if hp.name != "vc":
            raise ValueError("VoiceConverter needs the vc hyper parameters (got %r)" % (hp.name,))
        self.gen = generate.ParameterGenerator(model_g, hp, stats)
        self.hp, self.fs, self.order = hp, int(fs), int(hp.order)
        self.frame_period = float(getattr(hp, "frame_period", FRAME_PERIOD))
        self.hop = int(self.fs * (self.frame_period * 0.001))          # evaluation_vc.py:43
        self.alpha = generate.mcep_alpha(self.fs)
        self.windows = ops.windows_key(hp.windows)
        self.device = self.gen.device
        mean = np.asarray(stats["data_mean"], dtype=np.float64).reshape(-1)
        std = np.asarray(stats["data_std"], dtype=np.float64).reshape(-1)
        if mean.size != len(self.windows) * self.order:
            raise ValueError("the statistics have %d columns; hp.order = %d with %d windows needs %d"
                             % (mean.size, self.order, len(self.windows), len(self.windows) * self.order))
        self.mean = torch.from_numpy(mean).to(self.device)
        self.std = torch.from_numpy(std).to(self.device)

    def analyse(self, x, lengths):
        """The smoothed source mel-cepstra without c0, (B, T, order) float64 CUDA (a view), and the frame counts (host
        int64, CUDA int64).  test_vc_from_path smooths mc[:, 1:]; the smoothing treats each column on its own, so the
        smoothed (order + 1)-column chain of analysis without its column 0 has the same bits."""
        mc, host, frames = analysis.analyse_batch(x, lengths, self.fs, self.frame_period, self.order, "tts_acoustic")
        return mc[:, :, 1:], host, frames

    def convert(self, x, lengths):
        """x: (B, S) float64 CUDA source samples (int16 values, unscaled), zero-padded; lengths: int64 CUDA (B,).
        Returns {"waveform": (B, S) float64, 0 beyond each row's samples; "mc": (B, T, order) float32, the de-normalised
        converted statics (test_vc_from_path's outputs), 0 beyond each row's frames; "frames": host int64 (B,)}.  The
        analysis' read of the frame counts and its status word is the one host synchronisation; RuntimeError names the
        rule a row broke."""
        src, host, frames = self.analyse(x, lengths)
        xin, static = ops.vc_inputs(src, frames, self.windows, self.mean, self.std)
        pred = self.gen.generate(xin, frames)["mc"]
        b = ops.mc2b(pred, static, frames, self.alpha)
        y = ops.mlsa_filter(x, lengths, b, frames, self.alpha, self.hop)
        return {"waveform": y, "mc": pred, "frames": host}

    def convert_utterances(self, waves, batch_size, names=None):
        """1-D sample arrays (cast to float64) -> one {"waveform": float64 (S_i,), "mc": float32 (T_i, order)} per
        utterance, in input order.  The utterances are batched by generate.plan_batches over their sample counts; each
        result equals that utterance converted alone.  RuntimeError names the utterance (``names[i]``, or its index) that
        WORLD analysis refuses: too short for DIO, or with a sample that is not finite."""
        waves = [np.asarray(w).astype(np.float64) for w in waves]
        results = [None] * len(waves)
        for idx in generate.plan_batches([len(w) for w in waves], batch_size):
            x, lengths = analysis.pad_waves([waves[i] for i in idx], self.device)
            try:
                out = self.convert(x, lengths)
            except RuntimeError as e:
                raise self._name_refusal([waves[i] for i in idx], [i if names is None else names[i] for i in idx], e)
            y, mc = out["waveform"].cpu().numpy(), out["mc"].cpu().numpy()
            for j, i in enumerate(idx):
                results[i] = {"waveform": y[j, :len(waves[i])].copy(), "mc": mc[j, :out["frames"][j]].copy()}
        return results

    def _name_refusal(self, waves, names, err):
        """The batch's analysis refused a row: find it by analysing each utterance alone."""
        for w, name in zip(waves, names):
            try:
                x, lengths = analysis.pad_waves([w], self.device)
                self.analyse(x, lengths)
            except RuntimeError as e:
                return RuntimeError("utterance %s: %s" % (name, e))
        return err


# ---- the command (evaluation_vc.py:132-177) ----

def wav_files(data_dir, wav_dir):
    """[("eval", wavs), ("test", wavs)]: get_wav_files (evaluation_vc.py:121-129) of the evaluation split and the five
    held-out utterances of <data_dir>/X."""
    xd = join(data_dir, "X")
    as_wav = lambda files: [join(wav_dir, splitext(basename(f))[0] + ".wav") for f in files]
    return [("eval", as_wav(train.npy_files(xd, train=False))), ("test", as_wav(train.npy_files(xd, test=True)))]


def read_sources(wav_dir, files, frame_period):
    """(waves, fs) of the wavs, read as evaluation_vc.py reads them; ValueError naming the wav that is missing, not mono,
    at another rate than the first, or longer than modspec_smoothing's frames allow."""
    from scipy.io import wavfile
    waves = objective.read_wavs(wav_dir, files)
    fs = wavfile.read(files[0])[0] if files else 16000
    for f, w in zip(files, waves):
        T = ops.world_dio_frames(len(w), fs, frame_period)
        if T > analysis.SMOOTHING_N:
            raise ValueError("%s has %d frames; modspec_smoothing is defined for at most %d (%.2f s at %g ms)"
                             % (f, T, analysis.SMOOTHING_N, analysis.SMOOTHING_N * frame_period / 1000.0,
                                frame_period))
    return waves, fs


def parse_args(argv=None):
    from compat.docopt import docopt
    return docopt(__doc__, argv=argv)


def main(argv=None, hp=None):
    """``hp``: the hyper-parameter object to use instead of ``hparams.vc`` (``import hparams`` from the caller's path
    otherwise); --hparams is parsed into it either way."""
    args = parse_args(argv)
    if not args["--diffvc"]:
        raise SystemExit("gantts_b200.convert: " + NO_DIFFVC)
    if hp is None:
        import hparams
        hp = hparams.vc
    hp.parse(args["--hparams"])
    batch_size = int(args["--batch-size"]) if args["--batch-size"] is not None else int(hp.batch_size)
    try:
        generate.check_hparams(hp)
        if hp.name != "vc":
            raise ValueError("the vc hyper parameters are required (got %r)" % (hp.name,))
        if batch_size < 1:
            raise ValueError("--batch-size must be >= 1 (got %d)" % batch_size)
    except ValueError as e:
        raise SystemExit("gantts_b200.convert: %s" % e)
    checkpoint_path, data_dir, wav_dir, outputs_dir = (args["<checkpoint>"], args["<data_dir>"], args["<wav_dir>"],
                                                       args["<outputs_dir>"])
    splits = wav_files(data_dir, wav_dir)
    frame_period = float(getattr(hp, "frame_period", FRAME_PERIOD))
    try:
        waves, fs = read_sources(wav_dir, [p for _, files in splits for p in files], frame_period)
    except ValueError as e:
        raise SystemExit("gantts_b200.convert: %s" % e)
    if not torch.cuda.is_available():
        raise SystemExit("gantts_b200.convert: needs a CUDA device (there is no CPU path)")
    device = torch.device("cuda")

    stats = generate.load_stats(hp, data_dir)
    generate.derive_dims(hp, stats)
    model_g = getattr(models, hp.generator)(**hp.generator_params)
    train.load_checkpoint(model_g, checkpoint_path)
    conv = VoiceConverter(model_g.to(device), hp, stats, fs)

    start = 0
    for sub, files in splits:
        out_dir = join(outputs_dir, sub)
        os.makedirs(out_dir, exist_ok=True)
        try:
            results = conv.convert_utterances(waves[start:start + len(files)], batch_size, names=files)
        except RuntimeError as e:
            raise SystemExit("gantts_b200.convert: %s" % e)
        start += len(files)
        from scipy.io import wavfile
        for path, r in zip(files, results):
            dst = join(out_dir, splitext(basename(path))[0] + ".wav")
            wavfile.write(dst, fs, r["waveform"].astype(np.int16))
            print(dst)
    return 0


if __name__ == "__main__":
    sys.exit(main())
