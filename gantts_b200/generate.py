# coding: utf-8
"""Generate acoustic features from a trained generator, a batch of utterances per device pass.

usage: generate.py [options] <checkpoint> <inputs_dir> <dst_dir>

options:
    --hparams_name=<name>       Name of hyper params: vc, tts_acoustic or tts_duration [default: vc].
    --hparams=<parmas>          Hyper parameters to be overrided [default: ].
    --batch-size=<N>            Utterances per batch (default: hp.batch_size).
    --no-mge                    tts_acoustic: the generator was trained without MGE (de-normalise, then MLPG with the
                                variances of the statistics).
    --fs=<fs>                   Sampling frequency [default: 16000].
    --post-filter               tts_acoustic: apply Merlin's post filter to spectral features.
    --spectrogram               tts_acoustic: also write the power spectral envelope "sp" (mc2sp of mgc).
    -h, --help                  Show this help message and exit
"""
# The parameter generation of the reference's evaluation scripts (evaluation_vc.py:40-91, evaluation_tts.py:50-176) for a
# padded batch of any lengths: each utterance gets exactly what those scripts compute for it alone at B = 1 and T = its own
# length.  The length-exact pieces are the device kernels gantts_mlpg_ragged (MLPG over each row's own frames) and
# gantts_sru_fwd_lengths (SRU whose reverse direction starts at each row's last frame); the LSTM stacks already run on
# lengths and the MLP layers frame by frame.  Under tts_acoustic, gen_waveform's spectral steps (evaluation_tts.py:112-115:
# merlin_post_filter, mc2sp) run on the device too (gantts_mcep_postfilter, gantts_mcep_to_sp).  The command writes
# <dst_dir>/{eval,test}/<name>.npz, no audio: WORLD synthesis and decode_aperiodicity are not done here.
import os
import sys
from os.path import abspath, basename, join, splitext

import numpy as np
import torch

from . import _lib
from . import models
from . import multistream
from . import ops
from . import train

LSTM_MAX_B = 128            # sequences per call of the LSTM recurrence kernels (csrc/lstm.cu LSTM_MAX_B)
HIGHWAY_GENERATORS = ("In2OutHighwayNet", "In2OutRNNHighwayNet")
OUTPUT_NAMES = {"vc": ("mc",), "acoustic": ("mgc", "lf0", "vuv", "bap", "f0"), "duration": ("duration",)}
SPECTROGRAM_NAME = "sp"     # the extra acoustic output of spectrogram=True, after OUTPUT_NAMES["acoustic"]
POSTFILTER_COEF = 1.4       # gen_waveform's coef (evaluation_tts.py:103)
MAX_FFTLEN = 4096           # gantts_mcep_to_sp's largest FFT


# ---- statistics and input normalisation (evaluation_vc.py:61,142-144; evaluation_tts.py:153-156,210-212) ----

def _ty(hp):
    return "acoustic" if hp.name == "acoustic" else "duration"


def load_stats(hp, data_dir):
    """The statistics gantts_b200.train saved in data_dir (the parent of the inputs directory, train.load_data):
    vc {"data_mean", "data_std"}; TTS {"X_min", "X_max", "Y_mean", "Y_std"} of the acoustic or duration model."""
    if hp.name == "vc":
        return {"data_mean": np.load(join(data_dir, "data_mean.npy")),
                "data_std": np.sqrt(np.load(join(data_dir, "data_var.npy")))}
    ty = _ty(hp)
    return {"X_min": np.load(join(data_dir, "X_{}_data_min.npy".format(ty))),
            "X_max": np.load(join(data_dir, "X_{}_data_max.npy".format(ty))),
            "Y_mean": np.load(join(data_dir, "Y_{}_data_mean.npy".format(ty))),
            "Y_std": np.sqrt(np.load(join(data_dir, "Y_{}_data_var.npy".format(ty))))}


def output_stats(hp, stats):
    """(mean, std) of the generator's output columns."""
    if hp.name == "vc":
        return stats["data_mean"], stats["data_std"]
    return stats["Y_mean"], stats["Y_std"]


def normalize_input(x, hp, stats):
    """An utterance's input features as the evaluation scripts feed them to the generator, float32: vc
    P.scale(x, data_mean, data_std) = (x - mean) / std; TTS P.minmax_scale(x, X_min, X_max, feature_range=(0.01, 0.99))."""
    x = np.asarray(x)
    if hp.name == "vc":
        return ((x - stats["data_mean"]) / stats["data_std"]).astype(np.float32)
    min_, scale_ = train.minmax_scale_params(stats["X_min"], stats["X_max"])
    return (x * scale_ + min_).astype(np.float32)


def derive_dims(hp, stats):
    """in_dim / out_dim left None in the hparams, from the statistics (evaluation_vc.py:146-149, train.py:753-768)."""
    if hp.name == "vc":
        for k in ("in_dim", "out_dim"):
            if hp.generator_params[k] is None:
                hp.generator_params[k] = stats["data_mean"].shape[-1]
    else:
        train.derive_tts_dims(hp, stats["X_min"].shape[-1], stats["Y_mean"].shape[-1])


def mcep_alpha(fs):
    """pysptk.util.mcepalpha(fs) (evaluation_tts.py:105): the all-pass constant in arange(0, 1, 0.001) whose warped
    frequency axis is closest, in mean squared distance over 1000 points, to the mel scale on [0, fs/2)."""
    n = 1000
    mel = np.log1p((fs / 2.0) / n * np.arange(n) / 1000.0) * (1000.0 / np.log(2.0))
    mel /= mel[-1]
    alphas = np.arange(0.0, 1.0, 0.001)[:, None]
    omega = np.pi / n * np.arange(n)[None, :]
    warp = np.arctan((1 - alphas * alphas) * np.sin(omega) / ((1 + alphas * alphas) * np.cos(omega) - 2 * alphas))
    warp = np.where(warp < 0, warp + np.pi, warp)
    warp /= warp[:, -1:]
    return float(alphas[int(np.argmin(np.sum((mel - warp) ** 2, axis=1) / n)), 0])


def cheaptrick_fft_size(fs):
    """pyworld.get_cheaptrick_fft_size(fs) (evaluation_tts.py:106) at its default F0 floor of 71 Hz."""
    return 2 ** (1 + int(np.floor(np.log2(3.0 * fs / 71.0 + 1.0))))


def check_hparams(hp, mge_training=True, post_filter=False, spectrogram=False, fs=16000):
    """The configurations the evaluation scripts can run; raises ValueError naming the rule otherwise."""
    if hp.name not in OUTPUT_NAMES:
        raise ValueError("hp.name must be vc, acoustic or duration (got %r)" % (hp.name,))
    if hp.generator_add_noise:
        raise ValueError("hp.generator_add_noise=True (generator noise) is not supported")
    if hp.name != "vc" and hp.generator in HIGHWAY_GENERATORS:
        raise ValueError("%s runs its MLPG inside forward and cannot generate under the TTS hparams "
                         "(evaluation_tts.py calls the generator as model(x, lengths))" % hp.generator)
    if not mge_training and hp.name != "acoustic":
        raise ValueError("--no-mge applies to tts_acoustic only")
    for on, flag in ((post_filter, "--post-filter"), (spectrogram, "--spectrogram")):
        if on and hp.name != "acoustic":
            raise ValueError("%s applies to tts_acoustic only: it works on the generated mgc, which vc and duration "
                             "models do not produce" % flag)
    if fs <= 0:
        raise ValueError("--fs must be > 0 (got %d)" % fs)
    if spectrogram and cheaptrick_fft_size(fs) > MAX_FFTLEN:
        raise ValueError("--fs=%d needs a %d-point FFT; at most %d points are supported"
                         % (fs, cheaptrick_fft_size(fs), MAX_FFTLEN))


def plan_batches(lengths, batch_size, max_b=LSTM_MAX_B):
    """Indices of the utterances in batches of at most min(batch_size, max_b), longest first (ties in input order)."""
    if batch_size < 1:
        raise ValueError("batch size must be >= 1 (got %d)" % batch_size)
    order = sorted(range(len(lengths)), key=lambda i: (-int(lengths[i]), i))
    bs = min(int(batch_size), int(max_b))
    return [order[i:i + bs] for i in range(0, len(order), bs)]


class ParameterGenerator(object):
    """A trained generator in eval mode and the parameter generation of the evaluation scripts after it, on a padded
    device batch.  ``stats`` as ``load_stats`` returns them; ``mge_training`` picks gen_parameters' branch for
    tts_acoustic (evaluation_tts.py:64-98).  tts_acoustic only: ``post_filter`` replaces mgc with Merlin's post filter of
    it and ``spectrogram`` adds its power spectral envelope "sp", at the all-pass constant and FFT size of ``fs``
    (gen_waveform, evaluation_tts.py:103-115)."""

    def __init__(self, model_g, hp, stats, mge_training=True, post_filter=False, spectrogram=False, fs=16000):
        check_hparams(hp, mge_training, post_filter, spectrogram, fs)
        self.model, self.hp, self.stats, self.kind = model_g.eval(), hp, stats, hp.name
        self.post_filter, self.spectrogram = bool(post_filter), bool(spectrogram)
        if self.post_filter or self.spectrogram:
            self.alpha, self.fftlen = mcep_alpha(fs), cheaptrick_fft_size(fs)
        self.device = next(model_g.parameters()).device
        if self.device.type != "cuda":
            raise RuntimeError("gantts_b200: ParameterGenerator needs the generator on a CUDA device")
        self.windows = ops.windows_key(hp.windows)
        self.highway = model_g.include_parameter_generation()
        mean, std = output_stats(hp, stats)
        mean, std = np.asarray(mean, dtype=np.float64), np.asarray(std, dtype=np.float64)
        f32 = lambda a: torch.as_tensor(np.ascontiguousarray(a), dtype=torch.float32, device=self.device)
        self.var = self.in_affine = self.out_affine = None
        if self.highway:
            # x_s + Tx * MLPG(h) over the unit-variance solve of the static_dim columns, then inv_scale
            # (evaluation_vc.py:77,88-89)
            S = model_g.static_dim
            self.entries, self.ncols = [(0, S, True, 0)], S
            self.std_s, self.mean_s = f32(std[:S]), f32(mean[:S])
            return
        nw = len(hp.windows)
        streams = [True] * len(hp.stream_sizes)
        self.entries, self.ncols = multistream.mlpg_stream_entries(hp.stream_sizes, hp.has_dynamic_features, streams,
                                                                   nw)
        static_cols = multistream.static_feature_columns(nw, hp.stream_sizes, hp.has_dynamic_features, streams)
        if mge_training:
            # unit-variance MLPG on the normalised features, de-normalised after it (evaluation_tts.py:71-83,171;
            # evaluation_vc.py:82-89)
            self.out_affine = (f32(std[static_cols]), f32(mean[static_cols]))
        else:
            # de-normalised first, then MLPG with Y_var = Y_std ** 2 (evaluation_tts.py:86-98)
            self.in_affine = (f32(std), f32(mean))
            self.var = f32(std * std)

    def _generator_output(self, x, lengths):
        m = self.model
        if isinstance(m, models.SRURNN):
            h = m.gru(x, engine=m.engine, lengths=lengths)
            act = _lib.ACT_SIGMOID if m.last_sigmoid else _lib.ACT_NONE
            return ops.linear_act(h, m.hidden2out.weight, m.hidden2out.bias, act, engine=m.engine)
        return m(x, lengths)

    def _highway(self, x, lengths):
        from . import rnn
        m, S = self.model, self.model.static_dim
        x_s = x[:, :, :S]
        Tx = ops.linear_act(x_s, m.T.weight, m.T.bias, _lib.ACT_SIGMOID, engine=m.engine)
        if isinstance(m, models.In2OutHighwayNet):
            h = models._mlp(x, m.H, m.last_linear, m.dropout_p, False, _lib.ACT_NONE, m.engine)
        else:
            h = rnn.lstm_forward(m.lstm, x, lengths, False, m.engine)
            h = ops.linear_act(h, m.hidden2out.weight, m.hidden2out.bias, _lib.ACT_NONE, engine=m.engine)
        Gx = ops.mlpg_ragged(h, lengths, self.windows, self.entries, self.ncols)
        return torch.addcmul(self.mean_s, ops.highway_combine(x_s, Tx, Gx), self.std_s)

    def generate(self, x, lengths):
        """x: (B, T, D) normalised inputs (normalize_input), zero-padded, CUDA float32; lengths: int64 CUDA (B,).
        Returns {name: CUDA float32 tensor (B, T, ...)} with the names of OUTPUT_NAMES[hp.name] -- vc "mc"; acoustic
        "mgc", "lf0", "vuv" (B, T), "bap", "f0", with spectrogram also "sp" (B, T, fftlen/2 + 1); duration "duration" --
        de-normalised (mgc post-filtered under post_filter).  Frame t of row b is what the
        evaluation scripts compute for that utterance alone for t < lengths[b]; later frames are not part of the result.
        No host synchronisation."""
        ops.require_cuda(x)
        if x.dim() != 3 or lengths.dim() != 1 or lengths.numel() != x.shape[0]:
            raise RuntimeError("gantts_b200: generate needs x (B, T, D) and lengths (B,)")
        if x.shape[0] > LSTM_MAX_B:
            raise RuntimeError("gantts_b200: at most %d utterances per batch (LSTM_MAX_B)" % LSTM_MAX_B)
        with torch.no_grad():
            if self.highway:
                return {"mc": self._highway(x, lengths)}
            y = ops.mlpg_ragged(self._generator_output(x, lengths), lengths, self.windows, self.entries, self.ncols,
                                var=self.var, in_affine=self.in_affine, out_affine=self.out_affine)
            if self.kind == "vc":
                return {"mc": y}
            if self.kind == "duration":
                d = torch.round(y)                                  # evaluation_tts.py:172-176
                return {"duration": torch.where(d <= 0, torch.ones_like(d), d)}
            (_, _, _, o_lf0), (_, _, _, o_vuv), (_, _, _, o_bap) = self.entries[1:4]
            mgc, lf0, vuv, bap = y[:, :, :o_lf0], y[:, :, o_lf0:o_vuv], y[:, :, o_vuv], y[:, :, o_bap:]
            # gen_waveform (evaluation_tts.py:117-119): f0 = lf0, 0 where vuv < 0.5, exp of the nonzero values (a voiced
            # frame whose lf0 is exactly 0 stays 0)
            voiced = ~(vuv < 0.5).unsqueeze(-1) & (lf0 != 0)
            f0 = torch.where(voiced, torch.exp(lf0), torch.zeros_like(lf0))
            if self.post_filter:                                # evaluation_tts.py:112-113
                mgc = ops.mcep_postfilter(mgc, lengths, self.alpha, POSTFILTER_COEF)
            out = {"mgc": mgc, "lf0": lf0, "vuv": vuv, "bap": bap, "f0": f0}
            if self.spectrogram:                                # :115
                out[SPECTROGRAM_NAME] = ops.mc2sp(mgc, lengths, self.alpha, self.fftlen)
            return out

    def generate_utterances(self, arrays, batch_size):
        """Un-normalised input feature arrays (T_i, D) -> one dict of float32 numpy arrays of T_i frames per utterance,
        in input order, with the keys ``generate`` returns.  The utterances are sorted by length and batched
        (plan_batches); each batch makes one host-to-device and one device-to-host copy."""
        arrays = [normalize_input(a, self.hp, self.stats) for a in arrays]
        results = [None] * len(arrays)
        for idx in plan_batches([len(a) for a in arrays], batch_size):
            lens = [len(arrays[i]) for i in idx]
            T = max(lens)
            xb = np.zeros((len(idx), T, arrays[idx[0]].shape[-1]), dtype=np.float32)
            for j, i in enumerate(idx):
                xb[j, :lens[j]] = arrays[i]
            x = torch.from_numpy(xb).to(self.device)
            lengths = torch.tensor(lens, dtype=torch.int64).to(self.device)
            out = self.generate(x, lengths)
            names = list(out)
            widths = [1 if out[k].dim() == 2 else out[k].shape[-1] for k in names]
            host = torch.cat([out[k].reshape(len(idx), T, -1) for k in names], -1).cpu().numpy()
            for j, i in enumerate(idx):
                r, c = {}, 0
                for k, w in zip(names, widths):
                    a = host[j, :lens[j], c:c + w]
                    r[k] = np.ascontiguousarray(a[:, 0] if out[k].dim() == 2 else a)
                    c += w
                results[i] = r
        return results


# ---- the command (evaluation_vc.py:132-177 without the vocoder) ----

def utterance_files(inputs_dir):
    """[("eval", files), ("test", files)]: the evaluation split of the training command and its five held-out utterances
    (evaluation_vc.py:121-129,165-166 through train.py's NPYDataSource)."""
    return [("eval", train.npy_files(inputs_dir, train=False)), ("test", train.npy_files(inputs_dir, test=True))]


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
    post_filter, spectrogram = bool(args["--post-filter"]), bool(args["--spectrogram"])
    try:
        fs = int(args["--fs"])
    except ValueError:
        raise SystemExit("gantts_b200.generate: --fs must be an integer sampling frequency (got %r)" % args["--fs"])
    try:
        check_hparams(hp, mge_training, post_filter, spectrogram, fs)
        if batch_size < 1:
            raise ValueError("--batch-size must be >= 1 (got %d)" % batch_size)
    except ValueError as e:
        raise SystemExit("gantts_b200.generate: %s" % e)
    if not torch.cuda.is_available():
        raise SystemExit("gantts_b200.generate: needs a CUDA device (there is no CPU path)")
    device = torch.device("cuda")
    checkpoint_path, inputs_dir, dst_dir = args["<checkpoint>"], args["<inputs_dir>"], args["<dst_dir>"]

    stats = load_stats(hp, abspath(join(inputs_dir, os.pardir)))
    derive_dims(hp, stats)
    model_g = getattr(models, hp.generator)(**hp.generator_params)
    train.load_checkpoint(model_g, checkpoint_path)
    gen = ParameterGenerator(model_g.to(device), hp, stats, mge_training, post_filter, spectrogram, fs)

    for sub, files in utterance_files(inputs_dir):
        out_dir = join(dst_dir, sub)
        os.makedirs(out_dir, exist_ok=True)
        results = gen.generate_utterances([np.load(f) for f in files], batch_size)
        for f, r in zip(files, results):
            path = join(out_dir, splitext(basename(f))[0] + ".npz")
            np.savez(path, **r)
            print(path)
    return 0


if __name__ == "__main__":
    sys.exit(main())
