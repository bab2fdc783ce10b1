"""WORLD analysis of natural waveforms on the device, as the reference notebooks compute their natural features:
compute_static_features (Test VC.ipynb, Test RNN VC.ipynb) and compute_mgc_from_waveform (Test TTS.ipynb).

    f0, timeaxis = pyworld.dio(x, fs, frame_period=hp.frame_period)
    f0 = pyworld.stonemask(x, f0, timeaxis, fs)
    spectrogram = pyworld.cheaptrick(x, f0, timeaxis, fs)
    mc = pysptk.sp2mc(spectrogram, order=hp.order, alpha=pysptk.util.mcepalpha(fs))
    vc:           mc[:, 1:]
    tts_acoustic: P.modspec_smoothing(mc, fs / int(fs * hp.frame_period * 0.001), cutoff=50)

x is the wav's int16 samples cast to float64, unscaled, as the notebooks read them.  The notebooks also run pyworld.d4c
and discard it; it is not computed here."""
import numpy as np
import torch

from . import generate
from . import ops

SMOOTHING_N = 4096          # modspec_smoothing's default n
SMOOTHING_CUTOFF = 50.0     # the notebook's cutoff, Hz of modulation frequency
KINDS = ("vc", "tts_acoustic")


def modulation_rate(fs, frame_period):
    """modfs of compute_mgc_from_waveform: fs / int(fs * frame_period * 0.001), frames per second."""
    return fs / int(fs * (frame_period * 0.001))


def feature_width(kind, order):
    return order if kind == "vc" else order + 1


def pad_waves(waves, device):
    """(B, S) float64 CUDA batch of 1-D sample arrays, zero-padded, and their lengths (int64 CUDA)."""
    S = max(max(len(w) for w in waves), 1)
    xb = np.zeros((len(waves), S), dtype=np.float64)
    for i, w in enumerate(waves):
        xb[i, :len(w)] = w
    return (torch.from_numpy(xb).to(device),
            torch.tensor([len(w) for w in waves], dtype=torch.int64).to(device))


def analyse(waves, fs, frame_period, order, kind, device):
    """The natural features of a batch of waveforms (1-D arrays of samples, any dtype, cast to float64): returns (mc
    (B, T, D) float64 CUDA, 0 beyond each row's frames, D = order for vc and order + 1 for tts_acoustic; frame counts as
    a host int64 array; the same counts as int64 CUDA).  The read of the frame counts and the status word after the last
    kernel is the one host synchronisation; RuntimeError names the rule a row broke."""
    x, lengths = pad_waves([np.asarray(w).astype(np.float64) for w in waves], device)
    return analyse_batch(x, lengths, fs, frame_period, order, kind)


def analyse_batch(x, lengths, fs, frame_period, order, kind):
    """analyse on a padded device batch: x (B, S) float64 CUDA samples, lengths int64 CUDA (B,)."""
    if kind not in KINDS:
        raise ValueError("kind must be one of %s (got %r)" % (", ".join(KINDS), kind))
    T = ops.world_dio_frames(x.shape[1], fs, frame_period)
    if kind == "tts_acoustic" and T > SMOOTHING_N:
        raise ValueError("modspec_smoothing is defined for at most %d frames; the longest utterance has %d"
                         % (SMOOTHING_N, T))
    f0, info = ops.world_dio(x, lengths, fs, frame_period)
    f0 = ops.world_stonemask(x, lengths, f0, info, fs, frame_period)
    sp = ops.world_cheaptrick(x, lengths, f0, info, fs, frame_period, generate.cheaptrick_fft_size(fs))
    frames = info[:-1]
    mc = ops.sp2mc(sp, frames, order, generate.mcep_alpha(fs))
    if kind == "vc":
        mc = mc[:, :, 1:]
    else:
        mc = ops.modspec_smoothing(mc, frames, modulation_rate(fs, frame_period), SMOOTHING_N, SMOOTHING_CUTOFF)
    host = ops.world_analysis_check(info)
    return mc, host, frames
