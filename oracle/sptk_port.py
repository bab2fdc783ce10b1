"""CPU restatement of the spectral post-processing of reference evaluation_tts.py:103-115 (gen_waveform):
``nnmnkwii.postfilters.merlin_post_filter``, ``pysptk.mc2sp``, ``pysptk.util.mcepalpha`` and
``pyworld.get_cheaptrick_fft_size``.  TEST INFRASTRUCTURE ONLY.

pysptk, nnmnkwii and pyworld are third-party packages the reference does not vendor, so this is written from their
published definitions (SPTK's freqt / c2acr / mc2b / b2mc recursions, Merlin's formant enhancement): **parity unpinned**
against those packages.  It runs the literal chain -- freqt, FFT, c2acr, mc2b, b2mc -- and shares no code with the
product's operator builder (gantts_mcep_operator).  Every function takes one frame (M+1,) or a stack of frames (N, M+1)
and applies the per-frame chain to each frame (vectorised over frames only).
"""
import numpy as np


def freqt(c, m2, a):
    """SPTK freqt: the order-m2 cepstrum of the all-pass warp with parameter a of c (frames on the leading axes)."""
    c = np.asarray(c, dtype=np.float64)
    m1 = c.shape[-1] - 1
    b = 1.0 - a * a
    g = np.zeros(c.shape[:-1] + (m2 + 1,))
    for i in range(m1, -1, -1):
        d = g.copy()
        g[..., 0] = c[..., i] + a * d[..., 0]
        if m2 >= 1:
            g[..., 1] = b * d[..., 0] + a * d[..., 1]
        for j in range(2, m2 + 1):
            g[..., j] = d[..., j - 1] + a * (d[..., j] - g[..., j - 1])
    return g


def c2acr0(c, n):
    """c2acr(c, 0, n): the zeroth autocorrelation (1/n) sum_k exp(2 Re FFT_n(c zero-padded)[k])."""
    c = np.asarray(c, dtype=np.float64)
    x = np.zeros(c.shape[:-1] + (n,))
    x[..., :c.shape[-1]] = c
    return np.sum(np.exp(2.0 * np.fft.fft(x, axis=-1).real), axis=-1) / n


def mc2b(mc, alpha):
    b = np.array(mc, dtype=np.float64)
    for m in range(b.shape[-1] - 2, -1, -1):
        b[..., m] = b[..., m] - alpha * b[..., m + 1]
    return b


def b2mc(b, alpha):
    b = np.asarray(b, dtype=np.float64)
    mc = b.copy()
    for m in range(b.shape[-1] - 2, -1, -1):
        mc[..., m] = b[..., m] + alpha * b[..., m + 1]
    return mc


def merlin_post_filter(mgc, alpha, minimum_phase_order=511, fftlen=1024, coef=1.4):
    """nnmnkwii.postfilters.merlin_post_filter: weight the cepstrum from index 2 on by coef and restore the frame's
    energy r0 through c0 of the b coefficients."""
    mgc = np.asarray(mgc, dtype=np.float64)
    w = np.full(mgc.shape[-1], float(coef))
    w[:2] = 1.0
    r0 = c2acr0(freqt(mgc, minimum_phase_order, -alpha), fftlen)
    r0p = c2acr0(freqt(w * mgc, minimum_phase_order, -alpha), fftlen)
    b = mc2b(w * mgc, alpha)
    b[..., 0] += 0.5 * np.log(r0 / r0p)
    return b2mc(b, alpha)


def mc2sp(mc, alpha, fftlen):
    """pysptk.mc2sp: the power spectrum (fftlen/2 + 1 bins) of a mel-cepstrum."""
    c = freqt(mc, fftlen // 2, -alpha)
    c[..., 0] *= 2.0
    symc = np.zeros(c.shape[:-1] + (fftlen,))
    symc[..., 0] = c[..., 0]
    for i in range(1, c.shape[-1]):
        symc[..., i] = c[..., i]
        symc[..., fftlen - i] = c[..., i]
    return np.exp(np.fft.rfft(symc, axis=-1).real)


def mcepalpha(fs, start=0.0, stop=1.0, step=0.001, num_points=1000):
    """pysptk.util.mcepalpha: the all-pass constant whose warped frequency is closest to the mel scale at fs."""
    step_hz = (fs / 2.0) / num_points
    mel = 1000.0 / np.log(2.0) * np.log(1.0 + step_hz * np.arange(num_points) / 1000.0)
    mel /= mel[-1]
    best, best_alpha = np.inf, None
    for alpha in np.arange(start, stop, step):
        omega = np.pi / num_points * np.arange(num_points)
        warp = np.arctan((1 - alpha * alpha) * np.sin(omega) / ((1 + alpha * alpha) * np.cos(omega) - 2 * alpha))
        warp[warp < 0] += np.pi
        warp /= warp[-1]
        dist = np.sum((mel - warp) ** 2) / num_points
        if dist < best:
            best, best_alpha = dist, alpha
    return best_alpha


def cheaptrick_fft_size(fs, f0_floor=71.0):
    """pyworld.get_cheaptrick_fft_size."""
    return int(2 ** (1 + int(np.log2(3.0 * fs / f0_floor + 1))))
