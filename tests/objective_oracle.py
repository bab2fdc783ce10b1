"""The reference notebooks' objective measures restated in fp64 numpy (notebooks/Test VC.ipynb, Test RNN VC.ipynb,
Test TTS.ipynb: vis_gv, mean_modspec) -- the checker of csrc/modspec.cu.  TEST INFRASTRUCTURE.

nnmnkwii.preprocessing.modspec is restated from its published definition; parity with the package itself is unpinned
(it is not a dependency of this repository).  The float64 cast is the notebooks' arithmetic: they ran numpy 1.x, whose
FFT computed in double whatever the input, while numpy >= 2 keeps float32 input in single precision."""
import numpy as np


def modspec(x, n=4096, norm=None):
    """``nnmnkwii.preprocessing.modspec(x, n, norm)``: the power ``R * R + im * im`` of ``np.fft.rfft(x, n, axis=0)``,
    x ``(T, D)`` -> ``(n // 2 + 1, D)``.  numpy's ``n``: frames beyond n are cropped, shorter columns zero-padded."""
    s = np.fft.rfft(np.asarray(x, dtype=np.float64), n=n, axis=0, norm=norm)
    R, im = s.real, s.imag
    return R * R + im * im


def log_modspec(x, n=4096):
    """``np.log(P.modspec(mgc, n=n))`` of mean_modspec; a column whose power is exactly 0 gives -inf."""
    with np.errstate(divide="ignore"):
        return np.log(modspec(x, n))


def global_variance(x):
    """``np.var(mgc, axis=0)`` of vis_gv in float64 (ddof 0; no frames give NaN)."""
    x = np.asarray(x, dtype=np.float64)
    if len(x) == 0:
        return np.full(x.shape[1:], np.nan)
    return np.var(x, axis=0)
