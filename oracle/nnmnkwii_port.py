"""Restatement of the three nnmnkwii symbols the reference hot path calls.  TEST INFRASTRUCTURE.

nnmnkwii (pinned ``>= 0.0.14``, reference setup.py:63,66; depends on the cython package
``bandmat``) is NOT vendored under the reference checkout and is not installed in this image, so its
arithmetic is restated here from its published definition -- **parity unpinned** against the
package itself.  Call sites this follows:

  * ``nnmnkwii.paramgen.unit_variance_mlpg_matrix(windows, T)``
        reference train.py:49,511 ; evaluation_vc.py:27,70 ; tests/test_gantts.py:8,31,140
  * ``nnmnkwii.autograd.unit_variance_mlpg(R, means)``
        reference gantts/multistream.py:11,120 ; gantts/models.py:8,66,115 ;
        tests/test_gantts.py:9,156-159
  * ``nnmnkwii.preprocessing.delta_features(x, windows)``
        reference gantts/multistream.py:28

Definition (nnmnkwii docs, "unit variance MLPG"): every window ``(l, u, coef)`` defines a
``T x T`` band matrix ``W_w[t, t+k] = coef[k+l]``, ``k in [-l, u]``, entries that fall outside
``[0, T)`` dropped (zero boundary).  ``W`` stacks the window matrices **window-major**
(``num_windows*T x T``).  ``R = (W^T W)^-1 W^T`` is evaluated in float64 and returned as float32
with shape ``(T, num_windows*T)``.  ``unit_variance_mlpg(R, means)`` re-orders ``means``
``(B, T, num_windows*sd)`` -- feature layout ``[static sd | delta sd | delta-delta sd]`` -- to
window-major rows ``(B, num_windows*T, sd)`` and evaluates ``torch.matmul(R, .)``; the backward is
``R^T g`` re-ordered back, and ``R`` receives no gradient.
"""
import numpy as np
import torch


def window_matrices(windows, T, dtype=np.float64):
    """List of dense ``(T, T)`` window matrices with zero boundary handling."""
    mats = []
    for l, u, coef in windows:
        coef = np.asarray(coef, dtype=dtype)
        assert l >= 0 and u >= 0 and len(coef) == l + u + 1
        W = np.zeros((T, T), dtype=dtype)
        for k in range(-l, u + 1):
            c = coef[k + l]
            if c == 0.0:
                continue
            rows = np.arange(max(0, -k), min(T, T - k))
            W[rows, rows + k] = c
        mats.append(W)
    return mats


def normal_matrix(windows, T):
    """``P = sum_w W_w^T W_w`` (float64, dense; banded with half-bandwidth max(l+u))."""
    P = np.zeros((T, T), dtype=np.float64)
    for W in window_matrices(windows, T):
        P += W.T @ W
    return P


def unit_variance_mlpg_matrix(windows, T, dtype=np.float32):
    """Dense ``R = (W^T W)^-1 W^T`` as ``dtype`` (float32 by default) ``(T, num_windows*T)``.

    nnmnkwii computes the inverse through a banded Cholesky factorisation (bandmat); the
    result is the same matrix up to float64 round-off, then cast to ``dtype``.
    """
    T = int(T)
    mats = window_matrices(windows, T)
    P = np.zeros((T, T), dtype=np.float64)
    for W in mats:
        P += W.T @ W
    Wfull = np.vstack(mats)                       # (nw*T, T), window-major rows
    R = np.linalg.solve(P, Wfull.T)               # (T, nw*T)
    return np.ascontiguousarray(R.astype(dtype))


def _to_window_major(means, num_windows):
    B, T, D = means.shape
    sd = D // num_windows
    return means.contiguous().view(B, T, num_windows, sd).transpose(1, 2).reshape(
        B, num_windows * T, sd)


def _from_window_major(g, num_windows):
    B, WT, sd = g.shape
    T = WT // num_windows
    return g.view(B, num_windows, T, sd).transpose(1, 2).reshape(B, T, num_windows * sd)


class _UnitVarianceMLPG(torch.autograd.Function):
    @staticmethod
    def forward(ctx, means, R):
        squeeze = means.dim() == 2
        if squeeze:
            means = means.unsqueeze(0)
        nw = R.shape[1] // R.shape[0]
        ctx.nw, ctx.squeeze = nw, squeeze
        ctx.save_for_backward(R)
        out = torch.matmul(R, _to_window_major(means, nw))
        return out.squeeze(0) if squeeze else out

    @staticmethod
    def backward(ctx, grad_out):
        (R,) = ctx.saved_tensors
        if ctx.squeeze:
            grad_out = grad_out.unsqueeze(0)
        g = torch.matmul(R.t(), grad_out)
        g = _from_window_major(g, ctx.nw)
        return (g.squeeze(0) if ctx.squeeze else g), None


def unit_variance_mlpg(R, means):
    """``y = R . means`` (window-major), differentiable w.r.t. ``means`` only."""
    return _UnitVarianceMLPG.apply(means, R)


def delta_features(x, windows):
    """``hstack_w( correlate(x[:, d], coef_w, zero padded "same") )``; x is ``(T, D)``."""
    T, D = x.shape
    out = np.zeros((T, D * len(windows)), dtype=x.dtype)
    for wi, (l, u, coef) in enumerate(windows):
        for k in range(-l, u + 1):
            c = coef[k + l]
            lo, hi = max(0, -k), min(T, T - k)
            out[lo:hi, wi * D:(wi + 1) * D] += c * x[lo + k:hi + k]
    return out


def mlpg_solve_f64(windows, means):
    """Independent float64 ground truth: banded Cholesky solve of ``P y = W^T mu``.

    ``means``: ndarray ``(B, T, nw*sd)``.  Used to arbitrate float32 disagreements between the
    dense-R float32 path (the reference arithmetic) and the CUDA banded solver.
    """
    from scipy.linalg import cholesky_banded, cho_solve_banded
    means = np.asarray(means, dtype=np.float64)
    B, T, D = means.shape
    nw = len(windows)
    sd = D // nw
    mats = window_matrices(windows, T)
    P = np.zeros((T, T))
    for W in mats:
        P += W.T @ W
    hb = max(l + u for l, u, _ in windows)
    ab = np.zeros((hb + 1, T))
    for k in range(hb + 1):
        ab[k, :T - k] = np.diagonal(P, -k)
    c = cholesky_banded(ab, lower=True)
    out = np.empty((B, T, sd))
    for b in range(B):
        rhs = np.zeros((T, sd))
        for w, W in enumerate(mats):
            rhs += W.T @ means[b, :, w * sd:(w + 1) * sd]
        out[b] = cho_solve_banded((c, True), rhs)
    return out


def mlpg(mean_frames, variance_frames, windows):
    """``nnmnkwii.paramgen.mlpg(mean_frames, variance_frames, windows)`` restated (reference call sites
    evaluation_tts.py:70-72,92-94; the package is not vendored -> parity unpinned, but the unit-variance
    case must equal ``unit_variance_mlpg_matrix(windows, T) @ means``, which IS pinned by the goldens).

    mean_frames ``(T, nw*sd)``; variance_frames ``(nw*sd,)`` or ``(T, nw*sd)``.  Dense float64 solve of
    ``(sum_w W_w^T diag(1/var_w) W_w) y = sum_w W_w^T diag(1/var_w) mu_w`` per static dimension.
    """
    mu = np.asarray(mean_frames, dtype=np.float64)
    T, D = mu.shape
    nw = len(windows)
    sd = D // nw
    var = np.asarray(variance_frames, dtype=np.float64)
    if var.ndim == 1:
        var = np.tile(var, (T, 1))
    mats = window_matrices(windows, T)
    out = np.empty((T, sd))
    for d in range(sd):
        P = np.zeros((T, T))
        b = np.zeros(T)
        for w, W in enumerate(mats):
            tau = 1.0 / var[:, w * sd + d]
            P += W.T @ (tau[:, None] * W)
            b += W.T @ (tau * mu[:, w * sd + d])
        out[:, d] = np.linalg.solve(P, b)
    return out


# ------------------------------------------------------------------------------------------------------------------
# nnmnkwii.metrics (un-vendored; published definitions, parity unpinned against the package itself) -- the checker of
# the device-side distortions kernel (csrc/metrics.cu).  Written over a flat valid-frame selection, independently of the
# product's numpy shim (compat/nnmnkwii/metrics.py loops per utterance), so the two do not share code.
def _valid_frames(a, lengths):
    """(B, T, D) or (B, T) -> (n_valid_frames, D) float64 rows of the frames t < lengths[b]."""
    a = np.asarray(a, dtype=np.float64)
    if a.ndim == 2:
        a = a[:, :, None]
    B, T = a.shape[:2]
    lengths = [T] * B if lengths is None else [int(v) for v in lengths]
    keep = np.arange(T)[None, :] < np.asarray(lengths)[:, None]
    return a[keep]


def melcd(X, Y, lengths=None):
    """10 / ln(10) * sqrt(2) * mean over valid frames of the Euclidean distance (dB)."""
    d = _valid_frames(X, lengths) - _valid_frames(Y, lengths)
    return float(10.0 / np.log(10.0) * np.sqrt(2.0) * np.mean(np.sqrt(np.sum(d * d, axis=1))))


def mean_squared_error(X, Y, lengths=None):
    """sum of squared differences over valid frames / number of valid FRAMES."""
    d = _valid_frames(X, lengths) - _valid_frames(Y, lengths)
    return float(np.sum(d * d) / d.shape[0])


def lf0_mean_squared_error(src_f0, src_vuv, tgt_f0, tgt_vuv, lengths=None, linear_domain=False):
    """MSE of (log-)F0 over valid frames voiced in both; ZeroDivisionError when there is none."""
    sf, tf = _valid_frames(src_f0, lengths), _valid_frames(tgt_f0, lengths)
    both = (_valid_frames(src_vuv, lengths)[:, 0] + _valid_frames(tgt_vuv, lengths)[:, 0]) >= 2
    if linear_domain:
        sf, tf = np.exp(sf), np.exp(tf)
    n = int(np.count_nonzero(both))
    if n == 0:
        raise ZeroDivisionError("no frame voiced in both source and target")
    d = sf[both] - tf[both]
    return float(np.sum(d * d) / n)


def vuv_error(src_vuv, tgt_vuv, lengths=None):
    a, b = _valid_frames(src_vuv, lengths), _valid_frames(tgt_vuv, lengths)
    return float(np.count_nonzero(a != b) / a.shape[0])
