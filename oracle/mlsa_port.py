"""CPU restatement of the MLSA filter of reference evaluation_vc.py:95-101 (test_vc_from_path with diffvc=True):
SPTK's library ``mlsadf`` (mlsadf.c: mlsafir, mlsadf1, mlsadf2) at Pade order 5 and pysptk's ``Synthesizer`` frame loop,
in numpy fp64.  TEST INFRASTRUCTURE ONLY; it shares no code with the product's kernels (csrc/vc.cu).

pysptk cannot be installed here, so two conventions are restated from its published source and are NOT confirmed
against it:
  * the gain: pysptk.mlsadf wraps the library function, which does not apply exp(b[0]) (the SPTK command's -k option
    does), so the filter here has no gain either;
  * the frame loop: Synthesizer.synthesis filters hop t, the samples [t hop, (t+1) hop) of x truncated to its length,
    starting from b[max(t-1, 0)] and adding (b[t] - b[max(t-1, 0)]) / (the hop's sample count) after every sample;
    samples from T hop on stay 0.
tools/check_convert.py compares both with pysptk where it is installed.
"""
import numpy as np

MLSA_PADE5 = (1.0, 0.4999391, 0.1107098, 0.01369984, 0.0009564853, 0.00003041721)   # SPTK's pade[15..20]


def mlsa_delay_size(order, pd=5):
    """The doubles of one utterance's delay line: 3 (pd + 1) + pd (order + 2)."""
    return 3 * (pd + 1) + pd * (order + 2)


def _mlsafir(x, b, m, a, aa, d):
    """mlsafir on the delay lines d (rows..., stages, m + 2) and inputs x (rows..., stages), in place."""
    d[..., 0] = x
    d[..., 1] = aa * d[..., 0] + a * d[..., 1]
    for i in range(2, m + 1):
        d[..., i] += a * (d[..., i + 1] - d[..., i - 1])
    y = np.zeros(x.shape)
    for i in range(2, m + 1):
        y += d[..., i] * b[..., None, i]
    d[..., 2:] = d[..., 1:-1].copy()
    return y


def mlsadf(x, b, alpha, d, pd=5):
    """One sample of SPTK's mlsadf for every row: x (R,), b (R, M+1), d (R, mlsa_delay_size(M, pd)) updated in place.
    The five mlsafir stages of mlsadf2 each read the previous sample's output of the stage before them, so they are
    applied to all stages at once, in the order of SPTK's loop for the feedback sums."""
    m = b.shape[-1] - 1
    a, aa = alpha, 1.0 - alpha * alpha
    if pd != 5:
        raise ValueError("only SPTK's Pade order 5 is restated (got %d)" % pd)
    pade = MLSA_PADE5
    # mlsadf1: d[0 .. pd] the sections, pt = d[pd+1 .. 2pd+1]
    dd, pt = d[:, :pd + 1], d[:, pd + 1:2 * (pd + 1)]
    v_out = np.zeros(x.shape)
    for i in range(pd, 0, -1):
        dd[:, i] = aa * pt[:, i - 1] + a * dd[:, i]
        pt[:, i] = dd[:, i] * b[:, 1]
        v = pt[:, i] * pade[i]
        x = x + v if i & 1 else x - v
        v_out += v
    pt[:, 0] = x
    x = v_out + x
    # mlsadf2: the stages' delay lines, then pt
    base = 2 * (pd + 1)
    lines = d[:, base:base + pd * (m + 2)].reshape(len(x), pd, m + 2)
    pt = d[:, base + pd * (m + 2):]
    y = _mlsafir(pt[:, :pd].copy(), b, m, a, aa, lines)
    d[:, base:base + pd * (m + 2)] = lines.reshape(len(x), -1)
    v_out = np.zeros(x.shape)
    for i in range(pd, 0, -1):
        pt[:, i] = y[:, i - 1]
        v = pt[:, i] * pade[i]
        x = x + v if i & 1 else x - v
        v_out += v
    pt[:, 0] = x
    return v_out + x


def mlsa_synthesis(xs, bs, alpha, hop, pd=5):
    """Synthesizer(MLSADF(order=M, alpha=alpha), hopsize=hop).synthesis(x, b) for every pair (x, b) of the lists xs
    (S_r,) and bs (T_r, M+1), the rows run in lockstep; returns float64 arrays of S_r samples."""
    R = len(xs)
    m = bs[0].shape[-1] - 1
    S = np.array([len(x) for x in xs])
    T = np.array([len(b) for b in bs])
    end = np.minimum(S, T * hop)
    xp = np.zeros((R, max(int(S.max()), 1)))
    for r, x in enumerate(xs):
        xp[r, :len(x)] = x
    y = np.zeros_like(xp)
    d = np.zeros((R, mlsa_delay_size(m, pd)))
    bcur, inc = np.zeros((R, m + 1)), np.zeros((R, m + 1))
    for s in range(int(end.max()) if R else 0):
        if s % hop == 0:
            t = s // hop
            for r in range(R):
                if s < end[r]:
                    prev, cur = np.asarray(bs[r][max(t - 1, 0)], np.float64), np.asarray(bs[r][t], np.float64)
                    bcur[r] = prev
                    inc[r] = (cur - prev) / (min((t + 1) * hop, S[r]) - t * hop)
        out = mlsadf(xp[:, s], bcur, alpha, d, pd)
        live = s < end
        y[live, s] = out[live]
        bcur[live] += inc[live]
    return [y[r, :S[r]].copy() for r in range(R)]
