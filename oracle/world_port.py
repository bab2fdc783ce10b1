"""numpy fp64 restatement of WORLD's waveform synthesis as evaluation_tts.py's gen_waveform calls it
(pyworld.decode_aperiodicity, pyworld.synthesize), one utterance at a time, written as WORLD's sequential per-pulse loop.
Test infrastructure only: the product runs gantts_b200/csrc/world.cu.

Written from WORLD's published algorithm (codec.cpp DecodeAperiodicity; synthesis.cpp Synthesis, GetTimeBase,
GetOneFrameSegment; matlabfunctions.cpp randn, interp1).  Two places where a choice was made: the aperiodic ratio squares
the interpolated, clamped aperiodicity (WORLD's GetAperiodicRatio); a noise segment longer than fftlen keeps its first
fftlen zero-mean samples, where WORLD would write past its FFT buffer."""
import numpy as np

TWO_PI = 2.0 * np.pi
SAFE = 1e-12                    # kMySafeGuardMinimum
DEFAULT_F0 = 500.0              # kDefaultF0
SEED = (123456789, 362436069, 521288629, 88675123)
M32 = 0xFFFFFFFF


def band_count(fs):
    """GetNumberOfAperiodicities: int(min(15000, fs/2 - 3000) / 3000), 0 when negative."""
    return max(0, int(min(15000.0, fs / 2.0 - 3000.0) / 3000.0))


def y_length(frames, fs, frame_period):
    return int(frames * frame_period * fs / 1000)


# ---- randn ----

class Randn(object):
    """WORLD's randn: xorshift128, a draw the uint32 sum of w >> 4 over 12 outputs, / 2^28 - 6."""

    def __init__(self, state=SEED):
        self.s = list(state)

    def step(self):
        x, y, z, w = self.s
        t = (x ^ (x << 11)) & M32
        w2 = (w ^ (w >> 19)) ^ (t ^ (t >> 8))
        self.s = [y, z, w, w2 & M32]
        return self.s[3]

    def draw(self):
        tmp = 0
        for _ in range(12):
            tmp = (tmp + (self.step() >> 4)) & M32
        return tmp / 268435456.0 - 6.0

    def draws(self, count):
        return np.array([self.draw() for _ in range(int(count))], dtype=np.float64)


def _state_bits(s):
    return np.array([(s[q // 32] >> (q % 32)) & 1 for q in range(128)], dtype=np.uint8)


def _bits_state(v):
    return [int(sum(int(v[32 * k + i]) << i for i in range(32))) for k in range(4)]


def step_matrix():
    """The 128 x 128 GF(2) matrix of one xorshift step (column q: the step of unit state q)."""
    M = np.zeros((128, 128), dtype=np.uint8)
    for q in range(128):
        e = [0, 0, 0, 0]
        e[q // 32] = 1 << (q % 32)
        r = Randn(e)
        r.step()
        M[:, q] = _state_bits(r.s)
    return M


def gf2_matmul(A, B):
    return (A.astype(np.int64) @ B.astype(np.int64) % 2).astype(np.uint8)


def gf2_power(M, k):
    R = np.eye(128, dtype=np.uint8)
    while k:
        if k & 1:
            R = gf2_matmul(M, R)
        M = gf2_matmul(M, M)
        k >>= 1
    return R


def jump(state, steps, M=None):
    """The xorshift state `steps` steps after `state`, by a GF(2) matrix power."""
    M = step_matrix() if M is None else M
    return _bits_state(gf2_matmul(gf2_power(M, steps), _state_bits(state)[:, None])[:, 0])


# ---- decode_aperiodicity ----

def interp1(x, y, xi):
    """WORLD's interp1 (histc, then y[k] + s (y[k+1] - y[k])): k the last knot <= xi, clamped to len(x) - 2."""
    x, y, xi = (np.asarray(a, dtype=np.float64) for a in (x, y, xi))
    k = np.clip(np.searchsorted(x, xi, side="right") - 1, 0, len(x) - 2)
    h = x[k + 1] - x[k]
    s = (xi - x[k]) / h
    return y[k] + s * (y[k + 1] - y[k])


def decode_aperiodicity(bap, fs, fftlen):
    """pyworld.decode_aperiodicity: coded (F, nb) -> (F, fftlen/2 + 1) float64."""
    bap = np.asarray(bap, dtype=np.float64)
    nb = band_count(fs)
    if bap.ndim != 2 or bap.shape[1] != nb:
        raise ValueError("bap must have %d columns at fs = %d" % (nb, fs))
    K = fftlen // 2 + 1
    ap = np.full((len(bap), K), 1.0 - SAFE)
    freq = float(fs) / fftlen * np.arange(K)
    cx = np.concatenate([np.arange(nb + 1) * 3000.0, [fs / 2.0]])
    for t in range(len(bap)):
        tmp = 0.0
        for j in range(nb):
            tmp += bap[t, j]
        if tmp / nb > -0.5:
            continue
        cy = np.concatenate([[-60.0], bap[t], [-SAFE]])
        ap[t] = np.power(10.0, interp1(cx, cy, freq) / 20.0)
    return ap


# ---- time base ----

def time_base(f0, fs, frame_period, fftlen):
    """GetTimeBase: (pulse samples int64, fractional shifts in seconds, interpolated V/UV per sample, y_length)."""
    f0 = np.asarray(f0, dtype=np.float64).reshape(-1)
    F = len(f0)
    if F < 2:
        raise ValueError("WORLD synthesis needs at least 2 frames")
    Y = y_length(F, fs, frame_period)
    fp = frame_period / 1000.0
    lowest = fs // fftlen + 1.0
    t = np.arange(Y) / float(fs)
    ct = np.arange(F + 1) * fp
    cf = np.where(f0 < lowest, 0.0, f0)
    cv = np.where(cf == 0.0, 0.0, 1.0)
    cf = np.append(cf, cf[F - 1] * 2 - cf[F - 2])
    cv = np.append(cv, cv[F - 1] * 2 - cv[F - 2])
    fi = interp1(ct, cf, t)
    vi = interp1(ct, cv, t)
    vuv = np.where(vi > 0.5, 1.0, 0.0)
    fi = np.where(vuv == 0.0, DEFAULT_F0, fi)
    total = np.cumsum(TWO_PI * fi / fs)                   # sequential, as WORLD's loop
    wrap = np.fmod(total, TWO_PI)
    n = np.nonzero(np.abs(wrap[1:] - wrap[:-1]) > np.pi)[0]
    y1 = wrap[n] - TWO_PI
    y2 = wrap[n + 1]
    x = -y1 / (y2 - y1)
    return n.astype(np.int64), x / fs, vuv, Y


# ---- the responses ----

def min_phase(log_half):
    """GetMinimumPhaseSpectrum of a half log spectrum (n/2 + 1 bins) -> n/2 + 1 complex bins."""
    N = len(log_half) - 1
    n = 2 * N
    full = np.concatenate([log_half, log_half[N - 1:0:-1]])
    cep = np.fft.fft(full)
    cep = np.conj(cep)
    cep[1:N] *= 2.0
    cep[N + 1:] = 0.0
    s = np.fft.fft(cep)[:N + 1] / n
    return np.exp(s.real) * (np.cos(s.imag) + 1j * np.sin(s.imag))


def dc_remover(n):
    h = np.zeros(n)
    tot = 0.0
    for i in range(n // 2):
        h[i] = 0.5 - 0.5 * np.cos(TWO_PI * (i + 1.0) / (1.0 + n))
        h[n - i - 1] = h[i]
        tot += h[i] * 2.0
    return h / tot


def fftshift(r):
    n = len(r)
    return np.concatenate([r[n // 2:], r[:n // 2]])


def frames_at(n_i, fs, fp, F):
    q = (n_i / float(fs)) / fp
    ff = min(F - 1, int(np.floor(q)))
    fc = min(F - 1, int(np.ceil(q)))
    return ff, fc, q - ff


def envelope_ratio(sp, ap, n_i, fs, fp):
    ff, fc, w = frames_at(n_i, fs, fp, len(sp))
    safe = lambda a: np.maximum(0.001, np.minimum(0.999999999999, np.asarray(a, dtype=np.float64)))
    if ff == fc:
        return np.abs(np.asarray(sp[ff], dtype=np.float64)), safe(ap[ff]) ** 2
    env = (1.0 - w) * np.abs(np.asarray(sp[ff], np.float64)) + w * np.abs(np.asarray(sp[fc], np.float64))
    return env, ((1.0 - w) * safe(ap[ff]) + w * safe(ap[fc])) ** 2


def periodic_spectrum(env, ratio):
    """The periodic response's spectrum before the fractional shift: the minimum phase of 1/2 log(env (1 - r) + 1e-12)."""
    return min_phase(np.log(env * (1.0 - ratio) + SAFE) / 2.0)


def periodic_response(env, ratio, vuv, shift, fs, dcr):
    n = len(dcr)
    if vuv <= 0.5 or ratio[0] > 0.999:
        return np.zeros(n)
    X = periodic_spectrum(env, ratio)
    c = TWO_PI * shift * fs / n
    re2 = np.cos(c * np.arange(n // 2 + 1))
    im2 = np.sqrt(1.0 - re2 * re2)
    X = (X.real * re2 + X.imag * im2) + 1j * (X.imag * re2 - X.real * im2)
    r = fftshift(np.fft.irfft(X, n) * n)
    dc = np.sum(r[n // 2:])
    out = r.copy()
    out[:n // 2] = -dc * dcr[:n // 2]
    out[n // 2:] -= dc * dcr[n // 2:]
    return out


def aperiodic_response(env, ratio, vuv, noise, n):
    seg = np.zeros(n)
    if len(noise):
        kept = noise[:n]
        seg[:len(kept)] = kept - np.mean(noise)
    X = np.fft.rfft(seg) * min_phase(np.log(env * ratio) / 2.0 if vuv != 0.0 else np.log(env) / 2.0)
    return fftshift(np.fft.irfft(X, n) * n)


def synthesize(f0, sp, ap, fs, frame_period, details=False):
    """pyworld.synthesize(f0, sp, ap, fs, frame_period) -> y float64 (y_length,).  details: also return the pulse list
    (samples, shifts, V/UV at each pulse) and every pulse's response."""
    sp = np.asarray(sp, dtype=np.float64)
    ap = np.asarray(ap, dtype=np.float64)
    n = 2 * (sp.shape[1] - 1)
    idx, shifts, vuv, Y = time_base(f0, fs, frame_period, n)
    fp = frame_period / 1000.0
    dcr = dc_remover(n)
    y = np.zeros(Y)
    P = len(idx)
    stream = Randn().draws(idx[-1] - idx[0] if P else 0)   # pulse i draws from n_i - n_0 on, N_i values
    responses = []
    for i in range(P):
        Ni = int(idx[min(P - 1, i + 1)] - idx[i])
        env, ratio = envelope_ratio(sp, ap, idx[i], fs, fp)
        v = vuv[idx[i]]
        d0 = int(idx[i] - idx[0])
        noise = stream[d0:d0 + Ni]
        r = (periodic_response(env, ratio, v, shifts[i], fs, dcr) * np.sqrt(Ni) +
             aperiodic_response(env, ratio, v, noise, n)) / n
        off = int(idx[i]) - n // 2 + 1
        lo, hi = max(0, -off), min(n, Y - off)
        y[lo + off:hi + off] += r[lo:hi]                 # one add per sample, in pulse order
        if details:
            responses.append(r)
    if details:
        return y, {"index": idx, "shift": shifts, "vuv": vuv[idx].astype(np.uint8), "responses": responses}
    return y
