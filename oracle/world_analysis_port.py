"""numpy fp64 restatement of WORLD's waveform analysis as the reference notebooks call it (pyworld.dio, pyworld.stonemask,
pyworld.cheaptrick with pyworld's default options), of pysptk.sp2mc and of nnmnkwii.preprocessing.modspec_smoothing, one
utterance at a time.  Test infrastructure only: the product runs gantts_b200/csrc/world_analysis.cu.

Written from WORLD 0.2.3's published algorithm, the release oracle/world_port.py restates (dio.cpp, stonemask.cpp,
cheaptrick.cpp, common.cpp DCCorrection, matlabfunctions.cpp interp1 / interp1Q / randn).  Choices where WORLD is not
followed literally, shared with the kernels:
- DIO's DC removal sums the row in the fixed order of a 256-thread block (block_sum below) instead of WORLD's sequential
  loop, so the mean does not depend on how a row is split over threads;
- DIO's low-cut and Nuttall low-pass filters are direct FIR sums, taps in ascending order, without FMA.  WORLD multiplies
  zero-padded FFT spectra whose length covers both filters' support, so its product is the same linear convolution up to
  rounding (and a positive scale, fft_size, which no zero crossing depends on)."""
import numpy as np

from . import sptk_port
from . import world_port as W

F0_FLOOR = 71.0                 # pyworld's dio / cheaptrick default f0_floor
F0_CEIL = 800.0
CHANNELS_IN_OCTAVE = 2.0
ALLOWED_RANGE = 0.1
CUTOFF = 50.0                   # dio.cpp kCutOff: the low-cut filter, Hz
MAXIMUM_VALUE = 100000.0        # dio.cpp kMaximumValue
LOG2 = 0.69314718055994529      # kLog2
FLOOR_F0_STONEMASK = 40.0       # kFloorF0StoneMask
EPS = 2.220446049250313e-16     # kEps
Q1 = -0.15
THREADS = 256                   # the block whose reduction order block_sum follows


def matlab_round(x):
    return int(x + 0.5) if x > 0 else int(x - 0.5)


def block_sum(v, threads=THREADS):
    """The sum of v in a 256-thread block's fixed order (world.cu block_sum_f64): thread t adds v[t], v[t + 256], ... in
    turn; each warp adds its 32 partials by an xor butterfly (offsets 16 .. 1); the warps' sums are added in warp order."""
    v = np.asarray(v, dtype=np.float64)
    rows = -(-len(v) // threads)
    pad = np.zeros(max(rows, 1) * threads)
    pad[:len(v)] = v
    part = np.zeros(threads)
    for r in range(rows):
        part = part + pad[r * threads:(r + 1) * threads]
    lanes = part.reshape(threads // 32, 32)
    for o in (16, 8, 4, 2, 1):
        lanes = lanes + lanes[:, np.arange(32) ^ o]
    s = 0.0
    for w in range(threads // 32):
        s += lanes[w, 0]
    return s


# ---- DIO ----

def dio_frames(samples, fs, frame_period):
    """GetSamplesForDIO: int(1000 x_length / fs / frame_period) + 1."""
    return int(1000.0 * samples / fs / frame_period) + 1


def voice_range_minimum(frame_period):
    """FixF0Contour's window: int(0.5 + 1000 / frame_period / f0_floor) * 2 + 1; WORLD leaves f0 unset for F <= it."""
    return int(0.5 + 1000.0 / frame_period / F0_FLOOR) * 2 + 1


def band_boundaries():
    nb = 1 + int(np.log(F0_CEIL / F0_FLOOR) / LOG2 * CHANNELS_IN_OCTAVE)
    return np.array([F0_FLOOR * pow(2.0, (i + 1) / CHANNELS_IN_OCTAVE) for i in range(nb)])


def lowcut_taps(fs):
    """DesignLowCutFilter as a zero-phase kernel g[0 .. N-1], centre (N-1)/2: -hann / sum(hann), plus 1 at the centre."""
    N = matlab_round(fs / CUTOFF) * 2 + 1
    h = 0.5 - 0.5 * np.cos(np.arange(1, N + 1) * 2.0 * np.pi / (N + 1))
    tot = 0.0
    for v in h:
        tot += v
    g = -h / tot
    g[(N - 1) // 2] += 1.0
    return g


def nuttall(n):
    tmp = np.arange(n) / (n - 1.0)
    return (0.355768 - 0.487396 * np.cos(2.0 * np.pi * tmp) + 0.144232 * np.cos(4.0 * np.pi * tmp)
            - 0.012604 * np.cos(6.0 * np.pi * tmp))


def half_lengths(fs):
    """Each band's half_average_length: matlab_round(fs / boundary / 2); its Nuttall window has 4 h taps."""
    return [matlab_round(fs / b / 2.0) for b in band_boundaries()]


def _fir(taps, src, first, count):
    """out[i] = sum_k taps[k] src[first + i - k], k ascending, from 0.0, no FMA (the kernels' order)."""
    acc = np.zeros(count)
    for k, t in enumerate(taps):
        acc = acc + t * src[first - k:first - k + count]
    return acc


def band_signals(x, fs):
    """The low-passed signal of every band (the Y = L + 1 samples DIO searches): [(boundary, s)]."""
    x = np.asarray(x, dtype=np.float64)
    L = len(x)
    Y = L + 1
    mean = block_sum(x) / Y
    y = np.append(x - mean, -mean)                         # WORLD's y has L + 1 samples, the last 0 before the mean
    g = lowcut_taps(fs)
    c = (len(g) - 1) // 2
    hs = half_lengths(fs)
    P = 2 * max(hs)                                        # z is needed on [-P, L + P]
    ext = np.zeros(Y + 2 * P + 2 * c)
    ext[P + c:P + c + Y] = y                               # y[m] at m + P + c
    z = _fir(g, ext, 2 * c, Y + 2 * P)                     # z[m] at m + P
    out = []
    for b, h in zip(band_boundaries(), hs):
        out.append((b, _fir(nuttall(4 * h), z, P + 2 * h, Y)))
    return out


def fine_edges(f):
    """ZeroCrossingEngine's crossings of f from > 0 to <= 0, refined linearly: e - f[e-1] / (f[e] - f[e-1])."""
    e = np.nonzero((f[:-1] > 0.0) & (f[1:] <= 0.0))[0] + 1
    return e - f[e - 1] / (f[e] - f[e - 1])


def four_edges(s):
    """Negative-going, positive-going, peak and dip crossings (GetFourZeroCrossingIntervals)."""
    d = (-s[:-1]) - (-s[1:])
    return [fine_edges(s), fine_edges(-s), fine_edges(d), fine_edges(-d)]


def band_candidates(s, fs, boundary, t):
    """(candidate f0, score / (candidate + 1e-12)) of one band at the frame times t."""
    F = len(t)
    sets = []
    for fe in four_edges(s):
        if len(fe) - 1 - 2 <= 0:
            return np.zeros(F), np.full(F, MAXIMUM_VALUE / 1e-12)
        sets.append(W.interp1((fe[:-1] + fe[1:]) / 2.0 / fs, fs / (fe[1:] - fe[:-1]), t))
    a, b, c, d = sets
    cand = (a + b + c + d) / 4.0
    score = np.sqrt(((a - cand) * (a - cand) + (b - cand) * (b - cand) + (c - cand) * (c - cand)
                     + (d - cand) * (d - cand)) / 3.0)
    bad = (cand > boundary) | (cand < boundary / 2.0) | (cand > F0_CEIL) | (cand < F0_FLOOR)
    cand = np.where(bad, 0.0, cand)
    score = np.where(bad, MAXIMUM_VALUE, score)
    return cand, score / (cand + 1e-12)


def best_candidates(cands, scores):
    """GetBestF0Contour: per frame the first band with the least score."""
    best = cands[0].copy()
    tmp = scores[0].copy()
    for j in range(1, len(cands)):
        take = tmp > scores[j]
        tmp = np.where(take, scores[j], tmp)
        best = np.where(take, cands[j], best)
    return best


def _select_best(cur, past, cands, j):
    ref = (cur * 3.0 - past) / 2.0
    err = abs(ref - cands[0][j])
    best = cands[0][j]
    for i in range(1, len(cands)):
        e = abs(ref - cands[i][j])
        if e < err:
            err, best = e, cands[i][j]
    return 0.0 if abs(1.0 - best / ref) > ALLOWED_RANGE else best


def fix_f0_contour(best, cands, frame_period):
    """FixF0Contour: steps 1 and 2 (jumps and short voiced runs to 0), then steps 3 and 4 extend each voiced section
    forwards from its end and backwards from its start through the candidates."""
    F = len(best)
    vr = voice_range_minimum(frame_period)
    base = np.zeros(F)
    base[vr:F - vr] = best[vr:F - vr]
    s1 = np.zeros(F)
    for i in range(vr, F):
        s1[i] = base[i] if abs((base[i] - base[i - 1]) / (1e-12 + base[i])) < ALLOWED_RANGE else 0.0
    s2 = s1.copy()
    c = (vr - 1) // 2
    for i in range(c, F - c):
        if np.any(s1[i - c:i + c + 1] == 0):
            s2[i] = 0.0
    pos, neg = [], []
    for i in range(1, F):
        if s2[i] == 0 and s2[i - 1] != 0:
            neg.append(i - 1)
        elif s2[i - 1] == 0 and s2[i] != 0:
            pos.append(i)
    f = s2.copy()
    for i in range(len(neg)):
        limit = F - 1 if i == len(neg) - 1 else neg[i + 1]
        for j in range(neg[i], limit):
            f[j + 1] = _select_best(f[j], f[j - 1], cands, j + 1)
            if f[j + 1] == 0:
                break
    for i in range(len(pos) - 1, -1, -1):
        limit = 1 if i == 0 else pos[i - 1]
        for j in range(pos[i], limit, -1):
            f[j - 1] = _select_best(f[j], f[j + 1], cands, j - 1)
            if f[j - 1] == 0:
                break
    return f


def dio(x, fs, frame_period=5.0, details=False):
    """pyworld.dio(x, fs, frame_period=frame_period) -> (f0, temporal positions).  details: also the best candidate per
    frame and each band's candidates and scores."""
    F = dio_frames(len(x), fs, frame_period)
    if F <= voice_range_minimum(frame_period):
        raise ValueError("DIO needs more than %d frames (%d samples give %d)"
                         % (voice_range_minimum(frame_period), len(x), F))
    t = np.arange(F) * frame_period / 1000.0
    cands, scores = [], []
    for boundary, s in band_signals(x, fs):
        c, sc = band_candidates(s, fs, boundary, t)
        cands.append(c)
        scores.append(sc)
    best = best_candidates(cands, scores)
    f0 = fix_f0_contour(best, cands, frame_period)
    if details:
        return f0, t, {"best": best, "candidates": np.array(cands), "scores": np.array(scores)}
    return f0, t


# ---- StoneMask ----

def stonemask_fft_size(f0, fs):
    h = int(1.5 * fs / f0 + 1.0)
    return int(pow(2.0, 2.0 + int(np.log(h * 2.0 + 1.0) / LOG2)))


def _refine(x, fs, pos, f0):
    if f0 <= FLOOR_F0_STONEMASK or f0 > fs / 12.0:
        return 0.0
    h = int(1.5 * fs / f0 + 1.0)
    wlen = (2.0 * h + 1.0) / fs
    n = stonemask_fft_size(f0, fs)
    base = (np.arange(2 * h + 1) - h) / float(fs)
    raw = np.array([matlab_round(v) for v in (pos + base) * fs])
    tmp = (raw - 1.0) / fs - pos
    main = 0.42 + 0.5 * np.cos(2.0 * np.pi * tmp / wlen) + 0.08 * np.cos(4.0 * np.pi * tmp / wlen)
    diff = np.empty_like(main)
    diff[0] = -main[1] / 2.0
    diff[1:-1] = -(main[2:] - main[:-2]) / 2.0
    diff[-1] = main[-2] / 2.0
    seg = x[np.clip(raw - 1, 0, len(x) - 1)]
    Ms, Ds = np.fft.rfft(seg * main, n), np.fft.rfft(seg * diff, n)
    num = Ms.real * Ds.imag - Ms.imag * Ds.real
    pw = Ms.real * Ms.real + Ms.imag * Ms.imag
    nh = min(int(fs / 2.0 / f0), 6)
    numer = denom = 0.0
    for i in range(nh):
        k = matlab_round(f0 * n / fs * (i + 1))
        inst = 0.0 if pw[k] == 0.0 else k * fs / n + num[k] / pw[k] * fs / 2.0 / np.pi
        amp = np.sqrt(pw[k])
        numer += amp * inst
        denom += amp * (i + 1.0)
    mean = numer / (denom + 1e-12)
    return f0 if abs(mean - f0) > f0 * 0.2 else mean


def stonemask(x, f0, t, fs):
    """pyworld.stonemask(x, f0, temporal_positions, fs)."""
    x = np.asarray(x, dtype=np.float64)
    return np.array([_refine(x, fs, float(p), float(f)) for p, f in zip(t, f0)])


# ---- CheapTrick ----

def cheaptrick_f0_floor(fs, n):
    """GetF0FloorForCheapTrick: an f0 at or below it is analysed as 500 Hz."""
    return 3.0 * fs / (n - 3.0)


def current_f0(f0, fs, n):
    return np.where(np.asarray(f0, np.float64) <= cheaptrick_f0_floor(fs, n), W.DEFAULT_F0, f0)


def draw_counts(f0, fs, n):
    """randn draws of each frame: 2 h + 1 for the windowed waveform (h = round(1.5 fs / f0)), n/2 + 1 for the noise."""
    return np.array([2 * matlab_round(1.5 * fs / f) + 1 + n // 2 + 1 for f in current_f0(f0, fs, n)], np.int64)


def draw_offsets(f0, fs, n):
    """Each frame's first draw of the utterance's stream: the exclusive prefix sum of draw_counts."""
    c = draw_counts(f0, fs, n)
    return np.concatenate([[0], np.cumsum(c)[:-1]]).astype(np.int64)


def randn_stream(count, chunk=256):
    """Draws 0 .. count-1 of WORLD's randn after randn_reseed, vectorised over chunks of `chunk` draws whose starting
    states come from the GF(2) jump matrix of one chunk."""
    chunks = max(1, -(-int(count) // chunk))
    J = W.gf2_power(W.step_matrix(), 12 * chunk)
    states = np.zeros((chunks, 4), np.uint32)
    v = W._state_bits(W.SEED)
    for c in range(chunks):
        states[c] = W._bits_state(v)
        v = W.gf2_matmul(J, v[:, None])[:, 0]
    x, y, z, w = (states[:, i].copy() for i in range(4))
    out = np.zeros((chunks, chunk))
    for d in range(chunk):
        tmp = np.zeros(chunks, np.uint32)
        for _ in range(12):
            t = x ^ (x << np.uint32(11))
            x, y, z = y, z, w
            w = (w ^ (w >> np.uint32(19))) ^ (t ^ (t >> np.uint32(8)))
            tmp = tmp + (w >> np.uint32(4))
        out[:, d] = tmp / 268435456.0 - 6.0
    return out.reshape(-1)[:int(count)]


def _interp1q(x0, dx, y, xi):
    """WORLD's interp1Q on the grid x0 + k dx: y[b] + (y[b+1] - y[b]) f, b = int((xi - x0) / dx), the last slope 0."""
    q = (xi - x0) / dx
    base = q.astype(np.int64)
    dy = np.append(y[1:] - y[:-1], 0.0)
    return y[base] + dy[base] * (q - base)


def _frame(x, fs, f0, pos, n, draws):
    N = n // 2
    h = matlab_round(1.5 * fs / f0)
    base = np.arange(-h, h + 1)
    origin = matlab_round(pos * fs + 0.001)
    idx = np.clip(origin + base, 0, len(x) - 1)
    win = 0.5 * np.cos(np.pi * (base / 1.5 / fs) * f0) + 0.5
    win = win / np.sqrt(np.sum(win * win))
    wav = x[idx] * win + draws[:2 * h + 1] * 1e-12
    wav = wav - win * (np.sum(wav) / np.sum(win))
    X = np.fft.rfft(wav, n)
    p = X.real * X.real + X.imag * X.imag
    # DCCorrection
    ul = 2 + int(f0 * n / fs)
    rep = _interp1q(f0, -float(fs) / n, p[:ul + 1], np.arange(ul - 1) * fs / n)
    p[:ul - 1] = p[:ul - 1] + rep
    # LinearSmoothing over width 2 f0 / 3
    width = f0 * 2.0 / 3.0
    bd = int(width * n / fs) + 1
    mirror = np.concatenate([p[bd:0:-1], p[:N], p[N::-1][:bd + 1]])
    seg = np.cumsum(mirror * fs / n)
    origin_f = -(bd - 0.5) * fs / n
    axis = np.arange(N + 1) / n * fs - width / 2.0
    low = _interp1q(origin_f, float(fs) / n, seg, axis)
    high = _interp1q(origin_f, float(fs) / n, seg, axis + width)
    p = (high - low) / width
    p = p + np.abs(draws[2 * h + 1:2 * h + 1 + N + 1]) * EPS
    # SmoothingWithRecovery
    q = np.arange(1, N + 1) / float(fs)
    sl = np.concatenate([[1.0], np.sin(np.pi * f0 * q) / (np.pi * f0 * q)])
    cl = np.concatenate([[(1.0 - 2.0 * Q1) + 2.0 * Q1], (1.0 - 2.0 * Q1) + 2.0 * Q1 * np.cos(2.0 * np.pi * q * f0)])
    lp = np.log(p)
    cep = np.fft.fft(np.concatenate([lp, lp[N - 1:0:-1]])).real
    return np.exp(np.fft.irfft(cep[:N + 1] * sl * cl / n, n)[:N + 1] * n)


def cheaptrick(x, f0, t, fs, n=None, stream=None):
    """pyworld.cheaptrick(x, f0, temporal_positions, fs) (q1 -0.15, f0_floor 71, fft_size get_cheaptrick_fft_size(fs))
    -> (F, n/2 + 1).  stream: randn_stream of at least the utterance's draws, when already made."""
    x = np.asarray(x, dtype=np.float64)
    n = n or sptk_port.cheaptrick_fft_size(fs)
    cf = current_f0(f0, fs, n)
    off = draw_offsets(f0, fs, n)
    total = int(off[-1] + draw_counts(f0, fs, n)[-1]) if len(off) else 0
    if stream is None:
        stream = randn_stream(total)
    return np.array([_frame(x, fs, float(f), float(p), n, stream[o:]) for f, p, o in zip(cf, t, off)])


# ---- sp2mc and modulation-spectrum smoothing ----

def sp2mc(sp, order, alpha):
    """pysptk.sp2mc: the log power, its inverse real FFT (the real cepstrum), c[0] halved, freqt to order with alpha."""
    c = np.fft.irfft(np.log(np.asarray(sp, dtype=np.float64)), axis=-1)
    c[..., 0] /= 2.0
    return sptk_port.freqt(c, order, alpha)


def smoothing_bin(n, modfs, cutoff=50.0):
    """The first modulation-frequency bin modspec_smoothing removes: int(n * cutoff / modfs)."""
    return int(n * (cutoff / modfs))


def modspec_smoothing(x, modfs, n=4096, cutoff=50.0):
    """nnmnkwii.preprocessing.modspec_smoothing(x, modfs, n, cutoff=cutoff): each column's n-point real FFT along time
    with the bins from int(n cutoff / modfs) on set to 0, back by the inverse real FFT, the first T frames.  Only
    defined for T <= n."""
    x = np.asarray(x, dtype=np.float64)
    if x.shape[0] > n:
        raise ValueError("modspec_smoothing: %d frames, more than n = %d" % (x.shape[0], n))
    X = np.fft.rfft(x, n, axis=0)
    X[smoothing_bin(n, modfs, cutoff):] = 0.0
    return np.fft.irfft(X, n, axis=0)[:x.shape[0]]
