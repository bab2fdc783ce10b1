"""torch.autograd bindings of the C-ABI ops.  Every op requires CUDA float32 tensors; there is no
CPU path (the product must fail loudly rather than fall back)."""
import ctypes

import numpy as np
import torch

from . import _lib
from . import config

LEAKY_SLOPE = 0.01          # nn.LeakyReLU() default used by the reference (gantts/models.py:37,132)


_raw_stream = getattr(torch._C, "_cuda_getCurrentRawStream", None)


def _stream():
    """cudaStream_t of torch's current stream on the current device (the raw getter is ~20x cheaper than building a
    torch.cuda.Stream object; it is called once per native launch)."""
    if _raw_stream is not None:
        return ctypes.c_void_p(_raw_stream(torch.cuda.current_device()))
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def require_cuda(*tensors):
    for t in tensors:
        if t is None:
            continue
        if not t.is_cuda:
            raise RuntimeError("gantts_b200: CUDA tensor required (got a %s tensor); this package has "
                               "no CPU fallback" % t.device.type)
        if t.dtype != torch.float32:
            raise RuntimeError("gantts_b200: float32 tensor required (got %s)" % t.dtype)


def _rows2d(x):
    """View (…, D) as (rows, D) with unit column stride; returns (tensor2d, row_stride)."""
    D = x.shape[-1]
    x2 = x.reshape(-1, D)
    if x2.stride(1) != 1 or (x2.shape[0] > 1 and x2.stride(0) < D):
        x2 = x2.contiguous()
    return x2, (x2.stride(0) if x2.shape[0] > 1 else D)


_ws_cache = {}


def workspace(nbytes, device, tag="ws"):
    """Cached per-(device, tag) scratch buffer, grown geometrically (stream-ordered reuse on the
    current stream only)."""
    key = (device.index, tag)
    buf = _ws_cache.get(key)
    if buf is None or buf.numel() < nbytes:
        buf = torch.empty(max(int(nbytes * 1.25), 1 << 20), dtype=torch.uint8, device=device)
        _ws_cache[key] = buf
    return buf


# ------------------------------------------------------------------------------------- MLPG
STANDARD_WINDOWS = {
    1: [(0, 0, (1.0,))],
    2: [(0, 0, (1.0,)), (1, 1, (-0.5, 0.0, 0.5))],
    3: [(0, 0, (1.0,)), (1, 1, (-0.5, 0.0, 0.5)), (1, 1, (1.0, -2.0, 1.0))],
}
_registered_windows = {}
_table_cache = {}
_validated_R = set()


def windows_key(windows):
    return tuple((int(l), int(u), tuple(float(c) for c in coef)) for l, u, coef in windows)


def register_windows(windows):
    """Declare the delta windows behind the R matrices of a given window count (the defaults are
    the reference's hparams windows, hparams.py:22-26,183-187)."""
    _registered_windows[len(windows)] = windows_key(windows)


def windows_for(num_windows):
    w = _registered_windows.get(num_windows)
    if w is None:
        if num_windows not in STANDARD_WINDOWS:
            raise RuntimeError("gantts_b200: no windows registered for num_windows=%d" % num_windows)
        w = windows_key(STANDARD_WINDOWS[num_windows])
    return w


def mlpg_table_full_host(windows, T):
    """The coefficient table the kernels read, float32 (T, GANTTS_MLPG_TABLE_COLS): rows of P^-1 within +-24 taps
    followed by the rows of the banded Cholesky factor of P; host fp64 computation inside the C library."""
    lib = _lib.load()
    w = _lib.make_windows(windows)
    tab = np.zeros((int(T), _lib.MLPG_TABLE_COLS), dtype=np.float32)
    _lib.check(lib.gantts_mlpg_table(ctypes.byref(w), int(T), tab.ctypes.data))
    return tab


def mlpg_table_host(windows, T):
    """Rows of P^-1 within +-24 taps, float32 (T, 49)."""
    return np.ascontiguousarray(mlpg_table_full_host(windows, T)[:, :_lib.MLPG_NTAPS])


def mlpg_table(windows, T, device):
    key = (windows_key(windows), int(T), device.index)
    t = _table_cache.get(key)
    if t is None:
        t = torch.from_numpy(mlpg_table_full_host(windows, T)).to(device)
        _table_cache[key] = t
    return t


def mlpg_table_device(windows, T, device):
    """mlpg_table_full_host(windows, T) built on `device` instead: a (T, GANTTS_MLPG_TABLE_COLS) float32 CUDA tensor,
    bit-identical to the host table, enqueued on the current stream with no host synchronisation.  It does not repeat the
    host builder's checks that P is positive definite and P^-1 decays within the taps: validate a window set once with
    the host builder."""
    lib = _lib.load()
    w = _lib.make_windows(windows)
    with torch.cuda.device(device):
        tab = torch.empty(int(T), _lib.MLPG_TABLE_COLS, dtype=torch.float32, device=device)
        _lib.check(lib.gantts_mlpg_table_device(ctypes.byref(w), int(T), tab.data_ptr(), _stream()))
    return tab


def _validate_R(R, windows, T):
    """One-time check per (num_windows, T) that a dense R handed in by the caller really is
    (W^T W)^-1 W^T for the registered windows (the kernels never read R on the hot path)."""
    key = (windows, int(T))
    if key in _validated_R:
        return
    tab = mlpg_table_host(windows, T)
    t = int(T) // 2
    row = R[t].detach().float().cpu().numpy()
    K = _lib.MLPG_HALF_TAPS
    worst = 0.0
    for w, (l, u, coef) in enumerate(windows):
        for r in range(max(0, t - K + 2), min(int(T), t + K - 1)):
            exp = 0.0
            for k in range(-l, u + 1):
                c = r + k
                j = c - t + K
                if 0 <= c < T and 0 <= j < _lib.MLPG_NTAPS:
                    exp += tab[t, j] * coef[k + l]
            worst = max(worst, abs(exp - row[w * int(T) + r]))
    if worst > 1e-4:
        raise RuntimeError("gantts_b200: the R matrix does not match the registered delta windows "
                           "(max deviation %.3g); call gantts_b200.ops.register_windows(...)" % worst)
    _validated_R.add(key)


def windows_from_R(R):
    """(windows, T) for a dense MLPG matrix R of shape (T, num_windows*T) (reference train.py:511)."""
    T = int(R.shape[0])
    nw = int(R.shape[1]) // T
    if nw * T != int(R.shape[1]):
        raise RuntimeError("gantts_b200: R must have shape (T, num_windows*T)")
    windows = windows_for(nw)
    _validate_R(R, windows, T)
    return windows, T


class _MLPG(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, table, streams, windows, ncols_out):
        require_cuda(x, table)
        lib = _lib.load()
        B, T, D = x.shape
        if x.stride(2) != 1:
            x = x.contiguous()
        out = torch.empty(B, T, ncols_out, dtype=torch.float32, device=x.device)
        _lib.check(lib.gantts_mlpg_fwd(x.data_ptr(), x.stride(0), x.stride(1), out.data_ptr(),
                                       out.stride(0), out.stride(1), table.data_ptr(),
                                       ctypes.byref(streams), ctypes.byref(windows), B, T, _stream()))
        ctx.table, ctx.streams, ctx.windows = table, streams, windows
        ctx.in_shape = (B, T, D)
        return out

    @staticmethod
    def backward(ctx, go):
        require_cuda(go)
        lib = _lib.load()
        B, T, D = ctx.in_shape
        if go.stride(2) != 1:
            go = go.contiguous()
        gi = torch.zeros(B, T, D, dtype=torch.float32, device=go.device)
        _lib.check(lib.gantts_mlpg_bwd(go.data_ptr(), go.stride(0), go.stride(1), gi.data_ptr(),
                                       gi.stride(0), gi.stride(1), ctx.table.data_ptr(),
                                       ctypes.byref(ctx.streams), ctypes.byref(ctx.windows), B, T, 0,
                                       _stream()))
        return gi, None, None, None, None


def mlpg(x, windows, stream_entries, ncols_out):
    """x: (B, T, D) CUDA float32.  stream_entries: [(in_start, sd, dyn, out_start)]."""
    squeeze = x.dim() == 2
    if squeeze:
        x = x.unsqueeze(0)
    table = mlpg_table(windows, x.shape[1], x.device)
    out = _MLPG.apply(x, table, _lib.make_streams(stream_entries), _lib.make_windows(windows), ncols_out)
    return out.squeeze(0) if squeeze else out


def mlpg_var(mean, variance, windows):
    """nnmnkwii.paramgen.mlpg on the device (reference evaluation_tts.py:70-72,92-94): mean (T, nw*sd) or
    (B, T, nw*sd) CUDA float32, variance (nw*sd,) [time-invariant], (T, nw*sd) or (B, T, nw*sd);
    returns the static trajectory (…, T, sd)."""
    require_cuda(mean, variance)
    lib = _lib.load()
    squeeze = mean.dim() == 2
    if squeeze:
        mean = mean.unsqueeze(0)
    B, T, D = mean.shape
    nw = len(windows)
    if D % nw:
        raise RuntimeError("gantts_b200: feature width %d is not a multiple of the window count %d" % (D, nw))
    sd = D // nw
    if mean.stride(2) != 1:
        mean = mean.contiguous()
    variance = variance.contiguous()
    if variance.shape[-1] != D:
        raise RuntimeError("gantts_b200: variance width %d != mean width %d" % (variance.shape[-1], D))
    if variance.dim() == 1:
        v_bs, v_ts = 0, 0
    elif variance.dim() == 2:
        v_bs, v_ts = 0, variance.stride(0)
    else:
        v_bs, v_ts = variance.stride(0), variance.stride(1)
    if variance.dim() >= 2 and variance.shape[-2] != T:
        raise RuntimeError("gantts_b200: variance has %d frames, mean has %d" % (variance.shape[-2], T))
    w = _lib.make_windows(windows)
    out = torch.empty(B, T, sd, dtype=torch.float32, device=mean.device)
    nbytes = lib.gantts_mlpg_var_workspace_bytes(ctypes.byref(w), B, T, sd)
    ws = workspace(nbytes, mean.device, "mlpg_var")
    _lib.check(lib.gantts_mlpg_var(mean.data_ptr(), mean.stride(0), mean.stride(1), variance.data_ptr(), v_bs, v_ts,
                                   out.data_ptr(), out.stride(0), out.stride(1), ctypes.byref(w), B, T, sd,
                                   ws.data_ptr(), ws.numel(), _stream()))
    return out.squeeze(0) if squeeze else out


def _column_vector(v, n, device, what):
    """None, or `v` as a contiguous float32 CUDA vector of n values."""
    if v is None:
        return None
    v = torch.as_tensor(v, dtype=torch.float32, device=device).reshape(-1).contiguous()
    if v.numel() != n:
        raise RuntimeError("gantts_b200: %s has %d values, expected %d" % (what, v.numel(), n))
    return v


def mlpg_ragged(x, lengths, windows, stream_entries, ncols_out, var=None, in_affine=None, out_affine=None):
    """Length-exact multi-stream MLPG of generation (gantts_mlpg_ragged): row b of the padded batch x (B, T, D) CUDA
    float32 is solved over its own lengths[b] frames (int64 CUDA (B,)), as the evaluation scripts solve each utterance
    alone; frames at or beyond lengths[b] are 0.  stream_entries: [(in_start, sd, dyn, out_start)], static-only streams
    pass through.  var: (D,) time-invariant variances or None (unit).  in_affine / out_affine: (scale, shift) over the
    input columns (applied before the solve) / the ncols_out output columns (after it), or None.  No host sync."""
    require_cuda(x)
    lib = _lib.load()
    if not (torch.is_tensor(lengths) and lengths.is_cuda and lengths.dtype == torch.int64):
        raise RuntimeError("gantts_b200: mlpg_ragged needs int64 CUDA lengths")
    B, T, D = x.shape
    if x.stride(2) != 1:
        x = x.contiguous()
    lengths = lengths.contiguous()
    dev = x.device
    var = _column_vector(var, D, dev, "var")
    isc, ish = (None, None) if in_affine is None else (_column_vector(in_affine[0], D, dev, "input scale"),
                                                      _column_vector(in_affine[1], D, dev, "input shift"))
    osc, osh = (None, None) if out_affine is None else (_column_vector(out_affine[0], ncols_out, dev, "output scale"),
                                                       _column_vector(out_affine[1], ncols_out, dev, "output shift"))
    s, w = _lib.make_streams(stream_entries), _lib.make_windows(windows)
    nbytes = lib.gantts_mlpg_ragged_workspace_bytes(ctypes.byref(s), ctypes.byref(w), lengths.data_ptr(), B, T)
    if nbytes == 0:
        _lib.check(_lib.GANTTS_E_BADARG)
    ws = workspace(nbytes, dev, "mlpg_ragged")
    out = torch.empty(B, T, ncols_out, dtype=torch.float32, device=dev)
    ptr = lambda t: t.data_ptr() if t is not None else None
    _lib.check(lib.gantts_mlpg_ragged(x.data_ptr(), x.stride(0), x.stride(1), ptr(var), ptr(isc), ptr(ish),
                                      out.data_ptr(), out.stride(0), out.stride(1), ptr(osc), ptr(osh),
                                      ctypes.byref(s), ctypes.byref(w), lengths.data_ptr(), B, T, ws.data_ptr(),
                                      ws.numel(), _stream()))
    return out


# ----------------------------------------------------------------- mel-cepstrum post-processing
POSTFILTER_FFTLEN = 1024    # merlin_post_filter's defaults: fftlen 1024, minimum-phase order 511 (evaluation_tts.py:113)
_mcep_op_cache = {}


def mcep_operator_host(alpha, order, fftlen, kind):
    """The (fftlen/2 + 1, order + 1) float64 matrix of gantts_mcep_operator: row k maps a mel-cepstrum to its log power at
    bin k, for merlin_post_filter's energy (kind _lib.MCEP_R0) or for mc2sp (_lib.MCEP_SP).  Host computation."""
    lib = _lib.load()
    op = np.zeros((int(fftlen) // 2 + 1, int(order) + 1), dtype=np.float64)
    _lib.check(lib.gantts_mcep_operator(float(alpha), int(order), int(fftlen), int(kind), op.ctypes.data))
    return op


def _mcep_operator(alpha, order, fftlen, kind, device):
    key = (float(alpha), int(order), int(fftlen), int(kind), device.index)
    op = _mcep_op_cache.get(key)
    if op is None:
        op = torch.from_numpy(mcep_operator_host(alpha, order, fftlen, kind)).to(device)
        _mcep_op_cache[key] = op
    return op


def _mcep_args(mc, lengths, what):
    require_cuda(mc)
    if not (torch.is_tensor(lengths) and lengths.is_cuda and lengths.dtype == torch.int64):
        raise RuntimeError("gantts_b200: %s needs int64 CUDA lengths" % what)
    if mc.dim() != 3:
        raise RuntimeError("gantts_b200: %s needs mc (B, T, M+1)" % what)
    if mc.stride(2) != 1:
        mc = mc.contiguous()
    return mc, lengths.contiguous()


def mcep_postfilter(mc, lengths, alpha, coef=1.4):
    """nnmnkwii.postfilters.merlin_post_filter(mc, alpha, coef=coef) on every frame t < lengths[b] of row b
    (gantts_mcep_postfilter): mc (B, T, M+1) CUDA float32, lengths int64 CUDA (B,).  Returns (B, T, M+1) float32 with 0
    beyond each length.  The operator is built once per (alpha, order, device) and cached.  No host sync."""
    mc, lengths = _mcep_args(mc, lengths, "mcep_postfilter")
    lib = _lib.load()
    B, T, M1 = mc.shape
    op = _mcep_operator(alpha, M1 - 1, POSTFILTER_FFTLEN, _lib.MCEP_R0, mc.device)
    out = torch.empty(B, T, M1, dtype=torch.float32, device=mc.device)
    _lib.check(lib.gantts_mcep_postfilter(mc.data_ptr(), mc.stride(0), mc.stride(1), out.data_ptr(), out.stride(0),
                                          out.stride(1), op.data_ptr(), float(coef), lengths.data_ptr(), B, T, M1 - 1,
                                          op.shape[0], _stream()))
    return out


def mc2sp(mc, lengths, alpha, fftlen):
    """pysptk.mc2sp(mc, alpha, fftlen) on every frame t < lengths[b] of row b (gantts_mcep_to_sp): the power spectral
    envelope (B, T, fftlen/2 + 1) float32, 0 beyond each length.  The operator is cached per (alpha, order, fftlen,
    device).  No host sync."""
    mc, lengths = _mcep_args(mc, lengths, "mc2sp")
    lib = _lib.load()
    B, T, M1 = mc.shape
    op = _mcep_operator(alpha, M1 - 1, fftlen, _lib.MCEP_SP, mc.device)
    sp = torch.empty(B, T, op.shape[0], dtype=torch.float32, device=mc.device)
    _lib.check(lib.gantts_mcep_to_sp(mc.data_ptr(), mc.stride(0), mc.stride(1), sp.data_ptr(), sp.stride(0),
                                     sp.stride(1), op.data_ptr(), lengths.data_ptr(), B, T, M1 - 1, op.shape[0],
                                     _stream()))
    return sp


# ------------------------------------------------------------- global variance and modulation spectrum
def _feature_args(x, lengths, what):
    require_cuda(x)
    if not (torch.is_tensor(lengths) and lengths.is_cuda and lengths.dtype == torch.int64):
        raise RuntimeError("gantts_b200: %s needs int64 CUDA lengths" % what)
    if x.dim() != 3 or lengths.dim() != 1 or lengths.numel() != x.shape[0]:
        raise RuntimeError("gantts_b200: %s needs x (B, T, D) and lengths (B,)" % what)
    if x.stride(2) != 1:
        x = x.contiguous()
    return x, lengths.contiguous()


def modspec(x, lengths, n, out_sum=None):
    """np.log(nnmnkwii.preprocessing.modspec(x[b, :lengths[b]], n)) of every row b (gantts_modspec): x (B, T, D) CUDA
    float32, any batch and time strides (a column slice is read in place), lengths int64 CUDA (B,).  Returns the
    (B, n/2 + 1, D) float64 log power.  out_sum: None, or a (n/2 + 1, D) float64 CUDA tensor to which the rows are added
    one at a time in row order.  No host sync."""
    x, lengths = _feature_args(x, lengths, "modspec")
    lib = _lib.load()
    B, T, D = x.shape
    K = int(n) // 2 + 1
    if out_sum is not None and not (out_sum.is_cuda and out_sum.dtype == torch.float64 and out_sum.device == x.device
                                    and tuple(out_sum.shape) == (K, D) and out_sum.is_contiguous()):
        raise RuntimeError("gantts_b200: modspec's out_sum must be a contiguous float64 (%d, %d) tensor on %s"
                           % (K, D, x.device))
    out = torch.empty(B, K, D, dtype=torch.float64, device=x.device)
    _lib.check(lib.gantts_modspec(x.data_ptr(), x.stride(0), x.stride(1), lengths.data_ptr(), B, T, D, int(n),
                                  out.data_ptr(), None if out_sum is None else out_sum.data_ptr(), _stream()))
    return out


def global_variance(x, lengths):
    """np.var(x[b, :lengths[b]].astype(np.float64), axis=0) of every row b (gantts_global_variance): x (B, T, D) CUDA
    float32, lengths int64 CUDA (B,).  Returns (B, D) float64.  No host sync."""
    x, lengths = _feature_args(x, lengths, "global_variance")
    lib = _lib.load()
    B, T, D = x.shape
    out = torch.empty(B, D, dtype=torch.float64, device=x.device)
    _lib.check(lib.gantts_global_variance(x.data_ptr(), x.stride(0), x.stride(1), lengths.data_ptr(), B, T, D,
                                          out.data_ptr(), _stream()))
    return out


# ------------------------------------------------------------- phone rows and state durations to frames
def _durations(dur, what):
    require_cuda(dur)
    if dur.dim() != 3:
        raise RuntimeError("gantts_b200: %s needs durations (B, P, S)" % what)
    return dur if dur.stride(2) == 1 else dur.contiguous()


def state_frame_offsets(dur, phone_lengths):
    """Each phone's first frame (gantts_state_frame_offsets): dur (B, P, S) CUDA float32 state durations, any batch and
    phone strides; phone_lengths int64 CUDA (B,).  Returns (offsets int64 CUDA (B, P+1), frame_lengths int64 CUDA (B,),
    frame_lengths as a host numpy array).  Makes the one host synchronisation of the duration-to-frames chain: a single
    device-to-host copy of the frame lengths and the status word, because the frame count sizes the acoustic batch.
    Raises RuntimeError naming the rule when a duration is not a finite integer in [1, 2^24] or a row is too long."""
    dur = _durations(dur, "state_frame_offsets")
    if not (torch.is_tensor(phone_lengths) and phone_lengths.is_cuda and phone_lengths.dtype == torch.int64):
        raise RuntimeError("gantts_b200: state_frame_offsets needs int64 CUDA phone lengths")
    lib = _lib.load()
    B, P, S = dur.shape
    phone_lengths = phone_lengths.contiguous()
    offsets = torch.empty(B, P + 1, dtype=torch.int64, device=dur.device)
    buf = torch.empty(B + 1, dtype=torch.int64, device=dur.device)     # frame lengths, then the status word
    _lib.check(lib.gantts_state_frame_offsets(dur.data_ptr(), dur.stride(0), dur.stride(1), phone_lengths.data_ptr(),
                                              B, P, S, offsets.data_ptr(), buf.data_ptr(), buf[B:].data_ptr(),
                                              _stream()))
    host = buf.cpu().numpy()
    status = int(host[B])
    if status & _lib.FRAMES_BAD_DURATION:
        raise RuntimeError("gantts_b200: state_frame_offsets: a state duration is not a finite integer in [1, %d]"
                           % _lib.MAX_FRAMES)
    if status & _lib.FRAMES_TOO_LONG:
        raise RuntimeError("gantts_b200: state_frame_offsets: a row has more than %d frames (max %d)"
                           % (_lib.MAX_FRAMES, int(host[:B].max())))
    return offsets, buf[:B], host[:B].copy()


def expand_state_frames(phone_x, dur, offsets, frame_lengths, scale, min_, T):
    """The acoustic model's inputs (gantts_expand_state_frames): every phone's row of phone_x (B, P, L) CUDA float32
    repeated over its frames and followed by Merlin's nine "full" subphone features of its durations dur (B, P, S), then
    fl(fl(v * scale) + min_) per column in float32 (generate.normalize_input's arithmetic; scale 1 and min_ 0 give the raw
    features).  offsets, frame_lengths: state_frame_offsets' device tensors; scale, min_: (L+9,) float32.  Returns
    (B, T, L+9) float32, 0 at and beyond each row's frame length.  No host sync."""
    require_cuda(phone_x)
    dur = _durations(dur, "expand_state_frames")
    if phone_x.dim() != 3 or phone_x.shape[:2] != dur.shape[:2]:
        raise RuntimeError("gantts_b200: expand_state_frames needs phone_x (B, P, L) and dur (B, P, S)")
    if phone_x.stride(2) != 1:
        phone_x = phone_x.contiguous()
    B, P, L = phone_x.shape
    S = dur.shape[2]
    W = L + _lib.SUBPHONE_FEATURES
    for t, shape in ((offsets, (B, P + 1)), (frame_lengths, (B,))):
        if not (t.is_cuda and t.dtype == torch.int64 and tuple(t.shape) == shape and t.is_contiguous()):
            raise RuntimeError("gantts_b200: expand_state_frames needs state_frame_offsets' contiguous int64 offsets "
                               "(B, P+1) and frame lengths (B,)")
    dev = phone_x.device
    scale, min_ = _column_vector(scale, W, dev, "scale"), _column_vector(min_, W, dev, "min")
    lib = _lib.load()
    out = torch.empty(B, int(T), W, dtype=torch.float32, device=dev)
    _lib.check(lib.gantts_expand_state_frames(phone_x.data_ptr(), phone_x.stride(0), phone_x.stride(1), dur.data_ptr(),
                                              dur.stride(0), dur.stride(1), offsets.data_ptr(), frame_lengths.data_ptr(),
                                              scale.data_ptr(), min_.data_ptr(), B, P, L, S, int(T), out.data_ptr(),
                                              _stream()))
    return out


# ------------------------------------------------------------- WORLD waveform synthesis
WORLD_CHUNK_BYTES = 256 << 20   # per-pulse response buffer of world_synthesize: pulses beyond it run in further chunks


def world_band_count(fs):
    """WORLD's number of coded aperiodicity bands at fs: floor(min(15000, fs/2 - 3000) / 3000), 0 below 12 kHz."""
    return int(_lib.load().gantts_world_band_count(int(fs)))


def world_y_length(frames, fs, frame_period):
    """int(frames * frame_period * fs / 1000): the samples pyworld.synthesize makes of `frames` frames."""
    return int(_lib.load().gantts_world_y_length(int(frames), int(fs), float(frame_period)))


def _world_rows(x, lengths, what, width=None):
    """x (B, T) or (B, T, width) CUDA float32 -> (x, lengths) with a unit last stride."""
    require_cuda(x)
    if not (torch.is_tensor(lengths) and lengths.is_cuda and lengths.dtype == torch.int64):
        raise RuntimeError("gantts_b200: %s needs int64 CUDA lengths" % what)
    if x.dim() != 3 or (width is not None and x.shape[2] != width) or lengths.dim() != 1 \
            or lengths.numel() != x.shape[0]:
        raise RuntimeError("gantts_b200: %s needs x (B, T, %s) and lengths (B,)" % (what, width or "K"))
    return (x if x.stride(2) == 1 else x.contiguous()), lengths.contiguous()


def world_decode_aperiodicity(bap, lengths, fs, fftlen):
    """pyworld.decode_aperiodicity(bap[b, :lengths[b]], fs, fftlen) of every row b (gantts_world_decode_aperiodicity):
    bap (B, T, nb) CUDA float32 with nb = world_band_count(fs), lengths int64 CUDA (B,).  Returns (B, T, fftlen/2 + 1)
    float64, 0 beyond each length.  No host sync."""
    bap, lengths = _world_rows(bap, lengths, "world_decode_aperiodicity")
    B, T, nb = bap.shape
    ap = torch.empty(B, T, int(fftlen) // 2 + 1, dtype=torch.float64, device=bap.device)
    _lib.check(_lib.load().gantts_world_decode_aperiodicity(bap.data_ptr(), bap.stride(0), bap.stride(1),
                                                            lengths.data_ptr(), B, T, nb, int(fs), int(fftlen),
                                                            ap.data_ptr(), _stream()))
    return ap


def world_time_base(f0, lengths, fs, frame_period, fftlen):
    """WORLD's pulse locations of every row (gantts_world_time_base): f0 (B, T) or (B, T, 1) CUDA float32 in Hz, lengths
    int64 CUDA (B,).  Returns a dict: "index" int32, "shift" float64 (seconds), "vuv" uint8, each (B, cap) CUDA with the
    pulses of row b in its first counts[b] entries, and "counts", "y_lengths" as host int64 arrays.  Makes one host
    synchronisation, the read of the counts, the y_lengths and the status word; raises RuntimeError naming the rule when
    a valid f0 is not finite or a row has fewer than 2 frames."""
    if f0.dim() == 2:
        f0 = f0.unsqueeze(-1)
    f0, lengths = _world_rows(f0, lengths, "world_time_base", 1)
    B, T, _ = f0.shape
    lib = _lib.load()
    cap = world_y_length(T, fs, frame_period)
    dev = f0.device
    index = torch.empty(B, max(cap, 1), dtype=torch.int32, device=dev)
    shift = torch.empty(B, max(cap, 1), dtype=torch.float64, device=dev)
    vuv = torch.empty(B, max(cap, 1), dtype=torch.uint8, device=dev)
    info = torch.empty(2 * B + 1, dtype=torch.int64, device=dev)
    _lib.check(lib.gantts_world_time_base(f0.data_ptr(), f0.stride(0), f0.stride(1), lengths.data_ptr(), B, T, int(fs),
                                          float(frame_period), int(fftlen), cap, index.data_ptr(), shift.data_ptr(),
                                          vuv.data_ptr(), info.data_ptr(), _stream()))
    host = info.cpu().numpy()
    status = int(host[2 * B])
    if status & _lib.WORLD_BAD_F0:
        raise RuntimeError("gantts_b200: world_time_base: an f0 value within a row's length is not finite")
    if status & _lib.WORLD_SHORT:
        raise RuntimeError("gantts_b200: world_time_base: a row has fewer than 2 frames (WORLD synthesis needs 2)")
    return {"index": index, "shift": shift, "vuv": vuv, "info": info, "cap": cap,
            "counts": host[:B].copy(), "y_lengths": host[B:2 * B].copy()}


def world_randn(count, device):
    """Draws 0 .. count-1 of WORLD's randn after randn_reseed, float64 CUDA (count,), bit for bit (gantts_world_randn).
    No host sync."""
    lib = _lib.load()
    out = torch.empty(int(count), dtype=torch.float64, device=device)
    nbytes = lib.gantts_world_randn_workspace_bytes(int(count))
    ws = workspace(nbytes, device, "world_randn")
    _lib.check(lib.gantts_world_randn(int(count), out.data_ptr(), ws.data_ptr(), nbytes, _stream()))
    return out


def world_synthesize(f0, sp, ap, lengths, fs, frame_period, pulses=None, noise=None):
    """pyworld.synthesize(f0[b, :F], sp[b, :F], ap[b, :F], fs, frame_period) of every row b, F = lengths[b]
    (gantts_world_time_base, gantts_world_randn, gantts_world_synthesize): f0 (B, T) or (B, T, 1) CUDA float32 in Hz, sp
    (B, T, fftlen/2 + 1) CUDA float32, ap the same shape in float64 (world_decode_aperiodicity), lengths int64 CUDA (B,).
    Returns (y (B, Ymax) float64 CUDA with 0 beyond each row's y_length, y_lengths as a host int64 array).  The time
    base's read of the pulse counts is the one host synchronisation; pulses: that time base, when already made.
    noise: world_randn of at least Ymax draws, when already made (the stream is the same for every call)."""
    sp, lengths = _world_rows(sp, lengths, "world_synthesize")
    B, T, K = sp.shape
    if not (torch.is_tensor(ap) and ap.is_cuda and ap.dtype == torch.float64 and tuple(ap.shape) == (B, T, K)):
        raise RuntimeError("gantts_b200: world_synthesize needs ap (B, T, K) float64 CUDA, the shape of sp")
    if ap.stride(2) != 1:
        ap = ap.contiguous()
    n = 2 * (K - 1)
    if pulses is None:
        pulses = world_time_base(f0, lengths, fs, frame_period, n)
    lib = _lib.load()
    y_lengths = pulses["y_lengths"]
    y_max = max(int(y_lengths.max()), 1)
    total = int(pulses["counts"].sum())
    if noise is None:
        noise = world_randn(y_max, sp.device)
    elif not (noise.is_cuda and noise.dtype == torch.float64 and noise.dim() == 1 and noise.numel() >= y_max
              and noise.is_contiguous()):
        raise RuntimeError("gantts_b200: world_synthesize's noise must be world_randn's contiguous float64 CUDA draws, "
                           "at least %d of them" % y_max)
    chunk = max(1, min(total, WORLD_CHUNK_BYTES // (8 * n)))
    nbytes = lib.gantts_world_synthesize_workspace_bytes(B, n, chunk)
    if nbytes == 0:
        raise RuntimeError("gantts_b200: world_synthesize: fftlen = %d must be a power of two in [64, 4096]" % n)
    ws = workspace(nbytes, sp.device, "world_synthesize")
    y = torch.empty(B, y_max, dtype=torch.float64, device=sp.device)
    _lib.check(lib.gantts_world_synthesize(sp.data_ptr(), sp.stride(0), sp.stride(1), ap.data_ptr(), ap.stride(0),
                                           ap.stride(1), lengths.data_ptr(), pulses["index"].data_ptr(),
                                           pulses["shift"].data_ptr(), pulses["vuv"].data_ptr(),
                                           pulses["info"].data_ptr(), pulses["cap"], total, noise.data_ptr(), B, T,
                                           int(fs), float(frame_period), n, y_max, y.data_ptr(), ws.data_ptr(), nbytes,
                                           _stream()))
    return y, y_lengths


# ------------------------------------------------------------- WORLD analysis, sp2mc and modulation-spectrum smoothing
def world_dio_frames(samples, fs, frame_period):
    """WORLD's GetSamplesForDIO: the frames pyworld.dio makes of `samples` samples."""
    return int(_lib.load().gantts_world_dio_frames(int(samples), int(fs), float(frame_period)))


def _waves(x, lengths, what):
    if not (torch.is_tensor(x) and x.is_cuda and x.dtype == torch.float64 and x.dim() == 2):
        raise RuntimeError("gantts_b200: %s needs x (B, S) float64 CUDA" % what)
    if not (torch.is_tensor(lengths) and lengths.is_cuda and lengths.dtype == torch.int64 and lengths.dim() == 1
            and lengths.numel() == x.shape[0]):
        raise RuntimeError("gantts_b200: %s needs int64 CUDA lengths (B,)" % what)
    return (x if x.stride(1) == 1 else x.contiguous()), lengths.contiguous()


def _frames_f0(f0, info, B, what):
    if not (torch.is_tensor(f0) and f0.is_cuda and f0.dtype == torch.float64 and f0.dim() == 2 and f0.shape[0] == B):
        raise RuntimeError("gantts_b200: %s needs f0 (B, T) float64 CUDA" % what)
    if not (torch.is_tensor(info) and info.is_cuda and info.dtype == torch.int64 and tuple(info.shape) == (B + 1,)):
        raise RuntimeError("gantts_b200: %s needs world_dio's info, int64 CUDA (B + 1,)" % what)
    return f0.contiguous()


def world_dio(x, lengths, fs, frame_period):
    """pyworld.dio(x[b, :lengths[b]], fs, frame_period=frame_period) of every row b (gantts_world_dio): x (B, S) float64
    CUDA.  Returns (f0 (B, T) float64 CUDA, T = world_dio_frames(S), 0 beyond each row's frames; info int64 CUDA (B + 1,):
    each row's frame count, then the status word that world_stonemask and world_cheaptrick add to).  No host sync: read
    info with world_analysis_check.  Frame j is at j frame_period / 1000 s."""
    x, lengths = _waves(x, lengths, "world_dio")
    lib = _lib.load()
    B, S = x.shape
    T = world_dio_frames(S, fs, frame_period)
    nbytes = lib.gantts_world_dio_workspace_bytes(B, S, int(fs), float(frame_period))
    if nbytes == 0:
        raise RuntimeError("gantts_b200: world_dio: B = %d, S = %d, fs = %d, frame_period = %g out of range"
                           % (B, S, fs, frame_period))
    ws = workspace(nbytes, x.device, "world_dio")
    f0 = torch.empty(B, T, dtype=torch.float64, device=x.device)
    info = torch.empty(B + 1, dtype=torch.int64, device=x.device)
    _lib.check(lib.gantts_world_dio(x.data_ptr(), x.stride(0), lengths.data_ptr(), B, S, int(fs), float(frame_period),
                                    f0.data_ptr(), info.data_ptr(), ws.data_ptr(), nbytes, _stream()))
    return f0, info


def world_stonemask(x, lengths, f0, info, fs, frame_period):
    """pyworld.stonemask(x[b, :lengths[b]], f0[b], timeaxis, fs) of every row over its info[b] frames
    (gantts_world_stonemask): f0 and info world_dio's.  Returns (B, T) float64 CUDA.  No host sync."""
    x, lengths = _waves(x, lengths, "world_stonemask")
    B, S = x.shape
    f0 = _frames_f0(f0, info, B, "world_stonemask")
    out = torch.empty_like(f0)
    _lib.check(_lib.load().gantts_world_stonemask(x.data_ptr(), x.stride(0), lengths.data_ptr(), f0.data_ptr(),
                                                  info.data_ptr(), B, S, f0.shape[1], int(fs), float(frame_period),
                                                  out.data_ptr(), info[B:].data_ptr(), _stream()))
    return out


def world_cheaptrick(x, lengths, f0, info, fs, frame_period, fftlen):
    """pyworld.cheaptrick(x[b, :lengths[b]], f0[b], timeaxis, fs) with q1 -0.15, f0_floor 71 and fft_size fftlen
    (generate.cheaptrick_fft_size(fs) is pyworld's) of every row over its info[b] frames (gantts_world_randn,
    gantts_world_cheaptrick).  Returns (B, T, fftlen/2 + 1) float64 CUDA, 0 beyond each row's frames.  No host sync."""
    x, lengths = _waves(x, lengths, "world_cheaptrick")
    B, S = x.shape
    f0 = _frames_f0(f0, info, B, "world_cheaptrick")
    T = f0.shape[1]
    lib = _lib.load()
    count = int(lib.gantts_world_cheaptrick_draws(T, int(fs), int(fftlen)))
    if count < 1:
        raise RuntimeError("gantts_b200: world_cheaptrick: fftlen = %d must be a power of two in [64, 4096]" % fftlen)
    noise = world_randn(count, x.device)
    offsets = torch.empty(B, T, dtype=torch.int64, device=x.device)
    sp = torch.empty(B, T, int(fftlen) // 2 + 1, dtype=torch.float64, device=x.device)
    _lib.check(lib.gantts_world_cheaptrick(x.data_ptr(), x.stride(0), lengths.data_ptr(), f0.data_ptr(),
                                           info.data_ptr(), B, S, T, int(fs), float(frame_period), int(fftlen),
                                           noise.data_ptr(), count, offsets.data_ptr(), sp.data_ptr(),
                                           info[B:].data_ptr(), _stream()))
    return sp


def world_analysis_check(info):
    """The one host synchronisation of the analysis chain: copies world_dio's info (frame counts and the status word that
    every analysis kernel adds to) and returns the frame counts as a host int64 array.  Raises RuntimeError naming the
    rule when a status bit is set."""
    host = info.cpu().numpy()
    B = len(host) - 1
    status = int(host[B])
    if status & _lib.ANALYSIS_BAD_INPUT:
        raise RuntimeError("gantts_b200: WORLD analysis: a sample within a row's length, or an f0, is not finite, or an "
                           "f0 is beyond what CheapTrick's fft size can analyse")
    if status & _lib.ANALYSIS_SHORT:
        raise RuntimeError("gantts_b200: WORLD analysis: a row is too short for DIO (%d frames; FixF0Contour needs "
                           "more frames than its window)" % int(host[:B].min()))
    if status & _lib.ANALYSIS_FFT:
        raise RuntimeError("gantts_b200: WORLD analysis: a StoneMask window needs an FFT over 4096 points")
    return host[:B].copy()


def sp2mc(sp, lengths, order, alpha):
    """pysptk.sp2mc(sp[b, t], order, alpha) for t < lengths[b] (gantts_sp2mc): sp (B, T, K) float64 CUDA.  Returns
    (B, T, order + 1) float64 CUDA, 0 beyond each length.  The operator is cached per (alpha, order, fftlen, device).
    No host sync."""
    if not (torch.is_tensor(sp) and sp.is_cuda and sp.dtype == torch.float64 and sp.dim() == 3):
        raise RuntimeError("gantts_b200: sp2mc needs sp (B, T, K) float64 CUDA")
    if not (torch.is_tensor(lengths) and lengths.is_cuda and lengths.dtype == torch.int64):
        raise RuntimeError("gantts_b200: sp2mc needs int64 CUDA lengths")
    sp = sp.contiguous()
    B, T, K = sp.shape
    key = (float(alpha), int(order), 2 * (K - 1), "sp2mc", sp.device.index)
    op = _mcep_op_cache.get(key)
    if op is None:
        op = torch.from_numpy(sp2mc_operator_host(alpha, order, 2 * (K - 1))).to(sp.device)
        _mcep_op_cache[key] = op
    mc = torch.empty(B, T, int(order) + 1, dtype=torch.float64, device=sp.device)
    _lib.check(_lib.load().gantts_sp2mc(sp.data_ptr(), op.data_ptr(), lengths.contiguous().data_ptr(), B, T, int(order),
                                        K, mc.data_ptr(), _stream()))
    return mc


def sp2mc_operator_host(alpha, order, fftlen):
    """The (fftlen/2 + 1, order + 1) float64 matrix of gantts_sp2mc_operator: column m maps a frame's log power to
    pysptk.sp2mc's coefficient m.  Host computation."""
    op = np.zeros((int(fftlen) // 2 + 1, int(order) + 1), dtype=np.float64)
    _lib.check(_lib.load().gantts_sp2mc_operator(float(alpha), int(order), int(fftlen), op.ctypes.data))
    return op


def smoothing_bin(n, modfs, cutoff=50.0):
    """The first modulation-frequency bin modspec_smoothing removes: int(n * cutoff / modfs)."""
    return int(n * (float(cutoff) / float(modfs)))


def modspec_smoothing(x, lengths, modfs, n=4096, cutoff=50.0):
    """nnmnkwii.preprocessing.modspec_smoothing(x[b, :lengths[b]], modfs, n=n, cutoff=cutoff) of every row b
    (gantts_modspec_smoothing): x (B, T, D) float64 CUDA with T <= n.  Returns (B, T, D) float64 CUDA, 0 beyond each
    length.  No host sync."""
    if not (torch.is_tensor(x) and x.is_cuda and x.dtype == torch.float64 and x.dim() == 3):
        raise RuntimeError("gantts_b200: modspec_smoothing needs x (B, T, D) float64 CUDA")
    if not (torch.is_tensor(lengths) and lengths.is_cuda and lengths.dtype == torch.int64):
        raise RuntimeError("gantts_b200: modspec_smoothing needs int64 CUDA lengths")
    x = x.contiguous()
    B, T, D = x.shape
    out = torch.empty_like(x)
    _lib.check(_lib.load().gantts_modspec_smoothing(x.data_ptr(), lengths.contiguous().data_ptr(), B, T, D, int(n),
                                                    smoothing_bin(n, modfs, cutoff), out.data_ptr(), _stream()))
    return out


# ------------------------------------------------------------- voice conversion with the difference MLSA filter
def _int64_lengths(lengths, B, what):
    if not (torch.is_tensor(lengths) and lengths.is_cuda and lengths.dtype == torch.int64 and lengths.dim() == 1
            and lengths.numel() == B):
        raise RuntimeError("gantts_b200: %s needs int64 CUDA lengths (B,)" % what)
    return lengths.contiguous()


def vc_inputs(mc, lengths, windows, mean, std):
    """The generator's inputs of test_vc_from_path (gantts_vc_inputs) for every frame t < lengths[b] of row b:
    P.delta_features(mc[b, :L], windows).astype(np.float32) and P.scale of it by mean, std (float64, as
    generate.normalize_input scales).  mc (B, T, D) float64 CUDA, any batch and time strides (a column slice is read in
    place); windows: any window set ops.windows_key accepts.  Returns (xin (B, T, len(windows) D) float32, the static block
    (B, T, D) float32, the first window's D columns), 0 beyond each length.  No host sync."""
    if not (torch.is_tensor(mc) and mc.is_cuda and mc.dtype == torch.float64 and mc.dim() == 3):
        raise RuntimeError("gantts_b200: vc_inputs needs mc (B, T, D) float64 CUDA")
    if mc.stride(2) != 1:
        mc = mc.contiguous()
    B, T, D = mc.shape
    lengths = _int64_lengths(lengths, B, "vc_inputs")
    windows = windows_key(windows)
    W = len(windows) * D
    col = lambda v: torch.as_tensor(v, dtype=torch.float64, device=mc.device).reshape(-1).contiguous()
    mean, std = col(mean), col(std)
    if mean.numel() != W or std.numel() != W:
        raise RuntimeError("gantts_b200: vc_inputs: mean and std need %d values (got %d, %d)"
                           % (W, mean.numel(), std.numel()))
    n = len(windows)
    l = (ctypes.c_int * n)(*[w[0] for w in windows])
    u = (ctypes.c_int * n)(*[w[1] for w in windows])
    taps = [c for w in windows for c in w[2]]
    coef = (ctypes.c_double * max(len(taps), 1))(*taps)
    xin = torch.empty(B, T, W, dtype=torch.float32, device=mc.device)
    stat = torch.empty(B, T, D, dtype=torch.float32, device=mc.device)
    _lib.check(_lib.load().gantts_vc_inputs(mc.data_ptr(), mc.stride(0), mc.stride(1), lengths.data_ptr(), B, T, D, n,
                                            l, u, coef, mean.data_ptr(), std.data_ptr(), xin.data_ptr(),
                                            stat.data_ptr(), _stream()))
    return xin, stat


def mc2b(pred, src, lengths, alpha):
    """pysptk.mc2b([0, pred - src], alpha) of every frame t < lengths[b] of row b (gantts_mc2b), the difference
    filter's coefficients of test_vc_from_path: pred, src (B, T, M) CUDA float32 (the converted and the source statics).
    Returns (B, T, M + 1) float64, 0 beyond each length.  No host sync."""
    require_cuda(pred, src)
    if pred.dim() != 3 or tuple(src.shape) != tuple(pred.shape):
        raise RuntimeError("gantts_b200: mc2b needs pred and src of one shape (B, T, M)")
    pred = pred if pred.stride(2) == 1 else pred.contiguous()
    src = src if src.stride(2) == 1 else src.contiguous()
    B, T, M = pred.shape
    lengths = _int64_lengths(lengths, B, "mc2b")
    b = torch.empty(B, T, M + 1, dtype=torch.float64, device=pred.device)
    _lib.check(_lib.load().gantts_mc2b(pred.data_ptr(), pred.stride(0), pred.stride(1), src.data_ptr(), src.stride(0),
                                       src.stride(1), lengths.data_ptr(), B, T, M, float(alpha), b.data_ptr(),
                                       _stream()))
    return b


def mlsa_filter(x, lengths, b, frames, alpha, hop):
    """Synthesizer(MLSADF(order=M, alpha=alpha), hopsize=hop).synthesis(x[r, :lengths[r]], b[r, :frames[r]]) of every
    row r (gantts_mlsa_filter): x (B, S) float64 CUDA samples, b (B, T, M + 1) float64 CUDA (mc2b's), lengths and frames
    int64 CUDA (B,).  SPTK's mlsadf at Pade order 5 without the gain exp(b[0]); M <= 63.  Returns (B, S) float64, 0 at and
    beyond min(lengths[r], frames[r] hop).  No host sync."""
    x, lengths = _waves(x, lengths, "mlsa_filter")
    B, S = x.shape
    if not (torch.is_tensor(b) and b.is_cuda and b.dtype == torch.float64 and b.dim() == 3 and b.shape[0] == B):
        raise RuntimeError("gantts_b200: mlsa_filter needs b (B, T, M + 1) float64 CUDA")
    b = b.contiguous()
    frames = _int64_lengths(frames, B, "mlsa_filter")
    y = torch.empty(B, S, dtype=torch.float64, device=x.device)
    _lib.check(_lib.load().gantts_mlsa_filter(x.data_ptr(), x.stride(0), lengths.data_ptr(), b.data_ptr(),
                                              frames.data_ptr(), B, S, b.shape[1], b.shape[2] - 1, float(alpha),
                                              int(hop), y.data_ptr(), _stream()))
    return y


# ------------------------------------------------------------- mini-batches from a corpus on the device
def corpus_gather(X, Y, offsets, lengths, t, x_out=None, y_out=None, status=None):
    """One padded mini-batch from a packed corpus on the device (gantts_corpus_gather): X (N, Dx), Y (N, Dy) contiguous
    CUDA float32, the utterances' frames one after another; offsets, lengths contiguous int64 CUDA (b,), row r the
    utterance at frames [offsets[r], offsets[r] + lengths[r]).  Returns (x (b, t, Dx), y (b, t, Dy)) float32, 0 at and
    beyond each row's length, written into x_out / y_out when given (contiguous, of those shapes).  status: None, or an
    int64 CUDA scalar into which GANTTS_CORPUS_BAD_ROW is OR-ed when a row lies outside the corpus or is longer than t
    (that row is written as 0).  One launch, no host sync."""
    require_cuda(X, Y, x_out, y_out)
    if X.dim() != 2 or Y.dim() != 2 or X.shape[0] != Y.shape[0] or not (X.is_contiguous() and Y.is_contiguous()):
        raise RuntimeError("gantts_b200: corpus_gather needs contiguous X (N, Dx) and Y (N, Dy) of the same N")
    for v in (offsets, lengths):
        if not (torch.is_tensor(v) and v.is_cuda and v.dtype == torch.int64 and v.dim() == 1 and v.is_contiguous()):
            raise RuntimeError("gantts_b200: corpus_gather needs contiguous int64 CUDA offsets and lengths (b,)")
    if offsets.numel() != lengths.numel():
        raise RuntimeError("gantts_b200: corpus_gather: offsets and lengths differ in length")
    if status is not None and not (status.is_cuda and status.dtype == torch.int64 and status.numel() == 1):
        raise RuntimeError("gantts_b200: corpus_gather's status must be an int64 CUDA scalar")
    b, t, dev = offsets.numel(), int(t), X.device
    out = []
    for given, D in ((x_out, X.shape[1]), (y_out, Y.shape[1])):
        if given is None:
            given = torch.empty(b, t, D, dtype=torch.float32, device=dev)
        elif tuple(given.shape) != (b, t, D) or not given.is_contiguous():
            raise RuntimeError("gantts_b200: corpus_gather's outputs must be contiguous (%d, %d, %d)" % (b, t, D))
        out.append(given)
    lib = _lib.load()
    _lib.check(lib.gantts_corpus_gather(X.data_ptr(), Y.data_ptr(), X.shape[0], X.shape[1], Y.shape[1],
                                        offsets.data_ptr(), lengths.data_ptr(), b, t, out[0].data_ptr(),
                                        out[1].data_ptr(), None if status is None else status.data_ptr(), _stream()))
    return out[0], out[1]


def distortion_sums(y, y_hat, lengths, mean, std, mcd=(0, 0), bap=(0, 0), lf0_col=-1, vuv_col=-1,
                    lf0_linear=True, mse=(0, 0)):
    """Eight sums behind the objective metrics of reference train.py:399-432 (see include/gantts_b200.h,
    gantts_distortions).  y, y_hat: (B, T, D) CUDA float32; lengths: int64 CUDA (B,); mean/std: (D,) CUDA.
    Returns a CUDA float32 tensor of 8 values (no host synchronisation here)."""
    require_cuda(y, y_hat, mean, std)
    lib = _lib.load()
    B, T, D = y.shape
    if y.stride(2) != 1:
        y = y.contiguous()
    if y_hat.stride(2) != 1:
        y_hat = y_hat.contiguous()
    cols = _lib.DistortionColsT(int(mcd[0]), int(mcd[1]), int(bap[0]), int(bap[1]), int(lf0_col), int(vuv_col),
                                1 if lf0_linear else 0, int(mse[0]), int(mse[1]))
    out = torch.empty(8, dtype=torch.float32, device=y.device)
    ws = workspace(lib.gantts_distortions_workspace_bytes(), y.device, "distortions")
    _lib.check(lib.gantts_distortions(y.data_ptr(), y.stride(0), y.stride(1), y_hat.data_ptr(), y_hat.stride(0),
                                      y_hat.stride(1), lengths.data_ptr(), B, T, D, mean.contiguous().data_ptr(),
                                      std.contiguous().data_ptr(), ctypes.byref(cols), out.data_ptr(),
                                      ws.data_ptr(), ws.numel(), _stream()))
    return out


def unit_variance_mlpg(R, means):
    """Drop-in for nnmnkwii.autograd.unit_variance_mlpg(R, means) (reference
    gantts/multistream.py:120, gantts/models.py:66,115): means (B, T, nw*sd) or (T, nw*sd)."""
    windows, T = windows_from_R(R)
    if means.shape[-2] != T:
        raise RuntimeError("gantts_b200: means has %d frames but R was built for T=%d" % (means.shape[-2], T))
    nw = len(windows)
    D = means.shape[-1]
    if D % nw:
        raise RuntimeError("gantts_b200: feature dim %d not divisible by num_windows %d" % (D, nw))
    sd = D // nw
    return mlpg(means, windows, [(0, sd, True, 0)], sd)


# ---------------------------------------------------------------------------- column gather
_cols_cache = {}


def _cols_tensor(cols, device):
    key = (tuple(cols), device.index)
    t = _cols_cache.get(key)
    if t is None:
        t = torch.tensor(list(cols), dtype=torch.int32, device=device)
        _cols_cache[key] = t
    return t


class _GatherCols(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, cols):
        require_cuda(x)
        lib = _lib.load()
        x2, rs = _rows2d(x)
        rows = x2.shape[0]
        out = torch.empty(x.shape[:-1] + (len(cols),), dtype=torch.float32, device=x.device)
        ct = _cols_tensor(cols, x.device)
        _lib.check(lib.gantts_gather_cols(x2.data_ptr(), rs, out.data_ptr(), len(cols), ct.data_ptr(),
                                          len(cols), rows, _stream()))
        ctx.cols, ctx.in_shape = cols, tuple(x.shape)
        return out

    @staticmethod
    def backward(ctx, go):
        lib = _lib.load()
        go = go.contiguous()
        gi = torch.zeros(ctx.in_shape, dtype=torch.float32, device=go.device)
        rows = gi.numel() // ctx.in_shape[-1]
        ct = _cols_tensor(ctx.cols, go.device)
        _lib.check(lib.gantts_scatter_cols_add(go.data_ptr(), len(ctx.cols), gi.data_ptr(),
                                               ctx.in_shape[-1], ct.data_ptr(), len(ctx.cols), rows,
                                               _stream()))
        return gi, None


def gather_cols(x, cols):
    cols = tuple(int(c) for c in cols)
    if len(cols) == 0:
        raise RuntimeError("gantts_b200: empty column selection")
    return _GatherCols.apply(x, cols)


# ------------------------------------------------------------------------------ masks/losses
def sequence_mask(lengths, max_len):
    lib = _lib.load()
    if not lengths.is_cuda:
        raise RuntimeError("gantts_b200: CUDA lengths tensor required; this package has no CPU fallback")
    lengths = lengths.long().contiguous().view(-1)
    B = lengths.numel()
    mask = torch.empty(B, int(max_len), dtype=torch.float32, device=lengths.device)
    _lib.check(lib.gantts_sequence_mask(lengths.data_ptr(), mask.data_ptr(), B, int(max_len), _stream()))
    return mask


class _MaskedSSE(torch.autograd.Function):
    """sums = [sum(((a-b)*m)^2), sum(m)]"""

    @staticmethod
    def forward(ctx, a, b, mask):
        require_cuda(a, b, mask)
        lib = _lib.load()
        a2, ars = _rows2d(a)
        b2, brs = _rows2d(b)
        m = mask.reshape(-1).contiguous()
        rows, D = a2.shape
        if m.numel() != rows or b2.shape != a2.shape:
            raise RuntimeError("gantts_b200: masked MSE shape mismatch")
        sums = torch.empty(2, dtype=torch.float32, device=a.device)
        nb = lib.gantts_masked_sse_workspace_bytes()
        ws = workspace(nb, a.device, "red")
        _lib.check(lib.gantts_masked_sse_fwd(a2.data_ptr(), ars, b2.data_ptr(), brs, m.data_ptr(), rows, D,
                                             sums.data_ptr(), ws.data_ptr(), ws.numel(), _stream()))
        ctx.save_for_backward(a2, b2, m)
        ctx.strides = (ars, brs)
        ctx.shape = tuple(a.shape)
        return sums

    @staticmethod
    def backward(ctx, gsums):
        lib = _lib.load()
        a2, b2, m = ctx.saved_tensors
        rows, D = a2.shape
        scale = gsums[0:1].contiguous()
        ga = torch.empty(rows, D, dtype=torch.float32, device=a2.device)
        _lib.check(lib.gantts_masked_sse_bwd(a2.data_ptr(), ctx.strides[0], b2.data_ptr(), ctx.strides[1],
                                             m.data_ptr(), rows, D, scale.data_ptr(), ga.data_ptr(), D, 0,
                                             _stream()))
        return ga.view(ctx.shape), None, None


def masked_mse(inp, target, mask):
    """reference gantts/seqloss.py:41-43: sum((in*m - tgt*m)^2) / sum(m), m of shape (B, T, 1)."""
    sums = _MaskedSSE.apply(inp, target, mask)
    return sums[0] / sums[1]


class _MaskedBCE(torch.autograd.Function):
    """out = [-(log(arg) * m).sum(), count, sum(m)], arg = D+1e-20 (kind 0) or 1-D+1e-20 (kind 1)."""

    @staticmethod
    def forward(ctx, D, mask, kind):
        require_cuda(D, mask)
        lib = _lib.load()
        d = D.reshape(-1).contiguous()
        m = mask.reshape(-1).contiguous()
        if d.numel() != m.numel():
            raise RuntimeError("gantts_b200: masked BCE shape mismatch")
        out = torch.empty(3, dtype=torch.float32, device=D.device)
        ws = workspace(lib.gantts_masked_sse_workspace_bytes(), D.device, "red")
        _lib.check(lib.gantts_masked_bce_fwd(d.data_ptr(), m.data_ptr(), d.numel(), int(kind), out.data_ptr(),
                                             ws.data_ptr(), ws.numel(), _stream()))
        ctx.save_for_backward(d, m)
        ctx.kind, ctx.shape = int(kind), tuple(D.shape)
        return out

    @staticmethod
    def backward(ctx, gout):
        lib = _lib.load()
        d, m = ctx.saved_tensors
        scale = gout[0:1].contiguous()
        gD = torch.empty_like(d)
        _lib.check(lib.gantts_masked_bce_bwd(d.data_ptr(), m.data_ptr(), d.numel(), ctx.kind, scale.data_ptr(),
                                             gD.data_ptr(), _stream()))
        return gD.view(ctx.shape), None, None


def masked_bce(D, mask, kind):
    """Un-normalised adversarial BCE sum, correct-count and sum(mask) (reference train.py:258-271)."""
    return _MaskedBCE.apply(D, mask, kind)


# --------------------------------------------------------------------------- fused linear
class _LinearAct(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, W, b, act, slope, p, seed, engine):
        require_cuda(x, W, b)
        lib = _lib.load()
        x2, xrs = _rows2d(x)
        M, K = x2.shape
        N = W.shape[0]
        if W.shape[1] != K:
            raise RuntimeError("gantts_b200: linear shape mismatch (x has %d features, W expects %d)" % (K, W.shape[1]))
        Wc = W.contiguous()
        bc = b.contiguous() if b is not None else None
        y = torch.empty(M, N, dtype=torch.float32, device=x.device)
        nb = lib.gantts_linear_workspace_bytes(M, N, K, engine)
        ws = workspace(nb, x.device)
        _lib.check(lib.gantts_linear_fwd(x2.data_ptr(), xrs, Wc.data_ptr(), bc.data_ptr() if bc is not None else None,
                                         y.data_ptr(), N, M, N, K, act, slope, p, seed, engine,
                                         ws.data_ptr(), ws.numel(), _stream()))
        ctx.save_for_backward(x2, Wc, y)
        ctx.cfg = (xrs, act, slope, p, engine, b is not None, tuple(x.shape))
        return y.view(x.shape[:-1] + (N,))

    @staticmethod
    def backward(ctx, gy):
        lib = _lib.load()
        x2, W, y = ctx.saved_tensors
        xrs, act, slope, p, engine, has_bias, xshape = ctx.cfg
        M, K = x2.shape
        N = W.shape[0]
        gy2, gyrs = _rows2d(gy)
        need_gx, need_gW, need_gb = ctx.needs_input_grad[0], ctx.needs_input_grad[1], (has_bias and ctx.needs_input_grad[2])
        gz = torch.empty(M, N, dtype=torch.float32, device=gy.device)
        gx = torch.empty(M, K, dtype=torch.float32, device=gy.device) if need_gx else None
        gW = torch.empty(N, K, dtype=torch.float32, device=gy.device) if need_gW else None
        gb = torch.empty(N, dtype=torch.float32, device=gy.device) if need_gb else None
        nb = lib.gantts_linear_workspace_bytes(M, N, K, engine)
        ws = workspace(nb, gy.device)
        _lib.check(lib.gantts_linear_bwd(gy2.data_ptr(), gyrs, y.data_ptr(), N, x2.data_ptr(), xrs, W.data_ptr(),
                                         gz.data_ptr(), gx.data_ptr() if gx is not None else None, K,
                                         gW.data_ptr() if gW is not None else None,
                                         gb.data_ptr() if gb is not None else None,
                                         M, N, K, act, slope, p, 0, engine, ws.data_ptr(), ws.numel(), _stream()))
        return (gx.view(xshape) if gx is not None else None), gW, gb, None, None, None, None, None


_seed_state = [None, 0]      # [torch.initial_seed() the counter belongs to, draws since then]


def draw_seed():
    """62-bit dropout seed, reproducible under torch.manual_seed: splitmix64 of (torch.initial_seed(), number
    of draws since the last manual_seed).  Pure host arithmetic -- no tensor op, no synchronisation (the old
    form went through torch.randint(...).item() once per dropout layer)."""
    base = torch.initial_seed()
    if _seed_state[0] != base:
        _seed_state[0], _seed_state[1] = base, 0
    _seed_state[1] += 1
    z = (base + 0x9E3779B97F4A7C15 * _seed_state[1]) & 0xFFFFFFFFFFFFFFFF
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & 0xFFFFFFFFFFFFFFFF
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & 0xFFFFFFFFFFFFFFFF
    return (z ^ (z >> 31)) & ((1 << 62) - 1)


def peek_seeds(n):
    """The next `n` values draw_seed() will return (test hook: regenerate the masks of a step about to run)."""
    saved = list(_seed_state)
    out = [draw_seed() for _ in range(n)]
    _seed_state[0], _seed_state[1] = saved
    if _seed_state[0] is None:
        _seed_state[0], _seed_state[1] = torch.initial_seed(), 0
    return out


def dropout_mask(rows, cols, p, seed, device):
    """The dropout multiplier {0, 1/(1-p)} every engine applies for (seed, rows, cols): float32 (rows, cols).
    Test hook for injected-mask parity against the CPU checker (gantts_dropout on a tensor of ones)."""
    lib = _lib.load()
    ones = torch.ones(int(rows), int(cols), dtype=torch.float32, device=device)
    out = torch.empty_like(ones)
    _lib.check(lib.gantts_dropout(ones.data_ptr(), out.data_ptr(), int(rows), int(cols), float(p), int(seed),
                                  _stream()))
    return out


def mlp_dropout_masks(rows, hidden_dims, p, seed, device):
    """Masks of the hidden layers of an MLP run (mlp_stack / gantts_mlp_fwd) with dropout seed `seed`."""
    lib = _lib.load()
    return [dropout_mask(rows, n, p, lib.gantts_mlp_layer_seed(int(seed), l), device)
            for l, n in enumerate(hidden_dims)]


def linear_act(x, W, b, act=_lib.ACT_NONE, p=0.0, training=False, slope=LEAKY_SLOPE, engine=None, seed=None):
    """act(x W^T + b): the reference's Linear -> LeakyReLU(0.01) -> Dropout(p) hidden layer
    (gantts/models.py:137-139), ``last_linear`` (act NONE) or Linear -> Sigmoid."""
    eng = config.engine_id(engine)
    p_eff = float(p) if (training and act == _lib.ACT_LEAKY_DROPOUT) else 0.0
    if p_eff > 0.0 and seed is None:
        seed = draw_seed()
    return _LinearAct.apply(x, W, b, int(act), float(slope), p_eff, int(seed or 0), eng)


# ------------------------------------------------------------------ whole MLP (tensor cores)
class _MLPStack(torch.autograd.Function):
    """y = MLP(x) through gantts_mlp_fwd / gantts_mlp_bwd: one wgmma GEMM per layer and direction,
    activations resident as bf16 hi/lo planes (the tape)."""

    @staticmethod
    def forward(ctx, x, slope, p, last_act, seed, *params):
        require_cuda(x, *params)
        lib = _lib.load()
        L = len(params) // 2
        if L > _lib.MAX_LAYERS:
            raise RuntimeError("gantts_b200: at most %d layers" % _lib.MAX_LAYERS)
        x2, xrs = _rows2d(x)
        M = x2.shape[0]
        Ws = [params[2 * i].contiguous() for i in range(L)]
        bs = [params[2 * i + 1].contiguous() for i in range(L)]
        d = _lib.MlpT()
        d.num_layers = L
        d.dims[0] = x2.shape[1]
        for i in range(L):
            if Ws[i].shape[1] != d.dims[i]:
                raise RuntimeError("gantts_b200: MLP layer %d expects %d inputs, got %d" % (i, Ws[i].shape[1], d.dims[i]))
            d.dims[i + 1] = Ws[i].shape[0]
            d.W[i] = Ws[i].data_ptr()
            d.b[i] = bs[i].data_ptr()
        d.slope, d.dropout_p, d.last_act, d.seed = float(slope), float(p), int(last_act), int(seed)
        N = d.dims[L]
        y = torch.empty(M, N, dtype=torch.float32, device=x.device)
        tape = torch.empty(lib.gantts_mlp_tape_bytes(ctypes.byref(d), M), dtype=torch.uint8, device=x.device)
        _lib.check(lib.gantts_mlp_fwd(ctypes.byref(d), x2.data_ptr(), xrs, M, y.data_ptr(), N, tape.data_ptr(),
                                      tape.numel(), _stream()))
        ctx.save_for_backward(tape, y, *Ws, *bs)
        ctx.cfg = (d.dims[:L + 1], float(slope), float(p), int(last_act), int(seed), tuple(x.shape))
        return y.view(x.shape[:-1] + (N,))

    @staticmethod
    def backward(ctx, gy):
        lib = _lib.load()
        saved = ctx.saved_tensors
        tape, y = saved[0], saved[1]
        dims, slope, p, last_act, seed, xshape = ctx.cfg
        L = len(dims) - 1
        Ws, bs = saved[2:2 + L], saved[2 + L:2 + 2 * L]
        d = _lib.MlpT()
        d.num_layers = L
        for i, v in enumerate(dims):
            d.dims[i] = v
        for i in range(L):
            d.W[i], d.b[i] = Ws[i].data_ptr(), bs[i].data_ptr()
        d.slope, d.dropout_p, d.last_act, d.seed = slope, p, last_act, seed
        gy2, gyrs = _rows2d(gy)
        M = gy2.shape[0]
        dev = gy.device
        need_gx = ctx.needs_input_grad[0]
        gx = torch.empty(M, dims[0], dtype=torch.float32, device=dev) if need_gx else None
        gWs = [torch.empty_like(W) if ctx.needs_input_grad[5 + 2 * i] else None for i, W in enumerate(Ws)]
        gbs = [torch.empty_like(b) if ctx.needs_input_grad[6 + 2 * i] else None for i, b in enumerate(bs)]
        arr = lambda ts: (ctypes.c_void_p * L)(*[t.data_ptr() if t is not None else None for t in ts])
        ws = workspace(lib.gantts_mlp_workspace_bytes(ctypes.byref(d), M), dev, "mlp")
        _lib.check(lib.gantts_mlp_bwd(ctypes.byref(d), gy2.data_ptr(), gyrs, y.data_ptr(), dims[L], M,
                                      tape.data_ptr(), tape.numel(), gx.data_ptr() if gx is not None else None,
                                      dims[0], arr(gWs), arr(gbs), 0, ws.data_ptr(), ws.numel(), _stream()))
        grads = []
        for i in range(L):
            grads += [gWs[i], gbs[i]]
        return (gx.view(xshape) if gx is not None else None, None, None, None, None) + tuple(grads)


def mlp_stack(x, weights, biases, p=0.0, training=False, last_act=_lib.ACT_NONE, slope=LEAKY_SLOPE, seed=None):
    """Whole MLP (hidden: Linear -> LeakyReLU -> Dropout; last: Linear [-> sigmoid]) on the tensor-core
    engine.  reference gantts/models.py:137-141."""
    p_eff = float(p) if training else 0.0
    if p_eff > 0.0 and seed is None:
        seed = draw_seed()
    params = []
    for W, b in zip(weights, biases):
        params += [W, b]
    return _MLPStack.apply(x, float(slope), p_eff, int(last_act), int(seed or 0), *params)


def highway_combine(x_static, Tx, Gx):
    """y = x_static + Tx * Gx (reference gantts/models.py:69)."""
    require_cuda(x_static, Tx, Gx)
    return torch.addcmul(x_static, Tx, Gx)
