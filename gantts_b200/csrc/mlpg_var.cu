// Inference-time parameter generation with real variances: nnmnkwii.paramgen.mlpg(mean_frames,
// variance_frames, windows) as called by the reference's evaluation scripts (evaluation_tts.py:70-72,
// 92-94; the package itself is not vendored, the maths is the published MLPG):
//     y = argmax N(W y; mu, Sigma)  <=>  (sum_w W_w^T diag(1/var_w) W_w) y = sum_w W_w^T diag(1/var_w) mu_w
// for every static dimension independently.  The system is banded SPD (half bandwidth hb = max_w(l_w + u_w),
// 2 for the reference windows).  One thread per (batch row, static dimension) assembles its band row by
// row, factors it (banded Cholesky) and substitutes forwards while walking t upwards, then substitutes
// backwards walking down; L and z live in a caller workspace laid out [t][slot][column] so that the
// threads of a warp (adjacent columns) touch adjacent addresses.  fp64 arithmetic like bandmat's.
// Latency-bound in T (sequential recurrence), parallel over B * sd columns; an inference-time op.
#include "common.cuh"

namespace gantts {

constexpr int MV_HB = GANTTS_MAX_WINDOW_TAPS - 1;   // largest half bandwidth of W^T W: l + u <= taps - 1

// The banded solve of one column: `mu(t, w)` is window w's mean at frame t, `tau(t, w)` its precision 1/var, both as
// doubles; `store(t, y)` receives the static trajectory.  The system is built over frames [0, T): its end boundary is T.
// L and z of frame t live in ws[t][slot][col] (slots = hb + 2, row pitch ncols).
template <class Mu, class Tau, class Store>
__device__ __forceinline__ void mlpg_band_solve(const gantts_windows_t& w, int T, int hb, double* __restrict__ ws,
                                                int64_t col, int64_t ncols, Mu mu, Tau tau, Store store) {
  const int slots = hb + 2;                               // L[i][i-hb..i] (hb+1 values) and z[i]
  // ring of the last MV_HB rows of L: Lr[r][k] = L[i-r-1][i-r-1-k]  (k = 0 is the diagonal)
  double Lr[MV_HB][MV_HB + 1];
  for (int r = 0; r < MV_HB; ++r)
    for (int k = 0; k <= MV_HB; ++k) Lr[r][k] = 0.0;
  double zr[MV_HB];
  for (int r = 0; r < MV_HB; ++r) zr[r] = 0.0;

  for (int i = 0; i < T; ++i) {
    // band row i of P (columns i-hb..i) and right-hand side
    double prow[MV_HB + 1];
    for (int k = 0; k <= MV_HB; ++k) prow[k] = 0.0;
    double rhs = 0.0;
    for (int wi = 0; wi < w.n; ++wi) {
      // rows t' of W_w touching column i: i - u <= t' <= i + l
      for (int tp = i - w.u[wi]; tp <= i + w.l[wi]; ++tp) {
        if (tp < 0 || tp >= T) continue;
        const double ci = (double)w.coef[wi][i - tp + w.l[wi]];
        const double ta = tau(tp, wi);
        rhs += ci * ta * mu(tp, wi);
        for (int k = 0; k <= hb; ++k) {
          const int j = i - k;                            // column j <= i
          const int off = j - tp + w.l[wi];
          if (j < 0 || off < 0 || off > w.l[wi] + w.u[wi]) continue;
          prow[k] += ci * ta * (double)w.coef[wi][off];
        }
      }
    }
    // Cholesky row: L[i][j] for j = i-hb..i   (lrow[k] = L[i][i-k])
    double lrow[MV_HB + 1];
    for (int k = 0; k <= MV_HB; ++k) lrow[k] = 0.0;
    for (int k = hb; k >= 0; --k) {
      const int j = i - k;
      if (j < 0) continue;
      double s = prow[k];
      // sum over m < j, m >= i - hb:  L[i][m] * L[j][m];  L[i][m] = lrow[i-m], L[j][m] = row j's entry (j-m)
      for (int m = i - hb; m < j; ++m) {
        if (m < 0) continue;
        const double lim = lrow[i - m];
        const double ljm = (k == 0) ? lim : Lr[k - 1][j - m];   // row j = i-k is ring slot k-1
        if (k == 0 || j - m <= hb) s -= lim * ljm;
      }
      if (k == 0) lrow[0] = sqrt(s);
      else lrow[k] = s / Lr[k - 1][0];
    }
    // forward substitution z[i] = (rhs - sum_{k>=1} L[i][i-k] z[i-k]) / L[i][i]
    double zz = rhs;
    for (int k = 1; k <= hb; ++k)
      if (i - k >= 0) zz -= lrow[k] * zr[k - 1];
    zz /= lrow[0];
    double* wrow = ws + ((int64_t)i * slots) * ncols + col;
    for (int k = 0; k <= hb; ++k) wrow[(int64_t)k * ncols] = lrow[k];
    wrow[(int64_t)(hb + 1) * ncols] = zz;
    // rotate the rings
    for (int r = MV_HB - 1; r > 0; --r) {
      for (int k = 0; k <= MV_HB; ++k) Lr[r][k] = Lr[r - 1][k];
      zr[r] = zr[r - 1];
    }
    for (int k = 0; k <= MV_HB; ++k) Lr[0][k] = lrow[k];
    zr[0] = zz;
  }
  // backward substitution L^T y = z: y[i] = (z[i] - sum_{k=1..hb} L[i+k][i] y[i+k]) / L[i][i]
  double yr[MV_HB];
  for (int r = 0; r < MV_HB; ++r) yr[r] = 0.0;
  // ring of L rows above: Lup[r][k] = L[i+r+1][i+r+1-k]
  for (int r = 0; r < MV_HB; ++r)
    for (int k = 0; k <= MV_HB; ++k) Lr[r][k] = 0.0;
  for (int i = T - 1; i >= 0; --i) {
    const double* wrow = ws + ((int64_t)i * slots) * ncols + col;
    double lrow[MV_HB + 1];
    for (int k = 0; k <= MV_HB; ++k) lrow[k] = k <= hb ? wrow[(int64_t)k * ncols] : 0.0;
    double yy = wrow[(int64_t)(hb + 1) * ncols];
    for (int k = 1; k <= hb; ++k)
      if (i + k < T) yy -= Lr[k - 1][k] * yr[k - 1];    // L[i+k][i] = row (i+k)'s entry k
    yy /= lrow[0];
    store(i, yy);
    for (int r = MV_HB - 1; r > 0; --r) {
      for (int k = 0; k <= MV_HB; ++k) Lr[r][k] = Lr[r - 1][k];
      yr[r] = yr[r - 1];
    }
    for (int k = 0; k <= MV_HB; ++k) Lr[0][k] = lrow[k];
    yr[0] = yy;
  }
}

__global__ void __launch_bounds__(128)
mlpg_var_kernel(const float* __restrict__ mean, int64_t m_bs, int64_t m_ts, const float* __restrict__ var,
                int64_t v_bs, int64_t v_ts, float* __restrict__ out, int64_t o_bs, int64_t o_ts,
                const gantts_windows_t w, int B, int T, int sd, int hb, double* __restrict__ ws) {
  const int64_t col = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t ncols = (int64_t)B * sd;
  if (col >= ncols) return;
  const int b = (int)(col / sd), d = (int)(col - (int64_t)b * sd);
  const float* mu = mean + b * m_bs + d;
  const float* vr = var + b * v_bs + d;
  float* o = out + b * o_bs + d;
  mlpg_band_solve(
      w, T, hb, ws, col, ncols,
      [&](int tp, int wi) { return (double)mu[(int64_t)tp * m_ts + (int64_t)wi * sd]; },
      [&](int tp, int wi) { return 1.0 / (double)vr[(int64_t)tp * v_ts + (int64_t)wi * sd]; },
      [&](int i, double y) { o[(int64_t)i * o_ts] = (float)y; });
}

// Length-exact multi-stream MLPG of generation (gantts_mlpg_ragged).  One thread per (batch row, static output column),
// columns enumerated stream by stream.  Row b's system is built over its own L = lengths[b] frames, so nothing a thread
// reads or writes depends on the padded T; frames [L, T) are written as 0.  The optional affine maps are applied as the
// means are read (prologue) and as the trajectory is stored (epilogue), in double like the solve.
struct MlpgRaggedParams {
  const float* in;
  int64_t i_bs, i_ts;
  const float* var;                          // [input columns] time-invariant variances, or null (unit)
  const float *in_scale, *in_shift;          // [input columns] or null
  const float *out_scale, *out_shift;        // [output columns] or null
  float* out;
  int64_t o_bs, o_ts;
  const int64_t* lengths;
  gantts_streams_t s;
  gantts_windows_t w;
  int B, T, n_static, hb;                    // n_static: static output columns of one row (sum of the streams' sd)
  double* ws;
};

__global__ void __launch_bounds__(128) mlpg_ragged_kernel(const MlpgRaggedParams p) {
  const int64_t col = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t ncols = (int64_t)p.B * p.n_static;
  if (col >= ncols) return;
  const int b = (int)(col / p.n_static);
  int d = (int)(col - (int64_t)b * p.n_static), st = 0;
  while (d >= p.s.sd[st]) d -= p.s.sd[st++];
  const int sd = p.s.sd[st], dyn = p.s.dyn[st], oc = p.s.out_start[st] + d;
  const int64_t Lraw = p.lengths[b];
  const int L = Lraw < 0 ? 0 : (Lraw > p.T ? p.T : (int)Lraw);
  const float* x = p.in + b * p.i_bs;
  float* o = p.out + b * p.o_bs + oc;
  const double osc = p.out_scale ? (double)p.out_scale[oc] : 1.0, osh = p.out_shift ? (double)p.out_shift[oc] : 0.0;
  // per window: input column, precision and prologue map of this thread's dimension
  const int nw = dyn ? p.w.n : 1;
  int ic[GANTTS_MAX_WINDOWS];
  double tw[GANTTS_MAX_WINDOWS], isc[GANTTS_MAX_WINDOWS], ish[GANTTS_MAX_WINDOWS];
#pragma unroll
  for (int wi = 0; wi < GANTTS_MAX_WINDOWS; ++wi) {
    const int c = p.s.in_start[st] + (wi < nw ? wi : 0) * sd + d;
    ic[wi] = c;
    tw[wi] = p.var ? 1.0 / (double)p.var[c] : 1.0;
    isc[wi] = p.in_scale ? (double)p.in_scale[c] : 1.0;
    ish[wi] = p.in_shift ? (double)p.in_shift[c] : 0.0;
  }
  auto mu = [&](int t, int wi) { return (double)x[(int64_t)t * p.i_ts + ic[wi]] * isc[wi] + ish[wi]; };
  auto store = [&](int t, double y) { o[(int64_t)t * p.o_ts] = (float)(y * osc + osh); };
  if (dyn) {
    mlpg_band_solve(p.w, L, p.hb, p.ws, col, ncols, mu, [&](int, int wi) { return tw[wi]; }, store);
  } else {
    for (int t = 0; t < L; ++t) store(t, mu(t, 0));
  }
  for (int t = L; t < p.T; ++t) o[(int64_t)t * p.o_ts] = 0.f;
}

static int windows_half_band(const gantts_windows_t* w) {
  int hb = 0;
  for (int i = 0; i < w->n; ++i)
    if (w->l[i] + w->u[i] > hb) hb = w->l[i] + w->u[i];
  return hb;
}

}  // namespace gantts

using namespace gantts;

extern "C" size_t gantts_mlpg_var_workspace_bytes(const gantts_windows_t* windows, int B, int T, int sd) {
  if (!windows || B < 1 || T < 1 || sd < 1) return 0;
  return (size_t)T * (size_t)(windows_half_band(windows) + 2) * (size_t)B * sd * sizeof(double) + 256;
}

extern "C" int gantts_mlpg_var(const float* mean, int64_t m_bstride, int64_t m_tstride, const float* var,
                               int64_t v_bstride, int64_t v_tstride, float* out, int64_t o_bstride,
                               int64_t o_tstride, const gantts_windows_t* windows, int B, int T, int sd,
                               void* workspace, size_t workspace_bytes, void* stream) {
  GANTTS_CHECK_ARG(mean && var && out && windows, "mlpg_var: null argument");
  GANTTS_CHECK_ARG(B >= 1 && T >= 1 && sd >= 1, "mlpg_var: bad sizes");
  GANTTS_CHECK_ARG(windows->n >= 1 && windows->n <= GANTTS_MAX_WINDOWS, "mlpg_var: bad window count");
  for (int i = 0; i < windows->n; ++i)
    GANTTS_CHECK_ARG(windows->l[i] >= 0 && windows->u[i] >= 0 &&
                         windows->l[i] + windows->u[i] + 1 <= GANTTS_MAX_WINDOW_TAPS,
                     "mlpg_var: window too wide");
  const int hb = windows_half_band(windows);
  const size_t need = gantts_mlpg_var_workspace_bytes(windows, B, T, sd);
  if (!workspace || workspace_bytes < need) {
    set_error("mlpg_var: workspace too small (%zu < %zu)", workspace_bytes, need);
    return GANTTS_E_WORKSPACE;
  }
  double* ws = reinterpret_cast<double*>((reinterpret_cast<uintptr_t>(workspace) + 255) / 256 * 256);
  const int64_t ncols = (int64_t)B * sd;
  mlpg_var_kernel<<<(unsigned)((ncols + 127) / 128), 128, 0, as_stream(stream)>>>(
      mean, m_bstride, m_tstride, var, v_bstride, v_tstride, out, o_bstride, o_tstride, *windows, B, T, sd, hb, ws);
  GANTTS_LAUNCH_CHECK("mlpg_var_kernel");
  return GANTTS_OK;
}

namespace gantts {

constexpr int MLPG_RAGGED_MAX_T = 1 << 24;

// The rules of gantts_mlpg_ragged's descriptors, shared by the workspace query and the call; sets the error message and
// returns the number of static output columns of one row, or 0.
static int mlpg_ragged_check(const gantts_streams_t* s, const gantts_windows_t* w, const int64_t* lengths_dev, int B,
                             int T) {
  if (!s || !w) {
    set_error("mlpg_ragged: null stream or window table");
    return 0;
  }
  if (!lengths_dev) {
    set_error("mlpg_ragged: null lengths: every row is solved over its own lengths_dev[b] frames");
    return 0;
  }
  if (B < 1) {
    set_error("mlpg_ragged: batch size B = %d must be >= 1", B);
    return 0;
  }
  if (T < 1 || T > MLPG_RAGGED_MAX_T) {
    set_error("mlpg_ragged: padded length T = %d must be in [1, %d]", T, MLPG_RAGGED_MAX_T);
    return 0;
  }
  if (s->n < 1 || s->n > GANTTS_MAX_STREAMS) {
    set_error("mlpg_ragged: stream count %d must be in [1, %d]", s->n, GANTTS_MAX_STREAMS);
    return 0;
  }
  if (w->n < 1 || w->n > GANTTS_MAX_WINDOWS) {
    set_error("mlpg_ragged: window count %d must be in [1, %d]", w->n, GANTTS_MAX_WINDOWS);
    return 0;
  }
  for (int i = 0; i < w->n; ++i)
    if (w->l[i] < 0 || w->u[i] < 0 || w->l[i] + w->u[i] + 1 > GANTTS_MAX_WINDOW_TAPS) {
      set_error("mlpg_ragged: window %d taps out of range (l = %d, u = %d, at most %d taps)", i, w->l[i], w->u[i],
                GANTTS_MAX_WINDOW_TAPS);
      return 0;
    }
  int64_t n_static = 0;
  for (int i = 0; i < s->n; ++i) {
    if (s->sd[i] < 1 || s->sd[i] > GANTTS_MAX_COLS) {
      set_error("mlpg_ragged: stream %d static width sd = %d must be in [1, %d]", i, s->sd[i], GANTTS_MAX_COLS);
      return 0;
    }
    if (s->in_start[i] < 0 || s->out_start[i] < 0) {
      set_error("mlpg_ragged: stream %d has a negative column start", i);
      return 0;
    }
    n_static += s->sd[i];
  }
  if (n_static * B > (int64_t)1 << 30) {
    set_error("mlpg_ragged: B * static columns = %lld exceeds 2^30", (long long)(n_static * B));
    return 0;
  }
  return (int)n_static;
}

}  // namespace gantts

extern "C" size_t gantts_mlpg_ragged_workspace_bytes(const gantts_streams_t* streams, const gantts_windows_t* windows,
                                                     const int64_t* lengths_dev, int B, int T) {
  const int n_static = mlpg_ragged_check(streams, windows, lengths_dev, B, T);
  if (!n_static) return 0;
  return (size_t)T * (size_t)(windows_half_band(windows) + 2) * (size_t)B * (size_t)n_static * sizeof(double) + 256;
}

extern "C" int gantts_mlpg_ragged(const float* in, int64_t in_bstride, int64_t in_tstride, const float* var,
                                  const float* in_scale, const float* in_shift, float* out, int64_t out_bstride,
                                  int64_t out_tstride, const float* out_scale, const float* out_shift,
                                  const gantts_streams_t* streams, const gantts_windows_t* windows,
                                  const int64_t* lengths_dev, int B, int T, void* workspace, size_t workspace_bytes,
                                  void* stream) {
  const int n_static = mlpg_ragged_check(streams, windows, lengths_dev, B, T);
  if (!n_static) return GANTTS_E_BADARG;
  GANTTS_CHECK_ARG(in && out, "mlpg_ragged: null input or output");
  GANTTS_CHECK_ARG((in_scale == nullptr) == (in_shift == nullptr) && (out_scale == nullptr) == (out_shift == nullptr),
                   "mlpg_ragged: an affine map needs both its scale and its shift");
  const size_t need = gantts_mlpg_ragged_workspace_bytes(streams, windows, lengths_dev, B, T);
  if (!workspace || workspace_bytes < need) {
    set_error("mlpg_ragged: workspace too small (%zu < %zu)", workspace_bytes, need);
    return GANTTS_E_WORKSPACE;
  }
  MlpgRaggedParams p{};
  p.in = in; p.i_bs = in_bstride; p.i_ts = in_tstride;
  p.var = var; p.in_scale = in_scale; p.in_shift = in_shift; p.out_scale = out_scale; p.out_shift = out_shift;
  p.out = out; p.o_bs = out_bstride; p.o_ts = out_tstride;
  p.lengths = lengths_dev;
  p.s = *streams; p.w = *windows;
  p.B = B; p.T = T; p.n_static = n_static; p.hb = windows_half_band(windows);
  p.ws = reinterpret_cast<double*>((reinterpret_cast<uintptr_t>(workspace) + 255) / 256 * 256);
  const int64_t ncols = (int64_t)B * n_static;
  mlpg_ragged_kernel<<<(unsigned)((ncols + 127) / 128), 128, 0, as_stream(stream)>>>(p);
  GANTTS_LAUNCH_CHECK("mlpg_ragged_kernel");
  return GANTTS_OK;
}
