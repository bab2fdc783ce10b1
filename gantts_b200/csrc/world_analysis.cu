// WORLD's waveform analysis on padded device batches, as the reference notebooks run it on the natural wavs (Test VC.ipynb,
// Test RNN VC.ipynb compute_static_features; Test TTS.ipynb compute_mgc_from_waveform): pyworld.dio, pyworld.stonemask,
// pyworld.cheaptrick with pyworld's defaults, pysptk.sp2mc and nnmnkwii.preprocessing.modspec_smoothing, all in fp64.
//
//   dio          a fixed-order mean per row; the low-cut filter and each band's Nuttall low-pass as direct FIR sums (taps
//                ascending, no FMA); per (band, row) one block finds the four kinds of zero crossing of a tile of samples
//                in parallel and compacts them in sample order by a ballot scan; per (frame, band) WORLD's interp1 of the
//                four interval series at the frame time and the candidate's score; per row the best band of every frame
//                in parallel, then FixF0Contour, whose steps 3 and 4 are sequential over frames, on one thread
//   stonemask    one block per (frame, row): the two windowed waveforms' real FFTs in shared memory (common.cuh)
//   cheaptrick   one block per (frame, row); frame t reads WORLD's randn stream from its draw offset, a prefix sum of the
//                earlier frames' draw counts, out of one copy of the stream made by gantts_world_randn (WORLD reseeds it
//                per utterance, so every row reads the same stream)
//   sp2mc        one block per (frame, row): log sp times the (K x M+1) operator of gantts_sp2mc_operator
//   smoothing    one block per (column, row): the column's real FFT, the bins from the cut-off on zeroed, the inverse
//
// The scalar arithmetic of DIO uses __dmul_rn / __dadd_rn / __dsub_rn so that it rounds as the C code does.  A row's
// results depend only on that row.  The status word (GANTTS_ANALYSIS_*) is the only value written with an atomic.
#include "common.cuh"

#include <math.h>

namespace gantts {

constexpr int WA_THREADS = 256;
constexpr int WA_TILE = 2048;               // samples per step of the crossing search
constexpr int WA_MAX_BANDS = 8;
constexpr int WA_MAX_FFT = 4096;
constexpr int WA_MIN_FS = 4000;
constexpr int WA_MAX_FS = 96000;
constexpr int WA_MAX_S = 1 << 28;
constexpr double WA_F0_FLOOR = 71.0;        // pyworld's dio / cheaptrick f0_floor
constexpr double WA_F0_CEIL = 800.0;
constexpr double WA_CHANNELS = 2.0;         // channels_in_octave
constexpr double WA_ALLOWED = 0.1;          // allowed_range
constexpr double WA_CUTOFF = 50.0;          // dio.cpp kCutOff
constexpr double WA_MAXV = 100000.0;        // dio.cpp kMaximumValue
constexpr double WA_LOG2 = 0.69314718055994529;
constexpr double WA_FLOOR_SM = 40.0;        // kFloorF0StoneMask
constexpr double WA_EPS = 2.220446049250313e-16;
constexpr double WA_Q1 = -0.15;

__host__ __device__ inline int wa_round(double x) { return x > 0 ? (int)(x + 0.5) : (int)(x - 0.5); }

__host__ __device__ inline int64_t dio_frames(int64_t samples, int fs, double fp) {
  return (int64_t)(1000.0 * (double)samples / fs / fp) + 1;
}

__host__ __device__ inline int dio_voice_range(double fp) { return (int)(0.5 + 1000.0 / fp / WA_F0_FLOOR) * 2 + 1; }

static int dio_bands() { return 1 + (int)(log(WA_F0_CEIL / WA_F0_FLOOR) / WA_LOG2 * WA_CHANNELS); }

__device__ __forceinline__ int wa_len(const int64_t* lengths, int b, int S) {
  const int64_t L = lengths[b];
  return L < 0 ? 0 : (L > S ? S : (int)L);
}

__device__ __forceinline__ void wa_flag(int64_t* status, int bit) {
  atomicOr(reinterpret_cast<unsigned long long*>(status), (unsigned long long)bit);
}

// ---------------------------------------------------------------------------------------------- DIO
struct DioParams {
  const double* x;
  int64_t xs;
  const int64_t* lengths;
  int B, S, T, fs, nb, N, P, Z;             // N low-cut taps, z on [-P, L + P] (Z = S + 1 + 2P per row)
  double fp;
  int h[WA_MAX_BANDS], nut_off[WA_MAX_BANDS];
  double boundary[WA_MAX_BANDS];
  int cap;                                  // fine edges per (row, band, kind)
  double* taps;                             // [N] low-cut kernel, then each band's Nuttall window
  double* mean;                             // [B]
  double* z;                                // [B][Z]
  double* edges;                            // [B][nb][4][cap]
  int* counts;                              // [B][nb][4]
  double* cand;                             // [B][nb][T]
  double* score;                            // [B][nb][T]
  double* work;                             // [B][2][T]
  double* f0;                               // [B][T]
  int64_t* info;                            // [B] frame counts, [1] status
};

__device__ __forceinline__ bool dio_row_ok(const DioParams& p, int b, int L) {
  return dio_frames(L, p.fs, p.fp) > dio_voice_range(p.fp);
}

// DesignLowCutFilter as a zero-phase kernel (-hann / sum, plus 1 at the centre), and every band's Nuttall window.
__global__ void __launch_bounds__(WA_THREADS) dio_taps_kernel(const DioParams p) {
  const int N = p.N;
  double* g = p.taps;
  // rounded as the C code rounds (no FMA contraction)
  for (int i = threadIdx.x; i < N; i += blockDim.x)
    g[i] = __dsub_rn(0.5, __dmul_rn(0.5, cos(__dmul_rn((double)(i + 1), 2.0 * WD_PI) / (N + 1))));
  for (int band = 0; band < p.nb; ++band) {
    const int n = 4 * p.h[band];
    double* w = p.taps + p.nut_off[band];
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      const double t = i / (n - 1.0);
      const double a = __dmul_rn(0.487396, cos(__dmul_rn(2.0 * WD_PI, t)));
      const double c = __dmul_rn(0.144232, cos(__dmul_rn(4.0 * WD_PI, t)));
      const double d = __dmul_rn(0.012604, cos(__dmul_rn(6.0 * WD_PI, t)));
      w[i] = __dsub_rn(__dadd_rn(__dsub_rn(0.355768, a), c), d);
    }
  }
  __syncthreads();
  __shared__ double tot;
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int i = 0; i < N; ++i) s += g[i];
    tot = s;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < N; i += blockDim.x) {
    const double v = -g[i] / tot;
    g[i] = i == (N - 1) / 2 ? v + 1.0 : v;
  }
}

// One block per row: the status, the frame count and the mean over the L + 1 samples WORLD filters (the last is 0).
__global__ void __launch_bounds__(WA_THREADS) dio_prepare_kernel(const DioParams p) {
  __shared__ double red[32];
  const int b = blockIdx.x;
  const int L = wa_len(p.lengths, b, p.S);
  const double* x = p.x + (int64_t)b * p.xs;
  bool bad = false;
  double part = 0.0;
  for (int i = threadIdx.x; i < L; i += blockDim.x) {
    bad |= !isfinite(x[i]);
    part = __dadd_rn(part, x[i]);
  }
  if (bad) wa_flag(p.info + p.B, GANTTS_ANALYSIS_BAD_INPUT);
  const double s = block_sum_f64(part, red);
  if (threadIdx.x == 0) {
    const int64_t F = dio_frames(L, p.fs, p.fp);
    p.info[b] = F;
    p.mean[b] = s / (double)(L + 1);
    if (!dio_row_ok(p, b, L)) wa_flag(p.info + p.B, GANTTS_ANALYSIS_SHORT);
  }
}

// z[m] = sum_j g[j] y[m + c - j], j ascending, for m in [-P, L + P]; y = x - mean on [0, L] (y[L] = -mean), else 0.
__global__ void __launch_bounds__(WA_THREADS) dio_lowcut_kernel(const DioParams p) {
  extern __shared__ double wa_smem[];
  const int b = blockIdx.y, N = p.N, c = (N - 1) / 2;
  const int L = wa_len(p.lengths, b, p.S);
  const int m0 = blockIdx.x * WA_THREADS - p.P;            // first output of the block
  if (!dio_row_ok(p, b, L) || m0 > L + p.P) return;
  double* g = wa_smem;
  double* y = g + N;                                     // y[m0 + c - (N - 1) + q], q < WA_THREADS + N - 1
  const double* x = p.x + (int64_t)b * p.xs;
  const double mean = p.mean[b];
  const int y0 = m0 + c - (N - 1);
  for (int i = threadIdx.x; i < N; i += blockDim.x) g[i] = p.taps[i];
  for (int q = threadIdx.x; q < WA_THREADS + N - 1; q += blockDim.x) {
    const int i = y0 + q;
    y[q] = (i < 0 || i > L) ? 0.0 : __dsub_rn(i < L ? x[i] : 0.0, mean);
  }
  __syncthreads();
  const int m = m0 + threadIdx.x;
  if (m > L + p.P) return;
  double acc = 0.0;
  const double* yy = y + threadIdx.x + (N - 1);          // y[m + c - j] = yy[-j]
  for (int j = 0; j < N; ++j) acc = __dadd_rn(acc, __dmul_rn(g[j], yy[-j]));
  p.z[(int64_t)b * p.Z + (m + p.P)] = acc;
}

// fine edge of a crossing from a > 0 to b <= 0 between samples e - 1 and e: e - a / (b - a)
__device__ __forceinline__ double fine_edge(int e, double a, double bb) {
  return __dsub_rn((double)e, __ddiv_rn(a, __dsub_rn(bb, a)));
}

// One block per (band, row): s[i] = sum_k w[k] z[i + 2h - k] over the Y = L + 1 samples, tile by tile, and the fine
// edges of its negative-going (s), positive-going (-s), peak (d) and dip (-d) crossings, d[i] = (-s[i]) - (-s[i+1]),
// compacted in sample order.
__global__ void __launch_bounds__(WA_THREADS) dio_band_kernel(const DioParams p) {
  extern __shared__ double wa_smem[];
  __shared__ int warp_cnt[4][WA_THREADS / 32];
  __shared__ int found[4];
  const int band = blockIdx.x, b = blockIdx.y, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int L = wa_len(p.lengths, b, p.S);
  if (!dio_row_ok(p, b, L)) return;
  const int Y = L + 1, h = p.h[band], K = 4 * h;
  double* w = wa_smem;                                   // [K]
  double* s = w + K;                                     // [WA_TILE + 2]
  for (int k = threadIdx.x; k < K; k += blockDim.x) w[k] = p.taps[p.nut_off[band] + k];
  if (threadIdx.x < 4) found[threadIdx.x] = 0;
  const double* z = p.z + (int64_t)b * p.Z + p.P + 2 * h;  // z[i + 2h - k] = z[i - k]
  double* edges = p.edges + ((int64_t)b * p.nb + band) * 4 * p.cap;
  __syncthreads();
  for (int i0 = 0; i0 < Y; i0 += WA_TILE) {
    const int cnt = min(WA_TILE + 2, Y - i0);
    for (int q = threadIdx.x; q < cnt; q += blockDim.x) {
      const double* zz = z + i0 + q;
      double acc = 0.0;
      for (int k = 0; k < K; ++k) acc = __dadd_rn(acc, __dmul_rn(w[k], zz[-k]));
      s[q] = acc;
    }
    __syncthreads();
    for (int q0 = 0; q0 < min(WA_TILE, cnt); q0 += blockDim.x) {
      const int q = q0 + threadIdx.x, i = i0 + q;
      bool f[4] = {false, false, false, false};
      double fe[4];
      if (q < WA_TILE && i + 1 < Y) {
        const double s0 = s[q], s1 = s[q + 1];
        f[0] = s0 > 0.0 && s1 <= 0.0;
        if (f[0]) fe[0] = fine_edge(i + 1, s0, s1);
        f[1] = -s0 > 0.0 && -s1 <= 0.0;
        if (f[1]) fe[1] = fine_edge(i + 1, -s0, -s1);
        if (i + 2 < Y) {
          const double d0 = __dsub_rn(-s0, -s1), d1 = __dsub_rn(-s1, -s[q + 2]);
          f[2] = d0 > 0.0 && d1 <= 0.0;
          if (f[2]) fe[2] = fine_edge(i + 1, d0, d1);
          f[3] = -d0 > 0.0 && -d1 <= 0.0;
          if (f[3]) fe[3] = fine_edge(i + 1, -d0, -d1);
        }
      }
      unsigned bal[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        bal[k] = __ballot_sync(0xffffffffu, f[k]);
        if (lane == 0) warp_cnt[k][warp] = __popc(bal[k]);
      }
      __syncthreads();
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        if (!f[k]) continue;
        int before = 0;
        for (int v = 0; v < warp; ++v) before += warp_cnt[k][v];
        const int r = found[k] + before + __popc(bal[k] & ((1u << lane) - 1u));
        if (r < p.cap) edges[(int64_t)k * p.cap + r] = fe[k];
      }
      __syncthreads();
      if (threadIdx.x < 4) {
        int t = 0;
        for (int v = 0; v < WA_THREADS / 32; ++v) t += warp_cnt[threadIdx.x][v];
        found[threadIdx.x] += t;
      }
      __syncthreads();
    }
  }
  if (threadIdx.x < 4) p.counts[((int64_t)b * p.nb + band) * 4 + threadIdx.x] = min(found[threadIdx.x], p.cap);
}

// WORLD's interp1 of the intervals fs / (fe[i+1] - fe[i]) at their locations (fe[i] + fe[i+1]) / 2 / fs, at t
__device__ double interval_at(const double* fe, int n, double fs, double t) {
  auto loc = [&](int i) { return __ddiv_rn(__ddiv_rn(__dadd_rn(fe[i], fe[i + 1]), 2.0), fs); };
  int lo = 0, hi = n;                                    // the number of locations <= t
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (loc(mid) <= t) lo = mid + 1; else hi = mid;
  }
  const int k = min(max(lo - 1, 0), n - 2);
  const double x0 = loc(k), x1 = loc(k + 1);
  const double y0 = __ddiv_rn(fs, __dsub_rn(fe[k + 1], fe[k])), y1 = __ddiv_rn(fs, __dsub_rn(fe[k + 2], fe[k + 1]));
  const double sl = __ddiv_rn(__dsub_rn(t, x0), __dsub_rn(x1, x0));
  return __dadd_rn(y0, __dmul_rn(sl, __dsub_rn(y1, y0)));
}

// One thread per (frame, band, row): the band's candidate and its score / (candidate + 1e-12).
__global__ void __launch_bounds__(WA_THREADS) dio_candidate_kernel(const DioParams p) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x, band = blockIdx.y, b = blockIdx.z;
  const int L = wa_len(p.lengths, b, p.S);
  if (!dio_row_ok(p, b, L) || j >= dio_frames(L, p.fs, p.fp)) return;
  const int* cnt = p.counts + ((int64_t)b * p.nb + band) * 4;
  const double* edges = p.edges + ((int64_t)b * p.nb + band) * 4 * p.cap;
  const int64_t o = ((int64_t)b * p.nb + band) * p.T + j;
  bool enough = true;
  for (int k = 0; k < 4; ++k) enough &= cnt[k] - 1 - 2 > 0;
  if (!enough) {
    p.cand[o] = 0.0;
    p.score[o] = WA_MAXV / 1e-12;
    return;
  }
  const double t = __ddiv_rn(__dmul_rn((double)j, p.fp), 1000.0);
  const double fs = (double)p.fs;
  double v[4];
  for (int k = 0; k < 4; ++k) v[k] = interval_at(edges + (int64_t)k * p.cap, cnt[k] - 1, fs, t);
  const double c = __ddiv_rn(__dadd_rn(__dadd_rn(__dadd_rn(v[0], v[1]), v[2]), v[3]), 4.0);
  double ss = 0.0;
  for (int k = 0; k < 4; ++k) {
    const double e = __dsub_rn(v[k], c);
    ss = __dadd_rn(ss, __dmul_rn(e, e));
  }
  double score = sqrt(__ddiv_rn(ss, 3.0));
  double cand = c;
  const double bd = p.boundary[band];
  if (cand > bd || cand < bd / 2.0 || cand > WA_F0_CEIL || cand < WA_F0_FLOOR) {
    cand = 0.0;
    score = WA_MAXV;
  }
  p.cand[o] = cand;
  p.score[o] = __ddiv_rn(score, __dadd_rn(cand, 1e-12));
}

__device__ double select_best_f0(const DioParams& p, int b, double cur, double past, int j) {
  const double ref = __ddiv_rn(__dsub_rn(__dmul_rn(cur, 3.0), past), 2.0);
  const double* cand = p.cand + (int64_t)b * p.nb * p.T + j;
  double err = fabs(__dsub_rn(ref, cand[0])), best = cand[0];
  for (int i = 1; i < p.nb; ++i) {
    const double e = fabs(__dsub_rn(ref, cand[(int64_t)i * p.T]));
    if (e < err) {
      err = e;
      best = cand[(int64_t)i * p.T];
    }
  }
  return fabs(__dsub_rn(1.0, __ddiv_rn(best, ref))) > WA_ALLOWED ? 0.0 : best;
}

// One block per row: GetBestF0Contour and FixF0Contour's steps 1 and 2 in parallel, steps 3 and 4 on thread 0.
__global__ void __launch_bounds__(WA_THREADS) dio_fix_kernel(const DioParams p) {
  const int b = blockIdx.x;
  const int L = wa_len(p.lengths, b, p.S);
  double* f0 = p.f0 + (int64_t)b * p.T;
  const int F = (int)dio_frames(L, p.fs, p.fp);
  if (!dio_row_ok(p, b, L)) {
    for (int j = threadIdx.x; j < p.T; j += blockDim.x) f0[j] = 0.0;
    return;
  }
  const int vr = dio_voice_range(p.fp), T = p.T;
  double* base = p.work + (int64_t)b * 2 * T;
  double* s1 = base + T;
  const double* cand = p.cand + (int64_t)b * p.nb * T;
  const double* score = p.score + (int64_t)b * p.nb * T;
  for (int j = threadIdx.x; j < T; j += blockDim.x) {
    double best = 0.0;
    if (j >= vr && j < F - vr) {
      double tmp = score[j];
      best = cand[j];
      for (int k = 1; k < p.nb; ++k)
        if (tmp > score[(int64_t)k * T + j]) {
          tmp = score[(int64_t)k * T + j];
          best = cand[(int64_t)k * T + j];
        }
    }
    base[j] = best;
    f0[j] = 0.0;
  }
  __syncthreads();
  for (int j = threadIdx.x; j < F; j += blockDim.x) {
    double v = 0.0;
    if (j >= vr) {
      const double r = __ddiv_rn(__dsub_rn(base[j], base[j - 1]), __dadd_rn(1e-12, base[j]));
      v = fabs(r) < WA_ALLOWED ? base[j] : 0.0;
    }
    s1[j] = v;
  }
  __syncthreads();
  const int c = (vr - 1) / 2;
  for (int j = threadIdx.x; j < F; j += blockDim.x) {
    double v = s1[j];
    if (j >= c && j < F - c)
      for (int q = j - c; q <= j + c; ++q)
        if (s1[q] == 0) {
          v = 0.0;
          break;
        }
    f0[j] = v;
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  // steps 3 and 4 in WORLD's order: every voiced section extended forwards from its last frame, then, last section
  // first, backwards from its first frame; a section's sweep reads what the sweeps before it wrote
  int next = -1;                                         // the end of the next section (FixStep3's limit)
  for (int i = 1; i < F; ++i)
    if (f0[i] == 0 && f0[i - 1] != 0) {
      next = i - 1;
      break;
    }
  int last_pos = -1;
  for (int i = 1; i < F; ++i)
    if (f0[i - 1] == 0 && f0[i] != 0) last_pos = i;
  // the section boundaries are those of step 2's contour, so find each next one on a copy (s1 is free now)
  for (int j = 0; j < F; ++j) s1[j] = f0[j];
  while (next >= 0) {
    int after = -1;
    for (int i = next + 2; i < F; ++i)
      if (s1[i] == 0 && s1[i - 1] != 0) {
        after = i - 1;
        break;
      }
    const int limit = after < 0 ? F - 1 : after;
    for (int j = next; j < limit; ++j) {
      f0[j + 1] = select_best_f0(p, b, f0[j], f0[j - 1], j + 1);
      if (f0[j + 1] == 0) break;
    }
    next = after;
  }
  for (int cur = last_pos; cur >= 0;) {
    int prev = -1;
    for (int i = cur - 1; i >= 1; --i)
      if (s1[i - 1] == 0 && s1[i] != 0) {
        prev = i;
        break;
      }
    const int limit = prev < 0 ? 1 : prev;
    for (int j = cur; j > limit; --j) {
      f0[j - 1] = select_best_f0(p, b, f0[j], f0[j + 1], j - 1);
      if (f0[j - 1] == 0) break;
    }
    cur = prev;
  }
}

// ---------------------------------------------------------------------------------------------- StoneMask
struct FrameParams {
  const double* x;
  int64_t xs;
  const int64_t* lengths;                   // samples
  const double* f0;                         // [B][T]
  const int64_t* frames;                    // [B] (DIO's info)
  int64_t* status;
  int B, S, T, fs, n, logN;
  double fp;
  const double* noise;                      // cheaptrick: the randn stream
  const int64_t* offsets;                   // cheaptrick: [B][T] first draw of each frame
  double* out;
};

__device__ __forceinline__ int frame_count(const FrameParams& p, int b) {
  const int64_t F = p.frames[b];
  return F < 0 ? 0 : (F > p.T ? p.T : (int)F);
}

__device__ __forceinline__ void block_twiddles(double2* w, int n) {
  for (int j = threadIdx.x; j < n / 2; j += blockDim.x) {
    double s, c;
    sincospi(-2.0 * (double)j / (double)n, &s, &c);
    w[j] = make_double2(c, s);
  }
}

// One block per (frame j, row b).  Shared memory: z [N] complex, w [N] complex, the main window [N]; n <= WA_MAX_FFT.
__global__ void __launch_bounds__(WA_THREADS) stonemask_kernel(const FrameParams p) {
  extern __shared__ double2 wa_smem2[];
  __shared__ double2 Mk[6], Dk[6];
  __shared__ int kk[6];
  const int j = blockIdx.x, b = blockIdx.y;
  double* out = p.out + (int64_t)b * p.T + j;
  const int L = wa_len(p.lengths, b, p.S);
  if (j >= frame_count(p, b) || L < 1) {
    if (threadIdx.x == 0) *out = 0.0;
    return;
  }
  const double fs = (double)p.fs, f0 = p.f0[(int64_t)b * p.T + j];
  if (!isfinite(f0) || f0 <= WA_FLOOR_SM || f0 > fs / 12.0) {
    if (threadIdx.x == 0) {
      *out = 0.0;
      if (!isfinite(f0)) wa_flag(p.status, GANTTS_ANALYSIS_BAD_INPUT);
    }
    return;
  }
  const int h = (int)(1.5 * fs / f0 + 1.0), len = 2 * h + 1;
  // WORLD's pow(2.0, 2.0 + (int)(log(2h + 1) / log 2)), as a shift: the device pow may round 2^k below the integer
  const int e = 2 + (int)(log(h * 2.0 + 1.0) / WA_LOG2);
  const int n = e > 12 ? WA_MAX_FFT * 2 : 1 << e, N = n / 2;
  if (n > WA_MAX_FFT) {
    if (threadIdx.x == 0) {
      *out = 0.0;
      wa_flag(p.status, GANTTS_ANALYSIS_FFT);
    }
    return;
  }
  int logN = 0;
  while ((1 << logN) < N) ++logN;
  double2* z = wa_smem2;
  double2* w = z + N;
  double* mw = reinterpret_cast<double*>(w + N);
  const double* x = p.x + (int64_t)b * p.xs;
  const double pos = (double)j * p.fp / 1000.0;
  const double wl = (2.0 * h + 1.0) / fs;
  auto raw = [&](int i) { return wa_round((pos + (double)(-h + i) / fs) * fs); };
  block_twiddles(w, n);
  for (int i = threadIdx.x; i < len; i += blockDim.x) {
    const double t = ((double)raw(i) - 1.0) / fs - pos;
    mw[i] = 0.42 + 0.5 * cos(2.0 * WD_PI * t / wl) + 0.08 * cos(4.0 * WD_PI * t / wl);
  }
  const int nh = min((int)(fs / 2.0 / f0), 6);
  if (threadIdx.x < nh) kk[threadIdx.x] = wa_round(f0 * n / fs * (threadIdx.x + 1));
  __syncthreads();
  auto xv = [&](int i) { return x[min(L - 1, max(0, raw(i) - 1))]; };
  auto dw = [&](int i) {
    return i == 0 ? -mw[1] / 2.0 : (i == len - 1 ? mw[len - 2] / 2.0 : -(mw[i + 1] - mw[i - 1]) / 2.0);
  };
  for (int pass = 0; pass < 2; ++pass) {
    for (int m = threadIdx.x; m < N; m += blockDim.x) {
      const int i0 = 2 * m, i1 = 2 * m + 1;
      const double a = i0 < len ? xv(i0) * (pass ? dw(i0) : mw[i0]) : 0.0;
      const double c = i1 < len ? xv(i1) * (pass ? dw(i1) : mw[i1]) : 0.0;
      z[brev_index(m, logN)] = make_double2(a, c);
    }
    __syncthreads();
    fft_radix2_stages(z, w, N);
    if (threadIdx.x < nh) (pass ? Dk : Mk)[threadIdx.x] = rfft_split(z, w, kk[threadIdx.x], N);
    __syncthreads();
  }
  if (threadIdx.x != 0) return;
  double numer = 0.0, denom = 0.0;
  for (int i = 0; i < nh; ++i) {
    const double2 M = Mk[i], D = Dk[i];
    const double num = M.x * D.y - M.y * D.x, pw = M.x * M.x + M.y * M.y;
    const double inst = pw == 0.0 ? 0.0 : (double)kk[i] * fs / n + num / pw * fs / 2.0 / WD_PI;
    const double amp = sqrt(pw);
    numer += amp * inst;
    denom += amp * (i + 1.0);
  }
  const double mean = numer / (denom + 1e-12);
  *out = fabs(mean - f0) > f0 * 0.2 ? f0 : mean;
}

// ---------------------------------------------------------------------------------------------- CheapTrick
__device__ __forceinline__ double ct_current_f0(double f0, double fs, int n) {
  return f0 <= 3.0 * fs / (n - 3.0) ? WD_DEFAULT_F0 : f0;
}

// an f0 CheapTrick can analyse at this fft size: DCCorrection reads bins up to 2 + int(f0 n / fs)
__device__ __forceinline__ bool ct_f0_ok(double f0, double fs, int n) {
  return isfinite(f0) && 2.0 + floor(f0 * n / fs) <= n / 2;
}

// One block per row, thread 0: each frame's first draw, the running sum of 2 round(1.5 fs / f0) + 1 + n/2 + 1.
__global__ void cheaptrick_offsets_kernel(const FrameParams p, int64_t* offsets) {
  const int b = blockIdx.x, F = frame_count(p, b);
  const double fs = (double)p.fs;
  int64_t off = 0;
  bool bad = false;
  for (int j = 0; j < F; ++j) {
    offsets[(int64_t)b * p.T + j] = off;
    const double f = ct_current_f0(p.f0[(int64_t)b * p.T + j], fs, p.n);
    bad |= !ct_f0_ok(f, fs, p.n);
    off += 2 * (int64_t)(ct_f0_ok(f, fs, p.n) ? wa_round(1.5 * fs / f) : 0) + 1 + p.n / 2 + 1;
  }
  if (bad) wa_flag(p.status, GANTTS_ANALYSIS_BAD_INPUT);
}

// WORLD's interp1Q on the grid x0 + k dx (length len): y[q] + (y[q+1] - y[q]) f, q = int((xi - x0) / dx)
__device__ __forceinline__ double interp1q(double x0, double dx, const double* y, int len, double xi) {
  const double q = (xi - x0) / dx;
  const int k = (int)q;
  const double dy = k < len - 1 ? y[k + 1] - y[k] : 0.0;
  return y[k] + dy * (q - k);
}

// One block per (frame j, row b).  Shared memory (doubles): z [n] (N complex), w [n], P [n + 2] (the power spectrum; N + 1
// complex for the inverse), A [3N + 2] (the window, the DC replica, the cumulative mirrored spectrum, the log envelope).
__global__ void __launch_bounds__(WA_THREADS) cheaptrick_kernel(const FrameParams p) {
  extern __shared__ double2 wa_smem2[];
  __shared__ double red[32];
  const int j = blockIdx.x, b = blockIdx.y, n = p.n, N = n / 2, logN = p.logN;
  double* out = p.out + ((int64_t)b * p.T + j) * (N + 1);
  const int L = wa_len(p.lengths, b, p.S);
  const double fs = (double)p.fs;
  const double f0 = j < frame_count(p, b) ? ct_current_f0(p.f0[(int64_t)b * p.T + j], fs, n) : 0.0;
  if (j >= frame_count(p, b) || L < 1 || !ct_f0_ok(f0, fs, n)) {
    for (int k = threadIdx.x; k <= N; k += blockDim.x) out[k] = 0.0;
    return;
  }
  double2* z = wa_smem2;
  double2* w = z + N;
  double* P = reinterpret_cast<double*>(w + N);
  double* A = P + n + 2;
  const double* x = p.x + (int64_t)b * p.xs;
  const double* r = p.noise + p.offsets[(int64_t)b * p.T + j];
  const int h = wa_round(1.5 * fs / f0), len = 2 * h + 1;
  const int origin = wa_round((double)j * p.fp / 1000.0 * fs + 0.001);
  block_twiddles(w, n);
  // F0-adaptive window, normalised to unit energy
  double part = 0.0;
  for (int i = threadIdx.x; i < len; i += blockDim.x) {
    const double v = 0.5 * cos(WD_PI * ((double)(i - h) / 1.5 / fs) * f0) + 0.5;
    A[i] = v;
    part += v * v;
  }
  const double avg = sqrt(block_sum_f64(part, red));
  double p1 = 0.0, p2 = 0.0;
  for (int i = threadIdx.x; i < len; i += blockDim.x) {
    const double v = A[i] / avg;
    const double u = x[min(L - 1, max(0, origin + i - h))] * v + r[i] * WD_SAFE;
    A[i] = v;
    P[i] = u;
    p1 += u;
    p2 += v;
  }
  const double s1 = block_sum_f64(p1, red), s2 = block_sum_f64(p2, red);
  const double coef = s1 / s2;
  for (int i = threadIdx.x; i < len; i += blockDim.x) P[i] -= A[i] * coef;
  __syncthreads();
  for (int m = threadIdx.x; m < N; m += blockDim.x)
    z[brev_index(m, logN)] = make_double2(2 * m < len ? P[2 * m] : 0.0, 2 * m + 1 < len ? P[2 * m + 1] : 0.0);
  __syncthreads();
  fft_radix2_stages(z, w, N);
  for (int k = threadIdx.x; k <= N; k += blockDim.x) {
    const double2 X = rfft_split(z, w, k, N);
    P[k] = X.x * X.x + X.y * X.y;
  }
  __syncthreads();
  // DCCorrection: the spectrum mirrored about f0 added below f0
  const int ul = 2 + (int)(f0 * n / fs);
  for (int i = threadIdx.x; i < ul - 1; i += blockDim.x)
    A[i] = interp1q(f0, -fs / n, P, ul + 1, (double)i * fs / n);
  __syncthreads();
  for (int i = threadIdx.x; i < ul - 1; i += blockDim.x) P[i] += A[i];
  __syncthreads();
  // LinearSmoothing over 2 f0 / 3: the cumulative sum of the mirrored spectrum, sequential as WORLD's loop
  const double width = f0 * 2.0 / 3.0;
  const int bd = (int)(width * n / fs) + 1, ms = N + 2 * bd + 1;
  if (threadIdx.x == 0) {
    double acc = 0.0;
    for (int i = 0; i < ms; ++i) {
      const double v = i < bd ? P[bd - i] : (i < N + bd ? P[i - bd] : P[N - (i - (N + bd))]);
      acc = (i == 0) ? v * fs / n : v * fs / n + acc;
      A[i] = acc;
    }
  }
  __syncthreads();
  const double origin_f = -(bd - 0.5) * fs / n, df = fs / n;
  for (int k = threadIdx.x; k <= N; k += blockDim.x) {
    const double ax = (double)k / n * fs - width / 2.0;
    const double lo = interp1q(origin_f, df, A, ms, ax), hi = interp1q(origin_f, df, A, ms, ax + width);
    P[k] = log((hi - lo) / width + fabs(r[len + k]) * WA_EPS);
  }
  __syncthreads();
  // SmoothingWithRecovery: the cepstrum of the even log spectrum, liftered, back, exp
  for (int m = threadIdx.x; m < N; m += blockDim.x) {
    const int j0 = 2 * m, j1 = 2 * m + 1;
    z[brev_index(m, logN)] = make_double2(P[j0 <= N ? j0 : n - j0], P[j1 <= N ? j1 : n - j1]);
  }
  __syncthreads();
  fft_radix2_stages(z, w, N);
  double2* X = reinterpret_cast<double2*>(P);
  for (int k = threadIdx.x; k <= N; k += blockDim.x) {
    const double c = rfft_split(z, w, k, N).x;
    double sl = 1.0, cl = (1.0 - 2.0 * WA_Q1) + 2.0 * WA_Q1;
    if (k > 0) {
      const double q = (double)k / fs;
      sl = sin(WD_PI * f0 * q) / (WD_PI * f0 * q);
      cl = (1.0 - 2.0 * WA_Q1) + 2.0 * WA_Q1 * cos(2.0 * WD_PI * q * f0);
    }
    X[k] = make_double2(c * sl * cl / n, 0.0);
  }
  __syncthreads();
  irfft_shift(X, z, w, A, n, N, logN, 0);
  for (int k = threadIdx.x; k <= N; k += blockDim.x) out[k] = exp(A[k]);
}

// ---------------------------------------------------------------------------------------------- sp2mc, smoothing
// One block per (frame t, row b): mc[m] = sum_k op[k][m] log sp[k], k ascending.
__global__ void __launch_bounds__(128) sp2mc_kernel(const double* sp, const double* op, const int64_t* frames, int T,
                                                    int K, int M1, double* mc) {
  extern __shared__ double wa_smem[];
  const int t = blockIdx.x, b = blockIdx.y;
  double* o = mc + ((int64_t)b * T + t) * M1;
  const int64_t F = frames[b];
  if (t >= F) {
    for (int m = threadIdx.x; m < M1; m += blockDim.x) o[m] = 0.0;
    return;
  }
  const double* s = sp + ((int64_t)b * T + t) * K;
  for (int k = threadIdx.x; k < K; k += blockDim.x) wa_smem[k] = log(s[k]);
  __syncthreads();
  for (int m = threadIdx.x; m < M1; m += blockDim.x) {
    double acc = 0.0;
    for (int k = 0; k < K; ++k) acc = fma(op[(int64_t)k * M1 + m], wa_smem[k], acc);
    o[m] = acc;
  }
}

// One block per (column d, row b): the column's n-point real FFT, bins kc.. zeroed, the inverse / n, its first L frames.
// Shared memory: z [N] complex, w [N] complex, X [N + 1] complex (also the inverse's output).
__global__ void __launch_bounds__(WA_THREADS) modspec_smoothing_kernel(const double* x, const int64_t* lengths, int T,
                                                                       int D, int n, int logN, int kc, double* out) {
  extern __shared__ double2 wa_smem2[];
  const int d = blockIdx.x, b = blockIdx.y, N = n / 2;
  const int64_t Lr = lengths[b];
  const int L = Lr < 0 ? 0 : (Lr > T ? T : (int)Lr);
  double2* z = wa_smem2;
  double2* w = z + N;
  double2* X = w + N;
  const double* col = x + (int64_t)b * T * D + d;
  double* o = out + (int64_t)b * T * D + d;
  block_twiddles(w, n);
  for (int m = threadIdx.x; m < N; m += blockDim.x) {
    const int t = 2 * m;
    z[brev_index(m, logN)] = make_double2(t < L ? col[(int64_t)t * D] : 0.0, t + 1 < L ? col[(int64_t)(t + 1) * D] : 0.0);
  }
  __syncthreads();
  fft_radix2_stages(z, w, N);
  for (int k = threadIdx.x; k <= N; k += blockDim.x) X[k] = k < kc ? rfft_split(z, w, k, N) : make_double2(0.0, 0.0);
  __syncthreads();
  double* y = reinterpret_cast<double*>(X);
  irfft_shift(X, z, w, y, n, N, logN, 0);
  const double inv = 1.0 / n;
  for (int t = threadIdx.x; t < T; t += blockDim.x) o[(int64_t)t * D] = t < L ? y[t] * inv : 0.0;
}

// ---------------------------------------------------------------------------------------------- host side
static bool wa_fft_ok(int n) { return n >= 64 && n <= WA_MAX_FFT && (n & (n - 1)) == 0; }

static int wa_log2(int v) {
  int k = 0;
  while ((1 << k) < v) ++k;
  return k;
}

// The DIO plan of a batch: bands, taps and the buffers' sizes.
struct DioPlan {
  DioParams p;
  size_t taps, mean, z, edges, counts, cand, work, total;
};

static void dio_plan(int B, int S, int fs, double fp, int T, DioPlan* q) {
  DioParams& p = q->p;
  p = DioParams{};
  p.B = B; p.S = S; p.T = T; p.fs = fs; p.fp = fp;
  p.nb = dio_bands();
  p.N = wa_round(fs / WA_CUTOFF) * 2 + 1;
  int off = p.N, hmax = 0;
  for (int i = 0; i < p.nb; ++i) {
    p.boundary[i] = WA_F0_FLOOR * pow(2.0, (i + 1) / WA_CHANNELS);
    p.h[i] = wa_round((double)fs / p.boundary[i] / 2.0);
    p.nut_off[i] = off;
    off += 4 * p.h[i];
    hmax = p.h[i] > hmax ? p.h[i] : hmax;
  }
  p.P = 2 * hmax;
  p.Z = S + 1 + 2 * p.P;
  p.cap = S / 2 + 2;
  q->taps = wd_align(sizeof(double) * (size_t)off);
  q->mean = wd_align(sizeof(double) * (size_t)B);
  q->z = wd_align(sizeof(double) * (size_t)B * p.Z);
  q->edges = wd_align(sizeof(double) * (size_t)B * p.nb * 4 * p.cap);
  q->counts = wd_align(sizeof(int) * (size_t)B * p.nb * 4);
  q->cand = wd_align(sizeof(double) * (size_t)B * p.nb * T);
  q->work = wd_align(sizeof(double) * (size_t)B * 2 * T);
  q->total = q->taps + q->mean + q->z + q->edges + q->counts + 2 * q->cand + q->work;
}

static int analysis_common_check(const char* what, int B, int S, int fs, double fp) {
  GANTTS_CHECK_ARG(B >= 1 && B <= 65535, "%s: batch size B = %d must be in [1, 65535]", what, B);
  GANTTS_CHECK_ARG(S >= 1 && S <= WA_MAX_S, "%s: padded length S = %d samples must be in [1, %d]", what, S, WA_MAX_S);
  GANTTS_CHECK_ARG(fs >= WA_MIN_FS && fs <= WA_MAX_FS, "%s: fs = %d must be in [%d, %d]", what, fs, WA_MIN_FS,
                   WA_MAX_FS);
  GANTTS_CHECK_ARG(isfinite(fp) && fp >= 1.0 && fp <= 100.0, "%s: frame_period = %g ms must be in [1, 100]", what, fp);
  return GANTTS_OK;
}

}  // namespace gantts

using namespace gantts;

extern "C" int64_t gantts_world_dio_frames(int64_t samples, int fs, double frame_period) {
  return fs >= 1 && frame_period > 0.0 && samples >= 0 ? dio_frames(samples, fs, frame_period) : 0;
}

extern "C" size_t gantts_world_dio_workspace_bytes(int B, int S, int fs, double frame_period) {
  if (analysis_common_check("world_dio", B, S, fs, frame_period) != GANTTS_OK) return 0;
  DioPlan q;
  dio_plan(B, S, fs, frame_period, (int)dio_frames(S, fs, frame_period), &q);
  return q.total;
}

extern "C" int gantts_world_dio(const double* x, int64_t x_bstride, const int64_t* lengths_dev, int B, int S, int fs,
                                double frame_period, double* f0, int64_t* info_dev, void* workspace,
                                size_t workspace_bytes, void* stream) {
  GANTTS_CHECK_ARG(x && lengths_dev && f0 && info_dev && workspace, "world_dio: null pointer: x, lengths_dev, f0, "
                   "info_dev and workspace are all required");
  const int rc = analysis_common_check("world_dio", B, S, fs, frame_period);
  if (rc != GANTTS_OK) return rc;
  GANTTS_CHECK_ARG(x_bstride >= S, "world_dio: x_bstride = %lld must be >= S = %d", (long long)x_bstride, S);
  DioPlan q;
  const int T = (int)dio_frames(S, fs, frame_period);
  dio_plan(B, S, fs, frame_period, T, &q);
  if (workspace_bytes < q.total) {
    set_error("world_dio: workspace of %zu bytes, %zu needed", workspace_bytes, q.total);
    return GANTTS_E_WORKSPACE;
  }
  DioParams p = q.p;
  char* ws = static_cast<char*>(workspace);
  p.taps = reinterpret_cast<double*>(ws); ws += q.taps;
  p.mean = reinterpret_cast<double*>(ws); ws += q.mean;
  p.z = reinterpret_cast<double*>(ws); ws += q.z;
  p.edges = reinterpret_cast<double*>(ws); ws += q.edges;
  p.counts = reinterpret_cast<int*>(ws); ws += q.counts;
  p.cand = reinterpret_cast<double*>(ws); ws += q.cand;
  p.score = reinterpret_cast<double*>(ws); ws += q.cand;
  p.work = reinterpret_cast<double*>(ws);
  p.x = x; p.xs = x_bstride; p.lengths = lengths_dev; p.f0 = f0; p.info = info_dev;
  cudaStream_t st = as_stream(stream);
  GANTTS_CUDA(cudaMemsetAsync(info_dev + B, 0, sizeof(int64_t), st));
  dio_taps_kernel<<<1, WA_THREADS, 0, st>>>(p);
  GANTTS_LAUNCH_CHECK("dio_taps_kernel");
  dio_prepare_kernel<<<(unsigned)B, WA_THREADS, 0, st>>>(p);
  GANTTS_LAUNCH_CHECK("dio_prepare_kernel");
  const size_t lc_smem = sizeof(double) * (size_t)(2 * p.N + WA_THREADS);
  GANTTS_CUDA(cudaFuncSetAttribute(dio_lowcut_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)lc_smem));
  dio_lowcut_kernel<<<dim3((unsigned)((p.Z + WA_THREADS - 1) / WA_THREADS), (unsigned)B), WA_THREADS, lc_smem, st>>>(p);
  GANTTS_LAUNCH_CHECK("dio_lowcut_kernel");
  int hmax = 0;
  for (int i = 0; i < p.nb; ++i) hmax = p.h[i] > hmax ? p.h[i] : hmax;
  const size_t band_smem = sizeof(double) * (size_t)(4 * hmax + WA_TILE + 2);
  GANTTS_CUDA(cudaFuncSetAttribute(dio_band_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)band_smem));
  dio_band_kernel<<<dim3((unsigned)p.nb, (unsigned)B), WA_THREADS, band_smem, st>>>(p);
  GANTTS_LAUNCH_CHECK("dio_band_kernel");
  dio_candidate_kernel<<<dim3((unsigned)((T + WA_THREADS - 1) / WA_THREADS), (unsigned)p.nb, (unsigned)B), WA_THREADS, 0,
                         st>>>(p);
  GANTTS_LAUNCH_CHECK("dio_candidate_kernel");
  dio_fix_kernel<<<(unsigned)B, WA_THREADS, 0, st>>>(p);
  GANTTS_LAUNCH_CHECK("dio_fix_kernel");
  return GANTTS_OK;
}

static int frame_op_check(const char* what, const double* x, int64_t x_bstride, const int64_t* lengths_dev,
                          const double* f0, const int64_t* frames_dev, int64_t* status_dev, const void* out, int B,
                          int S, int T, int fs, double frame_period) {
  GANTTS_CHECK_ARG(x && lengths_dev && f0 && frames_dev && status_dev && out, "%s: null pointer: x, lengths_dev, f0, "
                   "frames_dev, status_dev and the output are all required", what);
  const int rc = analysis_common_check(what, B, S, fs, frame_period);
  if (rc != GANTTS_OK) return rc;
  GANTTS_CHECK_ARG(x_bstride >= S, "%s: x_bstride = %lld must be >= S = %d", what, (long long)x_bstride, S);
  GANTTS_CHECK_ARG(T >= 1 && T <= WD_MAX_T, "%s: padded frames T = %d must be in [1, %d]", what, T, WD_MAX_T);
  return GANTTS_OK;
}

extern "C" int gantts_world_stonemask(const double* x, int64_t x_bstride, const int64_t* lengths_dev, const double* f0,
                                      const int64_t* frames_dev, int B, int S, int T, int fs, double frame_period,
                                      double* out, int64_t* status_dev, void* stream) {
  const int rc = frame_op_check("world_stonemask", x, x_bstride, lengths_dev, f0, frames_dev, status_dev, out, B, S, T,
                                fs, frame_period);
  if (rc != GANTTS_OK) return rc;
  FrameParams p{};
  p.x = x; p.xs = x_bstride; p.lengths = lengths_dev; p.f0 = f0; p.frames = frames_dev; p.status = status_dev;
  p.B = B; p.S = S; p.T = T; p.fs = fs; p.fp = frame_period; p.out = out;
  const size_t smem = sizeof(double) * (size_t)(5 * (WA_MAX_FFT / 2));
  GANTTS_CUDA(cudaFuncSetAttribute(stonemask_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  stonemask_kernel<<<dim3((unsigned)T, (unsigned)B), WA_THREADS, smem, as_stream(stream)>>>(p);
  GANTTS_LAUNCH_CHECK("stonemask_kernel");
  return GANTTS_OK;
}

// the draws one frame can take: 2 h + 1 (h <= n/2 - 1 above the f0 floor, round(0.003 fs) at 500 Hz) + n/2 + 1
static int64_t ct_draws_per_frame(int fs, int n) {
  const int h500 = wa_round(1.5 * fs / WD_DEFAULT_F0);
  return 2 * (int64_t)(h500 > n / 2 ? h500 : n / 2) + 1 + n / 2 + 1;
}

extern "C" int64_t gantts_world_cheaptrick_draws(int T, int fs, int fftlen) {
  return T >= 1 && fs >= 1 && wa_fft_ok(fftlen) ? (int64_t)T * ct_draws_per_frame(fs, fftlen) : 0;
}

extern "C" int gantts_world_cheaptrick(const double* x, int64_t x_bstride, const int64_t* lengths_dev, const double* f0,
                                       const int64_t* frames_dev, int B, int S, int T, int fs, double frame_period,
                                       int fftlen, const double* noise, int64_t noise_count, int64_t* offsets,
                                       double* sp, int64_t* status_dev, void* stream) {
  const int rc = frame_op_check("world_cheaptrick", x, x_bstride, lengths_dev, f0, frames_dev, status_dev, sp, B, S, T,
                                fs, frame_period);
  if (rc != GANTTS_OK) return rc;
  GANTTS_CHECK_ARG(wa_fft_ok(fftlen), "world_cheaptrick: fftlen = %d must be a power of two in [64, %d]", fftlen,
                   WA_MAX_FFT);
  GANTTS_CHECK_ARG(noise && offsets, "world_cheaptrick: null noise or offsets");
  const int64_t need = gantts_world_cheaptrick_draws(T, fs, fftlen);
  GANTTS_CHECK_ARG(noise_count >= need, "world_cheaptrick: %lld noise draws, %lld needed for T = %d frames",
                   (long long)noise_count, (long long)need, T);
  FrameParams p{};
  p.x = x; p.xs = x_bstride; p.lengths = lengths_dev; p.f0 = f0; p.frames = frames_dev; p.status = status_dev;
  p.B = B; p.S = S; p.T = T; p.fs = fs; p.fp = frame_period; p.n = fftlen; p.logN = wa_log2(fftlen / 2);
  p.noise = noise; p.offsets = offsets; p.out = sp;
  cudaStream_t st = as_stream(stream);
  cheaptrick_offsets_kernel<<<(unsigned)B, 1, 0, st>>>(p, offsets);
  GANTTS_LAUNCH_CHECK("cheaptrick_offsets_kernel");
  const size_t smem = sizeof(double) * (size_t)(2 * fftlen + fftlen + 2 + 3 * (fftlen / 2) + 2);
  GANTTS_CUDA(cudaFuncSetAttribute(cheaptrick_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  cheaptrick_kernel<<<dim3((unsigned)T, (unsigned)B), WA_THREADS, smem, st>>>(p);
  GANTTS_LAUNCH_CHECK("cheaptrick_kernel");
  return GANTTS_OK;
}

extern "C" int gantts_sp2mc(const double* sp, const double* op, const int64_t* frames_dev, int B, int T, int M, int K,
                            double* mc, void* stream) {
  GANTTS_CHECK_ARG(sp && op && frames_dev && mc, "sp2mc: null pointer: sp, op, frames_dev and mc are all required");
  GANTTS_CHECK_ARG(B >= 1 && B <= 65535, "sp2mc: batch size B = %d must be in [1, 65535]", B);
  GANTTS_CHECK_ARG(T >= 1 && T <= WD_MAX_T, "sp2mc: padded frames T = %d must be in [1, %d]", T, WD_MAX_T);
  GANTTS_CHECK_ARG(M >= 0 && M + 1 <= MCEP_MAX_COLS, "sp2mc: order M = %d: M + 1 must be in [1, %d]", M, MCEP_MAX_COLS);
  GANTTS_CHECK_ARG(K >= 2 && wa_fft_ok(2 * (K - 1)), "sp2mc: K = %d bins: 2 (K - 1) must be a power of two in [64, %d]",
                   K, WA_MAX_FFT);
  const size_t smem = sizeof(double) * (size_t)K;
  GANTTS_CUDA(cudaFuncSetAttribute(sp2mc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  sp2mc_kernel<<<dim3((unsigned)T, (unsigned)B), 128, smem, as_stream(stream)>>>(sp, op, frames_dev, T, K, M + 1, mc);
  GANTTS_LAUNCH_CHECK("sp2mc_kernel");
  return GANTTS_OK;
}

extern "C" int gantts_modspec_smoothing(const double* x, const int64_t* lengths_dev, int B, int T, int D, int n,
                                        int cutoff_bin, double* out, void* stream) {
  GANTTS_CHECK_ARG(x && lengths_dev && out, "modspec_smoothing: null pointer: x, lengths_dev and out are all required");
  GANTTS_CHECK_ARG(B >= 1 && B <= 65535, "modspec_smoothing: batch size B = %d must be in [1, 65535]", B);
  GANTTS_CHECK_ARG(D >= 1 && D <= 65535, "modspec_smoothing: width D = %d must be in [1, 65535]", D);
  GANTTS_CHECK_ARG(wa_fft_ok(n), "modspec_smoothing: n = %d must be a power of two in [64, %d]", n, WA_MAX_FFT);
  GANTTS_CHECK_ARG(T >= 1 && T <= n, "modspec_smoothing: padded length T = %d frames must be in [1, n = %d]: the "
                   "smoothing is defined for sequences of at most n frames", T, n);
  GANTTS_CHECK_ARG(cutoff_bin >= 0, "modspec_smoothing: cutoff_bin = %d must be >= 0", cutoff_bin);
  const size_t smem = sizeof(double2) * (size_t)(3 * (n / 2) + 1);
  GANTTS_CUDA(cudaFuncSetAttribute(modspec_smoothing_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  modspec_smoothing_kernel<<<dim3((unsigned)D, (unsigned)B), WA_THREADS, smem, as_stream(stream)>>>(
      x, lengths_dev, T, D, n, wa_log2(n / 2), cutoff_bin, out);
  GANTTS_LAUNCH_CHECK("modspec_smoothing_kernel");
  return GANTTS_OK;
}
