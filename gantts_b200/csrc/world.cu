// WORLD's waveform synthesis on padded device batches (evaluation_tts.py:103-130 gen_waveform: pyworld.decode_aperiodicity
// and pyworld.synthesize), all arithmetic in fp64.
//
//   decode_aperiodicity  coded band aperiodicity -> ap, per (frame, row)
//   time_base            f0 -> the pulse list of each row: one block per row; the accumulated phase is one sequential
//                        fp64 chain in sample order, as WORLD's loop runs it (a parallel scan rounds differently and can
//                        move a pulse by one sample near a 2 pi crossing); the increments, fmod, the detection and the
//                        compaction around it are parallel
//   randn                WORLD's randn stream (xorshift128, 12 outputs per draw), reseeded per utterance so the same for
//                        every row; thread c starts draw c * WD_CHUNK by GF(2) jump-ahead matrices built on the device
//   synthesize           one block per pulse: the periodic and aperiodic responses (seven n-point real FFTs in shared
//                        memory), written to a per-pulse buffer; then a gather adds, for every output sample, the
//                        responses covering it in ascending pulse order, as WORLD's loop adds them
//
// The time base computes without FMA contraction (__dmul_rn / __dadd_rn), so it is bit for bit the C loop's arithmetic and
// a pulse lands on the same sample.  A row's results depend only on that row.
#include "common.cuh"

#include <math.h>

namespace gantts {

constexpr int WD_THREADS = 256;
constexpr int WD_MIN_FFT = 64;
constexpr int WD_MAX_FFT = 4096;
constexpr int WD_MAX_T = 1 << 24;
constexpr int WD_MAX_BANDS = 5;          // min(15000, fs/2 - 3000) / 3000 <= 5
constexpr int WD_TILE = 2048;            // samples per step of the time base
constexpr int WD_CHUNK = 256;            // noise draws per thread
constexpr int WD_STEPS_PER_DRAW = 12;
constexpr double WD_PI = 3.1415926535897932384;
constexpr double WD_TWO_PI = 2.0 * WD_PI;
constexpr double WD_SAFE = 1e-12;        // WORLD's kMySafeGuardMinimum
constexpr double WD_DEFAULT_F0 = 500.0;  // WORLD's kDefaultF0: the pulse rate of unvoiced samples
constexpr double WD_BAND = 3000.0;       // WORLD's kFrequencyInterval
constexpr double WD_UPPER = 15000.0;     // WORLD's kUpperLimit

__device__ __forceinline__ int wd_length(const int64_t* lengths, int b, int T) {
  const int64_t L = lengths[b];
  return L < 0 ? 0 : (L > T ? T : (int)L);
}

__host__ __device__ inline int world_bands(int fs) {
  const double top = fmin(WD_UPPER, fs / 2.0 - WD_BAND);
  return top < WD_BAND ? 0 : (int)(top / WD_BAND);
}

// int(F * frame_period * fs / 1000), as pyworld.synthesize sizes its output
__host__ __device__ inline int64_t world_y_length(int64_t F, int fs, double frame_period) {
  return (int64_t)((double)F * frame_period * (double)fs / 1000.0);
}

// ---------------------------------------------------------------------------------------------- decode_aperiodicity
// One block per (frame t, row b).  Knots (0 Hz, -60 dB), (3000 j Hz, coded[j-1]), (fs/2, -1e-12), interpolated over bin
// frequency fs / n * k as WORLD's interp1, then 10^(dB/20); a frame whose mean coded value is above -0.5 keeps 1 - 1e-12.
__global__ void __launch_bounds__(WD_THREADS) world_decode_ap_kernel(const float* bap, int64_t bs, int64_t ts,
                                                                     const int64_t* lengths, int T, int nb, int fs,
                                                                     int n, double* ap) {
  __shared__ double kx[WD_MAX_BANDS + 2], ky[WD_MAX_BANDS + 2];
  __shared__ int unvoiced;
  const int t = blockIdx.x, b = blockIdx.y, K = n / 2 + 1;
  double* o = ap + ((int64_t)b * T + t) * K;
  if (t >= wd_length(lengths, b, T)) {
    for (int k = threadIdx.x; k < K; k += blockDim.x) o[k] = 0.0;
    return;
  }
  if (threadIdx.x == 0) {
    const float* c = bap + (int64_t)b * bs + (int64_t)t * ts;
    double s = 0.0;
    for (int j = 0; j < nb; ++j) {
      s = __dadd_rn(s, (double)c[j]);
      ky[j + 1] = (double)c[j];
      kx[j] = __dmul_rn((double)j, WD_BAND);
    }
    kx[nb] = __dmul_rn((double)nb, WD_BAND);
    kx[nb + 1] = fs / 2.0;
    ky[0] = -60.0;
    ky[nb + 1] = -WD_SAFE;
    unvoiced = s / nb > -0.5;
  }
  __syncthreads();
  const double df = (double)fs / (double)n;
  for (int k = threadIdx.x; k < K; k += blockDim.x) {
    if (unvoiced) {
      o[k] = 1.0 - WD_SAFE;
      continue;
    }
    const double f = __dmul_rn(df, (double)k);
    int j = 0;                                           // the last knot at or below f, at most the second to last
    while (j < nb && kx[j + 1] <= f) ++j;
    const double s = __ddiv_rn(__dsub_rn(f, kx[j]), __dsub_rn(kx[j + 1], kx[j]));
    const double db = __dadd_rn(ky[j], __dmul_rn(s, __dsub_rn(ky[j + 1], ky[j])));
    o[k] = pow(10.0, db / 20.0);
  }
}

// ---------------------------------------------------------------------------------------------- time base
struct TimeBaseParams {
  const float* f0;
  int64_t bs, ts;
  const int64_t* lengths;
  int B, T, fs, cap;
  double fp_ms, fp_s, lowest;
  int32_t* index;
  double* shift;
  uint8_t* vuv;
  int64_t* info;                         // [B] pulse counts, [B] y_lengths, [1] status
};

// coarse f0 and V/UV of frame i < F (f0 below lowest_f0 is unvoiced), or the extrapolated point at i = F
__device__ __forceinline__ void coarse_point(const TimeBaseParams& p, const float* f0, int F, int i, double* f,
                                             double* v) {
  auto at = [&](int j, double* fj, double* vj) {
    const double x = (double)f0[(int64_t)j * p.ts];
    *fj = x < p.lowest ? 0.0 : x;
    *vj = *fj == 0.0 ? 0.0 : 1.0;
  };
  if (i < F) {
    at(i, f, v);
    return;
  }
  double f1, v1, f2, v2;
  at(F - 1, &f1, &v1);
  at(F - 2, &f2, &v2);
  *f = __dsub_rn(__dmul_rn(f1, 2.0), f2);
  *v = __dsub_rn(__dmul_rn(v1, 2.0), v2);
}

__global__ void __launch_bounds__(WD_THREADS) world_time_base_kernel(const TimeBaseParams p) {
  __shared__ double ph[WD_TILE];         // increments, then the accumulated phase, then its fmod
  __shared__ uint8_t vv[WD_TILE];
  __shared__ int warp_cnt[WD_THREADS / 32];
  __shared__ double carry_psi;
  __shared__ uint8_t carry_vuv;
  __shared__ int64_t found_s;
  const int b = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int F = wd_length(p.lengths, b, p.T);
  const float* f0 = p.f0 + (int64_t)b * p.bs;
  const int64_t Y = world_y_length(F, p.fs, p.fp_ms);
  bool bad = false;
  for (int t = threadIdx.x; t < F; t += blockDim.x) bad |= !isfinite(f0[(int64_t)t * p.ts]);
  if (bad) atomicOr(reinterpret_cast<unsigned long long*>(p.info + 2 * p.B), (unsigned long long)GANTTS_WORLD_BAD_F0);
  if (threadIdx.x == 0) {
    p.info[p.B + b] = Y;
    found_s = 0;
    if (F < 2) atomicOr(reinterpret_cast<unsigned long long*>(p.info + 2 * p.B), (unsigned long long)GANTTS_WORLD_SHORT);
  }
  __syncthreads();
  if (F < 2) {
    if (threadIdx.x == 0) p.info[b] = 0;
    return;
  }
  int32_t* idx = p.index + (int64_t)b * p.cap;
  double* sh = p.shift + (int64_t)b * p.cap;
  uint8_t* vo = p.vuv + (int64_t)b * p.cap;
  double phi = 0.0;                                      // thread 0's running total
  for (int64_t n0 = 0; n0 < Y; n0 += WD_TILE) {
    const int cnt = (int)min((int64_t)WD_TILE, Y - n0);
    for (int j = threadIdx.x; j < cnt; j += blockDim.x) {
      // WORLD's interp1 of the coarse f0 and V/UV at t = n / fs over the axis i * frame_period, i = 0 .. F
      const double t = __ddiv_rn((double)(n0 + j), (double)p.fs);
      int i = (int)floor(t / p.fp_s);
      i = min(max(i, 0), F);
      while (i < F && __dmul_rn((double)(i + 1), p.fp_s) <= t) ++i;
      while (i > 0 && __dmul_rn((double)i, p.fp_s) > t) --i;
      i = min(i, F - 1);
      const double x0 = __dmul_rn((double)i, p.fp_s), x1 = __dmul_rn((double)(i + 1), p.fp_s);
      double fa, va, fb, vb;
      coarse_point(p, f0, F, i, &fa, &va);
      coarse_point(p, f0, F, i + 1, &fb, &vb);
      const double s = __ddiv_rn(__dsub_rn(t, x0), __dsub_rn(x1, x0));
      const double fi = __dadd_rn(fa, __dmul_rn(s, __dsub_rn(fb, fa)));
      const double vi = __dadd_rn(va, __dmul_rn(s, __dsub_rn(vb, va)));
      const bool voiced = vi > 0.5;
      vv[j] = voiced ? 1 : 0;
      ph[j] = __ddiv_rn(__dmul_rn(WD_TWO_PI, voiced ? fi : WD_DEFAULT_F0), (double)p.fs);
    }
    __syncthreads();
    if (threadIdx.x == 0) {                              // the sequential chain
#pragma unroll 8
      for (int j = 0; j < cnt; ++j) {
        phi = __dadd_rn(phi, ph[j]);
        ph[j] = phi;
      }
    }
    __syncthreads();
    for (int j = threadIdx.x; j < cnt; j += blockDim.x) ph[j] = fmod(ph[j], WD_TWO_PI);
    __syncthreads();
    // pulse at m = n0 + j - 1 when |psi[m+1] - psi[m]| > pi; in sample order by a block scan of the flags
    for (int j0 = 0; j0 < cnt; j0 += blockDim.x) {
      const int j = j0 + threadIdx.x;
      const int64_t m = n0 + j - 1;
      bool flag = false;
      double psi0 = 0.0, psi1 = 0.0;
      uint8_t v0 = 0;
      if (j < cnt && m >= 0) {
        psi1 = ph[j];
        psi0 = j == 0 ? carry_psi : ph[j - 1];
        v0 = j == 0 ? carry_vuv : vv[j - 1];
        flag = fabs(__dsub_rn(psi1, psi0)) > WD_PI;
      }
      const unsigned bal = __ballot_sync(0xffffffffu, flag);
      if (lane == 0) warp_cnt[warp] = __popc(bal);
      __syncthreads();
      int before = 0, total = 0;
      for (int w = 0; w < WD_THREADS / 32; ++w) {
        if (w < warp) before += warp_cnt[w];
        total += warp_cnt[w];
      }
      if (flag) {
        const int64_t r = found_s + before + __popc(bal & ((1u << lane) - 1u));
        const double y1 = __dsub_rn(psi0, WD_TWO_PI);
        const double x = -y1 / __dsub_rn(psi1, y1);
        idx[r] = (int32_t)m;
        sh[r] = x / (double)p.fs;
        vo[r] = v0;
      }
      __syncthreads();
      if (threadIdx.x == 0) found_s += total;
      __syncthreads();
    }
    if (threadIdx.x == 0) {
      carry_psi = ph[cnt - 1];
      carry_vuv = vv[cnt - 1];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) p.info[b] = found_s;
}

// ---------------------------------------------------------------------------------------------- randn
struct Xs128 {
  uint32_t x, y, z, w;
};

__host__ __device__ __forceinline__ uint32_t xs_step(Xs128& s) {
  const uint32_t t = s.x ^ (s.x << 11);
  s.x = s.y;
  s.y = s.z;
  s.z = s.w;
  s.w = (s.w ^ (s.w >> 19)) ^ (t ^ (t >> 8));
  return s.w;
}

// One draw of WORLD's randn: the sum of w >> 4 over 12 outputs, in uint32, / 2^28 - 6.
__device__ __forceinline__ double xs_draw(Xs128& s) {
  uint32_t tmp = 0;
#pragma unroll
  for (int i = 0; i < WD_STEPS_PER_DRAW; ++i) tmp += xs_step(s) >> 4;
  return tmp / 268435456.0 - 6.0;
}

__device__ __forceinline__ uint4 xs_pack(const Xs128& s) { return make_uint4(s.x, s.y, s.z, s.w); }

// M v over GF(2), M as its 128 columns (bit q of v = bit q % 32 of word q / 32 of (x, y, z, w))
__device__ __forceinline__ uint4 gf2_apply(const uint4* M, uint4 v) {
  uint4 a = make_uint4(0u, 0u, 0u, 0u);
  const uint32_t words[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int wd = 0; wd < 4; ++wd) {
#pragma unroll 8
    for (int bit = 0; bit < 32; ++bit) {
      const uint32_t m = 0u - ((words[wd] >> bit) & 1u);
      const uint4 c = M[wd * 32 + bit];
      a.x ^= c.x & m; a.y ^= c.y & m; a.z ^= c.z & m; a.w ^= c.w & m;
    }
  }
  return a;
}

// One block of 128 threads: jump[k] = J^(2^k), J = M^(12 WD_CHUNK) the state map of WD_CHUNK draws, M one xorshift step.
__global__ void __launch_bounds__(128) world_jump_kernel(int nmat, uint4* jump) {
  __shared__ uint4 A[128], R[128];
  const int j = threadIdx.x;
  const uint32_t e = 1u << (j & 31);
  Xs128 s{j < 32 ? e : 0u, (j >> 5) == 1 ? e : 0u, (j >> 5) == 2 ? e : 0u, (j >> 5) == 3 ? e : 0u};
  R[j] = xs_pack(s);                                     // identity
  xs_step(s);
  A[j] = xs_pack(s);                                     // M
  __syncthreads();
  for (unsigned ex = WD_STEPS_PER_DRAW * WD_CHUNK; ex; ex >>= 1) {
    if (ex & 1u) {                                       // R = A R (powers of M commute)
      const uint4 c = gf2_apply(A, R[j]);
      __syncthreads();
      R[j] = c;
      __syncthreads();
    }
    if (ex > 1u) {                                       // A = A A
      const uint4 c = gf2_apply(A, A[j]);
      __syncthreads();
      A[j] = c;
      __syncthreads();
    }
  }
  for (int k = 0; k < nmat; ++k) {
    jump[k * 128 + j] = R[j];
    const uint4 c = gf2_apply(R, R[j]);
    __syncthreads();
    R[j] = c;
    __syncthreads();
  }
}

// Thread c writes draws [c WD_CHUNK, (c + 1) WD_CHUNK) of the stream seeded as WORLD's randn_reseed.
__global__ void __launch_bounds__(WD_THREADS) world_randn_kernel(const uint4* jump, int64_t count, double* out) {
  const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t d0 = c * WD_CHUNK;
  if (d0 >= count) return;
  uint4 v = make_uint4(123456789u, 362436069u, 521288629u, 88675123u);
  for (int k = 0; (c >> k) != 0; ++k)
    if ((c >> k) & 1) v = gf2_apply(jump + k * 128, v);
  Xs128 s{v.x, v.y, v.z, v.w};
  const int nd = (int)min((int64_t)WD_CHUNK, count - d0);
  for (int i = 0; i < nd; ++i) out[d0 + i] = xs_draw(s);
}

static int world_jump_count(int64_t count) {
  const int64_t chunks = (count + WD_CHUNK - 1) / WD_CHUNK;
  int k = 1;
  while (((int64_t)1 << k) < chunks) ++k;
  return k;
}

// ---------------------------------------------------------------------------------------------- synthesis
struct SynthParams {
  const float* sp;
  int64_t sp_bs, sp_ts;
  const double* ap;
  int64_t ap_bs, ap_ts;
  const int64_t* lengths;
  const int32_t* index;
  const double* shift;
  const uint8_t* vuv;
  const int64_t* info;                   // time base: [B] pulse counts, [B] y_lengths
  const double* noise;
  const int64_t* row_start;              // [B + 1] first global pulse of each row
  const double2* tw;                     // [N] exp(-2 pi i j / n)
  const double* dcr;                     // [n] WORLD's DC remover
  double* resp;                          // [chunk][n]
  double* y;
  int64_t y_stride;
  int B, T, cap, fs, n, logN;
  double fp_s;
};

__global__ void __launch_bounds__(WD_THREADS) world_setup_kernel(const SynthParams p, double2* tw, double* dcr,
                                                                 int64_t* row_start) {
  __shared__ double tot;
  const int n = p.n, N = n / 2;
  for (int j = threadIdx.x; j < N; j += blockDim.x) {
    double s, c;
    sincospi(-2.0 * (double)j / (double)n, &s, &c);
    tw[j] = make_double2(c, s);
    dcr[j] = 0.5 - 0.5 * cos(WD_TWO_PI * (j + 1.0) / (1.0 + n));
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int j = 0; j < N; ++j) s += dcr[j] * 2.0;
    tot = s;
    int64_t r = 0;
    for (int b = 0; b < p.B; ++b) {
      row_start[b] = r;
      r += p.info[b];
    }
    row_start[p.B] = r;
  }
  __syncthreads();
  for (int j = threadIdx.x; j < N; j += blockDim.x) {
    const double h = dcr[j] / tot;
    dcr[j] = h;
    dcr[n - 1 - j] = h;
  }
}

__device__ __forceinline__ int brev_index(int m, int logN) { return logN ? (int)(__brev((unsigned)m) >> (32 - logN)) : 0; }

// Fixed-order block sum (every thread gets it): each thread's strided partial, a butterfly per warp, warps in order.
__device__ double block_sum_f64(double v, double* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.0;
  for (int w = 0; w < (int)(blockDim.x >> 5); ++w) s += red[w];
  __syncthreads();
  return s;
}

// WORLD's GetMinimumPhaseSpectrum of the half log spectrum u[0..N]: the FFT of the even sequence u[min(j, n - j)], its
// causal quefrencies 1 .. N-1 doubled and the anticausal ones zeroed, an FFT, and exp(. / n).  u may alias X.
__device__ void min_phase(double* u, double2* z, const double2* w, double2* X, int n, int N, int logN) {
  for (int m = threadIdx.x; m < N; m += blockDim.x) {
    const int j0 = 2 * m, j1 = 2 * m + 1;
    z[brev_index(m, logN)] = make_double2(u[j0 <= N ? j0 : n - j0], u[j1 <= N ? j1 : n - j1]);
  }
  __syncthreads();
  fft_radix2_stages(z, w, N);
  for (int q = threadIdx.x; q <= N; q += blockDim.x) {
    const double c = rfft_split(z, w, q, N).x;
    u[q] = (q == 0 || q == N) ? c : 2.0 * c;
  }
  __syncthreads();
  for (int m = threadIdx.x; m < N; m += blockDim.x) {
    const int j0 = 2 * m, j1 = 2 * m + 1;
    z[brev_index(m, logN)] = make_double2(j0 <= N ? u[j0] : 0.0, j1 <= N ? u[j1] : 0.0);
  }
  __syncthreads();
  fft_radix2_stages(z, w, N);
  const double inv_n = 1.0 / (double)n;                 // a power of two: exact, as WORLD's / fft_size
  for (int k = threadIdx.x; k <= N; k += blockDim.x) {
    const double2 S = rfft_split(z, w, k, N);
    const double e = exp(S.x * inv_n);
    double s, c;
    sincos(S.y * inv_n, &s, &c);
    X[k] = make_double2(e * c, e * s);
  }
  __syncthreads();
}

// out[(j + rot) mod n] = r[j], r[j] = sum_k X[k] e^{2 pi i j k / n} over the Hermitian X given on 0..N (the imaginary
// parts of X[0] and X[N] are ignored, as a real inverse FFT does): the unnormalised inverse real FFT, then rotated by rot
// (N: fftshift).  out may alias X.
__device__ void irfft_shift(const double2* X, double2* z, const double2* w, double* out, int n, int N, int logN,
                            int rot) {
  for (int k = threadIdx.x; k < N; k += blockDim.x) {
    const double2 a = k == 0 ? make_double2(X[0].x, 0.0) : X[k];
    const double2 c = k == 0 ? make_double2(X[N].x, 0.0) : X[N - k];
    const double ex = a.x + c.x, ey = a.y - c.y;        // X[k] + conj X[N-k]
    const double dx = a.x - c.x, dy = a.y + c.y;        // X[k] - conj X[N-k]
    const double2 tw = w[k];                             // times conj(w[k]) = exp(+2 pi i k / n)
    const double ox = dx * tw.x + dy * tw.y, oy = dy * tw.x - dx * tw.y;
    z[brev_index(k, logN)] = make_double2(ex - oy, -(ey + ox));   // conj(E + i O): the inverse by a forward FFT
  }
  __syncthreads();
  fft_radix2_stages(z, w, N);
  for (int m = threadIdx.x; m < N; m += blockDim.x) {
    const double2 v = z[m];
    out[(2 * m + rot) & (n - 1)] = v.x;
    out[(2 * m + 1 + rot) & (n - 1)] = -v.y;
  }
  __syncthreads();
}

__device__ __forceinline__ double safe_ap(double a) { return fmax(0.001, fmin(0.999999999999, a)); }

// One block per pulse g0 + blockIdx.x: resp[blockIdx.x][j] = (periodic[j] sqrt(N_i) + aperiodic[j]) / n.
// Shared memory (doubles): z [n] (N complex), w [n], X [n + 2] (N + 1 complex; also the real scratch u), p [n], red [32].
__global__ void __launch_bounds__(WD_THREADS) world_response_kernel(const SynthParams p, int64_t g0) {
  extern __shared__ double2 wd_smem[];
  const int n = p.n, N = n / 2, logN = p.logN;
  double2* z = wd_smem;
  double2* w = z + N;
  double2* X = w + N;
  double* u = reinterpret_cast<double*>(X);
  double* per = reinterpret_cast<double*>(X + N + 1);
  double* red = per + n;
  const int64_t g = g0 + blockIdx.x;
  int lo = 0, hi = p.B - 1;                              // the row: the last b with row_start[b] <= g
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (p.row_start[mid] <= g) lo = mid; else hi = mid - 1;
  }
  const int b = lo;
  const int64_t i = g - p.row_start[b], P = p.info[b];
  const int32_t* idx = p.index + (int64_t)b * p.cap;
  const int ni = idx[i];
  const int64_t Ni = i + 1 < P ? (int64_t)idx[i + 1] - ni : 0;
  const double vuv = (double)p.vuv[(int64_t)b * p.cap + i];
  const int F = wd_length(p.lengths, b, p.T);
  // envelope and aperiodic ratio between frames floor and ceil of (n_i / fs) / frame_period, both clamped to F - 1
  const double q = __ddiv_rn(__ddiv_rn((double)ni, (double)p.fs), p.fp_s);
  const int ff = min(F - 1, (int)floor(q)), fc = min(F - 1, (int)ceil(q));
  const double wi = q - ff;
  const bool same = ff == fc;
  const float* s0 = p.sp + (int64_t)b * p.sp_bs + (int64_t)ff * p.sp_ts;
  const float* s1 = p.sp + (int64_t)b * p.sp_bs + (int64_t)fc * p.sp_ts;
  const double* a0 = p.ap + (int64_t)b * p.ap_bs + (int64_t)ff * p.ap_ts;
  const double* a1 = p.ap + (int64_t)b * p.ap_bs + (int64_t)fc * p.ap_ts;
  // Rounded as WORLD's C loop rounds, without FMA contraction: where ap is clamped near 1, 1 - ratio is ~2e-12, so an
  // ulp of the interpolated ap moves it by ~1e-4 relative and the minimum-phase step spreads that over every bin.
  const double wc = __dsub_rn(1.0, wi);
  auto env_ratio = [&](int k, double* env, double* ratio) {
    if (same) {
      const double a = safe_ap(a0[k]);
      *env = fabs((double)s0[k]);
      *ratio = __dmul_rn(a, a);
    } else {
      const double a = __dadd_rn(__dmul_rn(wc, safe_ap(a0[k])), __dmul_rn(wi, safe_ap(a1[k])));
      *env = __dadd_rn(__dmul_rn(wc, fabs((double)s0[k])), __dmul_rn(wi, fabs((double)s1[k])));
      *ratio = __dmul_rn(a, a);
    }
  };
  for (int j = threadIdx.x; j < N; j += blockDim.x) w[j] = p.tw[j];
  double env, ratio;
  env_ratio(0, &env, &ratio);
  const bool periodic = vuv > 0.5 && !(ratio > 0.999);
  __syncthreads();

  if (periodic) {
    for (int k = threadIdx.x; k <= N; k += blockDim.x) {
      env_ratio(k, &env, &ratio);
      u[k] = log(__dadd_rn(__dmul_rn(env, __dsub_rn(1.0, ratio)), WD_SAFE)) / 2.0;
    }
    __syncthreads();
    min_phase(u, z, w, X, n, N, logN);
    // fractional delay: bin k times cos(ck) - i sqrt(1 - cos^2(ck)), c = 2 pi shift fs / n
    const double coef = WD_TWO_PI * p.shift[(int64_t)b * p.cap + i] * p.fs / n;
    for (int k = threadIdx.x; k <= N; k += blockDim.x) {
      const double re = X[k].x, im = X[k].y;
      // c * c rounded before the subtraction, as WORLD computes it: an FMA here would differ by up to an ulp of 1, which
      // the cancellation near ck = 0 turns into a relative error of the sine up to ~1e-6
      const double c = cos(coef * k), s = sqrt(__dsub_rn(1.0, __dmul_rn(c, c)));
      X[k] = make_double2(re * c + im * s, im * c - re * s);
    }
    __syncthreads();
    irfft_shift(X, z, w, per, n, N, logN, N);
    double part = 0.0;
    for (int j = N + threadIdx.x; j < n; j += blockDim.x) part += per[j];
    const double dc = block_sum_f64(part, red);
    for (int j = threadIdx.x; j < n; j += blockDim.x) per[j] = j < N ? -dc * p.dcr[j] : per[j] - dc * p.dcr[j];
  } else {
    for (int j = threadIdx.x; j < n; j += blockDim.x) per[j] = 0.0;
  }
  __syncthreads();

  // aperiodic: minimum phase of the noise envelope, times the spectrum of the pulse's zero-mean noise
  for (int k = threadIdx.x; k <= N; k += blockDim.x) {
    env_ratio(k, &env, &ratio);
    u[k] = vuv != 0.0 ? log(env * ratio) / 2.0 : log(env) / 2.0;
  }
  __syncthreads();
  min_phase(u, z, w, X, n, N, logN);
  const double* nz = p.noise + (ni - idx[0]);            // the row's draws n_i - n_0 onwards
  double part = 0.0;
  for (int64_t j = threadIdx.x; j < Ni; j += blockDim.x) part += nz[j];
  const double mean = Ni > 0 ? block_sum_f64(part, red) / (double)Ni : 0.0;
  const int kept = (int)min(Ni, (int64_t)n);             // draws beyond n would not fit the FFT frame
  for (int m = threadIdx.x; m < N; m += blockDim.x) {
    const int j0 = 2 * m, j1 = 2 * m + 1;
    z[brev_index(m, logN)] = make_double2(j0 < kept ? nz[j0] - mean : 0.0, j1 < kept ? nz[j1] - mean : 0.0);
  }
  __syncthreads();
  fft_radix2_stages(z, w, N);
  for (int k = threadIdx.x; k <= N; k += blockDim.x) {
    const double2 ns = rfft_split(z, w, k, N), m = X[k];
    X[k] = make_double2(m.x * ns.x - m.y * ns.y, m.x * ns.y + m.y * ns.x);
  }
  __syncthreads();
  irfft_shift(X, z, w, u, n, N, logN, N);
  const double sq = sqrt((double)Ni);
  double* r = p.resp + (int64_t)blockIdx.x * n;
  for (int j = threadIdx.x; j < n; j += blockDim.x) r[j] = (per[j] * sq + u[j]) / n;
}

// y[b][s] += the responses of this chunk's pulses of row b that cover s, in ascending pulse order (pulse i covers
// [n_i - n/2 + 1, n_i + n/2 + 1)).
__global__ void __launch_bounds__(WD_THREADS) world_overlap_add_kernel(const SynthParams p, int64_t g0, int64_t g1) {
  const int b = blockIdx.y;
  const int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= p.info[p.B + b]) return;
  const int64_t rs = p.row_start[b];
  const int64_t lo = max(g0, rs) - rs, hi = min(g1, p.row_start[b + 1]) - rs;
  if (lo >= hi) return;
  const int32_t* idx = p.index + (int64_t)b * p.cap;
  const int N = p.n / 2;
  int64_t a = lo, c = hi;                                // the first pulse with n_i >= s - N
  while (a < c) {
    const int64_t mid = (a + c) >> 1;
    if ((int64_t)idx[mid] < s - N) a = mid + 1; else c = mid;
  }
  double* ys = p.y + (int64_t)b * p.y_stride + s;
  double acc = *ys;
  for (int64_t i = a; i < hi && (int64_t)idx[i] <= s + N - 1; ++i)
    acc += p.resp[(rs + i - g0) * p.n + (s - (idx[i] - N + 1))];
  *ys = acc;
}

static bool wd_fft_ok(int n) { return n >= WD_MIN_FFT && n <= WD_MAX_FFT && (n & (n - 1)) == 0; }

static size_t wd_align(size_t x) { return (x + 255) & ~(size_t)255; }

// workspace of gantts_world_synthesize: twiddles, DC remover, row starts, then the response buffer
static size_t wd_fixed_bytes(int B, int n) {
  return wd_align(sizeof(double2) * (size_t)(n / 2)) + wd_align(sizeof(double) * (size_t)n) +
         wd_align(sizeof(int64_t) * (size_t)(B + 1));
}

static size_t wd_response_smem(int n) { return sizeof(double) * (size_t)(4 * n + 2 + 32); }

}  // namespace gantts

using namespace gantts;

extern "C" int gantts_world_band_count(int fs) { return fs >= 1 ? world_bands(fs) : 0; }

extern "C" int64_t gantts_world_y_length(int64_t frames, int fs, double frame_period) {
  return world_y_length(frames, fs, frame_period);
}

extern "C" int gantts_world_decode_aperiodicity(const float* bap, int64_t bap_bstride, int64_t bap_tstride,
                                                const int64_t* lengths_dev, int B, int T, int nb, int fs, int fftlen,
                                                double* ap, void* stream) {
  GANTTS_CHECK_ARG(bap && lengths_dev && ap, "world_decode_aperiodicity: null pointer: bap, lengths_dev and ap are all "
                   "required");
  GANTTS_CHECK_ARG(B >= 1 && B <= 65535, "world_decode_aperiodicity: batch size B = %d must be in [1, 65535]", B);
  GANTTS_CHECK_ARG(T >= 1 && T <= WD_MAX_T, "world_decode_aperiodicity: padded length T = %d must be in [1, %d]", T,
                   WD_MAX_T);
  GANTTS_CHECK_ARG(fs >= 1, "world_decode_aperiodicity: fs = %d must be >= 1", fs);
  GANTTS_CHECK_ARG(world_bands(fs) >= 1, "world_decode_aperiodicity: fs = %d has no aperiodicity band (fs >= 12000)",
                   fs);
  GANTTS_CHECK_ARG(nb == world_bands(fs), "world_decode_aperiodicity: nb = %d coded bands, but WORLD codes %d at fs = %d",
                   nb, world_bands(fs), fs);
  GANTTS_CHECK_ARG(wd_fft_ok(fftlen), "world_decode_aperiodicity: fftlen = %d must be a power of two in [%d, %d]",
                   fftlen, WD_MIN_FFT, WD_MAX_FFT);
  GANTTS_CHECK_ARG(bap_bstride >= 0 && bap_tstride >= 0, "world_decode_aperiodicity: strides bap_bstride = %lld and "
                   "bap_tstride = %lld must be >= 0", (long long)bap_bstride, (long long)bap_tstride);
  world_decode_ap_kernel<<<dim3((unsigned)T, (unsigned)B), WD_THREADS, 0, as_stream(stream)>>>(
      bap, bap_bstride, bap_tstride, lengths_dev, T, nb, fs, fftlen, ap);
  GANTTS_LAUNCH_CHECK("world_decode_ap_kernel");
  return GANTTS_OK;
}

static int world_common_check(const char* what, int B, int T, int fs, double frame_period, int fftlen) {
  GANTTS_CHECK_ARG(B >= 1 && B <= 65535, "%s: batch size B = %d must be in [1, 65535]", what, B);
  GANTTS_CHECK_ARG(T >= 1 && T <= WD_MAX_T, "%s: padded length T = %d must be in [1, %d]", what, T, WD_MAX_T);
  GANTTS_CHECK_ARG(fs >= 1, "%s: fs = %d must be >= 1", what, fs);
  GANTTS_CHECK_ARG(isfinite(frame_period) && frame_period > 0.0, "%s: frame_period = %g ms must be finite and > 0", what,
                   frame_period);
  GANTTS_CHECK_ARG(wd_fft_ok(fftlen), "%s: fftlen = %d must be a power of two in [%d, %d]", what, fftlen, WD_MIN_FFT,
                   WD_MAX_FFT);
  const int64_t Y = world_y_length(T, fs, frame_period);
  GANTTS_CHECK_ARG(Y >= 1 && Y <= INT32_MAX, "%s: T = %d frames make %lld samples: the samples of a row must be in "
                   "[1, %d]", what, T, (long long)Y, INT32_MAX);
  return GANTTS_OK;
}

extern "C" int gantts_world_time_base(const float* f0, int64_t f0_bstride, int64_t f0_tstride,
                                      const int64_t* lengths_dev, int B, int T, int fs, double frame_period, int fftlen,
                                      int cap, int32_t* pulse_index, double* pulse_shift, uint8_t* pulse_vuv,
                                      int64_t* info_dev, void* stream) {
  GANTTS_CHECK_ARG(f0 && lengths_dev && pulse_index && pulse_shift && pulse_vuv && info_dev,
                   "world_time_base: null pointer: f0, lengths_dev, pulse_index, pulse_shift, pulse_vuv and info_dev "
                   "are all required");
  const int rc = world_common_check("world_time_base", B, T, fs, frame_period, fftlen);
  if (rc != GANTTS_OK) return rc;
  GANTTS_CHECK_ARG(f0_bstride >= 0 && f0_tstride >= 0, "world_time_base: strides f0_bstride = %lld and f0_tstride = "
                   "%lld must be >= 0", (long long)f0_bstride, (long long)f0_tstride);
  const int64_t Y = world_y_length(T, fs, frame_period);
  GANTTS_CHECK_ARG(cap >= Y, "world_time_base: cap = %d pulses per row, but a row of T = %d frames has %lld samples",
                   cap, T, (long long)Y);
  TimeBaseParams p{};
  p.f0 = f0; p.bs = f0_bstride; p.ts = f0_tstride; p.lengths = lengths_dev;
  p.B = B; p.T = T; p.fs = fs; p.cap = cap;
  p.fp_ms = frame_period;
  p.fp_s = frame_period / 1000.0;
  p.lowest = (double)(fs / fftlen) + 1.0;               // WORLD's fs / fft_size + 1.0, an integer division
  p.index = pulse_index; p.shift = pulse_shift; p.vuv = pulse_vuv; p.info = info_dev;
  cudaStream_t st = as_stream(stream);
  GANTTS_CUDA(cudaMemsetAsync(info_dev + 2 * B, 0, sizeof(int64_t), st));
  world_time_base_kernel<<<(unsigned)B, WD_THREADS, 0, st>>>(p);
  GANTTS_LAUNCH_CHECK("world_time_base_kernel");
  return GANTTS_OK;
}

extern "C" size_t gantts_world_randn_workspace_bytes(int64_t count) {
  return count < 1 ? 0 : sizeof(uint4) * 128 * (size_t)world_jump_count(count);
}

extern "C" int gantts_world_randn(int64_t count, double* out, void* workspace, size_t workspace_bytes, void* stream) {
  GANTTS_CHECK_ARG(count >= 1 && count <= INT32_MAX, "world_randn: count = %lld must be in [1, %d]", (long long)count,
                   INT32_MAX);
  GANTTS_CHECK_ARG(out && workspace, "world_randn: null output or workspace");
  const size_t need = gantts_world_randn_workspace_bytes(count);
  if (workspace_bytes < need) {
    set_error("world_randn: workspace of %zu bytes, %zu needed", workspace_bytes, need);
    return GANTTS_E_WORKSPACE;
  }
  cudaStream_t st = as_stream(stream);
  uint4* jump = static_cast<uint4*>(workspace);
  world_jump_kernel<<<1, 128, 0, st>>>(world_jump_count(count), jump);
  GANTTS_LAUNCH_CHECK("world_jump_kernel");
  const int64_t threads = (count + WD_CHUNK - 1) / WD_CHUNK;
  world_randn_kernel<<<(unsigned)((threads + WD_THREADS - 1) / WD_THREADS), WD_THREADS, 0, st>>>(jump, count, out);
  GANTTS_LAUNCH_CHECK("world_randn_kernel");
  return GANTTS_OK;
}

extern "C" size_t gantts_world_synthesize_workspace_bytes(int B, int fftlen, int64_t chunk_pulses) {
  if (B < 1 || !wd_fft_ok(fftlen) || chunk_pulses < 1) return 0;
  return wd_fixed_bytes(B, fftlen) + sizeof(double) * (size_t)fftlen * (size_t)chunk_pulses;
}

extern "C" int gantts_world_synthesize(const float* sp, int64_t sp_bstride, int64_t sp_tstride, const double* ap,
                                      int64_t ap_bstride, int64_t ap_tstride, const int64_t* lengths_dev,
                                      const int32_t* pulse_index, const double* pulse_shift, const uint8_t* pulse_vuv,
                                      const int64_t* info_dev, int cap, int64_t total_pulses, const double* noise,
                                      int B, int T, int fs, double frame_period, int fftlen, int y_max, double* y,
                                      void* workspace, size_t workspace_bytes, void* stream) {
  GANTTS_CHECK_ARG(sp && ap && lengths_dev && pulse_index && pulse_shift && pulse_vuv && info_dev && noise && y &&
                   workspace, "world_synthesize: null pointer: sp, ap, lengths_dev, the pulse arrays, info_dev, noise, "
                   "y and workspace are all required");
  const int rc = world_common_check("world_synthesize", B, T, fs, frame_period, fftlen);
  if (rc != GANTTS_OK) return rc;
  GANTTS_CHECK_ARG(sp_bstride >= 0 && sp_tstride >= 0 && ap_bstride >= 0 && ap_tstride >= 0,
                   "world_synthesize: strides sp_bstride = %lld, sp_tstride = %lld, ap_bstride = %lld and ap_tstride = "
                   "%lld must be >= 0", (long long)sp_bstride, (long long)sp_tstride, (long long)ap_bstride,
                   (long long)ap_tstride);
  const int64_t Ycap = world_y_length(T, fs, frame_period);
  GANTTS_CHECK_ARG(cap >= Ycap, "world_synthesize: cap = %d pulses per row, but a row of T = %d frames has %lld samples",
                   cap, T, (long long)Ycap);
  GANTTS_CHECK_ARG(y_max >= 1 && y_max <= Ycap, "world_synthesize: y_max = %d must be in [1, %lld]", y_max,
                   (long long)Ycap);
  GANTTS_CHECK_ARG(total_pulses >= 0, "world_synthesize: total_pulses = %lld must be >= 0", (long long)total_pulses);
  const size_t fixed = wd_fixed_bytes(B, fftlen);
  const int64_t chunk = workspace_bytes > fixed ? (int64_t)((workspace_bytes - fixed) / (sizeof(double) * fftlen)) : 0;
  if (chunk < 1) {
    set_error("world_synthesize: workspace of %zu bytes holds no pulse response (%zu needed for one)", workspace_bytes,
              gantts_world_synthesize_workspace_bytes(B, fftlen, 1));
    return GANTTS_E_WORKSPACE;
  }
  const int n = fftlen, N = n / 2;
  char* ws = static_cast<char*>(workspace);
  double2* tw = reinterpret_cast<double2*>(ws);
  ws += wd_align(sizeof(double2) * (size_t)N);
  double* dcr = reinterpret_cast<double*>(ws);
  ws += wd_align(sizeof(double) * (size_t)n);
  int64_t* row_start = reinterpret_cast<int64_t*>(ws);
  ws += wd_align(sizeof(int64_t) * (size_t)(B + 1));
  SynthParams p{};
  p.sp = sp; p.sp_bs = sp_bstride; p.sp_ts = sp_tstride;
  p.ap = ap; p.ap_bs = ap_bstride; p.ap_ts = ap_tstride;
  p.lengths = lengths_dev; p.index = pulse_index; p.shift = pulse_shift; p.vuv = pulse_vuv; p.info = info_dev;
  p.noise = noise; p.row_start = row_start; p.tw = tw; p.dcr = dcr; p.resp = reinterpret_cast<double*>(ws);
  p.y = y; p.y_stride = y_max; p.B = B; p.T = T; p.cap = cap; p.fs = fs; p.n = n;
  p.logN = 0;
  while ((1 << p.logN) < N) ++p.logN;
  p.fp_s = frame_period / 1000.0;
  cudaStream_t st = as_stream(stream);
  GANTTS_CUDA(cudaMemsetAsync(y, 0, sizeof(double) * (size_t)B * (size_t)y_max, st));
  world_setup_kernel<<<1, WD_THREADS, 0, st>>>(p, tw, dcr, row_start);
  GANTTS_LAUNCH_CHECK("world_setup_kernel");
  const size_t smem = wd_response_smem(n);
  GANTTS_CUDA(cudaFuncSetAttribute(world_response_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const dim3 ola_grid((unsigned)((y_max + WD_THREADS - 1) / WD_THREADS), (unsigned)B);
  for (int64_t g0 = 0; g0 < total_pulses; g0 += chunk) {   // chunks in order: each sample's sum keeps pulse order
    const int64_t g1 = min(total_pulses, g0 + chunk);
    prof_begin(PROF_WORLD_RESPONSE, (double)(g1 - g0), st);
    world_response_kernel<<<(unsigned)(g1 - g0), WD_THREADS, smem, st>>>(p, g0);
    prof_end(st);
    GANTTS_LAUNCH_CHECK("world_response_kernel");
    prof_begin(PROF_WORLD_OLA, (double)B * (double)y_max, st);
    world_overlap_add_kernel<<<ola_grid, WD_THREADS, 0, st>>>(p, g0, g1);
    prof_end(st);
    GANTTS_LAUNCH_CHECK("world_overlap_add_kernel");
  }
  return GANTTS_OK;
}
