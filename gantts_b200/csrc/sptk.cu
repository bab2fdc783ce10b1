// Spectral post-processing of generated mel-cepstra (reference evaluation_tts.py:103-115 gen_waveform): Merlin's post
// filter (nnmnkwii.postfilters.merlin_post_filter) and the power spectral envelope (pysptk.mc2sp).
//
// Up to the final exp, both are linear in the frame: freqt (the all-pass frequency warp), then the real FFT of a
// symmetric or zero-padded cepstrum.  So each is one fixed K x (M+1) fp64 matrix, built on the host by
// gantts_mcep_operator, whose row k maps a frame to its log power at bin k (K = fftlen/2 + 1).  The kernels apply that
// matrix to every valid frame of a padded batch and run a per-bin epilogue: exp for the envelope; for the post filter the
// bin-weighted exp sums r0 of mc and of w*mc, from which only c0 changes (mc2b / b2mc are inverse linear maps and freqt
// sends e0 to e0, so b2mc(mc2b(w*mc) + d e0) = w*mc + d e0).
#include "common.cuh"

#include <math.h>

#include <vector>

namespace gantts {

constexpr int MCEP_MAX_COLS = 128;     // M + 1
constexpr int MCEP_FRAMES = 32;        // frames per block (8 warps x 4 frames)
constexpr int MCEP_BINS = 64;          // bins per staged operator tile (2 per lane)
constexpr int MCEP_THREADS = 256;
constexpr int MCEP_PITCH = MCEP_BINS + 1;   // doubles per staged operator row: the transposing store is 2-way at worst
constexpr int MCEP_MAX_T = 1 << 24;

struct McepParams {
  const float* mc;
  int64_t m_bs, m_ts;
  float* out;                           // post filter: [B][T][M+1]; envelope: [B][T][K]
  int64_t o_bs, o_ts;
  const double* op;                     // [K][M+1]
  const int64_t* lengths;
  double coef;
  int T, M1, K;
};

// One block per (32-frame tile, batch row).  Warp w owns frames 4w..4w+3 of the tile; lane l owns bins l and l + 32 of
// each operator tile.  Every sum a frame's result depends on runs in an order fixed by m and k alone, so a frame gives the
// same bits wherever it sits in the batch.
template <bool POSTFILTER>
__global__ void __launch_bounds__(MCEP_THREADS) mcep_kernel(const McepParams p) {
  extern __shared__ double mcep_smem[];
  const int b = blockIdx.y, t0 = blockIdx.x * MCEP_FRAMES, M1 = p.M1;
  const int64_t Lraw = p.lengths[b];
  const int L = Lraw < 0 ? 0 : (Lraw > p.T ? p.T : (int)Lraw);
  const int nf = min(MCEP_FRAMES, p.T - t0);             // frames of this tile inside [0, T)
  const int nv = max(0, min(nf, L - t0));                // of which valid
  const int width = POSTFILTER ? M1 : p.K;
  float* out = p.out + (int64_t)b * p.o_bs;
  for (int i = threadIdx.x; i < (nf - nv) * width; i += blockDim.x) {
    const int f = nv + i / width, c = i - (i / width) * width;
    out[(int64_t)(t0 + f) * p.o_ts + c] = 0.f;
  }
  if (nv == 0) return;

  double* xs = mcep_smem;                                   // [F][M1] the frames
  double* xw = xs + MCEP_FRAMES * M1;                       // [F][M1] w * frames (post filter)
  double* ot = xw + (POSTFILTER ? MCEP_FRAMES * M1 : 0);    // [M1][PITCH] operator tile, bin-contiguous
  const float* mc = p.mc + (int64_t)b * p.m_bs;
  for (int i = threadIdx.x; i < MCEP_FRAMES * M1; i += blockDim.x) {
    const int f = i / M1, m = i - f * M1;
    const double v = f < nv ? (double)mc[(int64_t)(t0 + f) * p.m_ts + m] : 0.0;
    xs[i] = v;
    if (POSTFILTER) xw[i] = m < 2 ? v : v * p.coef;
  }
  const int lane = threadIdx.x & 31, fr = (threadIdx.x >> 5) * 4;
  double su[4] = {0.0, 0.0, 0.0, 0.0}, sv[4] = {0.0, 0.0, 0.0, 0.0};
  for (int k0 = 0; k0 < p.K; k0 += MCEP_BINS) {
    __syncthreads();                                     // frames staged / previous tile consumed
    for (int i = threadIdx.x; i < MCEP_BINS * M1; i += blockDim.x) {
      const int kk = i / M1, m = i - kk * M1;
      ot[m * MCEP_PITCH + kk] = k0 + kk < p.K ? p.op[(int64_t)k0 * M1 + i] : 0.0;
    }
    __syncthreads();
    double u[4][2], v[4][2];
#pragma unroll
    for (int f = 0; f < 4; ++f) u[f][0] = u[f][1] = v[f][0] = v[f][1] = 0.0;
#pragma unroll 2
    for (int m = 0; m < M1; ++m) {
      const double o0 = ot[m * MCEP_PITCH + lane], o1 = ot[m * MCEP_PITCH + lane + 32];
#pragma unroll
      for (int f = 0; f < 4; ++f) {
        const double x = xs[(fr + f) * M1 + m];
        u[f][0] = fma(o0, x, u[f][0]);
        u[f][1] = fma(o1, x, u[f][1]);
        if (POSTFILTER) {
          const double y = xw[(fr + f) * M1 + m];
          v[f][0] = fma(o0, y, v[f][0]);
          v[f][1] = fma(o1, y, v[f][1]);
        }
      }
    }
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int k = k0 + lane + 32 * j;
      if (k >= p.K) continue;
      if (POSTFILTER) {
        // c2acr's sum over all n bins of the real spectrum: bins 0 and n/2 once, the others twice (the 1/n cancels)
        const double wk = (k == 0 || k == p.K - 1) ? 1.0 : 2.0;
#pragma unroll
        for (int f = 0; f < 4; ++f) {
          su[f] += wk * exp(u[f][j]);
          sv[f] += wk * exp(v[f][j]);
        }
      } else {
#pragma unroll
        for (int f = 0; f < 4; ++f)
          if (fr + f < nv) out[(int64_t)(t0 + fr + f) * p.o_ts + k] = (float)exp(u[f][j]);
      }
    }
  }
  if (POSTFILTER) {
#pragma unroll
    for (int f = 0; f < 4; ++f) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {                 // butterfly: every lane ends with the same bits
        su[f] += __shfl_xor_sync(0xffffffffu, su[f], o);
        sv[f] += __shfl_xor_sync(0xffffffffu, sv[f], o);
      }
      if (fr + f >= nv) continue;
      const double d = 0.5 * log(su[f] / sv[f]);         // keeps r0 of the filtered frame equal to r0 of the input
      float* o = out + (int64_t)(t0 + fr + f) * p.o_ts;
      for (int m = lane; m < M1; m += 32) o[m] = (float)(m == 0 ? xs[(fr + f) * M1] + d : xw[(fr + f) * M1 + m]);
    }
  }
}

static bool mcep_fftlen_ok(int n) { return n >= 64 && n <= 4096 && (n & (n - 1)) == 0; }

// The rules shared by both kernels; sets the error message and returns false when one fails.
static bool mcep_check(const char* what, const float* in, const void* out, const double* op, const int64_t* lengths_dev,
                       int B, int T, int M, int K) {
  if (!lengths_dev) {
    set_error("%s: null lengths: every row is processed over its own lengths_dev[b] frames", what);
    return false;
  }
  if (B < 1 || B > 65535) {
    set_error("%s: batch size B = %d must be in [1, 65535]", what, B);
    return false;
  }
  if (T < 1 || T > MCEP_MAX_T) {
    set_error("%s: padded length T = %d must be in [1, %d]", what, T, MCEP_MAX_T);
    return false;
  }
  if (M < 0 || M + 1 > MCEP_MAX_COLS) {
    set_error("%s: order M = %d: M + 1 must be in [1, %d]", what, M, MCEP_MAX_COLS);
    return false;
  }
  if (K < 2 || !mcep_fftlen_ok(2 * (K - 1))) {
    set_error("%s: K = %d bins: fftlen = 2 (K - 1) must be a power of two in [64, 4096]", what, K);
    return false;
  }
  if (!in || !out || !op) {
    set_error("%s: null input, output or operator", what);
    return false;
  }
  return true;
}

template <bool POSTFILTER>
static int mcep_launch(const McepParams& p, int B, void* stream) {
  auto fn = mcep_kernel<POSTFILTER>;
  const size_t smem = sizeof(double) * (size_t)p.M1 * ((POSTFILTER ? 2 : 1) * MCEP_FRAMES + MCEP_PITCH);
  GANTTS_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const dim3 grid((unsigned)((p.T + MCEP_FRAMES - 1) / MCEP_FRAMES), (unsigned)B);
  fn<<<grid, MCEP_THREADS, smem, as_stream(stream)>>>(p);
  GANTTS_LAUNCH_CHECK("mcep_kernel");
  return GANTTS_OK;
}

}  // namespace gantts

using namespace gantts;

extern "C" int gantts_mcep_operator(double alpha, int order, int fftlen, int kind, double* out) {
  GANTTS_CHECK_ARG(fabs(alpha) < 1.0, "mcep_operator: alpha = %g must satisfy |alpha| < 1", alpha);
  GANTTS_CHECK_ARG(order >= 0 && order + 1 <= MCEP_MAX_COLS, "mcep_operator: order M = %d: M + 1 must be in [1, %d]",
                   order, MCEP_MAX_COLS);
  GANTTS_CHECK_ARG(mcep_fftlen_ok(fftlen), "mcep_operator: fftlen = %d must be a power of two in [64, 4096]", fftlen);
  GANTTS_CHECK_ARG(kind == GANTTS_MCEP_R0 || kind == GANTTS_MCEP_SP,
                   "mcep_operator: kind %d must be GANTTS_MCEP_R0 (0) or GANTTS_MCEP_SP (1)", kind);
  GANTTS_CHECK_ARG(out != nullptr, "mcep_operator: null output");
  const int M1 = order + 1, n = fftlen, half = n / 2, K = half + 1;
  const int m2 = kind == GANTTS_MCEP_SP ? half : half - 1;   // freqt order: n/2 (mc2sp), n/2 - 1 (merlin_post_filter)
  // C[i][m]: coefficient i of freqt(e_m, m2, -alpha), the SPTK recursion run on each unit vector
  const double a = -alpha, bb = 1.0 - a * a;
  std::vector<double> C((size_t)(m2 + 1) * M1, 0.0), g(m2 + 1), d(m2 + 1);
  for (int m = 0; m < M1; ++m) {
    std::fill(g.begin(), g.end(), 0.0);
    for (int i = m; i >= 0; --i) {                        // coefficients above m are 0 and leave g at 0
      d = g;
      g[0] = (i == m ? 1.0 : 0.0) + a * d[0];
      if (m2 >= 1) g[1] = bb * d[0] + a * d[1];
      for (int j = 2; j <= m2; ++j) g[j] = d[j - 1] + a * (d[j] - g[j - 1]);
    }
    for (int i = 0; i <= m2; ++i) C[(size_t)i * M1 + m] = g[i];
  }
  // log power at bin k: 2 (c0 + sum_{0 < i < n/2} c_i cos(2 pi i k / n) [+ c_{n/2} (-1)^k / 2 for mc2sp's symmetric
  // cepstrum, whose Nyquist term is counted once])
  std::vector<double> cs(n), row(M1);
  for (int j = 0; j < n; ++j) cs[j] = cos(2.0 * M_PI * (double)j / (double)n);
  for (int k = 0; k < K; ++k) {
    for (int m = 0; m < M1; ++m) row[m] = C[m];
    for (int i = 1; i < half; ++i) {
      const double c = cs[((int64_t)i * k) & (n - 1)];
      const double* ci = &C[(size_t)i * M1];
      for (int m = 0; m < M1; ++m) row[m] += ci[m] * c;
    }
    if (kind == GANTTS_MCEP_SP) {
      const double h = (k & 1) ? -0.5 : 0.5;
      const double* ci = &C[(size_t)half * M1];
      for (int m = 0; m < M1; ++m) row[m] += ci[m] * h;
    }
    for (int m = 0; m < M1; ++m) out[(size_t)k * M1 + m] = 2.0 * row[m];
  }
  return GANTTS_OK;
}

extern "C" int gantts_mcep_postfilter(const float* mc, int64_t mc_bstride, int64_t mc_tstride, float* out,
                                      int64_t out_bstride, int64_t out_tstride, const double* op_r, double coef,
                                      const int64_t* lengths_dev, int B, int T, int M, int K, void* stream) {
  if (!mcep_check("mcep_postfilter", mc, out, op_r, lengths_dev, B, T, M, K)) return GANTTS_E_BADARG;
  GANTTS_CHECK_ARG(isfinite(coef), "mcep_postfilter: coef = %g must be finite", coef);
  McepParams p{};
  p.mc = mc; p.m_bs = mc_bstride; p.m_ts = mc_tstride;
  p.out = out; p.o_bs = out_bstride; p.o_ts = out_tstride;
  p.op = op_r; p.lengths = lengths_dev; p.coef = coef;
  p.T = T; p.M1 = M + 1; p.K = K;
  return mcep_launch<true>(p, B, stream);
}

extern "C" int gantts_mcep_to_sp(const float* mc, int64_t mc_bstride, int64_t mc_tstride, float* sp, int64_t sp_bstride,
                                 int64_t sp_tstride, const double* op_s, const int64_t* lengths_dev, int B, int T, int M,
                                 int K, void* stream) {
  if (!mcep_check("mcep_to_sp", mc, sp, op_s, lengths_dev, B, T, M, K)) return GANTTS_E_BADARG;
  McepParams p{};
  p.mc = mc; p.m_bs = mc_bstride; p.m_ts = mc_tstride;
  p.out = sp; p.o_bs = sp_bstride; p.o_ts = sp_tstride;
  p.op = op_s; p.lengths = lengths_dev; p.coef = 1.0;
  p.T = T; p.M1 = M + 1; p.K = K;
  return mcep_launch<false>(p, B, stream);
}
