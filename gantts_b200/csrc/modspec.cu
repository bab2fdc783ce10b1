// Objective measures of generated features (the reference notebooks' vis_gv and mean_modspec): the global variance of
// each feature column over an utterance's frames, and its log modulation spectrum, the log power of the column's
// n-point real FFT along time (nnmnkwii.preprocessing.modspec).
//
// Both kernels give a column the same bits wherever it sits: every sum runs in an order fixed by the column's own valid
// frames, never by the batch position, the padded length or the neighbouring columns.  That is why each column gets
// its own complex FFT (n/2 points of x[2j] + i x[2j+1] and the split step) rather than two columns sharing one.
#include "common.cuh"

#include <math.h>

namespace gantts {

constexpr int MS_THREADS = 256;
constexpr int MS_MIN_N = 64;
constexpr int MS_MAX_N = 8192;
constexpr int MS_MAX_T = 1 << 24;
constexpr int MS_MAX_D = 65535;
constexpr int GV_COLS = 32;            // columns per block (one per lane)
constexpr int GV_SLICES = 8;           // warps; warp w sums frames t = w (mod 8)
constexpr int FOLD_THREADS = 256;

struct FeatureParams {
  const float* x;
  int64_t x_bs, x_ts;
  const int64_t* lengths;
  int T, D;
};

__device__ __forceinline__ int clamped_length(const FeatureParams& p, int b) {
  const int64_t L = p.lengths[b];
  return L < 0 ? 0 : (L > p.T ? p.T : (int)L);
}

// One block per (column d, row b).  Shared memory: z[N] the column packed as N = n/2 complex values, in bit-reversed
// order, then its FFT; w[N] = exp(-2 pi i k / n).  Radix-2 decimation in time, then the real-FFT split
// X[k] = E[k] + w^k O[k], E = (Z[k] + conj Z[N-k]) / 2, O = (Z[k] - conj Z[N-k]) / 2i.
__global__ void __launch_bounds__(MS_THREADS) modspec_kernel(const FeatureParams p, int n, int log2n, double* out) {
  extern __shared__ double2 ms_smem[];
  const int d = blockIdx.x, b = blockIdx.y, N = n >> 1, logN = log2n - 1;
  double2* z = ms_smem;
  double2* w = z + N;
  const int L = min(clamped_length(p, b), n);            // frames beyond n are cropped, as np.fft.rfft(x, n) does
  const float* col = p.x + (int64_t)b * p.x_bs + d;
  for (int j = threadIdx.x; j < N; j += blockDim.x) {
    double s, c;
    sincospi(-2.0 * (double)j / (double)n, &s, &c);
    w[j] = make_double2(c, s);
    const int t = 2 * j;
    const double re = t < L ? (double)col[(int64_t)t * p.x_ts] : 0.0;
    const double im = t + 1 < L ? (double)col[(int64_t)(t + 1) * p.x_ts] : 0.0;
    z[__brev((unsigned)j) >> (32 - logN)] = make_double2(re, im);
  }
  __syncthreads();
  fft_radix2_stages(z, w, N);
  const int K = N + 1;
  double* o = out + (int64_t)b * K * p.D + d;
  for (int k = threadIdx.x; k < K; k += blockDim.x) {
    const double2 X = rfft_split(z, w, k, N);
    o[(int64_t)k * p.D] = log(X.x * X.x + X.y * X.y);
  }
}

// sum[i] += ms[b][i] for b = 0, 1, ..., B-1 in that order: a running mean over utterances added in a fixed order has the
// same bits however they were batched.
__global__ void __launch_bounds__(FOLD_THREADS) modspec_fold_kernel(const double* ms, int B, int64_t KD, double* sum) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= KD) return;
  double s = sum[i];
  for (int b = 0; b < B; ++b) s += ms[(int64_t)b * KD + i];
  sum[i] = s;
}

// One block per (32-column tile, row b).  Two passes over the valid frames in fp64: the mean, then the mean squared
// deviation (np.var, ddof 0).  Warp w sums frames w, w + 8, ...; the 8 partial sums are added in warp order.
__global__ void __launch_bounds__(GV_COLS * GV_SLICES) global_variance_kernel(const FeatureParams p, double* out) {
  __shared__ double part[GV_SLICES][GV_COLS];
  __shared__ double mean[GV_COLS];
  const int lane = threadIdx.x & 31, slice = threadIdx.x >> 5, b = blockIdx.y;
  const int d = blockIdx.x * GV_COLS + lane;
  const int L = clamped_length(p, b);
  const float* col = p.x + (int64_t)b * p.x_bs + d;
  double s = 0.0;
  if (d < p.D)
    for (int t = slice; t < L; t += GV_SLICES) s += (double)col[(int64_t)t * p.x_ts];
  part[slice][lane] = s;
  __syncthreads();
  if (slice == 0) {
    double tot = 0.0;
#pragma unroll
    for (int i = 0; i < GV_SLICES; ++i) tot += part[i][lane];
    mean[lane] = tot / (double)L;                        // L = 0: NaN, as np.var of no frames
  }
  __syncthreads();
  const double m = mean[lane];
  s = 0.0;
  if (d < p.D)
    for (int t = slice; t < L; t += GV_SLICES) {
      const double e = (double)col[(int64_t)t * p.x_ts] - m;
      s += e * e;
    }
  part[slice][lane] = s;                                 // the first sums were read before the last barrier
  __syncthreads();
  if (slice == 0 && d < p.D) {
    double tot = 0.0;
#pragma unroll
    for (int i = 0; i < GV_SLICES; ++i) tot += part[i][lane];
    out[(int64_t)b * p.D + d] = tot / (double)L;
  }
}

static bool modspec_n_ok(int n) { return n >= MS_MIN_N && n <= MS_MAX_N && (n & (n - 1)) == 0; }

// The rules shared by both entry points; sets the error message and returns false when one fails.
static bool feature_check(const char* what, const float* x, int64_t x_bstride, int64_t x_tstride,
                          const int64_t* lengths_dev, int B, int T, int D, const void* out) {
  if (!lengths_dev) {
    set_error("%s: null lengths: every row is processed over its own lengths_dev[b] frames", what);
    return false;
  }
  if (B < 1 || B > 65535) {
    set_error("%s: batch size B = %d must be in [1, 65535]", what, B);
    return false;
  }
  if (T < 1 || T > MS_MAX_T) {
    set_error("%s: padded length T = %d must be in [1, %d]", what, T, MS_MAX_T);
    return false;
  }
  if (D < 1 || D > MS_MAX_D) {
    set_error("%s: feature width D = %d must be in [1, %d]", what, D, MS_MAX_D);
    return false;
  }
  if (x_bstride < 0 || x_tstride < 0) {
    set_error("%s: strides x_bstride = %lld and x_tstride = %lld must be >= 0", what, (long long)x_bstride,
              (long long)x_tstride);
    return false;
  }
  if (!x || !out) {
    set_error("%s: null input or output", what);
    return false;
  }
  return true;
}

static FeatureParams feature_params(const float* x, int64_t x_bstride, int64_t x_tstride, const int64_t* lengths_dev,
                                    int T, int D) {
  FeatureParams p{};
  p.x = x; p.x_bs = x_bstride; p.x_ts = x_tstride;
  p.lengths = lengths_dev; p.T = T; p.D = D;
  return p;
}

}  // namespace gantts

using namespace gantts;

extern "C" int gantts_modspec(const float* x, int64_t x_bstride, int64_t x_tstride, const int64_t* lengths_dev, int B,
                              int T, int D, int n, double* out, double* sum_dev, void* stream) {
  if (!feature_check("modspec", x, x_bstride, x_tstride, lengths_dev, B, T, D, out)) return GANTTS_E_BADARG;
  GANTTS_CHECK_ARG(modspec_n_ok(n), "modspec: n = %d must be a power of two in [%d, %d]", n, MS_MIN_N, MS_MAX_N);
  int log2n = 0;
  while ((1 << log2n) < n) ++log2n;
  const FeatureParams p = feature_params(x, x_bstride, x_tstride, lengths_dev, T, D);
  const size_t smem = sizeof(double2) * (size_t)n;      // z and w, n/2 complex values each
  GANTTS_CUDA(cudaFuncSetAttribute(modspec_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  cudaStream_t st = as_stream(stream);
  modspec_kernel<<<dim3((unsigned)D, (unsigned)B), MS_THREADS, smem, st>>>(p, n, log2n, out);
  GANTTS_LAUNCH_CHECK("modspec_kernel");
  if (sum_dev) {
    const int64_t KD = (int64_t)(n / 2 + 1) * D;
    modspec_fold_kernel<<<(unsigned)((KD + FOLD_THREADS - 1) / FOLD_THREADS), FOLD_THREADS, 0, st>>>(out, B, KD,
                                                                                                       sum_dev);
    GANTTS_LAUNCH_CHECK("modspec_fold_kernel");
  }
  return GANTTS_OK;
}

extern "C" int gantts_global_variance(const float* x, int64_t x_bstride, int64_t x_tstride, const int64_t* lengths_dev,
                                      int B, int T, int D, double* out, void* stream) {
  if (!feature_check("global_variance", x, x_bstride, x_tstride, lengths_dev, B, T, D, out)) return GANTTS_E_BADARG;
  const FeatureParams p = feature_params(x, x_bstride, x_tstride, lengths_dev, T, D);
  const dim3 grid((unsigned)((D + GV_COLS - 1) / GV_COLS), (unsigned)B);
  global_variance_kernel<<<grid, GV_COLS * GV_SLICES, 0, as_stream(stream)>>>(p, out);
  GANTTS_LAUNCH_CHECK("global_variance_kernel");
  return GANTTS_OK;
}
