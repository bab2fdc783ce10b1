// Shared helpers for libgantts_b200.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "../../include/gantts_b200.h"

namespace gantts {

// Thread-local last-error message (gantts_last_error_string()).
void set_error(const char* fmt, ...);
int cuda_fail(cudaError_t e, const char* what);

#define GANTTS_CHECK_ARG(cond, ...)            \
  do {                                         \
    if (!(cond)) {                             \
      ::gantts::set_error(__VA_ARGS__);        \
      return GANTTS_E_BADARG;                  \
    }                                          \
  } while (0)

#define GANTTS_CUDA(call)                                        \
  do {                                                           \
    cudaError_t _e = (call);                                     \
    if (_e != cudaSuccess) return ::gantts::cuda_fail(_e, #call); \
  } while (0)

#define GANTTS_LAUNCH_CHECK(name)                                     \
  do {                                                                \
    cudaError_t _e = cudaGetLastError();                              \
    if (_e != cudaSuccess) return ::gantts::cuda_fail(_e, "launch " name); \
    ::gantts::count_launch();                                         \
  } while (0)

// Kernel-launch counter (gantts_launch_count) and optional CUDA-event profiling of selected kernels
// (gantts_profile_*): event pairs are recorded on the launching stream around each profiled launch.
void count_launch();
enum ProfKind { PROF_GEMM_KK = 0, PROF_GEMM_MN = 1, PROF_MLPG_FWD = 2, PROF_MLPG_BWD = 3, PROF_LSTM_FWD = 4,
                PROF_LSTM_BWD = 5, PROF_WORLD_RESPONSE = 6, PROF_WORLD_OLA = 7, PROF_KINDS = 8 };
void prof_begin(int kind, double work, cudaStream_t st);   // work: algorithmic flops or bytes
void prof_end(cudaStream_t st);

static inline cudaStream_t as_stream(void* s) { return reinterpret_cast<cudaStream_t>(s); }

// Programmatic dependent launch for the tensor-core GEMMs and the small streaming kernels of the fused step:
// a kernel launched through GANTTS_PDL_LAUNCH may become resident while its predecessor in the stream is still in its last
// wave; pdl_entry() at the top of the kernel (a) lets ITS successor do the same and (b) blocks until every prerequisite
// grid has completed and its writes are visible -- nothing the predecessor produced is touched before that.  Without the
// launch attribute (plain <<<>>> launches, the modular ops) both instructions are no-ops.  GANTTS_B200_PDL=0 disables.
__device__ __forceinline__ void pdl_entry() {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");
}
inline int pdl_enabled() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("GANTTS_B200_PDL");
    v = e ? atoi(e) : 1;
  }
  return v;
}
template <typename... KA, typename... A>
static inline void pdl_launch(void (*kern)(KA...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, A&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  cudaLaunchKernelEx(&cfg, kern, static_cast<KA>(args)...);       // errors surface through GANTTS_LAUNCH_CHECK
}
#define GANTTS_PDL_LAUNCH(kern, grid, block, smem, st, ...) \
  ::gantts::pdl_launch(kern, dim3(grid), dim3(block), (size_t)(smem), st, __VA_ARGS__)

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Block-wide sum of up to 4 values; result valid in thread 0.  smem: float[4][32].
template <int NV>
__device__ __forceinline__ void block_sum(float (&v)[NV], float* smem) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = (blockDim.x + 31) >> 5;
#pragma unroll
  for (int i = 0; i < NV; ++i) v[i] = warp_sum(v[i]);
  if (lane == 0) {
#pragma unroll
    for (int i = 0; i < NV; ++i) smem[i * 32 + warp] = v[i];
  }
  __syncthreads();
  if (warp == 0) {
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      float x = lane < nwarp ? smem[i * 32 + lane] : 0.f;
      v[i] = warp_sum(x);
    }
  }
}

// In-place radix-2 decimation-in-time FFT of N = n/2 complex points in shared memory, by the whole block: z holds the
// input in bit-reversed order, w[j] = exp(-2 pi i j / n) for j < N; butterflies of span h use the twiddle
// exp(-2 pi i pos / 2h) = w[pos * N / h].  Ends with a barrier.  (modspec.cu, world.cu)
__device__ __forceinline__ void fft_radix2_stages(double2* z, const double2* w, int N) {
  for (int h = 1; h < N; h <<= 1) {
    const int step = N / h;
    for (int i = threadIdx.x; i < N / 2; i += blockDim.x) {
      const int pos = i & (h - 1), i0 = ((i - pos) << 1) + pos, i1 = i0 + h;
      const double2 tw = w[pos * step], a = z[i0], v = z[i1];
      const double tr = tw.x * v.x - tw.y * v.y, ti = tw.x * v.y + tw.y * v.x;
      z[i0] = make_double2(a.x + tr, a.y + ti);
      z[i1] = make_double2(a.x - tr, a.y - ti);
    }
    __syncthreads();
  }
}

// Bin k (0 <= k <= N) of the n-point real FFT X of x from Z, the N-point FFT of x[2j] + i x[2j+1]:
// X[k] = E[k] + w^k O[k], E = (Z[k] + conj Z[N-k]) / 2, O = (Z[k] - conj Z[N-k]) / 2i.
__device__ __forceinline__ double2 rfft_split(const double2* z, const double2* w, int k, int N) {
  if (k == 0 || k == N)                                  // E[0] = Re Z[0], O[0] = Im Z[0], w^N = -1
    return make_double2(k == 0 ? z[0].x + z[0].y : z[0].x - z[0].y, 0.0);
  const double2 a = z[k], c = z[N - k];
  const double er = 0.5 * (a.x + c.x), ei = 0.5 * (a.y - c.y);
  const double orr = 0.5 * (a.y + c.y), oi = -0.5 * (a.x - c.x);
  const double2 tw = w[k];
  return make_double2(er + (tw.x * orr - tw.y * oi), ei + (tw.x * oi + tw.y * orr));
}

// Counter-based keep decision for dropout: one 32-bit mixing chain per FOUR adjacent columns
// (key = row * ceil(N/4) + col/4, 32-bit wrap-around arithmetic) gives word a (columns 4q, 4q+1) and, by one more
// multiply-xorshift round, word b (columns 4q+2, 4q+3); 16-bit field per element, low field = even column:
// keep iff field >= thresh, thresh = round(p * 65536).  Every engine (tensor-core GEMM epilogues, SIMT GEMM,
// LSTM inter-layer dropout, gantts_dropout) uses exactly this function, so they produce identical masks.
// Not torch's Philox stream (SURVEY.md 7, hard part 4).  (Round 1 hashed once per column PAIR: the epilogues are
// issue-bound and the hash was ~16 % of their instructions.)
struct DropBits {
  uint32_t a, b;
};
__device__ __forceinline__ DropBits dropout_quad_bits(uint64_t seed, uint32_t row, uint32_t quarter_n, uint32_t quad) {
  uint32_t x = (row * quarter_n + quad) * 0x9E3779B1u + static_cast<uint32_t>(seed);
  x ^= x >> 16; x *= 0x7feb352dU; x ^= x >> 15; x *= 0x846ca68bU; x ^= x >> 16;
  uint32_t y = x * 0x9E3779B1u;
  y ^= y >> 15;
  const uint32_t s = static_cast<uint32_t>(seed >> 32);
  DropBits r;
  r.a = x ^ s;
  r.b = y ^ s;
  return r;
}
// keep iff field >= thresh  <=>  word > drop_limit(thresh) for the HIGH field of `word`, (word << 16) > the same limit
// for the LOW field (thresh in [1, 65536]; 65536 = p 1.0 keeps nothing): one compare per element without extracting it.
__device__ __forceinline__ uint32_t drop_limit(uint32_t thresh) { return ((thresh - 1u) << 16) | 0xffffu; }
__device__ __forceinline__ bool dropout_keep(uint64_t seed, uint32_t row, uint32_t n_cols, uint32_t col,
                                             uint32_t thresh) {
  const DropBits q = dropout_quad_bits(seed, row, (n_cols + 3) >> 2, col >> 2);
  const uint32_t w = (col & 2) ? q.b : q.a;
  const uint32_t f = (col & 1) ? (w >> 16) : (w & 0xffffu);
  return f >= thresh;
}

}  // namespace gantts
