// Sequence mask, masked MSE, masked adversarial BCE and stream column gathers.
// HBM-bound streaming kernels: one pass over the operands, deterministic two-stage reductions
// (per-block partials in the caller's workspace, then a single-block finish), grid sized to a
// multiple of the SM count.  sse_fwd_bwd_kernel and bce_fwd_bwd_kernel are the one MaskedMSE and BCE forward of the
// library: the modular ops launch them for the sums alone and finish with reduce_finish_kernel; the fused step
// (gan_step.cu) launches them through launch_sse / launch_bce for the sums and the gradient, and reduces the partials
// in its finalize kernel.
#include "common.cuh"

namespace gantts {

constexpr int RED_THREADS = 256;
constexpr int RED_MAX_BLOCKS = 132 * 4;
constexpr int RED_NV = 4;   // values reduced together

struct RedWs {
  float partial[RED_MAX_BLOCKS][RED_NV];
};

__global__ void sequence_mask_kernel(const int64_t* __restrict__ lengths, float* __restrict__ mask,
                                     int B, int T) {
  pdl_entry();
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)B * T) return;
  int b = (int)(i / T), t = (int)(i - (int64_t)b * T);
  mask[i] = (int64_t)t < lengths[b] ? 1.f : 0.f;
}

// Column map of a stream: up to GANTTS_MAX_COLS column indices passed by value (n = 0: no map).
struct ColList {
  int n;
  int c[GANTTS_MAX_COLS];
};

// MaskedMSELoss forward sums (reference gantts/seqloss.py:41-43: criterion(input * mask_, target * mask_) summed,
// / mask.sum()) AND its gradient 2 * scale * (a m - b m) * m in one pass; (a*m - b*m)^2 is evaluated exactly like that
// (two products, one subtraction, one square).  ga == nullptr: sums only, scale is not read.  The gradient is STORED (not
// accumulated): this launch initialises the buffer.  bmap.n > 0: column d of the target is column bmap.c[d] of `b` (the
// fused step reads the static features straight out of y: get_static_features of multistream.py:56-79 without
// materialising y_static).  One warp per row (lanes stride over the columns: coalesced, no integer division).
__global__ void __launch_bounds__(RED_THREADS)
sse_fwd_bwd_kernel(const float* __restrict__ a, int64_t a_rs, const float* __restrict__ b, int64_t b_rs,
                   const float* __restrict__ mask, int64_t rows, int D, const float* __restrict__ scale,
                   float* __restrict__ ga, int64_t ga_rs, RedWs* ws, ColList bmap) {
  pdl_entry();
  __shared__ float sm[RED_NV * 32];
  __shared__ int sc[GANTTS_MAX_COLS];
  for (int i = threadIdx.x; i < bmap.n; i += RED_THREADS) sc[i] = bmap.c[i];
  __syncthreads();
  const bool mapped = bmap.n > 0;
  float v[RED_NV] = {0.f, 0.f, 0.f, 0.f};
  const float s2 = ga ? 2.f * scale[0] : 0.f;
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * RED_THREADS + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * RED_THREADS) >> 5;
  for (int64_t r = warp; r < rows; r += nwarps) {
    const float m = mask[r];
    const float* ar = a + r * a_rs;
    const float* br = b + r * b_rs;
#pragma unroll 4
    for (int d = lane; d < D; d += 32) {
      const float x = ar[d] * m - br[mapped ? sc[d] : d] * m;
      v[0] = fmaf(x, x, v[0]);
      if (ga) ga[r * ga_rs + d] = s2 * x * m;
    }
    if (lane == 0) v[1] += m;
  }
  block_sum<RED_NV>(v, sm);
  if (threadIdx.x == 0) {
#pragma unroll
    for (int k = 0; k < RED_NV; ++k) ws->partial[blockIdx.x][k] = v[k];
  }
}

__global__ void __launch_bounds__(RED_THREADS)
reduce_finish_kernel(const RedWs* ws, int nblocks, float* out, int nout) {
  __shared__ float sm[RED_NV * 32];
  float v[RED_NV] = {0.f, 0.f, 0.f, 0.f};
  for (int i = threadIdx.x; i < nblocks; i += RED_THREADS) {
#pragma unroll
    for (int k = 0; k < RED_NV; ++k) v[k] += ws->partial[i][k];
  }
  block_sum<RED_NV>(v, sm);
  if (threadIdx.x == 0)
    for (int k = 0; k < nout; ++k) out[k] = v[k];
}

__global__ void __launch_bounds__(RED_THREADS)
masked_sse_bwd_kernel(const float* __restrict__ a, int64_t a_rs, const float* __restrict__ b,
                      int64_t b_rs, const float* __restrict__ mask, int64_t rows, int D,
                      const float* __restrict__ scale, float* __restrict__ ga, int64_t ga_rs,
                      int accumulate) {
  const float s2 = 2.f * scale[0];
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * RED_THREADS + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * RED_THREADS) >> 5;
  for (int64_t r = warp; r < rows; r += nwarps) {
    const float m = mask[r];
    const float* ar = a + r * a_rs;
    const float* br = b + r * b_rs;
    float* gr = ga + r * ga_rs;
#pragma unroll 4
    for (int d = lane; d < D; d += 32) {
      const float g = s2 * (ar[d] * m - br[d] * m) * m;
      gr[d] = accumulate ? gr[d] + g : g;
    }
  }
}

// Adversarial BCE terms of reference train.py:262-270,307-308 for one or two halves of a stacked discriminator output,
// forward sums AND the gradient w.r.t. D in one pass: half 0 = rows [0, M) with kind0, half 1 = rows [M, 2M) with kind1
// (kind 0: -log(D + eps) * m, correct = D > 0.5; kind 1: -log(1 - D + eps) * m, correct = D < 0.5).  mask is [M] for
// both halves.  Blocks [0, nbh) serve half 0 and write ws0, blocks [nbh, 2 nbh) serve half 1 and write ws1.
// gD == nullptr: sums only, scale is not read.  logf (not __logf) to stay within 1e-6 of torch.
__global__ void __launch_bounds__(RED_THREADS)
bce_fwd_bwd_kernel(const float* __restrict__ Dv, const float* __restrict__ mask, int64_t M, int kind0, int kind1,
                   int nbh, const float* __restrict__ scale, float* __restrict__ gD, RedWs* ws0, RedWs* ws1) {
  pdl_entry();
  __shared__ float sm[RED_NV * 32];
  const int half = blockIdx.x >= nbh ? 1 : 0;
  const int kind = half ? kind1 : kind0;
  const int blk = blockIdx.x - half * nbh;
  const float* d = Dv + (int64_t)half * M;
  float* g = gD ? gD + (int64_t)half * M : nullptr;
  const float s = g ? scale[0] : 0.f;
  float v[RED_NV] = {0.f, 0.f, 0.f, 0.f};
  for (int64_t i = (int64_t)blk * RED_THREADS + threadIdx.x; i < M; i += (int64_t)nbh * RED_THREADS) {
    const float dv = d[i], m = mask[i];
    const float arg = kind == 0 ? (dv + 1e-20f) : (1.f - dv + 1e-20f);
    v[0] -= logf(arg) * m;
    const bool hit = kind == 0 ? (dv > 0.5f) : (dv < 0.5f);
    v[1] += hit ? m : 0.f;
    v[2] += m;
    if (g) g[i] = kind == 0 ? (-s * m / (dv + 1e-20f)) : (s * m / (1.f - dv + 1e-20f));
  }
  block_sum<RED_NV>(v, sm);
  if (threadIdx.x == 0) {
    RedWs* ws = half ? ws1 : ws0;
#pragma unroll
    for (int k = 0; k < RED_NV; ++k) ws->partial[blk][k] = v[k];
  }
}

__global__ void masked_bce_bwd_kernel(const float* __restrict__ Dv, const float* __restrict__ mask,
                                      int64_t rows, int kind, const float* __restrict__ scale,
                                      float* __restrict__ gD) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows) return;
  float d = Dv[i], m = mask[i], s = scale[0];
  // d/dD -(log(D+eps) m) = -m/(D+eps) ; d/dD -(log(1-D+eps) m) = m/(1-D+eps)
  gD[i] = kind == 0 ? (-s * m / (d + 1e-20f)) : (s * m / (1.f - d + 1e-20f));
}

__global__ void gather_cols_kernel(const float* __restrict__ in, int64_t in_rs, float* __restrict__ out,
                                   int64_t out_rs, const int32_t* __restrict__ cols, int ncols,
                                   int64_t rows) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t r = warp; r < rows; r += nwarps)
    for (int j = lane; j < ncols; j += 32) out[r * out_rs + j] = in[r * in_rs + cols[j]];
}

__global__ void scatter_cols_add_kernel(const float* __restrict__ go, int64_t go_rs,
                                        float* __restrict__ gi, int64_t gi_rs,
                                        const int32_t* __restrict__ cols, int ncols, int64_t rows) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t r = warp; r < rows; r += nwarps)
    for (int j = lane; j < ncols; j += 32) gi[r * gi_rs + cols[j]] += go[r * go_rs + j];   // cols distinct
}

static inline int grid_for(int64_t work, int threads) {
  int64_t b = (work + threads - 1) / threads;
  if (b < 1) b = 1;
  if (b > RED_MAX_BLOCKS) b = RED_MAX_BLOCKS;
  return (int)b;
}

static inline int bce_blocks(int64_t rows) { return grid_for(rows, RED_THREADS); }
static inline int sse_blocks(int64_t rows, int D) { return grid_for(rows * D, RED_THREADS * 4); }

// The fused step's launches.  BCE of a stacked discriminator output: halves = 2 -> rows [0,M) kind0 into slot0 and rows
// [M,2M) kind1 into slot1
static int launch_bce(const float* Dv, const float* mask, int64_t M, int halves, int kind0, int kind1, const float* scale,
                      float* gD, RedWs* ws0, RedWs* ws1, cudaStream_t st) {
  const int nbh = bce_blocks(M);
  GANTTS_PDL_LAUNCH((bce_fwd_bwd_kernel), nbh * halves, RED_THREADS, 0, st, Dv, mask, M, kind0, kind1, nbh, scale, gD, ws0, ws1);
  GANTTS_LAUNCH_CHECK("bce_fwd_bwd_kernel");
  return GANTTS_OK;
}

static int launch_sse(const float* a, int64_t a_rs, const float* b, int64_t b_rs, const float* mask, int64_t rows, int D,
                      const float* scale, float* ga, int64_t ga_rs, RedWs* ws, cudaStream_t st,
                      const ColList* bmap = nullptr) {
  ColList none;
  none.n = 0;
  GANTTS_PDL_LAUNCH((sse_fwd_bwd_kernel), sse_blocks(rows, D), RED_THREADS, 0, st, a, a_rs, b, b_rs, mask, rows, D, scale, ga, ga_rs, ws,
                                                                 bmap ? *bmap : none);
  GANTTS_LAUNCH_CHECK("sse_fwd_bwd_kernel");
  return GANTTS_OK;
}

}  // namespace gantts

using namespace gantts;

extern "C" int gantts_sequence_mask(const int64_t* lengths_dev, float* mask, int B, int T, void* stream) {
  GANTTS_CHECK_ARG(lengths_dev && mask && B >= 1 && T >= 1, "sequence_mask: bad arguments");
  int64_t n = (int64_t)B * T;
  GANTTS_PDL_LAUNCH((sequence_mask_kernel), (unsigned)((n + 255) / 256), 256, 0, as_stream(stream), lengths_dev, mask, B, T);
  GANTTS_LAUNCH_CHECK("sequence_mask_kernel");
  return GANTTS_OK;
}

extern "C" size_t gantts_masked_sse_workspace_bytes(void) { return sizeof(RedWs); }

extern "C" int gantts_masked_sse_fwd(const float* a, int64_t a_rs, const float* b, int64_t b_rs,
                                     const float* mask, int64_t rows, int D, float* sums_dev,
                                     void* workspace, size_t workspace_bytes, void* stream) {
  GANTTS_CHECK_ARG(a && b && mask && sums_dev && rows >= 1 && D >= 1, "masked_sse_fwd: bad arguments");
  if (!workspace || workspace_bytes < sizeof(RedWs)) {
    set_error("masked_sse_fwd: workspace too small (%zu < %zu)", workspace_bytes, sizeof(RedWs));
    return GANTTS_E_WORKSPACE;
  }
  const int nb = sse_blocks(rows, D);
  RedWs* ws = static_cast<RedWs*>(workspace);
  ColList none;
  none.n = 0;
  sse_fwd_bwd_kernel<<<nb, RED_THREADS, 0, as_stream(stream)>>>(a, a_rs, b, b_rs, mask, rows, D, nullptr, nullptr, 0, ws,
                                                                none);
  GANTTS_LAUNCH_CHECK("sse_fwd_bwd_kernel");
  reduce_finish_kernel<<<1, RED_THREADS, 0, as_stream(stream)>>>(ws, nb, sums_dev, 2);
  GANTTS_LAUNCH_CHECK("reduce_finish_kernel");
  return GANTTS_OK;
}

extern "C" int gantts_masked_sse_bwd(const float* a, int64_t a_rs, const float* b, int64_t b_rs,
                                     const float* mask, int64_t rows, int D, const float* scale_dev,
                                     float* grad_a, int64_t ga_rs, int accumulate, void* stream) {
  GANTTS_CHECK_ARG(a && b && mask && scale_dev && grad_a && rows >= 1 && D >= 1,
                   "masked_sse_bwd: bad arguments");
  int nb = grid_for(rows * D, RED_THREADS * 4);
  masked_sse_bwd_kernel<<<nb, RED_THREADS, 0, as_stream(stream)>>>(a, a_rs, b, b_rs, mask, rows, D,
                                                                  scale_dev, grad_a, ga_rs, accumulate);
  GANTTS_LAUNCH_CHECK("masked_sse_bwd_kernel");
  return GANTTS_OK;
}

extern "C" int gantts_masked_bce_fwd(const float* D, const float* mask, int64_t rows, int kind,
                                     float* out_dev, void* workspace, size_t workspace_bytes,
                                     void* stream) {
  GANTTS_CHECK_ARG(D && mask && out_dev && rows >= 1 && (kind == 0 || kind == 1),
                   "masked_bce_fwd: bad arguments");
  if (!workspace || workspace_bytes < sizeof(RedWs)) {
    set_error("masked_bce_fwd: workspace too small");
    return GANTTS_E_WORKSPACE;
  }
  const int nb = bce_blocks(rows);
  RedWs* ws = static_cast<RedWs*>(workspace);
  bce_fwd_bwd_kernel<<<nb, RED_THREADS, 0, as_stream(stream)>>>(D, mask, rows, kind, kind, nb, nullptr, nullptr, ws,
                                                                nullptr);
  GANTTS_LAUNCH_CHECK("bce_fwd_bwd_kernel");
  reduce_finish_kernel<<<1, RED_THREADS, 0, as_stream(stream)>>>(ws, nb, out_dev, 3);
  GANTTS_LAUNCH_CHECK("reduce_finish_kernel");
  return GANTTS_OK;
}

extern "C" int gantts_masked_bce_bwd(const float* D, const float* mask, int64_t rows, int kind,
                                     const float* scale_dev, float* grad_D, void* stream) {
  GANTTS_CHECK_ARG(D && mask && scale_dev && grad_D && rows >= 1 && (kind == 0 || kind == 1),
                   "masked_bce_bwd: bad arguments");
  masked_bce_bwd_kernel<<<(unsigned)((rows + 255) / 256), 256, 0, as_stream(stream)>>>(D, mask, rows, kind,
                                                                                     scale_dev, grad_D);
  GANTTS_LAUNCH_CHECK("masked_bce_bwd_kernel");
  return GANTTS_OK;
}

extern "C" int gantts_gather_cols(const float* in, int64_t in_rs, float* out, int64_t out_rs,
                                  const int32_t* cols_dev, int ncols, int64_t rows, void* stream) {
  GANTTS_CHECK_ARG(in && out && cols_dev && ncols >= 1 && rows >= 1, "gather_cols: bad arguments");
  int nb = grid_for(rows * ncols, 256 * 4);
  gather_cols_kernel<<<nb, 256, 0, as_stream(stream)>>>(in, in_rs, out, out_rs, cols_dev, ncols, rows);
  GANTTS_LAUNCH_CHECK("gather_cols_kernel");
  return GANTTS_OK;
}

extern "C" int gantts_scatter_cols_add(const float* gout, int64_t go_rs, float* gin, int64_t gi_rs,
                                       const int32_t* cols_dev, int ncols, int64_t rows, void* stream) {
  GANTTS_CHECK_ARG(gout && gin && cols_dev && ncols >= 1 && rows >= 1, "scatter_cols_add: bad arguments");
  int nb = grid_for(rows * ncols, 256 * 4);
  scatter_cols_add_kernel<<<nb, 256, 0, as_stream(stream)>>>(gout, go_rs, gin, gi_rs, cols_dev, ncols, rows);
  GANTTS_LAUNCH_CHECK("scatter_cols_add_kernel");
  return GANTTS_OK;
}
