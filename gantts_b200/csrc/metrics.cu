// Objective distortions logged every mini-batch by the reference training loop (train.py:399-432,
// compute_distortions -> split_streams -> inv_scale -> nnmnkwii.metrics.{melcd, lf0_mean_squared_error,
// vuv_error, mean_squared_error}): the reference pulls both (B, T, D) tensors to the host and loops over
// utterances in numpy.  Here ONE streaming pass over the two static-domain tensors (one warp per frame,
// HBM-bound: 2 * D * 4 bytes per frame) produces the eight sums all four metrics are made of; the host
// reads 32 bytes.  De-normalisation (x * std + mean, per static column) and the V/UV binarisation
// (> 0.5, train.py:374-377) happen in registers.  Deterministic two-stage reduction.  The epoch log (epochlog.cu)
// launches the same partial kernel with a static-column map, which reads the target straight out of the fused step's
// input y, and finishes with the same distortions_totals, so its sums are bitwise those of gantts_distortions.
#include "common.cuh"

namespace gantts {

constexpr int MET_THREADS = 256;
constexpr int MET_MAX_BLOCKS = 132 * 4;
constexpr int MET_NV = 8;

struct MetWs {
  float partial[MET_MAX_BLOCKS][MET_NV];
};

__global__ void __launch_bounds__(MET_THREADS)
distortions_partial_kernel(const float* __restrict__ y, int64_t y_bs, int64_t y_ts, const float* __restrict__ yh,
                           int64_t yh_bs, int64_t yh_ts, const int64_t* __restrict__ lengths, int B, int T,
                           const float* __restrict__ mean, const float* __restrict__ stdv,
                           const gantts_distortion_cols_t c, const __grid_constant__ ColList ymap, MetWs* ws) {
  __shared__ float sm[4 * 32];
  __shared__ int ycol[GANTTS_MAX_COLS];
  for (int i = threadIdx.x; i < ymap.n; i += MET_THREADS) ycol[i] = ymap.c[i];
  __syncthreads();
  const bool mapped = ymap.n > 0;
  float v[MET_NV] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * MET_THREADS + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * MET_THREADS) >> 5;
  const int64_t frames = (int64_t)B * T;
  for (int64_t f = warp; f < frames; f += nwarps) {
    const int b = (int)(f / T), t = (int)(f - (int64_t)b * T);
    if ((int64_t)t >= lengths[b]) continue;
    const float* a = y + b * y_bs + t * y_ts;
    const float* h = yh + b * yh_bs + t * yh_ts;
    auto at = [&](int d) { return a[mapped ? ycol[d] : d]; };   // static column d of the target
    // cepstral groups: sum_d (de-normalised difference)^2 -> sqrt per frame
    float s0 = 0.f, s1 = 0.f, s2 = 0.f;
    for (int d = c.mcd_start + lane; d < c.mcd_start + c.mcd_count; d += 32) {
      const float z = (at(d) * stdv[d] + mean[d]) - (h[d] * stdv[d] + mean[d]);
      s0 = fmaf(z, z, s0);
    }
    for (int d = c.bap_start + lane; d < c.bap_start + c.bap_count; d += 32) {
      const float z = (at(d) * stdv[d] + mean[d]) - (h[d] * stdv[d] + mean[d]);
      s1 = fmaf(z, z, s1);
    }
    for (int d = c.mse_start + lane; d < c.mse_start + c.mse_count; d += 32) {
      const float z = (at(d) * stdv[d] + mean[d]) - (h[d] * stdv[d] + mean[d]);
      s2 = fmaf(z, z, s2);
    }
    s0 = warp_sum(s0);
    s1 = warp_sum(s1);
    s2 = warp_sum(s2);
    if (lane == 0) {
      if (c.mcd_count > 0) v[0] += sqrtf(s0);
      if (c.bap_count > 0) v[1] += sqrtf(s1);
      v[6] += s2;
      v[5] += 1.f;
      if (c.vuv_col >= 0) {
        const int k = c.vuv_col;
        const bool va = at(k) * stdv[k] + mean[k] > 0.5f, vh = h[k] * stdv[k] + mean[k] > 0.5f;
        if (va != vh) v[4] += 1.f;
        if (va && vh && c.lf0_col >= 0) {
          const int l = c.lf0_col;
          float fa = at(l) * stdv[l] + mean[l], fh = h[l] * stdv[l] + mean[l];
          if (c.lf0_linear) {
            fa = expf(fa);
            fh = expf(fh);
          }
          const float z = fa - fh;
          v[2] = fmaf(z, z, v[2]);
          v[3] += 1.f;
        }
      }
    }
  }
  // two block_sum<4> passes (the helper reduces up to four values)
  float lo4[4] = {v[0], v[1], v[2], v[3]}, hi4[4] = {v[4], v[5], v[6], v[7]};
  block_sum<4>(lo4, sm);
  __syncthreads();
  block_sum<4>(hi4, sm);
  if (threadIdx.x == 0) {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      ws->partial[blockIdx.x][k] = lo4[k];
      ws->partial[blockIdx.x][4 + k] = hi4[k];
    }
  }
}

// The fp64 finish of the blocks' eight sums in a fixed order (each thread's blocks, the warp shuffle, then the warps in
// turn); returns the eight totals in shared memory, valid in every thread of the block.
__device__ __forceinline__ const double* distortions_totals(const MetWs* ws, int nblocks) {
  __shared__ double sm[MET_THREADS / 32][MET_NV];
  __shared__ double tot[MET_NV];
  double v[MET_NV] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (int i = threadIdx.x; i < nblocks; i += MET_THREADS) {
#pragma unroll
    for (int k = 0; k < MET_NV; ++k) v[k] += (double)ws->partial[i][k];
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < MET_NV; ++k) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
    if (lane == 0) sm[warp][k] = v[k];
  }
  __syncthreads();
  if (threadIdx.x < MET_NV) {
    double s = 0;
    for (int w = 0; w < MET_THREADS / 32; ++w) s += sm[w][threadIdx.x];
    tot[threadIdx.x] = s;
  }
  __syncthreads();
  return tot;
}

__global__ void __launch_bounds__(MET_THREADS)
distortions_finish_kernel(const MetWs* ws, int nblocks, float* out) {
  const double* tot = distortions_totals(ws, nblocks);
  if (threadIdx.x < MET_NV) out[threadIdx.x] = (float)tot[threadIdx.x];
}

// one warp per frame, at most MET_MAX_BLOCKS blocks (the partials MetWs holds)
static inline int distortions_blocks(int B, int T) {
  const int nb = grid_for((int64_t)B * T * 32, MET_THREADS);
  return nb < MET_MAX_BLOCKS ? nb : MET_MAX_BLOCKS;
}

}  // namespace gantts

using namespace gantts;

extern "C" size_t gantts_distortions_workspace_bytes(void) { return sizeof(MetWs); }

extern "C" int gantts_distortions(const float* y, int64_t y_bs, int64_t y_ts, const float* y_hat, int64_t yh_bs,
                                  int64_t yh_ts, const int64_t* lengths_dev, int B, int T, int D,
                                  const float* mean_dev, const float* std_dev, const gantts_distortion_cols_t* cols,
                                  float* out8_dev, void* workspace, size_t workspace_bytes, void* stream) {
  GANTTS_CHECK_ARG(y && y_hat && lengths_dev && mean_dev && std_dev && cols && out8_dev,
                   "distortions: null argument");
  GANTTS_CHECK_ARG(B >= 1 && T >= 1 && D >= 1, "distortions: bad sizes");
  const gantts_distortion_cols_t& c = *cols;
  GANTTS_CHECK_ARG(c.mcd_start >= 0 && c.mcd_count >= 0 && c.mcd_start + c.mcd_count <= D && c.bap_start >= 0 &&
                       c.bap_count >= 0 && c.bap_start + c.bap_count <= D && c.mse_start >= 0 && c.mse_count >= 0 &&
                       c.mse_start + c.mse_count <= D && c.lf0_col < D && c.vuv_col < D,
                   "distortions: column groups outside [0, D)");
  if (!workspace || workspace_bytes < sizeof(MetWs)) {
    set_error("distortions: workspace too small (%zu < %zu)", workspace_bytes, sizeof(MetWs));
    return GANTTS_E_WORKSPACE;
  }
  MetWs* ws = static_cast<MetWs*>(workspace);
  const int nb = distortions_blocks(B, T);
  ColList none;
  none.n = 0;
  distortions_partial_kernel<<<nb, MET_THREADS, 0, as_stream(stream)>>>(y, y_bs, y_ts, y_hat, yh_bs, yh_ts, lengths_dev, B,
                                                                         T, mean_dev, std_dev, c, none, ws);
  GANTTS_LAUNCH_CHECK("distortions_partial_kernel");
  distortions_finish_kernel<<<1, MET_THREADS, 0, as_stream(stream)>>>(ws, nb, out8_dev);
  GANTTS_LAUNCH_CHECK("distortions_finish_kernel");
  return GANTTS_OK;
}
