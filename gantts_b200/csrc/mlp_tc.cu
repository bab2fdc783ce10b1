// Whole-MLP forward / backward on the tensor-core engine with activations resident as bf16 hi/lo planes
// (include/gantts_b200.h: gantts_mlp_*).  Replaces reference gantts/models.py:137-141 (MLP.forward)
// and its autograd backward with one GEMM launch per layer and direction:
//   forward  l: H_{l+1} = Dropout(LeakyReLU(H_l W_l^T + b_l))  epilogue writes the next layer's planes
//   backward l: gW_l = gZ_l^T H_l (MN-major GEMM, split over rows), gb_l = colsum(gZ_l),
//               gZ_{l-1} = (gZ_l W_l) * act'(H_l)              epilogue writes the next gradient's planes
// No fp32 activation ever round-trips through HBM between layers; the tape the caller keeps for the
// backward holds the same planes the forward consumed (4 B per activation element, like fp32).
#include "common.cuh"

namespace gantts {

// gz = gy (* y (1-y) for a sigmoid output) -> planes
__global__ void grad_out_to_planes_kernel(const float* __restrict__ gy, int64_t gy_rs,
                                          const float* __restrict__ y, int64_t y_rs, int64_t rows, int cols,
                                          __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo,
                                          int64_t pitch, int sigmoid) {
  if (cols < 32) {     // narrow outputs (the discriminator's single column): one thread per element
    const int64_t total = rows * cols;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
         i += (int64_t)gridDim.x * blockDim.x) {
      const int64_t r = i / cols;
      const int c = (int)(i - r * cols);
      float v = gy[r * gy_rs + c];
      if (sigmoid) {
        const float yy = y[r * y_rs + c];
        v *= yy * (1.f - yy);
      }
      const __nv_bfloat16 h = __float2bfloat16_rn(v);
      hi[r * pitch + c] = h;
      lo[r * pitch + c] = __float2bfloat16_rn(v - __bfloat162float(h));
    }
    return;
  }
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t r = warp; r < rows; r += nwarps)
    for (int c = lane; c < cols; c += 32) {
      float v = gy[r * gy_rs + c];
      if (sigmoid) {
        const float yy = y[r * y_rs + c];
        v *= yy * (1.f - yy);
      }
      const __nv_bfloat16 h = __float2bfloat16_rn(v);
      hi[r * pitch + c] = h;
      lo[r * pitch + c] = __float2bfloat16_rn(v - __bfloat162float(h));
    }
}

// out[i] (+)= sum_z partial[z * stride + off + i], i < n
__global__ void splitk_reduce_strided_kernel(const float* __restrict__ partial, int nsplit, int stride, int off, int n,
                                             float* __restrict__ out, int accumulate) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float s = 0.f;
  for (int z = 0; z < nsplit; ++z) s += partial[(int64_t)z * stride + off + i];
  out[i] = accumulate ? out[i] + s : s;
}

// Column sums of a planes matrix (hi + lo): partial[chunk][col].
__global__ void __launch_bounds__(256)
colsum_planes_partial_kernel(const __nv_bfloat16* __restrict__ hi, const __nv_bfloat16* __restrict__ lo,
                             int64_t pitch, int64_t M, int N, int64_t rows_per_chunk,
                             float* __restrict__ partial) {
  __shared__ float sm[8][33];
  const int cx = threadIdx.x & 31, ry = threadIdx.x >> 5;
  const int col = blockIdx.x * 32 + cx;
  const int64_t rbeg = (int64_t)blockIdx.y * rows_per_chunk;
  const int64_t rend = rbeg + rows_per_chunk < M ? rbeg + rows_per_chunk : M;
  float s = 0.f;
  if (col < N)
    for (int64_t r = rbeg + ry; r < rend; r += 8)
      s += __bfloat162float(hi[r * pitch + col]) + __bfloat162float(lo[r * pitch + col]);
  sm[ry][cx] = s;
  __syncthreads();
  if (ry == 0 && col < N) {
    float t = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) t += sm[k][cx];
    partial[(int64_t)blockIdx.y * N + col] = t;
  }
}

// All weight matrices of an MLP -> bf16 hi/lo planes, both [N][K] (forward operand) and transposed
// [K][N] (operand of gx = gz W), in ONE launch.
struct WeightSplitList {
  int n;
  const float* W[GANTTS_MAX_LAYERS];
  int N[GANTTS_MAX_LAYERS], K[GANTTS_MAX_LAYERS];
  __nv_bfloat16 *hi[GANTTS_MAX_LAYERS], *lo[GANTTS_MAX_LAYERS];       // [N][pitch]
  __nv_bfloat16 *thi[GANTTS_MAX_LAYERS], *tlo[GANTTS_MAX_LAYERS];     // [K][tpitch]
  int64_t pitch[GANTTS_MAX_LAYERS], tpitch[GANTTS_MAX_LAYERS];
  int64_t off[GANTTS_MAX_LAYERS + 1];
};

// 32 x 32 tiles through shared memory so that BOTH the [N][K] planes and the transposed [K][N] planes are
// written with coalesced 64-byte row segments (a per-element kernel scattered 2-byte stores into the
// transposed planes: 11 us per launch for 3.4 MB of generator weights).  off[] counts tiles per layer.
__global__ void __launch_bounds__(256) split_weights_kernel(WeightSplitList wl) {
  pdl_entry();
  __shared__ uint16_t th[32][34], tl[32][34];
  const int cx = threadIdx.x & 31, ry = threadIdx.x >> 5;
  for (int64_t tile = blockIdx.x; tile < wl.off[wl.n]; tile += gridDim.x) {
    int l = 0;
    while (l + 1 < wl.n && tile >= wl.off[l + 1]) ++l;
    const int N = wl.N[l], K = wl.K[l];
    const int tk = (K + 31) / 32;
    const int64_t tt = tile - wl.off[l];
    const int r0 = (int)(tt / tk) * 32, c0 = (int)(tt % tk) * 32;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int r = r0 + ry + 8 * i, c = c0 + cx;
      uint16_t hb = 0, lb = 0;
      if (r < N && c < K) {
        const float v = wl.W[l][(int64_t)r * K + c];
        const __nv_bfloat16 h = __float2bfloat16_rn(v);
        const __nv_bfloat16 lo = __float2bfloat16_rn(v - __bfloat162float(h));
        wl.hi[l][r * wl.pitch[l] + c] = h;
        wl.lo[l][r * wl.pitch[l] + c] = lo;
        hb = __bfloat16_as_ushort(h);
        lb = __bfloat16_as_ushort(lo);
      }
      th[ry + 8 * i][cx] = hb;
      tl[ry + 8 * i][cx] = lb;
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int c = c0 + ry + 8 * i, r = r0 + cx;
      if (c < K && r < N) {
        wl.thi[l][(int64_t)c * wl.tpitch[l] + r] = __ushort_as_bfloat16(th[cx][ry + 8 * i]);
        wl.tlo[l][(int64_t)c * wl.tpitch[l] + r] = __ushort_as_bfloat16(tl[cx][ry + 8 * i]);
      }
    }
    __syncthreads();
  }
}

// ---------------------------------------------------------------------------- single-output last layer
// The discriminator ends in Linear(256 -> 1) + sigmoid (reference gantts/models.py:140-141 with out_dim=1):
// a GEMV, not a GEMM.  Forward: one warp per row reads the row's hi/lo planes once (HBM-bound) and
// produces y.  Backward: gz = gy * act'(y) per row; gW = sum_m gz[m] H[m][:], gb = sum gz (two-stage
// deterministic reduction) and the NEXT gradient planes gZ_prev = (gz w^T) * act'(H) directly.
constexpr int GEMV_THREADS = 256;
constexpr int GEMV_MAX_K = 1024;

__global__ void __launch_bounds__(GEMV_THREADS)
gemv_fwd_kernel(const __nv_bfloat16* __restrict__ hi, const __nv_bfloat16* __restrict__ lo, int64_t pitch,
                const float* __restrict__ w, const float* __restrict__ b, float* __restrict__ y, int64_t y_rs,
                int64_t M, int K, int sigmoid) {
  __shared__ float ws[GEMV_MAX_K];
  for (int i = threadIdx.x; i < K; i += GEMV_THREADS) ws[i] = w[i];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * GEMV_THREADS + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * GEMV_THREADS) >> 5;
  const float bias = b[0];
  for (int64_t r = warp; r < M; r += nwarps) {
    const uint32_t* hr = reinterpret_cast<const uint32_t*>(hi + r * pitch);
    const uint32_t* lr = reinterpret_cast<const uint32_t*>(lo + r * pitch);
    float acc = 0.f;
    for (int c = 2 * lane; c < K; c += 64) {
      const uint32_t h2 = hr[c >> 1], l2 = lr[c >> 1];
      const float a0 = __uint_as_float(h2 << 16) + __uint_as_float(l2 << 16);
      const float a1 = __uint_as_float(h2 & 0xffff0000u) + __uint_as_float(l2 & 0xffff0000u);
      acc = fmaf(a0, ws[c], acc);
      if (c + 1 < K) acc = fmaf(a1, ws[c + 1], acc);
    }
    acc = warp_sum(acc);
    if (lane == 0) {
      float z = acc + bias;
      y[r * y_rs] = sigmoid ? 1.f / (1.f + expf(-z)) : z;
    }
  }
}

// partial[block][0..K) = sum over the block's rows of gz[m] * H[m][:], partial[block][K] = sum gz (want_gw), and the
// previous layer's gradient planes (want_gz).  A block's rows depend on the grid and M alone, so the partials of a launch
// over M rows do not depend on which launches write the gradient planes of those rows.
__global__ void __launch_bounds__(GEMV_THREADS)
gemv_bwd_kernel(const float* __restrict__ gy, int64_t gy_rs, const float* __restrict__ y, int64_t y_rs,
                const __nv_bfloat16* __restrict__ hi, const __nv_bfloat16* __restrict__ lo, int64_t pitch,
                const uint32_t* __restrict__ code, int64_t code_pitch, const float* __restrict__ w,
                __nv_bfloat16* __restrict__ ghi, __nv_bfloat16* __restrict__ glo, int64_t gpitch,
                float* __restrict__ partial, int64_t M, int K, int sigmoid, float dpos, float dneg, float dzero,
                int want_gw, int want_gz) {
  __shared__ float ws[GEMV_MAX_K];
  __shared__ float gws[GEMV_THREADS / 32][GEMV_MAX_K + 1];
  for (int i = threadIdx.x; i < K; i += GEMV_THREADS) ws[i] = w[i];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (int i = lane; i <= K; i += 32) gws[wid][i] = 0.f;
  __syncthreads();
  const int64_t warp = ((int64_t)blockIdx.x * GEMV_THREADS + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * GEMV_THREADS) >> 5;
  float gsum = 0.f;
  for (int64_t r = warp; r < M; r += nwarps) {
    float g = gy[r * gy_rs];
    if (sigmoid) {
      const float yy = y[r * y_rs];
      g *= yy * (1.f - yy);
    }
    gsum += g;
    const uint32_t* hr = reinterpret_cast<const uint32_t*>(hi + r * pitch);
    const uint32_t* lr = reinterpret_cast<const uint32_t*>(lo + r * pitch);
    uint32_t* gh = reinterpret_cast<uint32_t*>(ghi + r * gpitch);
    uint32_t* gl = reinterpret_cast<uint32_t*>(glo + r * gpitch);
    for (int c = 2 * lane; c < K; c += 64) {
      if (want_gw) {
        const uint32_t h2 = hr[c >> 1], l2 = lr[c >> 1];
        const float a0 = __uint_as_float(h2 << 16) + __uint_as_float(l2 << 16);
        const float a1 = __uint_as_float(h2 & 0xffff0000u) + __uint_as_float(l2 & 0xffff0000u);
        gws[wid][c] = fmaf(g, a0, gws[wid][c]);
        if (c + 1 < K) gws[wid][c + 1] = fmaf(g, a1, gws[wid][c + 1]);
      }
      if (!want_gz) continue;
      // gZ_prev = (g * w) * act'(H), derivative class from the 2-bit code plane
      const uint32_t cw = code[r * code_pitch + (c >> 4)];
      const uint32_t c0 = (cw >> (2 * (c & 15))) & 3u, c1 = (cw >> (2 * ((c + 1) & 15))) & 3u;
      const float v0 = g * ws[c] * ((c0 & 1u) ? dzero : ((c0 & 2u) ? dneg : dpos));
      const float v1 = (c + 1 < K) ? g * ws[c + 1] * ((c1 & 1u) ? dzero : ((c1 & 2u) ? dneg : dpos)) : 0.f;
      const uint32_t hp = pack_bf16x2(v0, v1);
      gh[c >> 1] = hp;
      gl[c >> 1] = pack_bf16x2(v0 - __uint_as_float(hp << 16), v1 - __uint_as_float(hp & 0xffff0000u));
    }
  }
  if (want_gw) {
    if (lane == 0) gws[wid][K] = gsum;
    __syncthreads();
    for (int i = threadIdx.x; i <= K; i += GEMV_THREADS) {
      float s = 0.f;
#pragma unroll
      for (int q = 0; q < GEMV_THREADS / 32; ++q) s += gws[q][i];
      partial[(int64_t)blockIdx.x * (K + 1) + i] = s;
    }
  }
}

// ---- vectorised variants (K % 8 == 0): each lane owns 8 consecutive columns of every 256-column chunk
// (one 16-byte load per plane), several rows per warp in flight, weights and gW accumulators in registers.
__device__ __forceinline__ void unpack8(const uint4& h, const uint4& l, float (&a)[8]) {
  const uint32_t hh[4] = {h.x, h.y, h.z, h.w}, ll[4] = {l.x, l.y, l.z, l.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    a[2 * i] = __uint_as_float(hh[i] << 16) + __uint_as_float(ll[i] << 16);
    a[2 * i + 1] = __uint_as_float(hh[i] & 0xffff0000u) + __uint_as_float(ll[i] & 0xffff0000u);
  }
}

__device__ __forceinline__ uint4 ldg_stream16(const void* p) {
  uint4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p));
  return v;
}

template <int NCH, int RU>
__global__ void __launch_bounds__(GEMV_THREADS)
gemv_fwd_vec_kernel(const __nv_bfloat16* __restrict__ hi, const __nv_bfloat16* __restrict__ lo, int64_t pitch,
                    const float* __restrict__ w, const float* __restrict__ b, float* __restrict__ y, int64_t y_rs,
                    int64_t M, int K, int sigmoid) {
  pdl_entry();
  const int lane = threadIdx.x & 31;
  float wr[NCH][8];
#pragma unroll
  for (int ch = 0; ch < NCH; ++ch) {
    const int c = ch * 256 + lane * 8;
#pragma unroll
    for (int j = 0; j < 8; ++j) wr[ch][j] = c < K ? w[c + j] : 0.f;
  }
  const int64_t warp = ((int64_t)blockIdx.x * GEMV_THREADS + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * GEMV_THREADS) >> 5;
  const float bias = b[0];
  for (int64_t r0 = warp * RU; r0 < M; r0 += nwarps * RU) {
    uint4 h[RU][NCH], l[RU][NCH];
#pragma unroll
    for (int u = 0; u < RU; ++u) {
      const int64_t r = r0 + u < M ? r0 + u : M - 1;
#pragma unroll
      for (int ch = 0; ch < NCH; ++ch) {
        const int c = ch * 256 + lane * 8;
        if (c < K) {
          h[u][ch] = ldg_stream16(hi + r * pitch + c);
          l[u][ch] = ldg_stream16(lo + r * pitch + c);
        } else {
          h[u][ch] = make_uint4(0, 0, 0, 0);
          l[u][ch] = make_uint4(0, 0, 0, 0);
        }
      }
    }
    float acc[RU];
#pragma unroll
    for (int u = 0; u < RU; ++u) {
      acc[u] = 0.f;
#pragma unroll
      for (int ch = 0; ch < NCH; ++ch) {
        float a[8];
        unpack8(h[u][ch], l[u][ch], a);
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[u] = fmaf(a[j], wr[ch][j], acc[u]);
      }
    }
#pragma unroll
    for (int u = 0; u < RU; ++u) acc[u] = warp_sum(acc[u]);
    if (lane == 0) {
#pragma unroll
      for (int u = 0; u < RU; ++u)
        if (r0 + u < M) {
          const float z = acc[u] + bias;
          y[(r0 + u) * y_rs] = sigmoid ? 1.f / (1.f + expf(-z)) : z;
        }
    }
  }
}

template <int NCH, int RU>
__global__ void __launch_bounds__(GEMV_THREADS)
gemv_bwd_vec_kernel(const float* __restrict__ gy, int64_t gy_rs, const float* __restrict__ y, int64_t y_rs,
                    const __nv_bfloat16* __restrict__ hi, const __nv_bfloat16* __restrict__ lo, int64_t pitch,
                    const uint32_t* __restrict__ code, int64_t code_pitch, const float* __restrict__ w,
                    __nv_bfloat16* __restrict__ ghi, __nv_bfloat16* __restrict__ glo, int64_t gpitch,
                    float* __restrict__ partial, int64_t M, int K, int sigmoid, float dpos, float dneg, float dzero,
                    int want_gw, int want_gz) {
  pdl_entry();
  __shared__ float gws[GEMV_THREADS / 32][GEMV_MAX_K + 1];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  float wr[NCH][8], gw[NCH][8];
#pragma unroll
  for (int ch = 0; ch < NCH; ++ch) {
    const int c = ch * 256 + lane * 8;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      wr[ch][j] = c < K ? w[c + j] : 0.f;
      gw[ch][j] = 0.f;
    }
  }
  const int64_t warp = ((int64_t)blockIdx.x * GEMV_THREADS + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * GEMV_THREADS) >> 5;
  float gsum = 0.f;
  for (int64_t r0 = warp * RU; r0 < M; r0 += nwarps * RU) {
    uint4 h[RU][NCH], l[RU][NCH];
    uint32_t cw[RU][NCH];
    float g[RU];
#pragma unroll
    for (int u = 0; u < RU; ++u) {
      const bool ok = r0 + u < M;
      const int64_t r = ok ? r0 + u : M - 1;
      float gg = ok ? gy[r * gy_rs] : 0.f;
      if (sigmoid) {
        const float yy = y[r * y_rs];
        gg *= yy * (1.f - yy);
      }
      g[u] = gg;
#pragma unroll
      for (int ch = 0; ch < NCH; ++ch) {
        const int c = ch * 256 + lane * 8;
        if (c < K) {
          if (want_gw) {
            h[u][ch] = ldg_stream16(hi + r * pitch + c);
            l[u][ch] = ldg_stream16(lo + r * pitch + c);
          }
          if (want_gz) cw[u][ch] = __ldg(code + r * code_pitch + (c >> 4)) >> (2 * (c & 15));
        }
      }
    }
#pragma unroll
    for (int u = 0; u < RU; ++u) {
      gsum += g[u];
      if (r0 + u >= M) continue;
      const int64_t r = r0 + u;
#pragma unroll
      for (int ch = 0; ch < NCH; ++ch) {
        const int c = ch * 256 + lane * 8;
        if (c >= K) continue;
        if (want_gw) {
          float a[8];
          unpack8(h[u][ch], l[u][ch], a);
#pragma unroll
          for (int j = 0; j < 8; ++j) gw[ch][j] = fmaf(g[u], a[j], gw[ch][j]);
        }
        if (!want_gz) continue;
        // gZ_prev = (g * w) * act'(H), derivative class from the 2-bit code plane
        uint32_t oh[4], ol[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const uint32_t c0 = (cw[u][ch] >> (4 * j)) & 3u, c1 = (cw[u][ch] >> (4 * j + 2)) & 3u;
          const float v0 = g[u] * wr[ch][2 * j] * ((c0 & 1u) ? dzero : ((c0 & 2u) ? dneg : dpos));
          const float v1 = g[u] * wr[ch][2 * j + 1] * ((c1 & 1u) ? dzero : ((c1 & 2u) ? dneg : dpos));
          oh[j] = pack_bf16x2(v0, v1);
          ol[j] = pack_bf16x2(v0 - __uint_as_float(oh[j] << 16), v1 - __uint_as_float(oh[j] & 0xffff0000u));
        }
        *reinterpret_cast<uint4*>(ghi + r * gpitch + c) = make_uint4(oh[0], oh[1], oh[2], oh[3]);
        *reinterpret_cast<uint4*>(glo + r * gpitch + c) = make_uint4(ol[0], ol[1], ol[2], ol[3]);
      }
    }
  }
  if (want_gw) {
#pragma unroll
    for (int ch = 0; ch < NCH; ++ch) {
      const int c = ch * 256 + lane * 8;
      if (c < K) {
#pragma unroll
        for (int j = 0; j < 8; ++j) gws[wid][c + j] = gw[ch][j];
      }
    }
    if (lane == 0) gws[wid][K] = gsum;
    __syncthreads();
    for (int i = threadIdx.x; i <= K; i += GEMV_THREADS) {
      float s = 0.f;
#pragma unroll
      for (int q = 0; q < GEMV_THREADS / 32; ++q) s += gws[q][i];
      partial[(int64_t)blockIdx.x * (K + 1) + i] = s;
    }
  }
}

// out_w[c] (+)= sum_b partial[b][c] (c < K), out_b[0] (+)= sum_b partial[b][K]; fixed summation order.
__global__ void __launch_bounds__(256)
gemv_partial_reduce_kernel(const float* __restrict__ partial, int blocks, int K, float* __restrict__ out_w,
                           float* __restrict__ out_b, int accumulate) {
  pdl_entry();
  __shared__ float sm[8][33];
  const int cl = threadIdx.x & 31, rg = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + cl;
  float s = 0.f;
  if (c <= K)
    for (int b = rg; b < blocks; b += 8) s += partial[(int64_t)b * (K + 1) + c];
  sm[rg][cl] = s;
  __syncthreads();
  if (rg == 0 && c <= K) {
    float t = 0.f;
#pragma unroll
    for (int q = 0; q < 8; ++q) t += sm[q][cl];
    float* o = c < K ? (out_w ? out_w + c : nullptr) : out_b;
    if (o) *o = accumulate ? *o + t : t;
  }
}

constexpr int GEMV_BLOCKS = 132 * 2;

constexpr int MLP_COLSUM_CHUNKS = 128;
// The backward walks down the stack with two gradient plane buffers, writing one while it reads the other.
constexpr int MLP_GRAD_BUFS = 2;

static int colsum_planes(const Planes& G, float* gb, int accumulate, float* partial, cudaStream_t st) {
  int chunks = MLP_COLSUM_CHUNKS;
  int64_t rpc = (G.rows + chunks - 1) / chunks;
  if (rpc < 8) rpc = 8;
  chunks = (int)((G.rows + rpc - 1) / rpc);
  dim3 grid((unsigned)((G.cols + 31) / 32), chunks);
  colsum_planes_partial_kernel<<<grid, 256, 0, st>>>(G.hi, G.lo, G.pitch, G.rows, (int)G.cols, rpc, partial);
  GANTTS_LAUNCH_CHECK("colsum_planes_partial_kernel");
  splitk_reduce_kernel<<<(unsigned)((G.cols + 1023) / 1024), 256, 0, st>>>(partial, chunks, G.cols, gb, accumulate);
  GANTTS_LAUNCH_CHECK("splitk_reduce_kernel(colsum planes)");
  return GANTTS_OK;
}

struct MlpTape {
  uint32_t* code[GANTTS_MAX_LAYERS];   // code[l]: activation-derivative codes of H[l] (l >= 1), [M][code_pitch[l]]
  int64_t code_pitch[GANTTS_MAX_LAYERS];
  Planes H[GANTTS_MAX_LAYERS];      // H[0] = input planes, H[l] = output of hidden layer l-1
  Planes W[GANTTS_MAX_LAYERS];      // [d_{l+1}][d_l]
  Planes Wt[GANTTS_MAX_LAYERS];     // [d_l][d_{l+1}]
};

static int check_mlp(const gantts_mlp_t* m, int64_t M) {
  GANTTS_CHECK_ARG(m, "mlp: null descriptor");
  GANTTS_CHECK_ARG(m->num_layers >= 1 && m->num_layers <= GANTTS_MAX_LAYERS, "mlp: bad layer count %d", m->num_layers);
  GANTTS_CHECK_ARG(M >= 1, "mlp: M must be >= 1");
  for (int l = 0; l <= m->num_layers; ++l) GANTTS_CHECK_ARG(m->dims[l] >= 1, "mlp: bad dim[%d]", l);
  for (int l = 0; l < m->num_layers; ++l) {
    GANTTS_CHECK_ARG(m->W[l] && m->b[l], "mlp: null weight/bias of layer %d", l);
    GANTTS_CHECK_ARG((reinterpret_cast<uintptr_t>(m->b[l]) & 15) == 0, "mlp: bias %d must be 16-byte aligned", l);
  }
  GANTTS_CHECK_ARG(m->dropout_p >= 0.f && m->dropout_p < 1.f, "mlp: dropout p out of [0,1)");
  GANTTS_CHECK_ARG(m->last_act == GANTTS_ACT_NONE || m->last_act == GANTTS_ACT_SIGMOID, "mlp: bad last_act");
  return GANTTS_OK;
}

static size_t carve_tape(const gantts_mlp_t* m, int64_t M, char* base, MlpTape* t) {
  char* cur = base;
  for (int l = 0; l < m->num_layers; ++l) {
    Planes p = carve_planes(cur, M, m->dims[l]);
    if (t) t->H[l] = p;
    const int64_t cp = ((m->dims[l] + 15) / 16 + 3) / 4 * 4;   // words per row, padded to 16 B
    if (t) {
      t->code[l] = reinterpret_cast<uint32_t*>(cur);
      t->code_pitch[l] = cp;
    }
    if (l >= 1) cur += ((size_t)M * cp * sizeof(uint32_t) + 255) / 256 * 256;
  }
  for (int l = 0; l < m->num_layers; ++l) {
    Planes a = carve_planes(cur, m->dims[l + 1], m->dims[l]);
    Planes b = carve_planes(cur, m->dims[l], m->dims[l + 1]);
    if (t) { t->W[l] = a; t->Wt[l] = b; }
  }
  return (size_t)(cur - base);
}

static inline uint64_t layer_seed(uint64_t seed, int l) { return seed + 0x9E3779B97F4A7C15ull * (uint64_t)(l + 1); }

}  // namespace gantts

using namespace gantts;

extern "C" uint64_t gantts_mlp_layer_seed(uint64_t seed, int layer) { return layer_seed(seed, layer); }

extern "C" size_t gantts_mlp_tape_bytes(const gantts_mlp_t* m, int64_t M) {
  if (!m || m->num_layers < 1 || m->num_layers > GANTTS_MAX_LAYERS || M < 1) return 0;
  return carve_tape(m, M, nullptr, nullptr) + 512;
}

namespace gantts {
// Gradient plane buffers of a backward.  With the weight gradients on a side stream (mlp_bwd_impl), dW_l still reads G_l
// while the input-gradient chain writes the layers below it: every layer's gradient gets its own buffer.
static int mlp_grad_bufs(const gantts_mlp_t* m, bool side) {
  return side && m->num_layers > MLP_GRAD_BUFS ? m->num_layers : MLP_GRAD_BUFS;
}

// upto = false: the workspace of M rows; true: enough for every row count in [1, M].  side: for a backward that runs the
// weight gradients on a side stream.
static size_t mlp_workspace_bytes(const gantts_mlp_t* m, int64_t M, bool upto, bool side = false) {
  if (!m || m->num_layers < 1 || m->num_layers > GANTTS_MAX_LAYERS || M < 1) return 0;
  int maxd = 0;
  size_t part = 0;
  for (int l = 0; l <= m->num_layers; ++l) maxd = m->dims[l] > maxd ? m->dims[l] : maxd;
  for (int l = 0; l < m->num_layers; ++l)       // one partial region per layer: reductions are deferred
    part += (upto ? mn_partial_bytes_upto(M, m->dims[l + 1], m->dims[l])
                  : mn_partial_bytes(M, m->dims[l + 1], m->dims[l], nullptr, nullptr)) + 256;
  return (size_t)2 * mlp_grad_bufs(m, side) * plane_bytes(M, maxd) + part +
         (size_t)MLP_COLSUM_CHUNKS * maxd * sizeof(float) + (size_t)GEMV_BLOCKS * (GEMV_MAX_K + 1) * sizeof(float) + 4096;
}
}  // namespace gantts

extern "C" size_t gantts_mlp_workspace_bytes(const gantts_mlp_t* m, int64_t M) { return mlp_workspace_bytes(m, M, false); }

// input_ready: the caller has already written the input planes into the tape (mlp_tape_input_planes) -- the fused
// step gathers the discriminator's input columns straight into planes instead of gathering to fp32 and splitting.
namespace gantts {
static int mlp_fwd_impl(const gantts_mlp_t* m, const float* x, int64_t x_rs, int64_t M, float* y, int64_t y_rs, void* tape,
                        size_t tape_bytes, void* stream, bool input_ready);
// The forward of an M-row batch in row windows, which may run on different streams (the fused step's real and fake
// halves of the stacked discriminator batch): mlp_split_weights writes the tape's weight planes once, then
// mlp_fwd_rows runs every layer over rows [r0, r1), from x's rows (split into the tape's input planes first) or, with
// x = nullptr, from input planes the caller wrote.  Dropout is keyed by the batch row, so each row's output, tape
// planes and derivative codes are those of one launch over all M rows, bit for bit.
static int mlp_split_weights(const gantts_mlp_t* m, int64_t M, void* tape, size_t tape_bytes, cudaStream_t st);
static int mlp_fwd_rows(const gantts_mlp_t* m, const float* x, int64_t x_rs, int64_t M, int64_t r0, int64_t r1, float* y,
                        int64_t y_rs, void* tape, size_t tape_bytes, cudaStream_t st);

// every weight matrix into its [N][K] and transposed [K][N] planes in the tape, one launch
static int split_weights(const gantts_mlp_t* m, const MlpTape& t, cudaStream_t st) {
  const int L = m->num_layers;
  WeightSplitList wl;
  wl.n = L;
  wl.off[0] = 0;
  for (int l = 0; l < L; ++l) {
    wl.W[l] = m->W[l];
    wl.N[l] = m->dims[l + 1];
    wl.K[l] = m->dims[l];
    wl.hi[l] = t.W[l].hi;
    wl.lo[l] = t.W[l].lo;
    wl.pitch[l] = t.W[l].pitch;
    wl.thi[l] = t.Wt[l].hi;
    wl.tlo[l] = t.Wt[l].lo;
    wl.tpitch[l] = t.Wt[l].pitch;
    wl.off[l + 1] = wl.off[l] + (int64_t)((m->dims[l + 1] + 31) / 32) * ((m->dims[l] + 31) / 32);
  }
  int nb = (int)wl.off[L];
  if (nb > num_sms() * 8) nb = num_sms() * 8;
  if (nb < 1) nb = 1;
  GANTTS_PDL_LAUNCH((split_weights_kernel), nb, 256, 0, st, wl);
  GANTTS_LAUNCH_CHECK("split_weights_kernel");
  return GANTTS_OK;
}

// every layer over rows [r0, r1) of the tape's batch, y's row r the batch's row r
static int fwd_layers(const gantts_mlp_t* m, const MlpTape& t, int64_t r0, int64_t r1, float* y, int64_t y_rs,
                      cudaStream_t st) {
  const int L = m->num_layers;
  const int64_t M = r1 - r0;
  y += r0 * y_rs;
  int rc;
  for (int l = 0; l < L; ++l) {
    const Planes A = plane_rows(t.H[l], r0, r1);
    EpiArgs e;
    e.bias = m->b[l];
    e.row0 = r0;
    if (l < L - 1) {
      const Planes O = plane_rows(t.H[l + 1], r0, r1);
      e.epi = EPI_PLANES_FWD;
      e.out_hi = O.hi;
      e.out_lo = O.lo;
      e.out_pitch = O.pitch;
      e.code = t.code[l + 1] + r0 * t.code_pitch[l + 1];
      e.code_pitch = t.code_pitch[l + 1];
      e.act = GANTTS_ACT_LEAKY_DROPOUT;
      e.slope = m->slope;
      e.p = m->dropout_p;
      e.seed = layer_seed(m->seed, l);
    } else {
      if (m->dims[L] == 1 && L >= 2 && m->dims[l] <= GEMV_MAX_K && (m->dims[l] & 1) == 0) {
        // single-output last layer: GEMV + sigmoid, one warp per row
        const int Kl = m->dims[l], sg = m->last_act == GANTTS_ACT_SIGMOID;
        if (Kl % 8 == 0 && Kl <= 256)
          GANTTS_PDL_LAUNCH((gemv_fwd_vec_kernel<1, 4>), 2 * GEMV_BLOCKS, GEMV_THREADS, 0, st, A.hi, A.lo, A.pitch, m->W[l],
                                                                          m->b[l], y, y_rs, M, Kl, sg);
        else if (Kl % 8 == 0 && Kl <= 512)
          gemv_fwd_vec_kernel<2, 2><<<2 * GEMV_BLOCKS, GEMV_THREADS, 0, st>>>(A.hi, A.lo, A.pitch, m->W[l],
                                                                          m->b[l], y, y_rs, M, Kl, sg);
        else if (Kl % 8 == 0)
          gemv_fwd_vec_kernel<4, 1><<<2 * GEMV_BLOCKS, GEMV_THREADS, 0, st>>>(A.hi, A.lo, A.pitch, m->W[l],
                                                                          m->b[l], y, y_rs, M, Kl, sg);
        else
          gemv_fwd_kernel<<<GEMV_BLOCKS, GEMV_THREADS, 0, st>>>(A.hi, A.lo, A.pitch, m->W[l], m->b[l], y,
                                                                y_rs, M, Kl, sg);
        GANTTS_LAUNCH_CHECK("gemv_fwd_kernel");
        continue;
      }
      e.epi = EPI_F32;
      e.C = y;
      e.ldc = y_rs;
      e.act = m->last_act;
    }
    if ((rc = launch_gemm_kk(A, t.W[l], e, st))) return rc;
  }
  return GANTTS_OK;
}

static int mlp_tape_input_planes(const gantts_mlp_t* m, int64_t M, void* tape, size_t tape_bytes, Planes* out) {
  int rc = check_mlp(m, M);
  if (rc) return rc;
  if (!tape || tape_bytes < gantts_mlp_tape_bytes(m, M)) {
    set_error("mlp_tape_input_planes: tape too small");
    return GANTTS_E_WORKSPACE;
  }
  MlpTape t;
  carve_tape(m, M, reinterpret_cast<char*>((reinterpret_cast<uintptr_t>(tape) + 255) / 256 * 256), &t);
  *out = t.H[0];
  return GANTTS_OK;
}
}  // namespace gantts

extern "C" int gantts_mlp_fwd(const gantts_mlp_t* m, const float* x, int64_t x_rs, int64_t M, float* y,
                              int64_t y_rs, void* tape, size_t tape_bytes, void* stream) {
  GANTTS_CHECK_ARG(m && x && x_rs >= m->dims[0], "mlp_fwd: bad input pointer/stride");
  return mlp_fwd_impl(m, x, x_rs, M, y, y_rs, tape, tape_bytes, stream, false);
}

static int gantts::mlp_fwd_impl(const gantts_mlp_t* m, const float* x, int64_t x_rs, int64_t M, float* y, int64_t y_rs,
                                void* tape, size_t tape_bytes, void* stream, bool input_ready) {
  int rc = check_mlp(m, M);
  if (rc) return rc;
  GANTTS_CHECK_ARG((x || input_ready) && y && y_rs >= m->dims[m->num_layers], "mlp_fwd: bad pointers/strides");
  size_t need = gantts_mlp_tape_bytes(m, M);
  if (!tape || tape_bytes < need) {
    set_error("mlp_fwd: tape too small (%zu < %zu)", tape_bytes, need);
    return GANTTS_E_WORKSPACE;
  }
  cudaStream_t st = as_stream(stream);
  MlpTape t;
  carve_tape(m, M, reinterpret_cast<char*>((reinterpret_cast<uintptr_t>(tape) + 255) / 256 * 256), &t);
  if (!input_ready && (rc = launch_split(x, x_rs, M, m->dims[0], t.H[0], 0, st))) return rc;
  if ((rc = split_weights(m, t, st))) return rc;
  return fwd_layers(m, t, 0, M, y, y_rs, st);
}

static int gantts::mlp_split_weights(const gantts_mlp_t* m, int64_t M, void* tape, size_t tape_bytes, cudaStream_t st) {
  int rc = check_mlp(m, M);
  if (rc) return rc;
  if (!tape || tape_bytes < gantts_mlp_tape_bytes(m, M)) {
    set_error("mlp_split_weights: tape too small");
    return GANTTS_E_WORKSPACE;
  }
  MlpTape t;
  carve_tape(m, M, reinterpret_cast<char*>((reinterpret_cast<uintptr_t>(tape) + 255) / 256 * 256), &t);
  return split_weights(m, t, st);
}

static int gantts::mlp_fwd_rows(const gantts_mlp_t* m, const float* x, int64_t x_rs, int64_t M, int64_t r0, int64_t r1,
                                float* y, int64_t y_rs, void* tape, size_t tape_bytes, cudaStream_t st) {
  int rc = check_mlp(m, M);
  if (rc) return rc;
  GANTTS_CHECK_ARG(r0 >= 0 && r0 < r1 && r1 <= M, "mlp_fwd_rows: bad row window [%lld, %lld) of %lld rows",
                   (long long)r0, (long long)r1, (long long)M);
  GANTTS_CHECK_ARG((!x || x_rs >= m->dims[0]) && y && y_rs >= m->dims[m->num_layers], "mlp_fwd_rows: bad pointers/strides");
  if (!tape || tape_bytes < gantts_mlp_tape_bytes(m, M)) {
    set_error("mlp_fwd_rows: tape too small");
    return GANTTS_E_WORKSPACE;
  }
  MlpTape t;
  carve_tape(m, M, reinterpret_cast<char*>((reinterpret_cast<uintptr_t>(tape) + 255) / 256 * 256), &t);
  if (x && (rc = launch_split(x + r0 * x_rs, x_rs, r1 - r0, m->dims[0], plane_rows(t.H[0], r0, r1), 0, st))) return rc;
  return fwd_layers(m, t, r0, r1, y, y_rs, st);
}

// gx_row0: the input gradient is only produced for rows [gx_row0, M) (the fused step stacks real | fake rows and
// needs the gradient w.r.t. the fake half only: the real half's input is data).
// chain_r0, chain_r1: the input-gradient chain -- the output gradient's planes, every layer's gradient planes, gx --
// covers rows [chain_r0, chain_r1) of the batch (chain_r1 < 0: M), while the weight gradients cover all M rows.  A
// windowed call reads the other rows' gradient planes as an earlier windowed call left them: the fused step runs the
// real half's chain with no weight gradients on its branch stream, then the fake half's with the weight gradients.  Each
// row's planes are those of one chain over all M rows, and so are the weight gradients, bit for bit.
namespace gantts {
static int mlp_bwd_impl(const gantts_mlp_t* m, const float* gy, int64_t gy_rs, const float* y, int64_t y_rs, int64_t M,
                        const void* tape, size_t tape_bytes, float* gx, int64_t gx_rs, int64_t gx_row0,
                        float* const* gW, float* const* gb, int accumulate, void* workspace, size_t workspace_bytes,
                        void* stream, int gx_accumulate = -1, bool gy_planes_ready = false, cudaStream_t side = nullptr,
                        int64_t chain_r0 = 0, int64_t chain_r1 = -1);
// Where mlp_bwd_impl expects the output-gradient planes when gy_planes_ready (linear output, not the GEMV tail): the
// producer of gy (the MLPG backward in the fused step) can write them directly instead of an fp32 matrix.
static int mlp_bwd_gy_planes(const gantts_mlp_t* m, int64_t M, void* workspace, size_t workspace_bytes, Planes* out);
}

static int gantts::mlp_bwd_gy_planes(const gantts_mlp_t* m, int64_t M, void* workspace, size_t workspace_bytes, Planes* out) {
  int rc = check_mlp(m, M);
  if (rc) return rc;
  if (!workspace || workspace_bytes < gantts_mlp_workspace_bytes(m, M)) {
    set_error("mlp_bwd_gy_planes: workspace too small");
    return GANTTS_E_WORKSPACE;
  }
  char* cur = reinterpret_cast<char*>((reinterpret_cast<uintptr_t>(workspace) + 255) / 256 * 256);   // = gbuf[0] of mlp_bwd_impl
  *out = carve_planes(cur, M, m->dims[m->num_layers]);
  return GANTTS_OK;
}

extern "C" int gantts_mlp_bwd(const gantts_mlp_t* m, const float* gy, int64_t gy_rs, const float* y,
                              int64_t y_rs, int64_t M, const void* tape, size_t tape_bytes, float* gx,
                              int64_t gx_rs, float* const* gW, float* const* gb, int accumulate,
                              void* workspace, size_t workspace_bytes, void* stream) {
  return mlp_bwd_impl(m, gy, gy_rs, y, y_rs, M, tape, tape_bytes, gx, gx_rs, 0, gW, gb, accumulate, workspace,
                      workspace_bytes, stream, -1);
}

static int gantts::mlp_bwd_impl(const gantts_mlp_t* m, const float* gy, int64_t gy_rs, const float* y, int64_t y_rs,
                                int64_t M, const void* tape, size_t tape_bytes, float* gx, int64_t gx_rs,
                                int64_t gx_row0, float* const* gW, float* const* gb, int accumulate, void* workspace,
                                size_t workspace_bytes, void* stream, int gx_accumulate, bool gy_planes_ready,
                                cudaStream_t side, int64_t chain_r0, int64_t chain_r1) {
  // gx_accumulate: -1 = like the parameter gradients, 0 = store, 1 = add to what gx holds (gx may be a column window of
  // a wider matrix with row stride gx_rs: the fused step scatters the input gradient into g_static this way)
  // side: the weight and bias gradients (their GEMMs, the GEMV tail's reduction, the split-K reduction) run on this
  // stream, each after the launch on `stream` that wrote the gradient planes it reads, while the input-gradient chain
  // stays on `stream`; the call joins the side stream back into `stream` before it returns.
  if (gx_accumulate < 0) gx_accumulate = accumulate;
  int rc = check_mlp(m, M);
  GANTTS_CHECK_ARG(gx_row0 >= 0 && gx_row0 < M, "mlp_bwd: bad gx_row0");
  if (rc) return rc;
  if (chain_r1 < 0) chain_r1 = M;
  GANTTS_CHECK_ARG(chain_r0 >= 0 && chain_r0 < chain_r1 && chain_r1 <= M, "mlp_bwd: bad chain rows [%lld, %lld)",
                   (long long)chain_r0, (long long)chain_r1);
  const bool windowed = chain_r0 > 0 || chain_r1 < M;
  GANTTS_CHECK_ARG(!windowed || !gy_planes_ready, "mlp_bwd: a row window needs gy, not gy planes");
  const int L = m->num_layers;
  GANTTS_CHECK_ARG(gy_planes_ready || (gy && gy_rs >= m->dims[L]), "mlp_bwd: bad gy");
  GANTTS_CHECK_ARG(!gy_planes_ready || (m->last_act == GANTTS_ACT_NONE && m->dims[L] > 1),
                   "mlp_bwd: gy planes are only accepted for a linear multi-column output");
  GANTTS_CHECK_ARG(m->last_act != GANTTS_ACT_SIGMOID || y, "mlp_bwd: sigmoid output needs y");
  if (!tape || tape_bytes < gantts_mlp_tape_bytes(m, M)) {
    set_error("mlp_bwd: tape too small");
    return GANTTS_E_WORKSPACE;
  }
  // windowed calls over the same batch keep a buffer per layer, so that their gradient planes meet at one address
  const bool per_layer = side != nullptr || windowed;
  size_t need = mlp_workspace_bytes(m, M, false, per_layer);
  if (!workspace || workspace_bytes < need) {
    set_error("mlp_bwd: workspace too small (%zu < %zu)", workspace_bytes, need);
    return GANTTS_E_WORKSPACE;
  }
  cudaStream_t st = as_stream(stream);
  // ws: the stream of the weight-gradient launches; fork(): it waits for what `stream` has issued so far
  const cudaStream_t ws = side ? side : st;
  auto fork = [&]() { return side ? stream_wait(side, st) : GANTTS_OK; };
  MlpTape t;
  carve_tape(m, M, reinterpret_cast<char*>((reinterpret_cast<uintptr_t>(const_cast<void*>(tape)) + 255) / 256 * 256), &t);
  int maxd = 0;
  for (int l = 0; l <= L; ++l) maxd = m->dims[l] > maxd ? m->dims[l] : maxd;
  char* cur = reinterpret_cast<char*>((reinterpret_cast<uintptr_t>(workspace) + 255) / 256 * 256);
  const int nbuf = mlp_grad_bufs(m, per_layer);
  char* gbuf[GANTTS_MAX_LAYERS > MLP_GRAD_BUFS ? GANTTS_MAX_LAYERS : MLP_GRAD_BUFS];
  for (int i = 0; i < nbuf; ++i) {
    gbuf[i] = cur;
    cur += 2 * plane_bytes(M, maxd);
  }
  float* colpart = reinterpret_cast<float*>(cur);
  cur += ((size_t)MLP_COLSUM_CHUNKS * maxd * sizeof(float) + 255) / 256 * 256;
  char* partial_cur = cur;
  ReduceList rl;

  float* gemv_part = reinterpret_cast<float*>(partial_cur);
  partial_cur += ((size_t)GEMV_BLOCKS * (GEMV_MAX_K + 1) * sizeof(float) + 255) / 256 * 256;
  int pp = 0;
  int l_start = L - 1;
  char* c0 = gbuf[pp];
  Planes G = carve_planes(c0, M, m->dims[L]);
  if (m->dims[L] == 1 && L >= 2 && m->dims[L - 1] <= GEMV_MAX_K && (m->dims[L - 1] & 1) == 0) {
    // single-output last layer: gW/gb by block partials, and the previous layer's gradient planes directly
    const int K1 = m->dims[L - 1];
    char* cg = gbuf[pp];
    G = carve_planes(cg, M, K1);
    const float ks = m->dropout_p > 0.f ? 1.f / (1.f - m->dropout_p) : 1.f;
    const int want = (gW && gW[L - 1]) || (gb && gb[L - 1]);
    // rows [r0, r1): their gradient planes (gz) and / or the block partials of gW, gb over them (gw)
    auto gemv_bwd = [&](int64_t r0, int64_t r1, int gw, int gz, cudaStream_t s) {
      const Planes H = plane_rows(t.H[L - 1], r0, r1), Gw = plane_rows(G, r0, r1);
#define GANTTS_GEMV_BWD_ARGS                                                                                     \
  gy + r0 * gy_rs, gy_rs, y ? y + r0 * y_rs : nullptr, y_rs, H.hi, H.lo, H.pitch,                              \
      t.code[L - 1] + r0 * t.code_pitch[L - 1], t.code_pitch[L - 1], m->W[L - 1], Gw.hi, Gw.lo, Gw.pitch,       \
      gemv_part, r1 - r0, K1, m->last_act == GANTTS_ACT_SIGMOID ? 1 : 0, ks, m->slope * ks,                     \
      m->dropout_p > 0.f ? 0.f : m->slope, gw, gz
      if (K1 % 8 == 0 && K1 <= 256)
        GANTTS_PDL_LAUNCH((gemv_bwd_vec_kernel<1, 4>), GEMV_BLOCKS, GEMV_THREADS, 0, s, GANTTS_GEMV_BWD_ARGS);
      else if (K1 % 8 == 0 && K1 <= 512)
        gemv_bwd_vec_kernel<2, 2><<<GEMV_BLOCKS, GEMV_THREADS, 0, s>>>(GANTTS_GEMV_BWD_ARGS);
      else if (K1 % 8 == 0)
        gemv_bwd_vec_kernel<4, 1><<<GEMV_BLOCKS, GEMV_THREADS, 0, s>>>(GANTTS_GEMV_BWD_ARGS);
      else
        gemv_bwd_kernel<<<GEMV_BLOCKS, GEMV_THREADS, 0, s>>>(GANTTS_GEMV_BWD_ARGS);
#undef GANTTS_GEMV_BWD_ARGS
      GANTTS_LAUNCH_CHECK("gemv_bwd_kernel");
      return GANTTS_OK;
    };
    // a window's chain writes its rows' planes; the partials of gW, gb come from one launch over all M rows, on the
    // weight-gradient stream, with the same row-to-block mapping as the single launch of an unwindowed call
    if (!windowed) {
      if ((rc = gemv_bwd(0, M, want, 1, st))) return rc;
    } else if ((rc = gemv_bwd(chain_r0, chain_r1, 0, 1, st))) {
      return rc;
    }
    if (want) {
      // partial rows are [K1 weights | 1 bias]: one column-parallel reduction for both
      if ((rc = fork())) return rc;
      if (windowed && (rc = gemv_bwd(0, M, 1, 0, ws))) return rc;
      GANTTS_PDL_LAUNCH((gemv_partial_reduce_kernel), (K1 + 1 + 31) / 32, 256, 0, ws, gemv_part, GEMV_BLOCKS, K1,
                                                                    gW ? gW[L - 1] : nullptr,
                                                                    gb ? gb[L - 1] : nullptr, accumulate);
      GANTTS_LAUNCH_CHECK("gemv_partial_reduce_kernel");
    }
    l_start = L - 2;
  } else if (!gy_planes_ready) {
    const int64_t rows = chain_r1 - chain_r0, total = rows * m->dims[L];
    int nb = (int)((total + 1023) / 1024);
    if (nb > num_sms() * 8) nb = num_sms() * 8;
    if (nb < 1) nb = 1;
    const Planes Gw = plane_rows(G, chain_r0, chain_r1);
    grad_out_to_planes_kernel<<<nb, 256, 0, st>>>(gy + chain_r0 * gy_rs, gy_rs, y ? y + chain_r0 * y_rs : nullptr, y_rs,
                                                  rows, m->dims[L], Gw.hi, Gw.lo, Gw.pitch,
                                                  m->last_act == GANTTS_ACT_SIGMOID ? 1 : 0);
    GANTTS_LAUNCH_CHECK("grad_out_to_planes_kernel");
  }
  for (int l = l_start; l >= 0; --l) {
    float* gbl = (gb && gb[l]) ? gb[l] : nullptr;
    if (((gW && gW[l]) || gbl) && (rc = fork())) return rc;
    if (gW && gW[l]) {
      // gW_l and (via the ones-MMA) gb_l from one launch; the split reductions of all layers are
      // summed by a single launch at the end
      float* partial = reinterpret_cast<float*>(partial_cur);
      partial_cur += mn_partial_bytes(M, m->dims[l + 1], m->dims[l], nullptr, nullptr) + 256;
      if ((rc = launch_gemm_mn(G, t.H[l], gW[l], gbl, accumulate, partial, ws, &rl))) return rc;
    } else if (gbl) {
      if ((rc = colsum_planes(G, gbl, accumulate, colpart, ws))) return rc;
    }
    if (l > 0) {
      char* c1 = gbuf[(pp + 1) % nbuf];
      Planes Gn = carve_planes(c1, M, m->dims[l]);
      const Planes O = plane_rows(Gn, chain_r0, chain_r1);
      EpiArgs e;
      e.epi = EPI_PLANES_BWD;
      e.out_hi = O.hi;
      e.out_lo = O.lo;
      e.out_pitch = O.pitch;
      e.code = t.code[l] + chain_r0 * t.code_pitch[l];
      e.code_pitch = t.code_pitch[l];
      e.slope = m->slope;
      e.p = m->dropout_p;
      if ((rc = launch_gemm_kk(plane_rows(G, chain_r0, chain_r1), t.Wt[l], e, st))) return rc;
      G = Gn;
      pp = (pp + 1) % nbuf;
    } else if (gx && (gx_row0 > chain_r0 ? gx_row0 : chain_r0) < chain_r1) {
      const int64_t g0 = gx_row0 > chain_r0 ? gx_row0 : chain_r0;
      EpiArgs e;
      e.epi = EPI_F32;
      e.C = gx + g0 * gx_rs;
      e.ldc = gx_rs;
      e.accumulate = gx_accumulate;
      if ((rc = launch_gemm_kk(plane_rows(G, g0, chain_r1), t.Wt[0], e, st))) return rc;
    }
  }
  if ((rc = flush_reduce(rl, accumulate, ws))) return rc;
  return side ? stream_wait(st, side) : GANTTS_OK;
}
