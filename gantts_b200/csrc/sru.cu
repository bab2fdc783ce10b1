// SRU (Simple Recurrent Unit, v1) recurrence -- the scan behind the third-party `cuda_functional.SRU`
// that reference gantts/models.py:144-167 (SRURNN) imports (github.com/taolei87/sru, NOT vendored, no
// reference test touches it: parity unpinned; restated from the published recurrence):
//   U = x W  with k = 3 (n_in == dirs*d) or 4 gates per hidden unit, laid out [.., column, k] (k fastest)
//   f = sigmoid(U_1 + b_f);  r = sigmoid(U_2 + b_r);  c_t = f c_{t-1} + (1 - f) U_0
//   h_t = r (g(c_t) mask) + (1 - r) x'_t,   x' = x (k == 3) or U_3 (k == 4),  g = tanh | relu | identity
// The GEMM is the tensor-core engine (caller); this kernel is the element-wise scan: one thread per
// (batch row, column) walking the T steps, columns [0,d) forward in time, [d,2d) backward.  HBM-bound.
#include "common.cuh"

namespace gantts {

struct SruParams {
  const float* u;       // [B][T][ncols*k]
  const float* x;       // [B][T][ncols] highway input when k == 3 (else null)
  const float* bias;    // [2*ncols]
  const float* mask_h;  // [B][ncols] output dropout mask (already scaled) or null
  float* h;             // [B][T][ncols]
  float* c;             // [B][T][ncols] cell states (saved for the backward)
  const float* dh;      // bwd
  float* du;            // bwd [B][T][ncols*k]
  float* dx;            // bwd [B][T][ncols] (+=) when k == 3
  float* dbias_part;    // bwd [B][2*ncols]
  const int64_t* lengths;  // fwd with lengths [B]
  int B, T, d, k, bidir, act;   // act: 0 identity, 1 tanh, 2 relu
};

__device__ __forceinline__ float sru_act(float c, int act) { return act == 1 ? tanhf(c) : (act == 2 ? fmaxf(c, 0.f) : c); }
__device__ __forceinline__ float sru_dact(float c, float val, int act) {
  return act == 1 ? (1.f - val * val) : (act == 2 ? (c > 0.f ? 1.f : 0.f) : 1.f);
}

// The scan is sequential in t only through c; everything it READS (U, x, saved c, dh) is known up front.  A
// plain loop issues one dependent HBM round trip per step (the stores to c / h keep the compiler from hoisting
// the next step's loads): measured 1.3 ms per layer at B=32, T=1000, 1024 columns, 15x the HBM time.  So the
// steps are processed in chunks of SRU_UNR: all loads of a chunk are issued first (independent, SRU_UNR deep
// per thread), then the recurrence runs on registers.
constexpr int SRU_UNR = 8;
constexpr int SRU_MAX_T = 1 << 24;   // of gantts_sru_fwd_lengths

// LEN = false: gantts_sru_fwd, every sequence runs over the padded T (the reverse direction starts at T - 1) and the
// cell states are saved.  LEN = true: gantts_sru_fwd_lengths, sequence b runs over its own L = lengths[b] frames (the
// reverse direction starts at L - 1 with a zero cell), h is 0 at and beyond L, and no cell state is kept.
template <int K, bool LEN>
__global__ void __launch_bounds__(128) sru_fwd_kernel(const SruParams p) {
  const int ncols = p.d * (p.bidir ? 2 : 1);
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= p.B * ncols) return;
  const int b = idx / ncols, col = idx - b * ncols;
  const bool rev = p.bidir && col >= p.d;
  const float bf = p.bias[col], br = p.bias[col + ncols];
  const float m = (!LEN && p.mask_h) ? p.mask_h[idx] : 1.f;    // eval mode: no mask
  int L = p.T;
  const int64_t base = (int64_t)b * p.T * ncols + col;       // element (b, t = 0, col)
  if (LEN) {
    const int64_t l = p.lengths[b];
    L = l < 0 ? 0 : (l > p.T ? p.T : (int)l);
    for (int t = L; t < p.T; ++t) p.h[base + (int64_t)t * ncols] = 0.f;
  }
  const int64_t tstep = rev ? -(int64_t)ncols : (int64_t)ncols;
  const int64_t first = rev ? base + (int64_t)(L - 1) * ncols : base;
  float c = 0.f;
  for (int s0 = 0; s0 < L; s0 += SRU_UNR) {
    float u0[SRU_UNR], u1[SRU_UNR], u2[SRU_UNR], xp[SRU_UNR];
#pragma unroll
    for (int j = 0; j < SRU_UNR; ++j) {
      u0[j] = u1[j] = u2[j] = xp[j] = 0.f;
      if (s0 + j < L) {
        const int64_t e = first + (int64_t)(s0 + j) * tstep;
        if (K == 4) {
          const float4 v = __ldg(reinterpret_cast<const float4*>(p.u + e * 4));
          u0[j] = v.x; u1[j] = v.y; u2[j] = v.z; xp[j] = v.w;
        } else {
          const float* up = p.u + e * 3;
          u0[j] = __ldg(up); u1[j] = __ldg(up + 1); u2[j] = __ldg(up + 2);
          xp[j] = __ldg(p.x + e);
        }
      }
    }
#pragma unroll
    for (int j = 0; j < SRU_UNR; ++j) {
      if (s0 + j < L) {
        const int64_t e = first + (int64_t)(s0 + j) * tstep;
        const float g1 = 1.f / (1.f + expf(-(u1[j] + bf)));
        const float g2 = 1.f / (1.f + expf(-(u2[j] + br)));
        c = (c - u0[j]) * g1 + u0[j];
        if (!LEN) p.c[e] = c;
        const float val = sru_act(c, p.act);
        p.h[e] = (val * m - xp[j]) * g2 + xp[j];
      }
    }
  }
}

template <int K>
__global__ void __launch_bounds__(128) sru_bwd_kernel(const SruParams p) {
  const int ncols = p.d * (p.bidir ? 2 : 1);
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= p.B * ncols) return;
  const int b = idx / ncols, col = idx - b * ncols;
  const bool rev = p.bidir && col >= p.d;
  const float bf = p.bias[col], br = p.bias[col + ncols];
  const float m = p.mask_h ? p.mask_h[idx] : 1.f;
  const int64_t base = (int64_t)b * p.T * ncols + col;
  const int64_t tstep = rev ? -(int64_t)ncols : (int64_t)ncols;      // forward-scan direction
  const int64_t first = rev ? base + (int64_t)(p.T - 1) * ncols : base;
  float dc = 0.f, gbf = 0.f, gbr = 0.f;
  // scan steps s = T-1 .. 0 (reverse of the forward order); element of step s is first + s * tstep
  for (int s0 = p.T - 1; s0 >= 0; s0 -= SRU_UNR) {
    float u0[SRU_UNR], u1[SRU_UNR], u2[SRU_UNR], xp[SRU_UNR], cs[SRU_UNR + 1], dhv[SRU_UNR], dxo[SRU_UNR];
#pragma unroll
    for (int j = 0; j < SRU_UNR; ++j) {
      u0[j] = u1[j] = u2[j] = xp[j] = cs[j] = dhv[j] = dxo[j] = 0.f;
      const int sidx = s0 - j;
      if (sidx >= 0) {
        const int64_t e = first + (int64_t)sidx * tstep;
        if (K == 4) {
          const float4 v = __ldg(reinterpret_cast<const float4*>(p.u + e * 4));
          u0[j] = v.x; u1[j] = v.y; u2[j] = v.z; xp[j] = v.w;
        } else {
          const float* up = p.u + e * 3;
          u0[j] = __ldg(up); u1[j] = __ldg(up + 1); u2[j] = __ldg(up + 2);
          xp[j] = __ldg(p.x + e);
          dxo[j] = p.dx[e];
        }
        cs[j] = p.c[e];
        dhv[j] = __ldg(p.dh + e);
      }
    }
    {
      const int sidx = s0 - SRU_UNR;                       // c of the step before the chunk's last one
      cs[SRU_UNR] = sidx >= 0 ? p.c[first + (int64_t)sidx * tstep] : 0.f;
    }
#pragma unroll
    for (int j = 0; j < SRU_UNR; ++j) {
      const int sidx = s0 - j;
      if (sidx >= 0) {
        const int64_t e = first + (int64_t)sidx * tstep;
        const float g1 = 1.f / (1.f + expf(-(u1[j] + bf)));
        const float g2 = 1.f / (1.f + expf(-(u2[j] + br)));
        const float c = cs[j];
        const float cprev = sidx > 0 ? cs[j + 1] : 0.f;
        const float val = sru_act(c, p.act);
        const float dg2 = dhv[j] * (val * m - xp[j]);
        const float dxp = dhv[j] * (1.f - g2);
        const float dct = dc + dhv[j] * g2 * m * sru_dact(c, val, p.act);
        const float du0 = dct * (1.f - g1);
        const float dg1 = dct * (cprev - u0[j]);
        dc = dct * g1;
        const float du1 = dg1 * g1 * (1.f - g1), du2 = dg2 * g2 * (1.f - g2);
        if (K == 4) {
          *reinterpret_cast<float4*>(p.du + e * 4) = make_float4(du0, du1, du2, dxp);
        } else {
          float* dup = p.du + e * 3;
          dup[0] = du0; dup[1] = du1; dup[2] = du2;
          p.dx[e] = dxo[j] + dxp;
        }
        gbf += du1; gbr += du2;
      }
    }
  }
  p.dbias_part[(int64_t)b * 2 * ncols + col] = gbf;
  p.dbias_part[(int64_t)b * 2 * ncols + ncols + col] = gbr;
}

// ---------------------------------------------------------------------------- SRU stack of the fused GAN step
// The fused step (gan_step.cu) runs U = (x * mask_x) W as one bf16x3 GEMM per layer and these scans around it.  The
// dropout masks of a layer are shared over time, so each thread draws its (b, col) keep decision once with the counter
// hash of gantts_dropout (thresh 0 / scale 1 = no mask).  Planes are bf16 hi/lo operand planes of the GEMM engine.
struct SruMask {
  uint64_t seed;
  uint32_t thresh;
  float scale;
};
__device__ __forceinline__ float sru_mask_value(const SruMask& m, int b, int n, int col) {
  return dropout_keep(m.seed, (uint32_t)b, (uint32_t)n, (uint32_t)col, m.thresh) ? m.scale : 0.f;
}
__device__ __forceinline__ void store_split(__nv_bfloat16* hi, __nv_bfloat16* lo, int64_t i, float v) {
  const __nv_bfloat16 h = __float2bfloat16_rn(v);
  hi[i] = h;
  lo[i] = __float2bfloat16_rn(v - __bfloat162float(h));
}

struct SruStepFwd {
  const float* u;                // [M][ncols*K] = U of this layer (GEMM output)
  const float* xh;               // highway input when K == 3 (the UNMASKED layer input), row stride xh_rs
  int64_t xh_rs;
  const float* bias;             // [2*ncols] forget | reset
  float* c;                      // [M][ncols] saved for the backward
  float* h;                      // [M][ncols] fp32 h (the next layer's highway input) or null
  __nv_bfloat16 *hi, *lo;        // operand planes of h * mask_x(next layer) [M][pitch]
  int64_t pitch;
  SruMask mh, mx;                // output mask on g(c_t) of this layer; input mask of the next layer
  int B, T, d, bidir, act;
};

// One thread per (batch row, column), sequential in t, loads of SRU_UNR steps in flight as in sru_fwd_kernel.
template <int K>
__global__ void __launch_bounds__(128) sru_step_fwd_kernel(const SruStepFwd p) {
  const int ncols = p.d * (p.bidir ? 2 : 1);
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= p.B * ncols) return;
  const int b = idx / ncols, col = idx - b * ncols;
  const bool rev = p.bidir && col >= p.d;
  const float bf = p.bias[col], br = p.bias[col + ncols];
  const float m = sru_mask_value(p.mh, b, ncols, col), mx = sru_mask_value(p.mx, b, ncols, col);
  const int64_t row0 = (int64_t)b * p.T;
  float c = 0.f;
  for (int s0 = 0; s0 < p.T; s0 += SRU_UNR) {
    float u0[SRU_UNR], u1[SRU_UNR], u2[SRU_UNR], xp[SRU_UNR];
#pragma unroll
    for (int j = 0; j < SRU_UNR; ++j) {
      u0[j] = u1[j] = u2[j] = xp[j] = 0.f;
      if (s0 + j < p.T) {
        const int64_t r = row0 + (rev ? p.T - 1 - (s0 + j) : s0 + j);
        const int64_t e = r * ncols + col;
        if (K == 4) {
          const float4 v = __ldg(reinterpret_cast<const float4*>(p.u + e * 4));
          u0[j] = v.x; u1[j] = v.y; u2[j] = v.z; xp[j] = v.w;
        } else {
          const float* up = p.u + e * 3;
          u0[j] = __ldg(up); u1[j] = __ldg(up + 1); u2[j] = __ldg(up + 2);
          xp[j] = __ldg(p.xh + r * p.xh_rs + col);
        }
      }
    }
#pragma unroll
    for (int j = 0; j < SRU_UNR; ++j) {
      if (s0 + j < p.T) {
        const int64_t r = row0 + (rev ? p.T - 1 - (s0 + j) : s0 + j);
        const int64_t e = r * ncols + col;
        const float g1 = 1.f / (1.f + expf(-(u1[j] + bf)));
        const float g2 = 1.f / (1.f + expf(-(u2[j] + br)));
        c = (c - u0[j]) * g1 + u0[j];
        p.c[e] = c;
        const float val = sru_act(c, p.act);
        const float h = (val * m - xp[j]) * g2 + xp[j];
        if (p.h) p.h[e] = h;
        store_split(p.hi, p.lo, r * p.pitch + col, h * mx);
      }
    }
  }
}

struct SruStepBwd {
  const float* u;                // [M][ncols*K]
  const float* xh;               // highway input when K == 3, row stride xh_rs
  int64_t xh_rs;
  const float* bias;
  const float* c;                // [M][ncols] from the forward
  const float* dx;               // [M][ncols]: dL/dh = dx * mask_x(upper layer) + dxp_in
  const float* dxp_in;           // highway gradient the upper layer left for this one, or null
  SruMask mxu, mh;               // input mask of the upper layer (none for the top layer); output mask of this layer
  __nv_bfloat16 *du_hi, *du_lo;  // dU as operand planes [M][du_pitch] of the two backward GEMMs
  int64_t du_pitch;
  float* dxp_out;                // K == 3: highway gradient (1 - r) dh for the layer below, or null; may alias dxp_in
  float* dbias_part;             // [B][2*ncols]
  int B, T, d, bidir, act;
};

// Reverse scan of sru_step_fwd_kernel (the arithmetic of sru_bwd_kernel).  dh is formed on load from the upper layer's
// input gradient and highway gradient; dxp_out may be the same buffer as dxp_in: each thread reads an element before it
// writes it, and no other thread touches it.
template <int K>
__global__ void __launch_bounds__(128) sru_step_bwd_kernel(const SruStepBwd p) {
  const int ncols = p.d * (p.bidir ? 2 : 1);
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= p.B * ncols) return;
  const int b = idx / ncols, col = idx - b * ncols;
  const bool rev = p.bidir && col >= p.d;
  const float bf = p.bias[col], br = p.bias[col + ncols];
  const float m = sru_mask_value(p.mh, b, ncols, col), mxu = sru_mask_value(p.mxu, b, ncols, col);
  const int64_t row0 = (int64_t)b * p.T;
  float dc = 0.f, gbf = 0.f, gbr = 0.f;
  for (int s0 = p.T - 1; s0 >= 0; s0 -= SRU_UNR) {
    float u0[SRU_UNR], u1[SRU_UNR], u2[SRU_UNR], xp[SRU_UNR], cs[SRU_UNR + 1], dhv[SRU_UNR];
#pragma unroll
    for (int j = 0; j < SRU_UNR; ++j) {
      u0[j] = u1[j] = u2[j] = xp[j] = cs[j] = dhv[j] = 0.f;
      const int sidx = s0 - j;
      if (sidx >= 0) {
        const int64_t r = row0 + (rev ? p.T - 1 - sidx : sidx);
        const int64_t e = r * ncols + col;
        if (K == 4) {
          const float4 v = __ldg(reinterpret_cast<const float4*>(p.u + e * 4));
          u0[j] = v.x; u1[j] = v.y; u2[j] = v.z; xp[j] = v.w;
        } else {
          const float* up = p.u + e * 3;
          u0[j] = __ldg(up); u1[j] = __ldg(up + 1); u2[j] = __ldg(up + 2);
          xp[j] = __ldg(p.xh + r * p.xh_rs + col);
        }
        cs[j] = __ldg(p.c + e);
        dhv[j] = p.dx[e] * mxu + (p.dxp_in ? p.dxp_in[e] : 0.f);
      }
    }
    {
      const int sidx = s0 - SRU_UNR;                       // c of the step before the chunk's last one
      cs[SRU_UNR] = sidx >= 0 ? __ldg(p.c + (row0 + (rev ? p.T - 1 - sidx : sidx)) * ncols + col) : 0.f;
    }
#pragma unroll
    for (int j = 0; j < SRU_UNR; ++j) {
      const int sidx = s0 - j;
      if (sidx >= 0) {
        const int64_t r = row0 + (rev ? p.T - 1 - sidx : sidx);
        const float g1 = 1.f / (1.f + expf(-(u1[j] + bf)));
        const float g2 = 1.f / (1.f + expf(-(u2[j] + br)));
        const float c = cs[j];
        const float cprev = sidx > 0 ? cs[j + 1] : 0.f;
        const float val = sru_act(c, p.act);
        const float dg2 = dhv[j] * (val * m - xp[j]);
        const float dxp = dhv[j] * (1.f - g2);
        const float dct = dc + dhv[j] * g2 * m * sru_dact(c, val, p.act);
        const float du0 = dct * (1.f - g1);
        const float dg1 = dct * (cprev - u0[j]);
        dc = dct * g1;
        const float du1 = dg1 * g1 * (1.f - g1), du2 = dg2 * g2 * (1.f - g2);
        const int64_t q = r * p.du_pitch + (int64_t)col * K;
        if (K == 4) {
          const uint32_t h01 = pack_bf16x2(du0, du1), h23 = pack_bf16x2(du2, dxp);
          const uint32_t l01 = pack_bf16x2(du0 - __uint_as_float(h01 << 16), du1 - __uint_as_float(h01 & 0xffff0000u));
          const uint32_t l23 = pack_bf16x2(du2 - __uint_as_float(h23 << 16), dxp - __uint_as_float(h23 & 0xffff0000u));
          *reinterpret_cast<uint2*>(p.du_hi + q) = make_uint2(h01, h23);
          *reinterpret_cast<uint2*>(p.du_lo + q) = make_uint2(l01, l23);
        } else {
          store_split(p.du_hi, p.du_lo, q, du0);
          store_split(p.du_hi, p.du_lo, q + 1, du1);
          store_split(p.du_hi, p.du_lo, q + 2, du2);
          if (p.dxp_out) p.dxp_out[r * ncols + col] = dxp;
        }
        gbf += du1; gbr += du2;
      }
    }
  }
  p.dbias_part[(int64_t)b * 2 * ncols + col] = gbf;
  p.dbias_part[(int64_t)b * 2 * ncols + ncols + col] = gbr;
}

// out[i] = sum over b = 0..B-1 (in that order) of part[b][i]: the bias gradient, deterministic.
__global__ void sru_bias_reduce_kernel(const float* __restrict__ part, int B, int n, float* __restrict__ out) {
  pdl_entry();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float s = 0.f;
  for (int b = 0; b < B; ++b) s += part[(int64_t)b * n + i];
  out[i] = s;
}

// Layer 0's GEMM operand: planes of x * mask_x, mask [B][cols] shared over the T rows of each sequence.  One warp per
// row, a lane converts pairs of columns (split_planes_kernel with the mask).
__global__ void sru_mask_split_kernel(const float* __restrict__ x, int64_t rs, int64_t rows, int cols, int T, SruMask mk,
                                      __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo, int64_t pitch) {
  pdl_entry();
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t r = warp; r < rows; r += nwarps) {
    const int b = (int)(r / T);
    const float* sr = x + r * rs;
    uint32_t* hr = reinterpret_cast<uint32_t*>(hi + r * pitch);
    uint32_t* lr = reinterpret_cast<uint32_t*>(lo + r * pitch);
    for (int c = 2 * lane; c < cols; c += 64) {
      const float a = sr[c] * sru_mask_value(mk, b, cols, c);
      const float v = (c + 1 < cols) ? sr[c + 1] * sru_mask_value(mk, b, cols, c + 1) : 0.f;
      const uint32_t hp = pack_bf16x2(a, v);
      hr[c >> 1] = hp;
      lr[c >> 1] = pack_bf16x2(a - __uint_as_float(hp << 16), v - __uint_as_float(hp & 0xffff0000u));
    }
  }
}

static inline SruMask sru_mask(uint64_t seed, float p) {
  SruMask m;
  m.seed = seed;
  m.thresh = p > 0.f ? (uint32_t)(p * 65536.f + 0.5f) : 0u;      // as gantts_dropout
  m.scale = p > 0.f ? 1.f / (1.f - p) : 1.f;
  return m;
}

// The two scans are the only kernels of the step launched WITHOUT programmatic dependent launch, and they do not trigger
// their successor early.  A scan is a few hundred long-lived blocks (B * ncols threads, 160 blocks at tts_acoustic);
// launched early, they become resident on the first SMs the previous GEMM's persistent CTAs free and pack several to an
// SM, and a GEMM launched early behind them holds the other SMs while it waits.  Measured at tts_acoustic (B = 20,
// T = 1000, H100 80GB HBM3 at 400 W): 28.5 ms per step with the scans under PDL, 23.1 ms with plain launches.
static int launch_sru_step_fwd(const SruStepFwd& p, int k, cudaStream_t st) {
  const int n = p.B * p.d * (p.bidir ? 2 : 1);
  if (k == 4) sru_step_fwd_kernel<4><<<(n + 127) / 128, 128, 0, st>>>(p);
  else sru_step_fwd_kernel<3><<<(n + 127) / 128, 128, 0, st>>>(p);
  GANTTS_LAUNCH_CHECK("sru_step_fwd_kernel");
  return GANTTS_OK;
}

static int launch_sru_step_bwd(const SruStepBwd& p, int k, cudaStream_t st) {
  const int ncols = p.d * (p.bidir ? 2 : 1), n = p.B * ncols;
  if (k == 4) sru_step_bwd_kernel<4><<<(n + 127) / 128, 128, 0, st>>>(p);
  else sru_step_bwd_kernel<3><<<(n + 127) / 128, 128, 0, st>>>(p);
  GANTTS_LAUNCH_CHECK("sru_step_bwd_kernel");
  return GANTTS_OK;
}

static int sru_check(const SruParams& p) {
  GANTTS_CHECK_ARG(p.B >= 1 && p.T >= 1 && p.d >= 1 && (p.k == 3 || p.k == 4), "sru: bad shape (B=%d T=%d d=%d k=%d)",
                   p.B, p.T, p.d, p.k);
  // one thread per (batch row, column): the launches count B * columns in int
  GANTTS_CHECK_ARG((int64_t)p.B * p.d * (p.bidir ? 2 : 1) <= ((int64_t)1 << 30),
                   "sru: B = %d and d = %d must be >= 1 with B * columns <= 2^30", p.B, p.d);
  GANTTS_CHECK_ARG(p.act >= 0 && p.act <= 2, "sru: bad activation %d", p.act);
  GANTTS_CHECK_ARG(p.u && p.bias && (p.k == 4 || p.x), "sru: null pointer");
  return GANTTS_OK;
}

}  // namespace gantts

using namespace gantts;

extern "C" int gantts_sru_fwd(const float* u, const float* x, const float* bias, const float* mask_h, float* h, float* c,
                              int B, int T, int d, int k, int bidir, int act, void* stream) {
  SruParams p{};
  p.u = u; p.x = x; p.bias = bias; p.mask_h = mask_h; p.h = h; p.c = c;
  p.B = B; p.T = T; p.d = d; p.k = k; p.bidir = bidir ? 1 : 0; p.act = act;
  int rc = sru_check(p);
  if (rc) return rc;
  GANTTS_CHECK_ARG(h && c, "sru_fwd: null output");
  const int n = B * d * (bidir ? 2 : 1);
  if (k == 4) sru_fwd_kernel<4, false><<<(n + 127) / 128, 128, 0, as_stream(stream)>>>(p);
  else sru_fwd_kernel<3, false><<<(n + 127) / 128, 128, 0, as_stream(stream)>>>(p);
  GANTTS_LAUNCH_CHECK("sru_fwd_kernel");
  return GANTTS_OK;
}

extern "C" int gantts_sru_fwd_lengths(const float* u, const float* x, const float* bias, const int64_t* lengths_dev,
                                      float* h, int B, int T, int d, int k, int bidir, int act, void* stream) {
  SruParams p{};
  p.u = u; p.x = x; p.bias = bias; p.h = h; p.lengths = lengths_dev;
  p.B = B; p.T = T; p.d = d; p.k = k; p.bidir = bidir ? 1 : 0; p.act = act;
  GANTTS_CHECK_ARG(lengths_dev, "sru_fwd_lengths: null lengths: sequence b runs over its own lengths_dev[b] frames");
  GANTTS_CHECK_ARG(T >= 1 && T <= SRU_MAX_T, "sru_fwd_lengths: padded length T = %d must be in [1, %d]", T, SRU_MAX_T);
  GANTTS_CHECK_ARG(B >= 1 && d >= 1 && (int64_t)B * d * (bidir ? 2 : 1) <= ((int64_t)1 << 30),
                   "sru_fwd_lengths: B = %d and d = %d must be >= 1 with B * columns <= 2^30", B, d);
  int rc = sru_check(p);
  if (rc) return rc;
  GANTTS_CHECK_ARG(h, "sru_fwd_lengths: null output");
  const int n = B * d * (bidir ? 2 : 1);
  if (k == 4) sru_fwd_kernel<4, true><<<(n + 127) / 128, 128, 0, as_stream(stream)>>>(p);
  else sru_fwd_kernel<3, true><<<(n + 127) / 128, 128, 0, as_stream(stream)>>>(p);
  GANTTS_LAUNCH_CHECK("sru_fwd_lengths_kernel");
  return GANTTS_OK;
}

extern "C" int gantts_sru_bwd(const float* u, const float* x, const float* bias, const float* mask_h, const float* c,
                              const float* dh, float* du, float* dx, float* dbias_part, int B, int T, int d, int k,
                              int bidir, int act, void* stream) {
  SruParams p{};
  p.u = u; p.x = x; p.bias = bias; p.mask_h = mask_h; p.c = const_cast<float*>(c); p.dh = dh; p.du = du; p.dx = dx;
  p.dbias_part = dbias_part;
  p.B = B; p.T = T; p.d = d; p.k = k; p.bidir = bidir ? 1 : 0; p.act = act;
  int rc = sru_check(p);
  if (rc) return rc;
  GANTTS_CHECK_ARG(c && dh && du && dbias_part && (k == 4 || dx), "sru_bwd: null pointer");
  const int n = B * d * (bidir ? 2 : 1);
  if (k == 4) sru_bwd_kernel<4><<<(n + 127) / 128, 128, 0, as_stream(stream)>>>(p);
  else sru_bwd_kernel<3><<<(n + 127) / 128, 128, 0, as_stream(stream)>>>(p);
  GANTTS_LAUNCH_CHECK("sru_bwd_kernel");
  return GANTTS_OK;
}
