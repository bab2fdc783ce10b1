// MLPG trajectory generation as stencil + row-variant FIR (see include/gantts_b200.h).
//
// Reference path replaced: nnmnkwii.paramgen.unit_variance_mlpg_matrix (train.py:510-513, a dense
// (T x 3T) matrix rebuilt on the CPU per batch) + nnmnkwii.autograd.unit_variance_mlpg (a dense fp32
// matmul, gantts/multistream.py:120, gantts/models.py:66,115).  y = R mu with R = P^-1 W^T is
// evaluated as  b = W^T mu  (<=5-tap stencil per window)  followed by  y_t = sum_j G[t][j] b_{t-K+j},
// G = rows of P^-1 truncated at +-K (entries beyond are < 3e-10 of the diagonal for the hparams
// windows).  Per-column arithmetic does not depend on which other columns are in the launch nor on
// the launch geometry (tiles depend on T only), which the reference test
// tests/test_gantts.py:156-159 (bitwise whole-vs-slice equality) requires.
//
// HBM-bound by design: algorithmic bytes per (b,t) = 4 * (sum of stream widths + output columns).
#include <cuda_bf16.h>
#include <math.h>

#include <vector>

#include "common.cuh"

namespace gantts {

constexpr int K_HALF = GANTTS_MLPG_HALF_TAPS;     // 24
constexpr int NTAPS = 2 * K_HALF + 1;             // 49
constexpr int TABW = GANTTS_MLPG_TABLE_COLS;      // floats per table row: 49 FIR taps, pad, Cholesky rows at 52 and 56
constexpr int GROW = 52;                          // taps padded to a float4 multiple
constexpr int TT = 64;                            // frames per block
constexpr int TC = 64;                            // columns per block
constexpr int HALO = 2;                           // max(l,u)
constexpr int MLPG_THREADS = 256;

struct ColInfo {
  int in_col;   // column of the window-0 component, -1 when the column is out of range
  int sd;
  int dyn;
};

__device__ __forceinline__ ColInfo find_col(const gantts_streams_t& st, int oc) {
  ColInfo ci{-1, 0, 0};
#pragma unroll 1
  for (int s = 0; s < st.n; ++s) {
    int d = oc - st.out_start[s];
    if (d >= 0 && d < st.sd[s]) {
      ci.in_col = st.in_start[s] + d;
      ci.sd = st.sd[s];
      ci.dyn = st.dyn[s];
    }
  }
  return ci;
}

// acc[i] = sum_j G[row0+i][j] * win[i+j], 8 rows at a time, window held in registers.
__device__ __forceinline__ void fir8(const float* __restrict__ gs, int grow0, const float* win,
                                     float* acc) {
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float4* g4 = reinterpret_cast<const float4*>(gs + (grow0 + i) * GROW);
    float a = 0.f;
#pragma unroll
    for (int q = 0; q < GROW / 4; ++q) {
      float4 g = g4[q];
      if (4 * q + 0 < NTAPS) a = fmaf(g.x, win[i + 4 * q + 0], a);
      if (4 * q + 1 < NTAPS) a = fmaf(g.y, win[i + 4 * q + 1], a);
      if (4 * q + 2 < NTAPS) a = fmaf(g.z, win[i + 4 * q + 2], a);
      if (4 * q + 3 < NTAPS) a = fmaf(g.w, win[i + 4 * q + 3], a);
    }
    acc[i] = a;
  }
}

__global__ void __launch_bounds__(MLPG_THREADS)
mlpg_fwd_kernel(const float* __restrict__ in, int64_t in_bs, int64_t in_ts,
                float* __restrict__ out, int64_t out_bs, int64_t out_ts,
                const float* __restrict__ table, gantts_streams_t st, gantts_windows_t win,
                int T, int ncols) {
  extern __shared__ __align__(16) float smem[];
  float* bv = smem;                                   // [(TT + 2K)][TC]
  float* gs = smem + (TT + 2 * K_HALF) * TC;          // [TT][GROW]
  const int b = blockIdx.z, t0 = blockIdx.y * TT, c0 = blockIdx.x * TC;
  const float* inb = in + (int64_t)b * in_bs;

  for (int i = threadIdx.x; i < TT * GROW; i += MLPG_THREADS) {
    int r = i / GROW, j = i - r * GROW, t = t0 + r;
    gs[i] = (t < T && j < NTAPS) ? table[(int64_t)t * TABW + j] : 0.f;
  }
  // Phase 1: b = W^T mu over [t0-K, t0+TT+K) (or the raw input for static streams).  Each thread owns ONE
  // column (stream lookup hoisted) and strides over rows; the non-zero window taps are compacted once per
  // block into a small shared table (7 taps for the hparams windows), so a row costs 7 coalesced loads.
  __shared__ int tap_dt[GANTTS_MAX_WINDOWS * GANTTS_MAX_WINDOW_TAPS];
  __shared__ int tap_w[GANTTS_MAX_WINDOWS * GANTTS_MAX_WINDOW_TAPS];
  __shared__ float tap_c[GANTTS_MAX_WINDOWS * GANTTS_MAX_WINDOW_TAPS];
  __shared__ int tap_n;
  if (threadIdx.x == 0) {
    int n = 0;
    for (int w = 0; w < win.n; ++w)
      for (int kk = 0; kk <= win.l[w] + win.u[w]; ++kk)
        if (win.coef[w][kk] != 0.f) {
          tap_dt[n] = -(kk - win.l[w]);
          tap_w[n] = w;
          tap_c[n] = win.coef[w][kk];
          ++n;
        }
    tap_n = n;
  }
  __syncthreads();
  {
    // taps outer, this thread's 28 rows inner and fully unrolled: 28 independent loads in flight per tap
    // (a row-outer loop serialises ~200 L2 round trips per thread: measured 52 us per launch at cfg2).
    // Per element the taps are still accumulated in ascending order, so the bits do not change.
    constexpr int RPT = (TT + 2 * K_HALF) / (MLPG_THREADS / TC);      // 28 rows per thread
    const int cx = threadIdx.x & (TC - 1), rg = threadIdx.x / TC;
    const ColInfo ci = find_col(st, c0 + cx);
    const float* colp = inb + (ci.in_col >= 0 ? ci.in_col : 0);
    const int ntap = tap_n;
    const int tb = t0 - K_HALF + rg;
    float v[RPT];
#pragma unroll
    for (int j = 0; j < RPT; ++j) v[j] = 0.f;
    if (ci.in_col >= 0) {
      if (!ci.dyn) {
#pragma unroll
        for (int j = 0; j < RPT; ++j) {
          const int t = tb + 4 * j;
          if (t >= 0 && t < T) v[j] = colp[(int64_t)t * in_ts];
        }
      } else {
#pragma unroll 1
        for (int i = 0; i < ntap; ++i) {
          const int dt = tap_dt[i];
          const float c = tap_c[i];
          const float* cp = colp + tap_w[i] * ci.sd;
          // loads first (all independent, each into its own register), then the FMAs: a fused
          // "if (ok) v = fma(c, load, v)" form compiles to one load register reused serially
          float xv[RPT];
#pragma unroll
          for (int j = 0; j < RPT; ++j) {
            const int t = tb + 4 * j, tt = t + dt;
            const bool ok = t >= 0 && t < T && tt >= 0 && tt < T;
            xv[j] = ok ? __ldg(cp + (int64_t)(ok ? tt : 0) * in_ts) : 0.f;
          }
#pragma unroll
          for (int j = 0; j < RPT; ++j) v[j] = fmaf(c, xv[j], v[j]);
        }
      }
    }
#pragma unroll
    for (int j = 0; j < RPT; ++j) bv[(rg + 4 * j) * TC + cx] = v[j];
  }
  __syncthreads();
  // Phase 2: FIR with the rows of P^-1.
  const int cx = threadIdx.x & (TC - 1), rg = threadIdx.x / TC;
  const int oc = c0 + cx;
  ColInfo ci = find_col(st, oc);
  if (ci.in_col < 0 || oc >= ncols) return;
  float* outb = out + (int64_t)b * out_bs + oc;
#pragma unroll 1
  for (int pass = 0; pass < TT / 32; ++pass) {
    const int r0 = rg * (TT / 4) + pass * 8;
    if (t0 + r0 >= T) break;
    if (!ci.dyn) {
#pragma unroll
      for (int i = 0; i < 8; ++i)
        if (t0 + r0 + i < T) outb[(int64_t)(t0 + r0 + i) * out_ts] = bv[(K_HALF + r0 + i) * TC + cx];
      continue;
    }
    float w[8 + 2 * K_HALF], acc[8];
#pragma unroll
    for (int j = 0; j < 8 + 2 * K_HALF; ++j) w[j] = bv[(r0 + j) * TC + cx];
    fir8(gs, r0, w, acc);
#pragma unroll
    for (int i = 0; i < 8; ++i)
      if (t0 + r0 + i < T) outb[(int64_t)(t0 + r0 + i) * out_ts] = acc[i];
  }
}

constexpr int ZROWS = TT + 2 * HALO;                  // 68 rows of z per block
constexpr int GIN_ROWS = ZROWS + 2 * K_HALF;          // 116 rows of upstream gradient

__global__ void __launch_bounds__(MLPG_THREADS)
mlpg_bwd_kernel(const float* __restrict__ go, int64_t go_bs, int64_t go_ts,
                float* __restrict__ gi, int64_t gi_bs, int64_t gi_ts,
                const float* __restrict__ table, gantts_streams_t st, gantts_windows_t win,
                int T, int ncols, int accumulate) {
  extern __shared__ __align__(16) float smem[];
  float* gv = smem;                                   // [GIN_ROWS][TC]   upstream gradient tile
  float* gs = gv + GIN_ROWS * TC;                     // [ZROWS (pad 72)][GROW]
  float* zs = gs + 72 * GROW;                         // [ZROWS (pad 72)][TC]
  const int b = blockIdx.z, t0 = blockIdx.y * TT, c0 = blockIdx.x * TC;
  const float* gob = go + (int64_t)b * go_bs;

  for (int i = threadIdx.x; i < 72 * GROW; i += MLPG_THREADS) {
    int r = i / GROW, j = i - r * GROW, t = t0 - HALO + r;
    gs[i] = (t >= 0 && t < T && j < NTAPS && r < ZROWS) ? table[(int64_t)t * TABW + j] : 0.f;
  }
  for (int i = threadIdx.x; i < GIN_ROWS * TC; i += MLPG_THREADS) {
    int r = i / TC, c = i - r * TC, t = t0 - HALO - K_HALF + r, oc = c0 + c;
    float v = 0.f;
    if (oc < ncols && t >= 0 && t < T) v = gob[(int64_t)t * go_ts + oc];
    gv[i] = v;
  }
  __syncthreads();
  // Phase 2: z = P^-1 g on rows [t0-HALO, t0+TT+HALO); rows outside [0,T) have all-zero taps.
  {
    const int cx = threadIdx.x & (TC - 1), rg = threadIdx.x / TC;
#pragma unroll 1
    for (int q = rg; q < 72 / 8; q += MLPG_THREADS / TC) {
      const int r0 = q * 8;
      float w[8 + 2 * K_HALF], acc[8];
#pragma unroll
      for (int j = 0; j < 8 + 2 * K_HALF; ++j) {
        int rr = r0 + j;
        w[j] = rr < GIN_ROWS ? gv[rr * TC + cx] : 0.f;
      }
      fir8(gs, r0, w, acc);
#pragma unroll
      for (int i = 0; i < 8; ++i) zs[(r0 + i) * TC + cx] = acc[i];
    }
  }
  __syncthreads();
  // Phase 3: grad wrt window w of stream column = sum_k coef_w[k+l] z_{t+k}; static: copy g.
  // One column per thread (stream lookup hoisted), rows strided, coalesced 128 B stores per warp.
  {
    const int cx = threadIdx.x & (TC - 1), rg = threadIdx.x / TC;
    const int oc = c0 + cx;
    const ColInfo ci = find_col(st, oc);
    if (ci.in_col >= 0 && oc < ncols) {
      float* gib = gi + (int64_t)b * gi_bs + ci.in_col;
#pragma unroll 2
      for (int r = rg; r < TT; r += MLPG_THREADS / TC) {
        const int t = t0 + r;
        if (t >= T) break;
        float* prow = gib + (int64_t)t * gi_ts;
        if (!ci.dyn) {
          const float v = gv[(HALO + K_HALF + r) * TC + cx];
          prow[0] = accumulate ? prow[0] + v : v;
        } else {
#pragma unroll
          for (int w = 0; w < GANTTS_MAX_WINDOWS; ++w) {
            if (w < win.n) {
              const int l = win.l[w], ntap = win.l[w] + win.u[w] + 1;
              float v = 0.f;
#pragma unroll
              for (int kk = 0; kk < GANTTS_MAX_WINDOW_TAPS; ++kk)
                if (kk < ntap) v = fmaf(win.coef[w][kk], zs[(HALO + r + kk - l) * TC + cx], v);
              float* q = prow + w * ci.sd;
              *q = accumulate ? *q + v : v;
            }
          }
        }
      }
    }
  }
}


// ---------------------------------------------------------------------------- substitution kernels (half bandwidth <= 2)
// y = P^-1 b by banded Cholesky substitution instead of the 49-tap FIR: P = L L^T is pentadiagonal for the hparams
// windows, so a forward and a backward sweep cost 2 x 3 flops per frame where the FIR costs 49.  Both sweeps are
// sequential in t; parallelism comes from (batch row, column, time chunk): a chunk of SC frames is solved from a zero
// state SW frames earlier (forward) / later (backward) -- the influence of the state decays like |r|^n with
// |r| = sqrt(L2/L0) = 0.389 for these windows (0.389^32 = 8e-14, below fp32 resolution); chunks that touch the ends of
// the utterance start from the exact boundary state.  One warp = 32 consecutive output columns (lane = column: every
// load and store is a coalesced row segment).  Each warp works in phases over a shared-memory strip of its chunk:
//   (1) right-hand side for every frame of the strip -- no recurrence, 8 frames x up to 12 rows of loads in flight;
//   (2) forward substitution in place;  (3) backward substitution in place (forward kernel: straight to the output);
//   (4) adjoint only: the window stencil of the solved strip.
// so the HBM/L2 latency is paid in phase (1) with deep memory-level parallelism and the serial phases touch shared
// memory only.  The per-column arithmetic depends on T only (chunking), not on which columns share the launch: the
// reference's bitwise whole-vs-slice property (tests/test_gantts.py:156-159) holds.
constexpr int SC = 32;                 // frames per chunk
constexpr int SW = 28;                 // warm-up frames on either side (the recursion forgets at ~0.46 per frame: 4e-10)
constexpr int SOLVE_WARPS = 4;         // the warps of a block work on the SAME chunk (different batch rows / column groups)
constexpr int SOLVE_ZROWS = SC + 4 + 2 * SW;                        // strip rows per warp (backward: [t0-2, t1+2) + warm-up)
constexpr int SOLVE_SMEM_FLOATS = SOLVE_ZROWS * 8 + SOLVE_WARPS * SOLVE_ZROWS * 32;   // Cholesky rows of the chunk + 4 strips

// In2OutHighwayNet's combine around the MLPG of the fused step (gantts_highway_t): one dynamic stream whose output column
// c is static column c, rows r = b * T + t.  Forward: y_hat_static = x_s + Tx * Gx, Gx kept for the backward.  Backward:
// the adjoint solves with Tx * g, and dz = g * Gx * Tx * (1 - Tx) leaves as the bf16 hi/lo planes of the gate's
// weight-gradient GEMM.  Separate roundings (no FMA contraction) as in the reference's eager arithmetic.
struct HighwayArgs {
  const float* x;                      // generator input; x_s = its first S columns
  int64_t x_rs;
  const float* tx;                     // [B*T][S] gate
  float* gx;                           // [B*T][S] MLPG output
  __nv_bfloat16 *dz_hi, *dz_lo;        // [B*T][dz_pitch]
  int64_t dz_pitch;
  int S;
};

__device__ __forceinline__ float highway_out(const HighwayArgs& hw, int64_t r, int c, float gxv) {
  return __fadd_rn(hw.x[r * hw.x_rs + c], __fmul_rn(hw.tx[r * hw.S + c], gxv));
}

__device__ __forceinline__ void highway_dz(const HighwayArgs& hw, int64_t r, int c, float g) {
  const int64_t i = r * hw.S + c;
  const float t = hw.tx[i];
  const float v = __fmul_rn(__fmul_rn(__fmul_rn(g, hw.gx[i]), __fsub_rn(1.f, t)), t);
  const __nv_bfloat16 h = __float2bfloat16_rn(v);
  hw.dz_hi[r * hw.dz_pitch + c] = h;
  hw.dz_lo[r * hw.dz_pitch + c] = __float2bfloat16_rn(v - __bfloat162float(h));
}

// FIR family: the combine and the backward's preparation as plain elementwise passes around the unchanged kernels.
__global__ void highway_combine_kernel(HighwayArgs hw, float* __restrict__ out, int64_t rows) {
  pdl_entry();
  const int64_t n = rows * hw.S;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / hw.S;
    const int c = (int)(i - r * hw.S);
    out[i] = highway_out(hw, r, c, hw.gx[i]);
  }
}

// dz from g, then g *= Tx in place (the adjoint that follows sees dL/dGx)
__global__ void highway_bwd_prep_kernel(HighwayArgs hw, float* __restrict__ g, int64_t rows) {
  pdl_entry();
  const int64_t n = rows * hw.S;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / hw.S;
    const int c = (int)(i - r * hw.S);
    const float gv = g[i];
    highway_dz(hw, r, c, gv);
    g[i] = __fmul_rn(gv, hw.tx[i]);
  }
}

struct SolveTaps {
  float c[GANTTS_MAX_WINDOWS][5];      // coefficient of mu_w[t - k] in b_t, k = -2..2 at index k + 2 (0 where absent)
  int nw;
  int std3;                            // the reference's windows: (0,0) | (1,1) with a zero centre tap | (1,1)
};

struct SolveItem {
  int b, cg, chunk;
  bool active;
};

// blocks are laid out chunk-major: ipc = ceil(B * ncg / SOLVE_WARPS) blocks per chunk
__device__ __forceinline__ SolveItem solve_item(int B, int ncg, int bpc) {
  SolveItem it;
  it.chunk = blockIdx.x / bpc;
  const int local = (blockIdx.x % bpc) * SOLVE_WARPS + (threadIdx.x >> 5);
  it.active = local < B * ncg;
  it.b = it.active ? local / ncg : 0;
  it.cg = it.active ? local % ncg : 0;
  return it;
}

// Cholesky rows of the strip [s, s+n) into shared memory, once per block: cf[i] = {1/L_tt, L[t][t-1], L[t][t-2], -},
// cb[i] = {1/L_tt, L[t+1][t], L[t+2][t], -}: one broadcast LDS.128 per substitution step.
__device__ __forceinline__ void strip_coefs(float4* cf, float4* cb, const float* __restrict__ table, int s, int n) {
  for (int i = threadIdx.x; i < n; i += 32 * SOLVE_WARPS) {
    const float4 a = __ldg(reinterpret_cast<const float4*>(table + (int64_t)(s + i) * TABW + 52));
    const float4 b = __ldg(reinterpret_cast<const float4*>(table + (int64_t)(s + i) * TABW + 56));
    cf[i] = a;
    cb[i] = make_float4(a.x, b.x, b.y, 0.f);
  }
  __syncthreads();
}

// forward substitution over rows [0, n) of the strip, in place (static columns are copied through)
__device__ __forceinline__ void strip_forward(float* zs, const float4* cf, int lane, int n, bool dyn) {
  float z1 = 0.f, z2 = 0.f;
#pragma unroll 4
  for (int i = 0; i < n; ++i) {
    const float4 c = cf[i];
    const float b = zs[i * 32 + lane];
    float z = (b - c.y * z1 - c.z * z2) * c.x;
    if (!dyn) z = b;
    z2 = z1;
    z1 = z;
    zs[i * 32 + lane] = z;
  }
}

// HW: highway combine at the output store (HighwayArgs): out = x_s + Tx * y, y itself goes to hw.gx.
template <bool STD3, bool HW>
__global__ void __launch_bounds__(32 * SOLVE_WARPS, 4)
mlpg_solve_fwd_kernel(const float* __restrict__ in, int64_t in_bs, int in_ts, float* __restrict__ out, int64_t out_bs,
                      int out_ts, const float* __restrict__ table, gantts_streams_t st, SolveTaps taps, int B, int T,
                      int ncols, int ncg, int bpc, HighwayArgs hw) {
  pdl_entry();
  extern __shared__ __align__(16) float smem[];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const SolveItem it = solve_item(B, ncg, bpc);
  float4* cf = reinterpret_cast<float4*>(smem);
  float4* cb = cf + SOLVE_ZROWS;
  float* zs = smem + SOLVE_ZROWS * 8 + (size_t)wib * SOLVE_ZROWS * 32;
  const int t0 = it.chunk * SC;
  const int t1 = t0 + SC < T ? t0 + SC : T;                 // outputs [t0, t1)
  const int s = t0 - SW > 0 ? t0 - SW : 0;                  // strip start (exact state when s == 0)
  const int e = t1 + SW < T ? t1 + SW : T;                  // strip end (exact state when e == T)
  const int n = e - s;
  strip_coefs(cf, cb, table, s, n);
  if (!it.active) return;
  const int oc = it.cg * 32 + lane;
  ColInfo ci = find_col(st, oc);
  const bool valid = ci.in_col >= 0 && oc < ncols;
  const bool dyn = valid && ci.dyn;
  // per-lane view of the windows: a static column is "window 0 with coefficient 1", an out-of-range lane reads column 0
  // of its batch row with all coefficients 0 -- no divergent branches in the gather below
  const float* colp = in + (int64_t)it.b * in_bs + (valid ? ci.in_col : 0);
  const int sd = dyn ? ci.sd : 0;
  // (1) b_t = sum_w sum_k coef_w[k+l] mu_w[t - k] over the strip, 8 frames per batch
  for (int i0 = 0; i0 < n; i0 += 8) {
    float bt[8];
    const int r0 = s + i0 - 2;                              // row of batch-window index q = 0 (q = u + 2 - k)
    const bool interior = r0 >= 0 && r0 + 11 < T;
    if (STD3) {
      const float c0 = taps.c[0][2];
      const float c1m = taps.c[1][1], c1p = taps.c[1][3];
      const float c2m = taps.c[2][1], c2z = taps.c[2][2], c2p = taps.c[2][3];
      float x0[8], x1[10], x2[10];           // rows t (q = 2..9) of window 0, rows t-1 .. t+1 (q = 1..10) of windows 1, 2
      if (interior) {
        const float* p0 = colp + (int64_t)(r0 + 2) * in_ts;
        const float* p1 = colp + sd + (int64_t)(r0 + 1) * in_ts;
        const float* p2 = p1 + sd;
#pragma unroll
        for (int q = 0; q < 10; ++q) {
          x1[q] = __ldg(p1);
          x2[q] = __ldg(p2);
          p1 += in_ts;
          p2 += in_ts;
        }
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          x0[u] = __ldg(p0);
          p0 += in_ts;
        }
      } else {                               // first / last batches of a sequence: rows outside [0, T) read as zero
#pragma unroll
        for (int q = 0; q < 10; ++q) {
          const int r = r0 + 1 + q;
          const int rc = r < 0 ? 0 : (r >= T ? T - 1 : r);
          const float* pr = colp + (int64_t)rc * in_ts;
          const float a1 = __ldg(pr + sd), a2 = __ldg(pr + 2 * sd), a0 = __ldg(pr);
          x1[q] = r == rc ? a1 : 0.f;
          x2[q] = r == rc ? a2 : 0.f;
          if (q >= 1 && q <= 8) x0[q - 1] = r == rc ? a0 : 0.f;
        }
      }
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        // k = -1 -> row t+1 (x[u+2]), k = +1 -> row t-1 (x[u])
        float v = c0 * x0[u];
        v = fmaf(c1m, x1[u + 2], v);
        v = fmaf(c1p, x1[u], v);
        v = fmaf(c2m, x2[u + 2], v);
        v = fmaf(c2z, x2[u + 1], v);
        v = fmaf(c2p, x2[u], v);
        bt[u] = dyn ? v : (valid ? x0[u] : 0.f);
      }
    } else {
#pragma unroll
      for (int u = 0; u < 8; ++u) bt[u] = 0.f;
#pragma unroll
      for (int w = 0; w < GANTTS_MAX_WINDOWS; ++w) {
        if (w >= taps.nw) continue;
        float xr[12];
        const float* wp = colp + w * sd + (int64_t)r0 * in_ts;
#pragma unroll
        for (int q = 0; q < 12; ++q) {
          const int r = r0 + q;
          xr[q] = (valid && (dyn || w == 0) && r >= 0 && r < T) ? __ldg(wp + (int64_t)q * in_ts) : 0.f;
        }
#pragma unroll
        for (int k = -2; k <= 2; ++k) {
          const float c = dyn ? taps.c[w][k + 2] : ((w == 0 && k == 0) ? 1.f : 0.f);
#pragma unroll
          for (int u = 0; u < 8; ++u) bt[u] = fmaf(c, xr[u + 2 - k], bt[u]);      // mu_w[t - k]
        }
      }
    }
#pragma unroll
    for (int u = 0; u < 8; ++u)
      if (i0 + u < n) zs[(i0 + u) * 32 + lane] = bt[u];
  }
  __syncwarp();
  // (2) forward substitution
  strip_forward(zs, cf, lane, n, dyn);
  // (3) backward substitution: warm-up rows [t1, e) silently, then [t0, t1) straight to the output
  float y1 = 0.f, y2 = 0.f;
#pragma unroll 4
  for (int i = n - 1; i >= t1 - s; --i) {
    const float4 c = cb[i];
    const float y = (zs[i * 32 + lane] - c.y * y1 - c.z * y2) * c.x;
    y2 = y1;
    y1 = y;
  }
  float* outp = out + (int64_t)it.b * out_bs + (valid ? oc : 0) + (int64_t)(t1 - 1) * out_ts;
#pragma unroll 4
  for (int i = t1 - s - 1; i >= t0 - s; --i) {
    const float4 c = cb[i];
    const float zt = zs[i * 32 + lane];
    float y = (zt - c.y * y1 - c.z * y2) * c.x;
    if (!dyn) y = zt;
    y2 = y1;
    y1 = y;
    if (HW) {
      if (valid) {
        const int64_t r = (int64_t)it.b * T + s + i;
        hw.gx[r * hw.S + oc] = y;
        *outp = highway_out(hw, r, oc, y);
      }
    } else if (valid) {
      *outp = y;
    }
    outp -= out_ts;
  }
}

// Adjoint: z = P^-1 g (same two sweeps on the upstream gradient), gi_w[t] = sum_k coef_w[k+l] z_{t+k}.
// HW: highway backward (HighwayArgs): the strip is loaded as Tx * g, and the chunk's own frames [t0, t1) emit dz.
template <bool STD3, bool HW>
__global__ void __launch_bounds__(32 * SOLVE_WARPS, 4)
mlpg_solve_bwd_kernel(const float* __restrict__ go, int64_t go_bs, int go_ts, float* __restrict__ gi, int64_t gi_bs,
                      int gi_ts, const float* __restrict__ table, gantts_streams_t st, SolveTaps taps, int B, int T, int ncols,
                      int ncg, int bpc, int accumulate, __nv_bfloat16* __restrict__ phi, __nv_bfloat16* __restrict__ plo,
                      int ppitch, HighwayArgs hw) {
  pdl_entry();
  extern __shared__ __align__(16) float smem[];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const SolveItem it = solve_item(B, ncg, bpc);
  float4* cf = reinterpret_cast<float4*>(smem);
  float4* cb = cf + SOLVE_ZROWS;
  float* zs = smem + SOLVE_ZROWS * 8 + (size_t)wib * SOLVE_ZROWS * 32;
  const int t0 = it.chunk * SC;
  const int t1 = t0 + SC < T ? t0 + SC : T;                 // gradient rows [t0, t1) are produced here
  const int lo = t0 - 2 > 0 ? t0 - 2 : 0;                   // z is needed on [t0-2, t1+2)
  const int hi = t1 + 2 < T ? t1 + 2 : T;
  const int s = lo - SW > 0 ? lo - SW : 0;
  const int e = hi + SW < T ? hi + SW : T;
  const int n = e - s;                                      // <= SC + 4 + 2 SW
  strip_coefs(cf, cb, table, s, n);
  if (!it.active) return;
  const int oc = it.cg * 32 + lane;
  ColInfo ci = find_col(st, oc);
  const bool valid = ci.in_col >= 0 && oc < ncols;
  const bool dyn = valid && ci.dyn;
  // (1) the strip of the upstream gradient
  if (HW) {
    const float* gop = go + (int64_t)it.b * go_bs + (valid ? oc : 0) + (int64_t)s * go_ts;
    const int64_t r0 = (int64_t)it.b * T + s;
    const float* txp = hw.tx + r0 * hw.S + (valid ? oc : 0);
#pragma unroll 8
    for (int i = 0; i < n; ++i) {
      float gv = 0.f;
      if (valid) {
        gv = __ldg(gop);
        if (s + i >= t0 && s + i < t1) highway_dz(hw, r0 + i, oc, gv);
        gv = __fmul_rn(gv, __ldg(txp));
      }
      zs[i * 32 + lane] = gv;
      gop += go_ts;
      txp += hw.S;
    }
  } else {
    const float* gop = go + (int64_t)it.b * go_bs + (valid ? oc : 0) + (int64_t)s * go_ts;
#pragma unroll 8
    for (int i = 0; i < n; ++i) {
      zs[i * 32 + lane] = valid ? __ldg(gop) : 0.f;
      gop += go_ts;
    }
  }
  __syncwarp();
  // (2) forward, (3) backward substitution in place
  strip_forward(zs, cf, lane, n, dyn);
  {
    float y1 = 0.f, y2 = 0.f;
#pragma unroll 4
    for (int i = n - 1; i >= lo - s; --i) {
      const float4 c = cb[i];
      const float zt = zs[i * 32 + lane];
      float y = (zt - c.y * y1 - c.z * y2) * c.x;
      if (!dyn) y = zt;
      y2 = y1;
      y1 = y;
      zs[i * 32 + lane] = y;
    }
  }
  __syncwarp();
  // (4) gi_w[t] = sum_k coef_w[k+l] z_{t+k} on [t0, t1): z outside [0, T) is zero
  if (!valid) return;
  if (STD3) {
    const float c0 = dyn ? taps.c[0][2] : 1.f;
    const float c1m = taps.c[1][1], c1p = taps.c[1][3];
    const float c2m = taps.c[2][1], c2z = taps.c[2][2], c2p = taps.c[2][3];
    const int sd = dyn ? ci.sd : 0;
    float zm = t0 - 1 >= 0 ? zs[(t0 - 1 - s) * 32 + lane] : 0.f;
    float zc = zs[(t0 - s) * 32 + lane];
    // planes output (phi != null): the gradient goes out as the bf16 hi/lo operand planes of the next GEMM, rows = b*T + t
    int64_t po = ((int64_t)it.b * T + t0) * ppitch + ci.in_col;
    float* gp = gi ? gi + (int64_t)it.b * gi_bs + ci.in_col + (int64_t)t0 * gi_ts : nullptr;
#pragma unroll 2
    for (int t = t0; t < t1; ++t) {
      const float zp = t + 1 < T ? zs[(t + 1 - s) * 32 + lane] : 0.f;
      // coefficient index k + 2 multiplies z_{t + k}
      const float v0 = c0 * zc;
      const float v1 = fmaf(c1p, zp, c1m * zm);
      const float v2 = fmaf(c2p, zp, fmaf(c2z, zc, c2m * zm));
      if (phi) {
        const __nv_bfloat16 h0 = __float2bfloat16_rn(v0);
        phi[po] = h0;
        plo[po] = __float2bfloat16_rn(v0 - __bfloat162float(h0));
        if (dyn) {
          const __nv_bfloat16 h1 = __float2bfloat16_rn(v1), h2 = __float2bfloat16_rn(v2);
          phi[po + sd] = h1;
          plo[po + sd] = __float2bfloat16_rn(v1 - __bfloat162float(h1));
          phi[po + 2 * sd] = h2;
          plo[po + 2 * sd] = __float2bfloat16_rn(v2 - __bfloat162float(h2));
        }
        po += ppitch;
      } else {
        gp[0] = accumulate ? gp[0] + v0 : v0;
        if (dyn) {
          gp[sd] = accumulate ? gp[sd] + v1 : v1;
          gp[2 * sd] = accumulate ? gp[2 * sd] + v2 : v2;
        }
        gp += gi_ts;
      }
      zm = zc;
      zc = zp;
    }
    return;
  }
  float* gib = gi ? gi + (int64_t)it.b * gi_bs + ci.in_col : nullptr;
#pragma unroll 2
  for (int t = t0; t < t1; ++t) {
    float zw[5];
#pragma unroll
    for (int k = -2; k <= 2; ++k) {
      const int tt = t + k;
      zw[k + 2] = (tt >= 0 && tt < T) ? zs[(tt - s) * 32 + lane] : 0.f;
    }
    const int64_t prow_p = ((int64_t)it.b * T + t) * ppitch + ci.in_col;
    float* prow = gib + (int64_t)t * gi_ts;
    if (!dyn) {
      if (phi) {
        const __nv_bfloat16 h = __float2bfloat16_rn(zw[2]);
        phi[prow_p] = h;
        plo[prow_p] = __float2bfloat16_rn(zw[2] - __bfloat162float(h));
      } else {
        prow[0] = accumulate ? prow[0] + zw[2] : zw[2];
      }
    } else {
#pragma unroll
      for (int w = 0; w < GANTTS_MAX_WINDOWS; ++w) {
        if (w < taps.nw) {
          float v = 0.f;
#pragma unroll
          for (int k = -2; k <= 2; ++k) v = fmaf(taps.c[w][k + 2], zw[2 + k], v);       // z_{t + k}
          if (phi) {
            const __nv_bfloat16 h = __float2bfloat16_rn(v);
            phi[prow_p + w * ci.sd] = h;
            plo[prow_p + w * ci.sd] = __float2bfloat16_rn(v - __bfloat162float(h));
          } else {
            float* q = prow + w * ci.sd;
            *q = accumulate ? *q + v : v;
          }
        }
      }
    }
  }
}

struct SolveGrid {
  int ncg, bpc;
  unsigned blocks;
  size_t smem;
};
static SolveGrid solve_grid(int B, int T, int ncols) {
  SolveGrid g;
  g.ncg = (ncols + 31) / 32;
  g.bpc = (B * g.ncg + SOLVE_WARPS - 1) / SOLVE_WARPS;
  g.blocks = (unsigned)(((T + SC - 1) / SC) * g.bpc);
  g.smem = (size_t)SOLVE_SMEM_FLOATS * sizeof(float);
  return g;
}

// True when the windows admit the substitution kernels: half bandwidth l + u <= 2 for every window, so that the Cholesky
// factor has the two sub-diagonals the table holds.  Wider windows take the FIR kernels.
static bool solve_taps(const gantts_windows_t* win, SolveTaps* tp) {
  int hb = 0;
  tp->nw = win->n;
  for (int w = 0; w < GANTTS_MAX_WINDOWS; ++w)
    for (int q = 0; q < 5; ++q) tp->c[w][q] = 0.f;
  for (int w = 0; w < win->n; ++w) {
    if (win->l[w] > 2 || win->u[w] > 2) return false;
    hb = win->l[w] + win->u[w] > hb ? win->l[w] + win->u[w] : hb;
    for (int k = -win->l[w]; k <= win->u[w]; ++k) tp->c[w][k + 2] = win->coef[w][k + win->l[w]];
  }
  // the sparsity pattern of the reference's windows (hparams.py: [1], [-0.5, 0, 0.5], [1, -2, 1]); any coefficients
  bool std3 = win->n == 3;
  for (int w = 0; w < 3 && std3; ++w) {
    std3 = tp->c[w][0] == 0.f && tp->c[w][4] == 0.f;
    if (w == 0) std3 = std3 && tp->c[0][1] == 0.f && tp->c[0][3] == 0.f;
    if (w == 1) std3 = std3 && tp->c[1][2] == 0.f;
  }
  tp->std3 = std3 ? 1 : 0;
  return hb <= 2;
}

static bool fits_i32(int64_t v) { return v >= 0 && v < ((int64_t)1 << 31); }

// mlpg_solve_{fwd,bwd}_kernel<STD3, HW> for the windows' sparsity pattern and the highway combine
template <bool BWD>
static auto solve_kernel(bool std3, bool hw) {
  if constexpr (BWD)
    return hw ? (std3 ? mlpg_solve_bwd_kernel<true, true> : mlpg_solve_bwd_kernel<false, true>)
              : (std3 ? mlpg_solve_bwd_kernel<true, false> : mlpg_solve_bwd_kernel<false, false>);
  else
    return hw ? (std3 ? mlpg_solve_fwd_kernel<true, true> : mlpg_solve_fwd_kernel<false, true>)
              : (std3 ? mlpg_solve_fwd_kernel<true, false> : mlpg_solve_fwd_kernel<false, false>);
}

// Algorithmic bytes of one MLPG pass, either direction: every input column read and every output column written once.
static double mlpg_bytes(const gantts_streams_t* st, const gantts_windows_t* win, int B, int T, int ncols) {
  int in_cols = 0;
  for (int s = 0; s < st->n; ++s) in_cols += st->sd[s] * (st->dyn[s] ? win->n : 1);
  return 4.0 * (double)B * T * (in_cols + ncols);
}

// One substitution-kernel launch: the forward (src = in, dst = out) or, with BWD, the adjoint (src = go, dst = gi; `tail`
// is the adjoint kernel's accumulate flag and output planes).  Returns GANTTS_E_UNSUPPORTED, having launched nothing,
// when the windows are wider than solve_taps admits or a row offset does not fit in int32: those shapes take the FIR
// kernels.
template <bool BWD, typename... Tail>
static int launch_solve(const float* src, int64_t src_bs, int64_t src_ts, float* dst, int64_t dst_bs, int64_t dst_ts,
                        const float* table, const gantts_streams_t* st, const gantts_windows_t* win, int B, int T,
                        int ncols, void* stream, const HighwayArgs* hw, Tail... tail) {
  SolveTaps tp;
  if (!solve_taps(win, &tp) || !fits_i32((int64_t)T * src_ts) || !fits_i32((int64_t)T * dst_ts))
    return GANTTS_E_UNSUPPORTED;
  const SolveGrid g = solve_grid(B, T, ncols);
  const auto fn = solve_kernel<BWD>(tp.std3, hw != nullptr);
  GANTTS_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)g.smem));
  // 50 KB per block: the full shared-memory carve-out lets 4 blocks (16 warps) share an SM
  GANTTS_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
  const cudaStream_t cs = as_stream(stream);
  prof_begin(BWD ? PROF_MLPG_BWD : PROF_MLPG_FWD, mlpg_bytes(st, win, B, T, ncols), cs);
  GANTTS_PDL_LAUNCH((fn), g.blocks, 32 * SOLVE_WARPS, g.smem, cs, src, src_bs, (int)src_ts, dst, dst_bs, (int)dst_ts,
                    table, *st, tp, B, T, ncols, g.ncg, g.bpc, tail..., hw ? *hw : HighwayArgs{});
  prof_end(cs);
  GANTTS_LAUNCH_CHECK("mlpg_solve_{fwd,bwd}_kernel");
  return GANTTS_OK;
}

static int check_layout(const gantts_streams_t* st, const gantts_windows_t* win, int* ncols) {
  GANTTS_CHECK_ARG(st && win, "mlpg: null stream/window table");
  GANTTS_CHECK_ARG(st->n >= 1 && st->n <= GANTTS_MAX_STREAMS, "mlpg: bad stream count %d", st->n);
  GANTTS_CHECK_ARG(win->n >= 1 && win->n <= GANTTS_MAX_WINDOWS, "mlpg: bad window count %d", win->n);
  int nc = 0;
  for (int s = 0; s < st->n; ++s) {
    GANTTS_CHECK_ARG(st->sd[s] > 0 && st->in_start[s] >= 0 && st->out_start[s] >= 0,
                     "mlpg: bad stream %d", s);
    nc = st->out_start[s] + st->sd[s] > nc ? st->out_start[s] + st->sd[s] : nc;
  }
  for (int w = 0; w < win->n; ++w)
    GANTTS_CHECK_ARG(win->l[w] >= 0 && win->l[w] <= HALO && win->u[w] >= 0 && win->u[w] <= HALO,
                     "mlpg: window %d taps out of range (l,u <= %d)", w, HALO);
  *ncols = nc;
  return GANTTS_OK;
}

}  // namespace gantts

using namespace gantts;

extern "C" int gantts_mlpg_table(const gantts_windows_t* win, int T, float* table_host) {
  GANTTS_CHECK_ARG(win && table_host && T >= 1, "mlpg_table: bad arguments");
  GANTTS_CHECK_ARG(win->n >= 1 && win->n <= GANTTS_MAX_WINDOWS, "mlpg_table: bad window count");
  int hb = 0;
  for (int w = 0; w < win->n; ++w) {
    GANTTS_CHECK_ARG(win->l[w] >= 0 && win->l[w] <= HALO && win->u[w] >= 0 && win->u[w] <= HALO,
                     "mlpg_table: window %d taps out of range", w);
    hb = win->l[w] + win->u[w] > hb ? win->l[w] + win->u[w] : hb;
  }
  // Lower band of P = sum_w W_w^T W_w:  band[d][j] = P[j+d][j], d = 0..hb.
  std::vector<double> band((size_t)(hb + 1) * T, 0.0);
  for (int w = 0; w < win->n; ++w) {
    const int l = win->l[w], u = win->u[w];
    for (int r = 0; r < T; ++r)
      for (int k1 = -l; k1 <= u; ++k1)
        for (int k2 = -l; k2 <= k1; ++k2) {          // column j = r+k2 <= i = r+k1
          int i = r + k1, j = r + k2;
          if (i < 0 || i >= T || j < 0 || j >= T) continue;
          band[(size_t)(i - j) * T + j] += (double)win->coef[w][k1 + l] * (double)win->coef[w][k2 + l];
        }
  }
  // Banded Cholesky P = L L^T, L stored in the same band layout.
  std::vector<double>& L = band;
  for (int j = 0; j < T; ++j) {
    double d = L[j];
    for (int k = 1; k <= hb && j - k >= 0; ++k) {
      double v = L[(size_t)k * T + (j - k)];
      d -= v * v;
    }
    if (!(d > 0.0)) {
      set_error("mlpg_table: normal matrix not positive definite at row %d", j);
      return GANTTS_E_UNSUPPORTED;
    }
    d = sqrt(d);
    L[j] = d;
    for (int i = j + 1; i <= j + hb && i < T; ++i) {
      double s = L[(size_t)(i - j) * T + j];
      for (int k = 1; k <= hb; ++k) {
        int c = j - k;
        if (c < 0 || i - c > hb) continue;
        s -= L[(size_t)(i - c) * T + c] * L[(size_t)(j - c) * T + c];
      }
      L[(size_t)(i - j) * T + j] = s / d;
    }
  }
  // Cholesky rows for the substitution kernels (half bandwidth <= 2): forward  z_i = (b_i - f1 z_{i-1} - f2 z_{i-2}) invd,
  // backward  y_i = (z_i - b1 y_{i+1} - b2 y_{i+2}) invd  with f1 = L[i][i-1], f2 = L[i][i-2], b1 = L[i+1][i], b2 = L[i+2][i]
  for (int t = 0; t < T; ++t) {
    float* row = table_host + (size_t)t * TABW;
    for (int j = NTAPS; j < TABW; ++j) row[j] = 0.f;
    auto Lat = [&](int i, int j) -> double {      // L[i][j], i >= j
      const int d = i - j;
      return (i < T && j >= 0 && d >= 0 && d <= hb) ? L[(size_t)d * T + j] : 0.0;
    };
    row[52] = (float)(1.0 / Lat(t, t));
    row[53] = (float)Lat(t, t - 1);
    row[54] = (float)Lat(t, t - 2);
    row[56] = (float)Lat(t + 1, t);
    row[57] = (float)Lat(t + 2, t);
  }
  std::vector<double> x(T);
  double worst_tail = 0.0;
  for (int t = 0; t < T; ++t) {
    // Solve P x = e_t restricted to where x can be non-negligible is not needed: full O(T*hb) solve.
    for (int i = 0; i < T; ++i) x[i] = 0.0;
    x[t] = 1.0;
    for (int i = t; i < T; ++i) {                     // forward substitution (zeros before t)
      double s = x[i];
      for (int k = 1; k <= hb && i - k >= t; ++k) s -= L[(size_t)k * T + (i - k)] * x[i - k];
      x[i] = s / L[i];
    }
    for (int i = T - 1; i >= 0; --i) {                // backward substitution
      double s = x[i];
      for (int k = 1; k <= hb && i + k < T; ++k) s -= L[(size_t)k * T + i] * x[i + k];
      x[i] = s / L[i];
    }
    for (int j = 0; j < NTAPS; ++j) {
      int c = t + j - K_HALF;
      table_host[(size_t)t * TABW + j] = (c >= 0 && c < T) ? (float)x[c] : 0.f;
    }
    double tail = 0.0;
    if (t - K_HALF - 1 >= 0) tail = fabs(x[t - K_HALF - 1]);
    if (t + K_HALF + 1 < T && fabs(x[t + K_HALF + 1]) > tail) tail = fabs(x[t + K_HALF + 1]);
    if (tail / x[t] > worst_tail) worst_tail = tail / x[t];
  }
  if (worst_tail > 1e-8) {
    set_error("mlpg_table: P^-1 decays too slowly for these windows (%.3g at lag %d)", worst_tail,
              K_HALF + 1);
    return GANTTS_E_UNSUPPORTED;
  }
  return GANTTS_OK;
}

// ---------------------------------------------------------------------------- the table built on the device
// gantts_mlpg_table's arithmetic, operation for operation: every product, sum and difference in float64 through the
// _rn intrinsics (no FMA contraction, which the host build does not emit either), IEEE division and square root.  Only
// the parallel structure differs, and no value depends on it.
namespace gantts {

constexpr int TABLE_DEV_THREADS = 256;
constexpr int TABLE_DEV_MAX_WARPS = 32;       // row solves in flight: scratch = warps x 32 x T doubles

// band[d * T + j] = P[j + d][j]: each entry sums its terms in the host's order (window, then frame r ascending: one
// (k1, k2) pair per frame), then thread 0 factors P = L L^T in place, column by column.
__global__ void __launch_bounds__(TABLE_DEV_THREADS)
mlpg_table_factor_kernel(gantts_windows_t win, int T, int hb, double* __restrict__ band) {
  for (int64_t e = threadIdx.x; e < (int64_t)(hb + 1) * T; e += TABLE_DEV_THREADS) {
    const int d = (int)(e / T), j = (int)(e - (int64_t)d * T), i = j + d;
    double acc = 0.0;
    if (i < T) {
      for (int w = 0; w < win.n; ++w) {
        const int l = win.l[w], u = win.u[w];
        const int r0 = i - u > 0 ? i - u : 0, r1 = j + l < T - 1 ? j + l : T - 1;
        for (int r = r0; r <= r1; ++r)
          acc = __dadd_rn(acc, __dmul_rn((double)win.coef[w][i - r + l], (double)win.coef[w][j - r + l]));
      }
    }
    band[e] = acc;
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  double* L = band;
  for (int j = 0; j < T; ++j) {
    double d = L[j];
    for (int k = 1; k <= hb && j - k >= 0; ++k) {
      const double v = L[(int64_t)k * T + (j - k)];
      d = __dsub_rn(d, __dmul_rn(v, v));
    }
    d = __dsqrt_rn(d);          // P not positive definite: NaN (the host builder rejects such windows)
    L[j] = d;
    for (int i = j + 1; i <= j + hb && i < T; ++i) {
      double s = L[(int64_t)(i - j) * T + j];
      for (int k = 1; k <= hb; ++k) {
        const int c = j - k;
        if (c < 0 || i - c > hb) continue;
        s = __dsub_rn(s, __dmul_rn(L[(int64_t)(i - c) * T + c], L[(int64_t)(j - c) * T + c]));
      }
      L[(int64_t)(i - j) * T + j] = __ddiv_rn(s, d);
    }
  }
}

__device__ __forceinline__ double band_at(const double* __restrict__ L, int T, int hb, int i, int j) {   // L[i][j], i >= j
  const int d = i - j;
  return (i < T && j >= 0 && d >= 0 && d <= hb) ? L[(int64_t)d * T + j] : 0.0;
}

// One lane per table row t: x = P^-1 e_t by the host's forward substitution (zeros before t) and backward substitution,
// stopped once the FIR taps of the row are written (x[i] for i < t - K does not feed them).  The 32 lanes of a warp walk
// the same frame i together (a lane whose row starts later contributes its zeros), so the scratch column z[i][lane] of
// the forward values is read and written in whole rows.
__global__ void __launch_bounds__(32 * 4)
mlpg_table_rows_kernel(int T, int hb, const double* __restrict__ L, double* __restrict__ zbuf, int nwarps,
                       float* __restrict__ table) {
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (warp >= nwarps) return;
  double* z = zbuf + (int64_t)warp * T * 32 + lane;
  for (int t0 = warp * 32; t0 < T; t0 += nwarps * 32) {
    const int t = t0 + lane;
    const bool on = t < T;
    if (on) {
      float* row = table + (int64_t)t * TABW;
      for (int j = 0; j < TABW; ++j) row[j] = 0.f;
      row[52] = __double2float_rn(__ddiv_rn(1.0, band_at(L, T, hb, t, t)));
      row[53] = __double2float_rn(band_at(L, T, hb, t, t - 1));
      row[54] = __double2float_rn(band_at(L, T, hb, t, t - 2));
      row[56] = __double2float_rn(band_at(L, T, hb, t + 1, t));
      row[57] = __double2float_rn(band_at(L, T, hb, t + 2, t));
    }
    double p[GANTTS_MAX_WINDOW_TAPS] = {0.0, 0.0, 0.0, 0.0, 0.0};   // p[k - 1] = x[i - k] (forward) / x[i + k] (backward)
    for (int i = t0; i < T; ++i) {
      double x = 0.0;
      if (i >= t) {
        double s = i == t ? 1.0 : 0.0;
#pragma unroll
        for (int k = 1; k < GANTTS_MAX_WINDOW_TAPS; ++k)
          if (k <= hb && i - k >= t) s = __dsub_rn(s, __dmul_rn(L[(int64_t)k * T + (i - k)], p[k - 1]));
        x = __ddiv_rn(s, L[i]);
      }
#pragma unroll
      for (int k = GANTTS_MAX_WINDOW_TAPS - 1; k > 0; --k) p[k] = p[k - 1];
      p[0] = x;
      z[(int64_t)i * 32] = x;
    }
#pragma unroll
    for (int k = 0; k < GANTTS_MAX_WINDOW_TAPS; ++k) p[k] = 0.0;
    const int stop = t0 - K_HALF > 0 ? t0 - K_HALF : 0;
    for (int i = T - 1; i >= stop; --i) {
      double s = i >= t0 ? z[(int64_t)i * 32] : 0.0;      // x[i] = 0 before the row's start
#pragma unroll
      for (int k = 1; k < GANTTS_MAX_WINDOW_TAPS; ++k)
        if (k <= hb && i + k < T) s = __dsub_rn(s, __dmul_rn(L[(int64_t)k * T + i], p[k - 1]));
      const double x = __ddiv_rn(s, L[i]);
#pragma unroll
      for (int k = GANTTS_MAX_WINDOW_TAPS - 1; k > 0; --k) p[k] = p[k - 1];
      p[0] = x;
      const int j = i - t + K_HALF;
      if (on && j >= 0 && j < NTAPS) table[(int64_t)t * TABW + j] = __double2float_rn(x);
    }
  }
}

}  // namespace gantts

extern "C" int gantts_mlpg_table_device(const gantts_windows_t* win, int T, float* table_dev, void* stream) {
  GANTTS_CHECK_ARG(win && table_dev && T >= 1, "mlpg_table_device: bad arguments");
  GANTTS_CHECK_ARG(win->n >= 1 && win->n <= GANTTS_MAX_WINDOWS, "mlpg_table_device: bad window count");
  int hb = 0;
  for (int w = 0; w < win->n; ++w) {
    GANTTS_CHECK_ARG(win->l[w] >= 0 && win->l[w] <= HALO && win->u[w] >= 0 && win->u[w] <= HALO,
                     "mlpg_table_device: window %d taps out of range", w);
    hb = win->l[w] + win->u[w] > hb ? win->l[w] + win->u[w] : hb;
  }
  static_assert(2 * HALO < GANTTS_MAX_WINDOW_TAPS, "the row solves keep hb <= 2 HALO previous values");
  const cudaStream_t st = as_stream(stream);
  const int groups = (T + 31) / 32, warps = groups < TABLE_DEV_MAX_WARPS ? groups : TABLE_DEV_MAX_WARPS;
  const size_t band_bytes = (size_t)(hb + 1) * T * sizeof(double), z_bytes = (size_t)warps * 32 * T * sizeof(double);
  void* scratch = nullptr;
  GANTTS_CUDA(cudaMallocAsync(&scratch, band_bytes + z_bytes, st));
  double* band = static_cast<double*>(scratch);
  mlpg_table_factor_kernel<<<1, TABLE_DEV_THREADS, 0, st>>>(*win, T, hb, band);
  GANTTS_LAUNCH_CHECK("mlpg_table_factor_kernel");
  mlpg_table_rows_kernel<<<(warps + 3) / 4, 32 * 4, 0, st>>>(T, hb, band, band + (size_t)(hb + 1) * T, warps, table_dev);
  GANTTS_LAUNCH_CHECK("mlpg_table_rows_kernel");
  GANTTS_CUDA(cudaFreeAsync(scratch, st));
  return GANTTS_OK;
}

namespace gantts {
static int check_highway(const HighwayArgs* hw, int ncols, int64_t bs, int64_t ts, int T) {
  if (!hw) return GANTTS_OK;
  GANTTS_CHECK_ARG(hw->x && hw->tx && hw->gx && hw->dz_hi && hw->dz_lo && hw->S == ncols && ts == hw->S &&
                       bs == (int64_t)T * hw->S,
                   "mlpg: highway combine needs contiguous [B][T][S] static features, S = %d", ncols);
  return GANTTS_OK;
}

static inline int elementwise_blocks(int64_t n) {
  int64_t b = (n + 255) / 256;
  if (b > 132 * 8) b = 132 * 8;
  return (int)(b < 1 ? 1 : b);
}

// hw != null: the In2OutHighwayNet combine, `out` receives y_hat_static and hw->gx the MLPG output.
static int mlpg_fwd_impl(const float* in, int64_t in_bs, int64_t in_ts, float* out, int64_t out_bs, int64_t out_ts,
                         const float* table_dev, const gantts_streams_t* st, const gantts_windows_t* win, int B, int T,
                         void* stream, const HighwayArgs* hw);
}  // namespace gantts

extern "C" int gantts_mlpg_fwd(const float* in, int64_t in_bs, int64_t in_ts, float* out,
                               int64_t out_bs, int64_t out_ts, const float* table_dev,
                               const gantts_streams_t* st, const gantts_windows_t* win, int B, int T,
                               void* stream) {
  return mlpg_fwd_impl(in, in_bs, in_ts, out, out_bs, out_ts, table_dev, st, win, B, T, stream, nullptr);
}

static int gantts::mlpg_fwd_impl(const float* in, int64_t in_bs, int64_t in_ts, float* out, int64_t out_bs,
                                 int64_t out_ts, const float* table_dev, const gantts_streams_t* st,
                                 const gantts_windows_t* win, int B, int T, void* stream, const HighwayArgs* hw) {
  int ncols = 0;
  int rc = check_layout(st, win, &ncols);
  if (rc) return rc;
  GANTTS_CHECK_ARG(in && out && table_dev && B >= 1 && T >= 1, "mlpg_fwd: bad arguments");
  if ((rc = check_highway(hw, ncols, out_bs, out_ts, T))) return rc;
  rc = launch_solve<false>(in, in_bs, in_ts, out, out_bs, out_ts, table_dev, st, win, B, T, ncols, stream, hw);
  if (rc != GANTTS_E_UNSUPPORTED) return rc;
  if (hw) {
    // FIR family: MLPG into Gx, then the combine as one elementwise pass
    if ((rc = mlpg_fwd_impl(in, in_bs, in_ts, hw->gx, (int64_t)T * hw->S, hw->S, table_dev, st, win, B, T, stream,
                            nullptr)))
      return rc;
    const int64_t rows = (int64_t)B * T;
    GANTTS_PDL_LAUNCH((highway_combine_kernel), elementwise_blocks(rows * hw->S), 256, 0, as_stream(stream), *hw, out, rows);
    GANTTS_LAUNCH_CHECK("highway_combine_kernel");
    return GANTTS_OK;
  }
  const size_t smem = ((TT + 2 * K_HALF) * TC + TT * GROW) * sizeof(float);
  static bool attr_done_dev[64] = {};
  int dev_id = -1;
  cudaGetDevice(&dev_id);
  const bool attr_done = dev_id >= 0 && dev_id < 64 && attr_done_dev[dev_id];
  if (!attr_done) {
    if (dev_id >= 0 && dev_id < 64) attr_done_dev[dev_id] = true;
    GANTTS_CUDA(cudaFuncSetAttribute(mlpg_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
    // 42 KB per block: with the full shared-memory carve-out 5 blocks fit per SM and the 512 blocks of a
    // cfg2 launch are resident in one wave (the default carve-out admitted 3)
    GANTTS_CUDA(cudaFuncSetAttribute(mlpg_fwd_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
  }
  dim3 grid((ncols + TC - 1) / TC, (T + TT - 1) / TT, B);
  prof_begin(PROF_MLPG_FWD, mlpg_bytes(st, win, B, T, ncols), as_stream(stream));
  mlpg_fwd_kernel<<<grid, MLPG_THREADS, smem, as_stream(stream)>>>(in, in_bs, in_ts, out, out_bs, out_ts,
                                                                  table_dev, *st, *win, T, ncols);
  prof_end(as_stream(stream));
  GANTTS_LAUNCH_CHECK("mlpg_fwd_kernel");
  return GANTTS_OK;
}

// MLPG backward whose result leaves as bf16 hi/lo operand planes [B*T][pitch] (fused step: the gradient w.r.t. y_hat
// is consumed by the generator's backward GEMMs only).  Returns GANTTS_E_UNSUPPORTED when the substitution kernel does
// not apply (the caller then takes the fp32 route).
// hw != null (both functions): the In2OutHighwayNet backward, go = dL/dy_hat_static; dz goes to hw's planes.
namespace gantts {
static int mlpg_bwd_planes(const float* go, int64_t go_bs, int64_t go_ts, __nv_bfloat16* phi, __nv_bfloat16* plo,
                           int64_t ppitch, const float* table_dev, const gantts_streams_t* st, const gantts_windows_t* win,
                           int B, int T, void* stream, const HighwayArgs* hw = nullptr) {
  int ncols = 0;
  int rc = check_layout(st, win, &ncols);
  if (rc) return rc;
  if ((rc = check_highway(hw, ncols, go_bs, go_ts, T))) return rc;
  if (!fits_i32((int64_t)B * T * ppitch)) return GANTTS_E_UNSUPPORTED;
  return launch_solve<true>(go, go_bs, go_ts, nullptr, 0, 0, table_dev, st, win, B, T, ncols, stream, hw, 0, phi, plo,
                            (int)ppitch);
}

// With hw and the FIR family, go is scaled by Tx in place before the unchanged adjoint runs on it.
static int mlpg_bwd_impl(const float* go, int64_t go_bs, int64_t go_ts, float* gi, int64_t gi_bs, int64_t gi_ts,
                         const float* table_dev, const gantts_streams_t* st, const gantts_windows_t* win, int B, int T,
                         int accumulate, void* stream, const HighwayArgs* hw);
}  // namespace gantts

extern "C" int gantts_mlpg_bwd(const float* go, int64_t go_bs, int64_t go_ts, float* gi,
                               int64_t gi_bs, int64_t gi_ts, const float* table_dev,
                               const gantts_streams_t* st, const gantts_windows_t* win, int B, int T,
                               int accumulate, void* stream) {
  return mlpg_bwd_impl(go, go_bs, go_ts, gi, gi_bs, gi_ts, table_dev, st, win, B, T, accumulate, stream, nullptr);
}

static int gantts::mlpg_bwd_impl(const float* go, int64_t go_bs, int64_t go_ts, float* gi, int64_t gi_bs, int64_t gi_ts,
                                 const float* table_dev, const gantts_streams_t* st, const gantts_windows_t* win, int B,
                                 int T, int accumulate, void* stream, const HighwayArgs* hw) {
  int ncols = 0;
  int rc = check_layout(st, win, &ncols);
  if (rc) return rc;
  GANTTS_CHECK_ARG(go && gi && table_dev && B >= 1 && T >= 1, "mlpg_bwd: bad arguments");
  if ((rc = check_highway(hw, ncols, go_bs, go_ts, T))) return rc;
  rc = launch_solve<true>(go, go_bs, go_ts, gi, gi_bs, gi_ts, table_dev, st, win, B, T, ncols, stream, hw, accumulate,
                          nullptr, nullptr, 0);
  if (rc != GANTTS_E_UNSUPPORTED) return rc;
  if (hw) {
    const int64_t rows = (int64_t)B * T;
    GANTTS_PDL_LAUNCH((highway_bwd_prep_kernel), elementwise_blocks(rows * hw->S), 256, 0, as_stream(stream), *hw,
                      const_cast<float*>(go), rows);
    GANTTS_LAUNCH_CHECK("highway_bwd_prep_kernel");
  }
  const size_t smem = (GIN_ROWS * TC + 72 * GROW + 72 * TC) * sizeof(float);
  static bool attr_done_dev[64] = {};
  int dev_id = -1;
  cudaGetDevice(&dev_id);
  const bool attr_done = dev_id >= 0 && dev_id < 64 && attr_done_dev[dev_id];
  if (!attr_done) {
    if (dev_id >= 0 && dev_id < 64) attr_done_dev[dev_id] = true;
    GANTTS_CUDA(cudaFuncSetAttribute(mlpg_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
    GANTTS_CUDA(cudaFuncSetAttribute(mlpg_bwd_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
  }
  dim3 grid((ncols + TC - 1) / TC, (T + TT - 1) / TT, B);
  prof_begin(PROF_MLPG_BWD, mlpg_bytes(st, win, B, T, ncols), as_stream(stream));
  mlpg_bwd_kernel<<<grid, MLPG_THREADS, smem, as_stream(stream)>>>(go, go_bs, go_ts, gi, gi_bs, gi_ts,
                                                                  table_dev, *st, *win, T, ncols, accumulate);
  prof_end(as_stream(stream));
  GANTTS_LAUNCH_CHECK("mlpg_bwd_kernel");
  return GANTTS_OK;
}
