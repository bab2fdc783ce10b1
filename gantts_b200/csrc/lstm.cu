// Persistent LSTM recurrence (include/gantts_b200.h: gantts_lstm_layer_fwd / _bwd).
//
// Replaces the cuDNN/ATen LSTM behind nn.LSTM in reference gantts/models.py:84-85,175-176,198-199
// (In2OutRNNHighwayNet, GRURNN -- which is an nn.LSTM --, LSTMRNN) with packed-sequence semantics
// (pack_padded_sequence / pad_packed_sequence, models.py:101-112,182-187,205-210): sequence b only runs
// for t < lengths[b], outputs beyond are zero, the reverse direction starts at t = lengths[b]-1.
//
// The input projections x W_ih^T + b_ih + b_hh of ALL time steps are one tensor-core GEMM (caller);
// this file holds the sequential part.  One cooperative launch per layer covers every time step and
// both directions: each CTA owns HS hidden units of one direction, keeps its slice of W_hh (4*HS rows)
// in shared memory for the whole sequence, reads h_{t-1} of all units from L2, and the CTAs of one
// direction meet at a grid barrier once per time step.  Recurrent mat-vec products are exact fp32 FFMA.
//   forward  step: pre = W_hh[slice] h_{t-1};  (i,f,o) = sigmoid, g = tanh;  c = f c + i g;  h = o tanh(c)
//   backward step: gate gradients for the own slice -> barrier -> dh_{t-1}[slice] = dgates W_hh[:, slice]
#include "common.cuh"

namespace gantts {

constexpr int LSTM_THREADS = 256;
constexpr int LSTM_BC = 16;       // batch rows per shared-memory chunk
constexpr int LSTM_MAX_B = 128;

struct LstmParams {
  const float* xproj;    // [B][T][ndir*4H]
  const float* W_hh;     // [4H][H] of direction 0; direction d's starts at W_hh + d * W_hh_dir (nn.LSTM keeps the
  int64_t W_hh_dir;      // directions as separate tensors: a stride, not a copy)
  const int64_t* lengths;
  float* h_out;          // [B][T][ndir*H]
  float* gates;          // [ndir][B][T][4H]
  float* cells;          // [ndir][B][T][H]
  const float* dh_out;   // bwd: [B][T][ndir*H]
  float* dxproj;         // bwd: [B][T][ndir*4H]
  unsigned int* bar;     // [ndir][2] {count, generation}
  int B, T, H, ndir, slices;
};

// Barrier among the `n` CTAs of one direction (all co-resident: cooperative launch).  One monotonically
// increasing arrival counter per direction: the k-th barrier completes when it reaches k * n -- no reset,
// no generation word, one atomic + one polling load per CTA and step.
__device__ __forceinline__ void dir_barrier(unsigned int* bar, unsigned int n, unsigned int& gen) {
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int target = (gen + 1) * n;
    __threadfence();
    atomicAdd(bar, 1u);
    const long long t0 = clock64();
    while (*reinterpret_cast<volatile unsigned int*>(bar) < target) {
      if (clock64() - t0 > 8000000000LL) {
        printf("gantts_b200: lstm grid barrier timeout (block %d)\n", blockIdx.x);
        __trap();
      }
    }
    __threadfence();
  }
  gen += 1;
  __syncthreads();
}

__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + expf(-x)); }

template <int HS>
__global__ void __launch_bounds__(LSTM_THREADS, 1) lstm_fwd_kernel(const LstmParams p) {
  constexpr int R = 4 * HS;                       // W_hh rows owned by this CTA
  constexpr int GROUPS = LSTM_THREADS / R;        // thread groups along the batch chunk
  constexpr int BPT = LSTM_BC / GROUPS;           // batch rows per thread
  extern __shared__ __align__(16) float sm[];
  const int H = p.H, HP = H + 4;
  float* Ws = sm;                                  // [R][HP]
  float* hs = Ws + R * HP;                         // [LSTM_BC][H]
  float* pre = hs + LSTM_BC * H;                   // [LSTM_BC][R]
  float* cst = pre + LSTM_BC * R;                  // [LSTM_MAX_B][HS]
  const int dir = blockIdx.x / p.slices, sl = blockIdx.x % p.slices, u0 = sl * HS;
  const int tid = threadIdx.x;
  const int ldx = p.ndir * 4 * H, ldh = p.ndir * H;
  const float* Wd = p.W_hh + (int64_t)dir * p.W_hh_dir;
  for (int i = tid; i < R * H; i += LSTM_THREADS) {
    const int r = i / H, k = i - r * H;
    const int g = r / HS, u = r - g * HS;
    Ws[r * HP + k] = (u0 + u < H) ? Wd[(int64_t)(g * H + u0 + u) * H + k] : 0.f;
  }
  for (int i = tid; i < LSTM_MAX_B * HS; i += LSTM_THREADS) cst[i] = 0.f;
  __syncthreads();
  unsigned int gen = 0;
  unsigned int* bar = p.bar + 2 * dir;
  float* gates_d = p.gates + (int64_t)dir * p.B * p.T * 4 * H;
  float* cells_d = p.cells + (int64_t)dir * p.B * p.T * H;
  const int r = tid % R, bl = tid / R;

  for (int step = 0; step < p.T; ++step) {
    const int t = dir == 0 ? step : p.T - 1 - step;
    const int tprev = dir == 0 ? t - 1 : t + 1;
    for (int cb = 0; cb < p.B; cb += LSTM_BC) {
      // h_{t-1} of all hidden units for this batch chunk (zeros at the first step)
      for (int i = tid; i < LSTM_BC * (H / 4); i += LSTM_THREADS) {
        const int bb = i / (H / 4), k4 = i - bb * (H / 4), b = cb + bb;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (step > 0 && b < p.B)
          v = *reinterpret_cast<const float4*>(p.h_out + ((int64_t)b * p.T + tprev) * ldh + dir * H + 4 * k4);
        reinterpret_cast<float4*>(hs)[bb * (H / 4) + k4] = v;
      }
      __syncthreads();
      // input projections of this step (independent of the recurrence): issue the loads now so that
      // their latency hides under the mat-vec
      float xq[4] = {0.f, 0.f, 0.f, 0.f};
      if (tid < LSTM_BC * HS) {
        const int bb = tid / HS, u = tid - bb * HS, b = cb + bb;
        if (b < p.B && u0 + u < H && (int64_t)t < p.lengths[b]) {
          const float* xp = p.xproj + ((int64_t)b * p.T + t) * ldx + dir * 4 * H + u0 + u;
          xq[0] = xp[0]; xq[1] = xp[H]; xq[2] = xp[2 * H]; xq[3] = xp[3 * H];
        }
      }
      float acc[BPT];
#pragma unroll
      for (int j = 0; j < BPT; ++j) acc[j] = 0.f;
      const float4* w4 = reinterpret_cast<const float4*>(Ws + r * HP);
      for (int k4 = 0; k4 < H / 4; ++k4) {
        const float4 w = w4[k4];
#pragma unroll
        for (int j = 0; j < BPT; ++j) {
          const float4 h = reinterpret_cast<const float4*>(hs + (bl + j * GROUPS) * H)[k4];
          acc[j] = fmaf(w.x, h.x, fmaf(w.y, h.y, fmaf(w.z, h.z, fmaf(w.w, h.w, acc[j]))));
        }
      }
#pragma unroll
      for (int j = 0; j < BPT; ++j) pre[(bl + j * GROUPS) * R + r] = acc[j];
      __syncthreads();
      if (tid < LSTM_BC * HS) {
        const int bb = tid / HS, u = tid - bb * HS, b = cb + bb;
        if (b < p.B && u0 + u < H) {
          const bool valid = (int64_t)t < p.lengths[b];
          const int64_t row = (int64_t)b * p.T + t;
          float hval = 0.f;
          if (valid) {
            const float gi = sigmoidf_(pre[bb * R + 0 * HS + u] + xq[0]);
            const float gf = sigmoidf_(pre[bb * R + 1 * HS + u] + xq[1]);
            const float gg = tanhf(pre[bb * R + 2 * HS + u] + xq[2]);
            const float go = sigmoidf_(pre[bb * R + 3 * HS + u] + xq[3]);
            const float c = gf * cst[b * HS + u] + gi * gg;
            cst[b * HS + u] = c;
            hval = go * tanhf(c);
            float* gp = gates_d + row * 4 * H + u0 + u;
            gp[0] = gi; gp[H] = gf; gp[2 * H] = gg; gp[3 * H] = go;
            cells_d[row * H + u0 + u] = c;
          }
          p.h_out[row * ldh + dir * H + u0 + u] = hval;     // zero beyond the length (pad_packed_sequence)
        }
      }
      __syncthreads();
    }
    if (step + 1 < p.T) dir_barrier(bar, p.slices, gen);
  }
}

template <int HS>
__global__ void __launch_bounds__(LSTM_THREADS, 1) lstm_bwd_kernel(const LstmParams p) {
  constexpr int OUTS = LSTM_BC * HS;                 // (batch row, hidden unit) outputs per chunk
  constexpr int SPLIT = LSTM_THREADS / OUTS;         // threads sharing one output (row ranges)
  extern __shared__ __align__(16) float sm[];
  const int H = p.H, G4 = 4 * H, GP = G4 + 4;
  float* Wt = sm;                                    // [HS][GP]   Wt[k][row] = W_hh[row][u0+k]
  float* dgs = Wt + HS * GP;                         // [LSTM_BC][GP]
  float* red = dgs + LSTM_BC * GP;                   // [SPLIT][OUTS]
  float* dhr = red + SPLIT * OUTS;                   // [LSTM_MAX_B][HS]  dL/dh_t (recurrent part)
  float* dcs = dhr + LSTM_MAX_B * HS;                // [LSTM_MAX_B][HS]  dL/dc_t carried
  const int dir = blockIdx.x / p.slices, sl = blockIdx.x % p.slices, u0 = sl * HS;
  const int tid = threadIdx.x;
  const int ldx = p.ndir * 4 * H, ldh = p.ndir * H;
  const float* Wd = p.W_hh + (int64_t)dir * p.W_hh_dir;
  for (int i = tid; i < HS * G4; i += LSTM_THREADS) {
    const int row = i / HS, k = i - row * HS;
    Wt[k * GP + row] = (u0 + k < H) ? Wd[(int64_t)row * H + u0 + k] : 0.f;
  }
  for (int i = tid; i < LSTM_MAX_B * HS; i += LSTM_THREADS) { dhr[i] = 0.f; dcs[i] = 0.f; }
  __syncthreads();
  unsigned int gen = 0;
  unsigned int* bar = p.bar + 2 * dir;
  const float* gates_d = p.gates + (int64_t)dir * p.B * p.T * 4 * H;
  const float* cells_d = p.cells + (int64_t)dir * p.B * p.T * H;

  for (int step = 0; step < p.T; ++step) {
    const int t = dir == 0 ? p.T - 1 - step : step;  // reverse of the forward recurrence order
    const int tprev = dir == 0 ? t - 1 : t + 1;      // forward-order predecessor (holds c_{prev})
    // phase A: gate gradients of the own hidden units
    for (int i = tid; i < p.B * HS; i += LSTM_THREADS) {
      const int b = i / HS, u = i - b * HS;
      if (u0 + u >= H) continue;
      const int64_t len = p.lengths[b];
      const int64_t row = (int64_t)b * p.T + t;
      float* dxp = p.dxproj + row * ldx + dir * 4 * H + u0 + u;
      float di = 0.f, df = 0.f, dg = 0.f, d_og = 0.f;
      if ((int64_t)t < len) {
        const float* gp = gates_d + row * 4 * H + u0 + u;
        const float gi = gp[0], gf = gp[H], gg = gp[2 * H], go = gp[3 * H];
        const float c = cells_d[row * H + u0 + u];
        const bool first = dir == 0 ? (t == 0) : ((int64_t)t == len - 1);
        const float cprev = first ? 0.f : cells_d[((int64_t)b * p.T + tprev) * H + u0 + u];
        const float dh = p.dh_out[row * ldh + dir * H + u0 + u] + dhr[i];
        const float tc = tanhf(c);
        const float dct = dcs[i] + dh * go * (1.f - tc * tc);
        d_og = dh * tc * go * (1.f - go);
        di = dct * gg * gi * (1.f - gi);
        dg = dct * gi * (1.f - gg * gg);
        df = dct * cprev * gf * (1.f - gf);
        dcs[i] = dct * gf;
      }
      dxp[0] = di; dxp[H] = df; dxp[2 * H] = dg; dxp[3 * H] = d_og;
    }
    if (step + 1 == p.T) break;
    dir_barrier(bar, p.slices, gen);
    // phase B: dh_{prev}[b][own units] = sum_row dgates_t[b][row] * W_hh[row][unit]
    for (int cb = 0; cb < p.B; cb += LSTM_BC) {
      for (int i = tid; i < LSTM_BC * (G4 / 4); i += LSTM_THREADS) {
        const int bb = i / (G4 / 4), r4 = i - bb * (G4 / 4), b = cb + bb;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (b < p.B)
          v = *reinterpret_cast<const float4*>(p.dxproj + ((int64_t)b * p.T + t) * ldx + dir * 4 * H + 4 * r4);
        *reinterpret_cast<float4*>(dgs + bb * GP + 4 * r4) = v;
      }
      __syncthreads();
      const int out = tid % OUTS, part = tid / OUTS;
      const int bb = out / HS, k = out - bb * HS;
      const int rows_per = G4 / SPLIT;
      const float4* w4 = reinterpret_cast<const float4*>(Wt + k * GP + part * rows_per);
      const float4* d4 = reinterpret_cast<const float4*>(dgs + bb * GP + part * rows_per);
      float acc = 0.f;
      for (int i = 0; i < rows_per / 4; ++i) {
        const float4 w = w4[i], d = d4[i];
        acc = fmaf(w.x, d.x, fmaf(w.y, d.y, fmaf(w.z, d.z, fmaf(w.w, d.w, acc))));
      }
      red[part * OUTS + out] = acc;
      __syncthreads();
      if (tid < OUTS) {
        float s = 0.f;
#pragma unroll
        for (int q = 0; q < SPLIT; ++q) s += red[q * OUTS + tid];
        const int b = cb + bb;
        if (b < p.B) dhr[b * HS + k] = s;
      }
      __syncthreads();
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Register-resident variants (HS = 8, H <= 512).  The shared-memory kernels above re-read the CTA's W_hh
// slice from shared memory once per thread group and step (8 x 64 KB per step: ~2 us of shared-memory
// bandwidth).  Here every thread keeps its 64 weights in REGISTERS for the whole sequence:
//   forward : thread (r = tid % 32, kq = tid / 32) owns W_hh[row r][kq*KR .. +KR); per step it forms the
//             partial dot products of all 16 batch rows of the chunk (h_{t-1} from shared memory, one
//             broadcast LDS.128 per 4 FMAs), the 8 k-ranges are summed in the gate stage;
//   backward: thread owns rows {tid + 256 i} of W_hh[:, u0 .. u0+8); per step it accumulates
//             dh_prev[b][k] partials for 8 batch rows x 8 units in registers (scalar conflict-free LDS of
//             the staged gate gradients, 8 FMAs per load), a butterfly reduction over the warp (62
//             shuffles for 64 values) and an 8-way shared-memory sum finish it.
// Both are FMA-bound at ~1 us per step and chunk instead of shared-memory-bound at 2-4 us.
template <int KR>
__global__ void __launch_bounds__(LSTM_THREADS, 1) lstm_fwd_reg_kernel(const LstmParams p) {
  constexpr int HS = 8, R = 32, NKQ = LSTM_THREADS / R;     // 8 k-ranges
  constexpr int HPAD = NKQ * KR;                            // >= H, zero padded
  constexpr int NQ = LSTM_BC * (HPAD / 4) / LSTM_THREADS;   // float4 loads of h_{t-1} per thread and chunk
  extern __shared__ __align__(16) float sm[];
  const int H = p.H;
  float* hs = sm;                                           // [LSTM_BC][HPAD]
  float* part = hs + LSTM_BC * HPAD;                        // [NKQ][LSTM_BC][R]
  float* cst = part + NKQ * LSTM_BC * R;                    // [LSTM_MAX_B][HS]
  const int dir = blockIdx.x / p.slices, sl = blockIdx.x % p.slices, u0 = sl * HS;
  const int tid = threadIdx.x;
  const int ldx = p.ndir * 4 * H, ldh = p.ndir * H;
  const float* Wd = p.W_hh + (int64_t)dir * p.W_hh_dir;
  const int r = tid % R, kq = tid / R;
  float w[KR];
  {
    const int g = r / HS, u = r - g * HS;
    const bool row_ok = u0 + u < H;
    const float* wr = Wd + (int64_t)(g * H + u0 + u) * H;
#pragma unroll
    for (int j = 0; j < KR; ++j) {
      const int k = kq * KR + j;
      w[j] = (row_ok && k < H) ? wr[k] : 0.f;
    }
  }
  for (int i = tid; i < LSTM_MAX_B * HS; i += LSTM_THREADS) cst[i] = 0.f;
  for (int i = tid; i < LSTM_BC * HPAD; i += LSTM_THREADS) hs[i] = 0.f;
  int sofs[NQ];                                             // smem offset bb * HPAD + 4 * k4, -1 if unused
#pragma unroll
  for (int q = 0; q < NQ; ++q) {
    const int i = tid + q * LSTM_THREADS;
    const int bb = i / (H / 4), k4 = i - bb * (H / 4);
    sofs[q] = bb < LSTM_BC ? bb * HPAD + 4 * k4 : -1;
  }
  __syncthreads();
  unsigned int gen = 0;
  unsigned int* bar = p.bar + 2 * dir;
  float* gates_d = p.gates + (int64_t)dir * p.B * p.T * 4 * H;
  float* cells_d = p.cells + (int64_t)dir * p.B * p.T * H;

  for (int step = 0; step < p.T; ++step) {
    const int t = dir == 0 ? step : p.T - 1 - step;
    const int tprev = dir == 0 ? t - 1 : t + 1;
    for (int cb = 0; cb < p.B; cb += LSTM_BC) {
      // all of this thread's h_{t-1} loads are issued before the first store (a load->store loop compiles
      // to one L2 round trip per iteration: 8 serial round trips per step in the ncu source view)
      float4 hv[NQ];
#pragma unroll
      for (int q = 0; q < NQ; ++q) {
        hv[q] = make_float4(0.f, 0.f, 0.f, 0.f);
        const int so = sofs[q];
        if (so >= 0) {
          const int bb = so / HPAD, b = cb + bb;
          if (step > 0 && b < p.B)
            hv[q] = __ldcg(reinterpret_cast<const float4*>(p.h_out + ((int64_t)b * p.T + tprev) * ldh + dir * H +
                                                           (so - bb * HPAD)));
        }
      }
#pragma unroll
      for (int q = 0; q < NQ; ++q)
        if (sofs[q] >= 0) *reinterpret_cast<float4*>(hs + sofs[q]) = hv[q];
      __syncthreads();
      float xq[4] = {0.f, 0.f, 0.f, 0.f};
      if (tid < LSTM_BC * HS) {
        const int bb = tid / HS, u = tid - bb * HS, b = cb + bb;
        if (b < p.B && u0 + u < H && (int64_t)t < p.lengths[b]) {
          const float* xp = p.xproj + ((int64_t)b * p.T + t) * ldx + dir * 4 * H + u0 + u;
          xq[0] = xp[0]; xq[1] = xp[H]; xq[2] = xp[2 * H]; xq[3] = xp[3 * H];
        }
      }
      float acc[LSTM_BC];
#pragma unroll
      for (int b = 0; b < LSTM_BC; ++b) acc[b] = 0.f;
      const float* hk = hs + kq * KR;
#pragma unroll
      for (int j4 = 0; j4 < KR / 4; ++j4) {
#pragma unroll
        for (int b = 0; b < LSTM_BC; ++b) {
          const float4 h = *reinterpret_cast<const float4*>(hk + b * HPAD + 4 * j4);
          acc[b] = fmaf(w[4 * j4], h.x, fmaf(w[4 * j4 + 1], h.y, fmaf(w[4 * j4 + 2], h.z, fmaf(w[4 * j4 + 3], h.w, acc[b]))));
        }
      }
#pragma unroll
      for (int b = 0; b < LSTM_BC; ++b) part[(kq * LSTM_BC + b) * R + r] = acc[b];
      __syncthreads();
      if (tid < LSTM_BC * HS) {
        const int bb = tid / HS, u = tid - bb * HS, b = cb + bb;
        if (b < p.B && u0 + u < H) {
          const bool valid = (int64_t)t < p.lengths[b];
          const int64_t row = (int64_t)b * p.T + t;
          float hval = 0.f;
          if (valid) {
            float pre[4] = {xq[0], xq[1], xq[2], xq[3]};
#pragma unroll
            for (int q = 0; q < NKQ; ++q) {
#pragma unroll
              for (int g = 0; g < 4; ++g) pre[g] += part[(q * LSTM_BC + bb) * R + g * HS + u];
            }
            const float gi = sigmoidf_(pre[0]);
            const float gf = sigmoidf_(pre[1]);
            const float gg = tanhf(pre[2]);
            const float go = sigmoidf_(pre[3]);
            const float c = gf * cst[b * HS + u] + gi * gg;
            cst[b * HS + u] = c;
            hval = go * tanhf(c);
            float* gp = gates_d + row * 4 * H + u0 + u;
            gp[0] = gi; gp[H] = gf; gp[2 * H] = gg; gp[3 * H] = go;
            cells_d[row * H + u0 + u] = c;
          }
          p.h_out[row * ldh + dir * H + u0 + u] = hval;
        }
      }
      __syncthreads();
    }
    if (step + 1 < p.T) dir_barrier(bar, p.slices, gen);
  }
}

// Sum v[0..63] over the 32 lanes of a warp; afterwards lane L holds the totals of indices
// idx(L) + {0, 1} with idx(L) = 32*b4 + 16*b3 + 8*b2 + 4*b1 + 2*b0 (bN = bit N of L) in v[0], v[1].
__device__ __forceinline__ void warp_reduce64(float (&v)[64], int lane) {
#pragma unroll
  for (int half = 32, bit = 16; half >= 2; half >>= 1, bit >>= 1) {
    const bool upper = (lane & bit) != 0;
#pragma unroll
    for (int i = 0; i < half; ++i) {
      const float send = upper ? v[i] : v[i + half];
      const float keep = upper ? v[i + half] : v[i];
      v[i] = keep + __shfl_xor_sync(0xffffffffu, send, bit);
    }
  }
}

template <int RPT>
__global__ void __launch_bounds__(LSTM_THREADS, 1) lstm_bwd_reg_kernel(const LstmParams p) {
  constexpr int HS = 8, HB = 8;                       // hidden units per CTA, batch rows per register pass
  extern __shared__ __align__(16) float sm[];
  const int H = p.H, G4 = 4 * H;
  constexpr int GPAD = RPT * LSTM_THREADS;            // >= 4H, zero padded
  float* dgs = sm;                                    // [LSTM_BC][GPAD]
  float* red = dgs + LSTM_BC * GPAD;                  // [8 warps][64]
  float* dhr = red + 8 * 64;                          // [LSTM_MAX_B][HS]
  float* dcs = dhr + LSTM_MAX_B * HS;                 // [LSTM_MAX_B][HS]
  const int dir = blockIdx.x / p.slices, sl = blockIdx.x % p.slices, u0 = sl * HS;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int ldx = p.ndir * 4 * H, ldh = p.ndir * H;
  const float* Wd = p.W_hh + (int64_t)dir * p.W_hh_dir;
  float w[RPT][HS];
#pragma unroll
  for (int i = 0; i < RPT; ++i) {
    const int row = i * LSTM_THREADS + tid;
#pragma unroll
    for (int k = 0; k < HS; ++k) w[i][k] = (row < G4 && u0 + k < H) ? Wd[(int64_t)row * H + u0 + k] : 0.f;
  }
  for (int i = tid; i < LSTM_MAX_B * HS; i += LSTM_THREADS) { dhr[i] = 0.f; dcs[i] = 0.f; }
  for (int i = tid; i < LSTM_BC * GPAD; i += LSTM_THREADS) dgs[i] = 0.f;
  __syncthreads();
  unsigned int gen = 0;
  unsigned int* bar = p.bar + 2 * dir;
  const float* gates_d = p.gates + (int64_t)dir * p.B * p.T * 4 * H;
  const float* cells_d = p.cells + (int64_t)dir * p.B * p.T * H;

  for (int step = 0; step < p.T; ++step) {
    const int t = dir == 0 ? p.T - 1 - step : step;
    const int tprev = dir == 0 ? t - 1 : t + 1;
    // phase A: gate gradients of the own hidden units (as in lstm_bwd_kernel)
    for (int i = tid; i < p.B * HS; i += LSTM_THREADS) {
      const int b = i / HS, u = i - b * HS;
      if (u0 + u >= H) continue;
      const int64_t len = p.lengths[b];
      const int64_t row = (int64_t)b * p.T + t;
      float* dxp = p.dxproj + row * ldx + dir * 4 * H + u0 + u;
      float di = 0.f, df = 0.f, dg = 0.f, d_og = 0.f;
      if ((int64_t)t < len) {
        const float* gp = gates_d + row * 4 * H + u0 + u;
        const float gi = gp[0], gf = gp[H], gg = gp[2 * H], go = gp[3 * H];
        const float c = cells_d[row * H + u0 + u];
        const bool first = dir == 0 ? (t == 0) : ((int64_t)t == len - 1);
        const float cprev = first ? 0.f : cells_d[((int64_t)b * p.T + tprev) * H + u0 + u];
        const float dh = p.dh_out[row * ldh + dir * H + u0 + u] + dhr[i];
        const float tc = tanhf(c);
        const float dct = dcs[i] + dh * go * (1.f - tc * tc);
        d_og = dh * tc * go * (1.f - go);
        di = dct * gg * gi * (1.f - gi);
        dg = dct * gi * (1.f - gg * gg);
        df = dct * cprev * gf * (1.f - gf);
        dcs[i] = dct * gf;
      }
      dxp[0] = di; dxp[H] = df; dxp[2 * H] = dg; dxp[3 * H] = d_og;
    }
    if (step + 1 == p.T) break;
    dir_barrier(bar, p.slices, gen);
    // phase B: dh_prev[b][own units] = sum_row dgates_t[b][row] * W_hh[row][unit]
    for (int cb = 0; cb < p.B; cb += LSTM_BC) {
      // gate gradients of ALL units for the chunk: four batch rows (RPT/4 float4 each per thread) are in
      // flight before the first store -- no integer division, no load->store serialisation
      constexpr int RQ = RPT / 4;
#pragma unroll 1
      for (int bb0 = 0; bb0 < LSTM_BC; bb0 += 4) {
        float4 v[4][RQ];
#pragma unroll
        for (int rr = 0; rr < 4; ++rr) {
#pragma unroll
          for (int q = 0; q < RQ; ++q) {
            const int r4 = tid + q * LSTM_THREADS, b = cb + bb0 + rr;
            v[rr][q] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (r4 < G4 / 4 && b < p.B)
              v[rr][q] = __ldcg(reinterpret_cast<const float4*>(p.dxproj + ((int64_t)b * p.T + t) * ldx +
                                                                dir * 4 * H + 4 * r4));
          }
        }
#pragma unroll
        for (int rr = 0; rr < 4; ++rr) {
#pragma unroll
          for (int q = 0; q < RQ; ++q)
            *reinterpret_cast<float4*>(dgs + (bb0 + rr) * GPAD + 4 * (tid + q * LSTM_THREADS)) = v[rr][q];
        }
      }
      __syncthreads();
#pragma unroll 1
      for (int hb = 0; hb < LSTM_BC; hb += HB) {
        float acc[64];
#pragma unroll
        for (int i = 0; i < 64; ++i) acc[i] = 0.f;
#pragma unroll
        for (int i = 0; i < RPT; ++i) {
#pragma unroll
          for (int b = 0; b < HB; ++b) {
            const float d = dgs[(hb + b) * GPAD + i * LSTM_THREADS + tid];
#pragma unroll
            for (int k = 0; k < HS; ++k) acc[b * HS + k] = fmaf(d, w[i][k], acc[b * HS + k]);
          }
        }
        warp_reduce64(acc, lane);
        const int idx = ((lane & 16) ? 32 : 0) + ((lane & 8) ? 16 : 0) + ((lane & 4) ? 8 : 0) + ((lane & 2) ? 4 : 0) +
                        ((lane & 1) ? 2 : 0);
        red[warp * 64 + idx] = acc[0];
        red[warp * 64 + idx + 1] = acc[1];
        __syncthreads();
        if (tid < 64) {
          float s = 0.f;
#pragma unroll
          for (int q = 0; q < 8; ++q) s += red[q * 64 + tid];
          const int b = cb + hb + tid / HS;
          if (b < p.B) dhr[b * HS + (tid % HS)] = s;
        }
        __syncthreads();
      }
    }
  }
}

// hprev[b][t][:] = h[b][t -/+ 1][dir*H : (dir+1)*H] (forward-order predecessor), 0 at the first step and
// beyond the length: the operand of dW_hh = dgates^T h_prev.
__global__ void lstm_hprev_kernel(const float* __restrict__ h, const int64_t* __restrict__ lengths,
                                  float* __restrict__ hprev, int B, int T, int H, int ndir, int dir) {
  const int64_t total = (int64_t)B * T * H;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int k = (int)(i % H);
    const int64_t row = i / H;
    const int t = (int)(row % T), b = (int)(row / T);
    const int64_t len = lengths[b];
    const int tp = dir == 0 ? t - 1 : t + 1;
    float v = 0.f;
    if ((int64_t)t < len && tp >= 0 && (int64_t)tp < len) v = h[((int64_t)b * T + tp) * (ndir * H) + dir * H + k];
    hprev[i] = v;
  }
}

// y = keep ? x / (1-p) : 0 with the counter-hash mask of the GEMM epilogues (inter-layer LSTM dropout,
// nn.LSTM(dropout=p)); the backward applies the same function to the gradient.
__global__ void dropout_kernel(const float* __restrict__ x, float* __restrict__ y, int64_t rows, int cols,
                               uint32_t thresh, float keep_scale, uint64_t seed) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t r = warp; r < rows; r += nwarps)
    for (int c = lane; c < cols; c += 32) {
      const bool keep = dropout_keep(seed, (uint32_t)r, (uint32_t)cols, (uint32_t)c, thresh);
      y[r * cols + c] = keep ? x[r * cols + c] * keep_scale : 0.f;
    }
}

static int lstm_check(int B, int T, int H, int ndir) {
  GANTTS_CHECK_ARG(B >= 1 && B <= LSTM_MAX_B, "lstm: batch %d out of [1,%d]", B, LSTM_MAX_B);
  GANTTS_CHECK_ARG(T >= 1 && H >= 4 && (H % 4) == 0, "lstm: bad T/H (H must be a multiple of 4)");
  GANTTS_CHECK_ARG(ndir == 1 || ndir == 2, "lstm: ndir must be 1 or 2");
  return GANTTS_OK;
}

static int lstm_pick_hs(int H, int ndir, int* slices) {
  int sms = 132;
  int dev = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  for (int hs = 8; hs <= 16; hs *= 2) {
    int s = (H + hs - 1) / hs;
    if (s * ndir <= sms) {
      *slices = s;
      return hs;
    }
  }
  return 0;
}

// The kernel lstm_run launches for one layer: HS hidden units per CTA, `slices` CTAs per direction, the register-resident
// kernels when HS = 8 and H <= 512 (64 weights per thread), the shared-memory kernels otherwise, and its dynamic shared
// memory.
struct LstmPlan {
  int hs, slices;
  const void* fn;
  size_t smem;
};

// GANTTS_E_UNSUPPORTED, with the error set, when the current device cannot run the recurrence of this shape.
static int lstm_plan(bool bwd, int H, int ndir, LstmPlan* pl) {
  pl->hs = lstm_pick_hs(H, ndir, &pl->slices);
  if (pl->hs == 0) {
    set_error("lstm: hidden size %d x %d directions does not fit one wave of CTAs", H, ndir);
    return GANTTS_E_UNSUPPORTED;
  }
  const size_t HS = pl->hs;
  if (HS == 8 && H <= 512) {
    const size_t KR = H <= 256 ? 32 : 64, RPT = 4 * H <= 4 * LSTM_THREADS ? 4 : 8;
    if (!bwd) {
      pl->fn = KR == 32 ? (const void*)lstm_fwd_reg_kernel<32> : (const void*)lstm_fwd_reg_kernel<64>;
      pl->smem = (LSTM_BC * 8 * KR + 8 * LSTM_BC * 32 + LSTM_MAX_B * 8) * sizeof(float);
    } else {
      pl->fn = RPT == 4 ? (const void*)lstm_bwd_reg_kernel<4> : (const void*)lstm_bwd_reg_kernel<8>;
      pl->smem = (LSTM_BC * RPT * LSTM_THREADS + 8 * 64 + 2 * LSTM_MAX_B * 8) * sizeof(float);
    }
  } else if (!bwd) {
    pl->fn = HS == 8 ? (const void*)lstm_fwd_kernel<8> : (const void*)lstm_fwd_kernel<16>;
    pl->smem = (4 * HS * (H + 4) + (size_t)LSTM_BC * H + LSTM_BC * 4 * HS + LSTM_MAX_B * HS) * sizeof(float);
  } else {
    pl->fn = HS == 8 ? (const void*)lstm_bwd_kernel<8> : (const void*)lstm_bwd_kernel<16>;
    pl->smem = (HS * (4 * H + 4) + (size_t)LSTM_BC * (4 * H + 4) + LSTM_THREADS + 2 * LSTM_MAX_B * HS) * sizeof(float);
  }
  if (pl->smem > 227 * 1024) {
    set_error("lstm: the %s of hidden size %d x %d directions (%d units per CTA) needs %zu B of shared memory per CTA, "
              "more than the 227 KB limit", bwd ? "backward" : "forward", H, ndir, pl->hs, pl->smem);
    return GANTTS_E_UNSUPPORTED;
  }
  return GANTTS_OK;
}

// One layer's recurrence (forward or backward) in one cooperative launch of the planned kernel; p.slices is chosen here.
// The barrier counters at p.bar are zeroed on the stream before the launch.
static int lstm_run(bool bwd, LstmParams& p, cudaStream_t st) {
  LstmPlan pl;
  const int rc = lstm_plan(bwd, p.H, p.ndir, &pl);
  if (rc) return rc;
  p.slices = pl.slices;
  GANTTS_CUDA(cudaFuncSetAttribute(pl.fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pl.smem));
  GANTTS_CUDA(cudaMemsetAsync(p.bar, 0, 4 * sizeof(unsigned int), st));
  void* args[] = {&p};
  dim3 grid(p.slices * p.ndir), block(LSTM_THREADS);
  // work = recurrent-matmul flops: 2 * B * T * dirs * 4H * H forward, twice that backward (dh and the gate chain)
  const double H = p.H;
  prof_begin(bwd ? PROF_LSTM_BWD : PROF_LSTM_FWD, (bwd ? 2.0 : 1.0) * 8.0 * p.B * (double)p.T * p.ndir * H * H, st);
  cudaError_t e = cudaLaunchCooperativeKernel(pl.fn, grid, block, args, pl.smem, st);
  prof_end(st);
  if (e != cudaSuccess) return cuda_fail(e, "cudaLaunchCooperativeKernel(lstm)");
  count_launch();
  return GANTTS_OK;
}

// A layer that trains needs both launches; the backward is the larger one, but check both.
static int lstm_check_trainable(int H, int ndir) {
  LstmPlan pl;
  int rc = lstm_plan(false, H, ndir, &pl);
  return rc ? rc : lstm_plan(true, H, ndir, &pl);
}

// ---------------------------------------------------------------------------- LSTM stack of the fused GAN step
// The fused step (gan_step.cu) runs xproj = planes(in) W_ih^T + (b_ih + b_hh) as one bf16x3 GEMM per layer, the
// recurrence above, and these element-wise kernels around them.  Planes are bf16 hi/lo operand planes of the GEMM engine.

// Planes of h * mask, mask = gantts_dropout(ones[rows][cols], p, seed) (thresh 0 / scale 1: no mask): the next layer's
// GEMM operand, or hidden2out's input on the top layer.  One warp per row, a lane converts pairs of columns.
__global__ void lstm_planes_kernel(const float* __restrict__ h, int64_t rows, int cols, uint64_t seed, uint32_t thresh,
                                   float scale, __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo,
                                   int64_t pitch) {
  pdl_entry();
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t r = warp; r < rows; r += nwarps) {
    const float* hr_in = h + r * cols;
    uint32_t* hr = reinterpret_cast<uint32_t*>(hi + r * pitch);
    uint32_t* lr = reinterpret_cast<uint32_t*>(lo + r * pitch);
    for (int c = 2 * lane; c < cols; c += 64) {
      const float m0 = dropout_keep(seed, (uint32_t)r, (uint32_t)cols, (uint32_t)c, thresh) ? scale : 0.f;
      const float m1 = dropout_keep(seed, (uint32_t)r, (uint32_t)cols, (uint32_t)(c + 1), thresh) ? scale : 0.f;
      const float a = hr_in[c] * m0, v = (c + 1 < cols) ? hr_in[c + 1] * m1 : 0.f;
      const uint32_t hp = pack_bf16x2(a, v);
      hr[c >> 1] = hp;
      lr[c >> 1] = pack_bf16x2(a - __uint_as_float(hp << 16), v - __uint_as_float(hp & 0xffff0000u));
    }
  }
}

// Planes of hprev (the values of lstm_hprev_kernel for direction `dir`): the right operand of dW_hh = dgates^T hprev.
__global__ void lstm_hprev_planes_kernel(const float* __restrict__ h, const int64_t* __restrict__ lengths, int B, int T,
                                         int H, int ndir, int dir, __nv_bfloat16* __restrict__ hi,
                                         __nv_bfloat16* __restrict__ lo, int64_t pitch) {
  pdl_entry();
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t r = warp; r < (int64_t)B * T; r += nwarps) {
    const int t = (int)(r % T), b = (int)(r / T);
    const int64_t len = lengths[b];
    const int tp = dir == 0 ? t - 1 : t + 1;
    const bool ok = (int64_t)t < len && tp >= 0 && (int64_t)tp < len;
    const float* src = h + ((int64_t)b * T + tp) * (ndir * H) + dir * H;
    uint32_t* hr = reinterpret_cast<uint32_t*>(hi + r * pitch);
    uint32_t* lr = reinterpret_cast<uint32_t*>(lo + r * pitch);
    for (int c = 2 * lane; c < H; c += 64) {      // H is a multiple of 4
      const float a = ok ? src[c] : 0.f, v = ok ? src[c + 1] : 0.f;
      const uint32_t hp = pack_bf16x2(a, v);
      hr[c >> 1] = hp;
      lr[c >> 1] = pack_bf16x2(a - __uint_as_float(hp << 16), v - __uint_as_float(hp & 0xffff0000u));
    }
  }
}

// out[l][d * 4H + i] = b_ih[l][d][i] + b_hh[l][d][i] for every layer and direction (the xproj GEMM's bias), one launch.
struct LstmBiasList {
  int n, len;                             // n = layers * ndir vectors of len = 4H
  const float* a[2 * GANTTS_MAX_LSTM_LAYERS];
  const float* b[2 * GANTTS_MAX_LSTM_LAYERS];
  float* out[2 * GANTTS_MAX_LSTM_LAYERS];
};
__global__ void lstm_bias_sum_kernel(LstmBiasList bl) {
  pdl_entry();
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < (int64_t)bl.n * bl.len;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int v = (int)(i / bl.len), e = (int)(i - (int64_t)v * bl.len);
    bl.out[v][e] = bl.a[v][e] + bl.b[v][e];
  }
}

}  // namespace gantts

using namespace gantts;

extern "C" size_t gantts_lstm_workspace_bytes(void) { return 256; }

extern "C" int gantts_lstm_layer_supported(int H, int ndir, int train) {
  GANTTS_CHECK_ARG(H >= 4 && (H % 4) == 0 && (ndir == 1 || ndir == 2), "lstm: bad H/ndir (H must be a multiple of 4)");
  LstmPlan pl;
  return train ? lstm_check_trainable(H, ndir) : lstm_plan(false, H, ndir, &pl);
}

extern "C" int gantts_lstm_layer_fwd(const float* xproj, const float* W_hh, const int64_t* lengths_dev, float* h_out,
                                     float* gates, float* cells, int B, int T, int H, int ndir, void* workspace,
                                     size_t workspace_bytes, void* stream) {
  int rc = lstm_check(B, T, H, ndir);
  if (rc) return rc;
  GANTTS_CHECK_ARG(xproj && W_hh && lengths_dev && h_out && gates && cells, "lstm_fwd: null pointer");
  GANTTS_CHECK_ARG(workspace && workspace_bytes >= 256, "lstm_fwd: workspace too small");
  LstmParams p{};
  p.xproj = xproj; p.lengths = lengths_dev; p.h_out = h_out; p.gates = gates; p.cells = cells;
  p.W_hh = W_hh;
  p.W_hh_dir = (int64_t)4 * H * H;
  p.bar = static_cast<unsigned int*>(workspace);
  p.B = B; p.T = T; p.H = H; p.ndir = ndir;
  return lstm_run(false, p, as_stream(stream));
}

extern "C" int gantts_lstm_layer_bwd(const float* dh_out, const float* W_hh, const int64_t* lengths_dev,
                                     const float* gates, const float* cells, float* dxproj, int B, int T, int H,
                                     int ndir, void* workspace, size_t workspace_bytes, void* stream) {
  int rc = lstm_check(B, T, H, ndir);
  if (rc) return rc;
  GANTTS_CHECK_ARG(dh_out && W_hh && lengths_dev && gates && cells && dxproj, "lstm_bwd: null pointer");
  GANTTS_CHECK_ARG(workspace && workspace_bytes >= 256, "lstm_bwd: workspace too small");
  LstmParams p{};
  p.lengths = lengths_dev; p.gates = const_cast<float*>(gates); p.cells = const_cast<float*>(cells);
  p.W_hh = W_hh;
  p.W_hh_dir = (int64_t)4 * H * H;
  p.dh_out = dh_out; p.dxproj = dxproj;
  p.bar = static_cast<unsigned int*>(workspace);
  p.B = B; p.T = T; p.H = H; p.ndir = ndir;
  return lstm_run(true, p, as_stream(stream));
}

extern "C" int gantts_lstm_hprev(const float* h, const int64_t* lengths_dev, float* hprev, int B, int T, int H,
                                 int ndir, int dir, void* stream) {
  GANTTS_CHECK_ARG(h && lengths_dev && hprev && B >= 1 && T >= 1 && H >= 1 && (dir == 0 || dir == 1) && dir < ndir,
                   "lstm_hprev: bad arguments");
  int64_t total = (int64_t)B * T * H;
  int nb = (int)((total + 1023) / 1024);
  if (nb > 132 * 8) nb = 132 * 8;
  lstm_hprev_kernel<<<nb, 256, 0, as_stream(stream)>>>(h, lengths_dev, hprev, B, T, H, ndir, dir);
  GANTTS_LAUNCH_CHECK("lstm_hprev_kernel");
  return GANTTS_OK;
}

extern "C" int gantts_dropout(const float* x, float* y, int64_t rows, int cols, float p, uint64_t seed, void* stream) {
  GANTTS_CHECK_ARG(x && y && rows >= 1 && cols >= 1 && p >= 0.f && p < 1.f, "dropout: bad arguments");
  const uint32_t thresh = (uint32_t)(p * 65536.f + 0.5f);
  int nb = (int)((rows * cols + 1023) / 1024);
  if (nb > 132 * 8) nb = 132 * 8;
  if (nb < 1) nb = 1;
  dropout_kernel<<<nb, 256, 0, as_stream(stream)>>>(x, y, rows, cols, thresh, p > 0.f ? 1.f / (1.f - p) : 1.f, seed);
  GANTTS_LAUNCH_CHECK("dropout_kernel");
  return GANTTS_OK;
}
