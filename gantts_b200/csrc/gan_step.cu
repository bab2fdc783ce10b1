// Fused GAN training step (include/gantts_b200.h: gantts_gan_step): the whole mini-batch of reference
// train.py:528-580 -- batch prologue, apply_generator (:336-355), update_discriminator (:245-279),
// update_generator (:282-320) with both clip_grad_norm_ + Adagrad steps -- enqueued on ONE stream by one
// C call, with no host synchronisation: every loss is a device scalar.
//
// Semantics kept from the reference (SURVEY.md 3.2):
//   * the fake-term gradient of loss_d reaches the generator (y_hat_static is not detached, one
//     zero_grad per step): it is accumulated into the SAME upstream buffer as the gradient of loss_g,
//     so the generator/MLPG backward runs ONCE on the summed gradient (gradients are linear; the
//     reference runs it twice and adds the results);
//   * three discriminator forwards with independent dropout masks; the discriminator is updated
//     BEFORE the third forward used by the adversarial loss;
//   * losses are normalised by the number of valid frames, BCE uses log(D + 1e-20) verbatim.
// Real and fake discriminator batches are stacked into one 2M-row batch (one GEMM per layer).
#include <nvtx3/nvToolsExt.h>

#include "common.cuh"

namespace gantts {

// NVTX range per phase of the step (header-only NVTX3: a no-op unless a profiler is attached; `ncu --nvtx` and nsys
// show the phases of one gantts_gan_step call on the timeline).
struct NvtxRange {
  explicit NvtxRange(const char* name) { nvtxRangePushA(name); }
  ~NvtxRange() { nvtxRangePop(); }
};

enum ScalarSlot {
  S_REAL = 0,      // [0..2]  real: loss sum, correct count, sum(mask)
  S_FAKE = 3,      // [3..5]
  S_ADV = 6,       // [6..8]
  S_MGE = 9,       // [9..10] sse, sum(mask)
  S_MSE = 11,      // [11..12]
  S_DSUMSQ = 13,
  S_GSUMSQ = 14,
  S_INV_T = 15,    // 1 / frames
  S_ADV_SCALE = 16,
  S_MGE_SCALE = 17,
  S_MSE_SCALE = 18,
  S_COUNT = 32
};

struct ColList {
  int n;
  int c[GANTTS_MAX_COLS];
};

__global__ void gather_cols_list_kernel(const float* __restrict__ in, int64_t in_rs, float* __restrict__ out,
                                        int64_t out_rs, ColList cols, int64_t rows) {
  __shared__ int sc[GANTTS_MAX_COLS];
  for (int i = threadIdx.x; i < cols.n; i += blockDim.x) sc[i] = cols.c[i];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t r = warp; r < rows; r += nwarps)
    for (int j = lane; j < cols.n; j += 32) out[r * out_rs + j] = in[r * in_rs + sc[j]];
}

// Column gather of up to two row blocks straight into bf16 hi/lo operand planes (the discriminator's input: rows
// [0, rows_a) = selected columns of `a`, rows [rows_a, rows_a + rows_b) = selected columns of `b`): replaces
// gather -> fp32 matrix -> split_planes.  One warp per row, a lane converts PAIRS of columns (4-byte stores).
__global__ void gather_planes_kernel(const float* __restrict__ a, int64_t a_rs, ColList ca, int64_t rows_a,
                                     const float* __restrict__ b, int64_t b_rs, ColList cb, int64_t rows_b,
                                     __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo, int64_t pitch) {
  pdl_entry();
  __shared__ int sa[GANTTS_MAX_COLS], sb[GANTTS_MAX_COLS];
  for (int i = threadIdx.x; i < ca.n; i += blockDim.x) sa[i] = ca.c[i];
  for (int i = threadIdx.x; i < cb.n; i += blockDim.x) sb[i] = cb.c[i];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t r = warp; r < rows_a + rows_b; r += nwarps) {
    const bool first = r < rows_a;
    const float* src = first ? a + r * a_rs : b + (r - rows_a) * b_rs;
    const int* sc = first ? sa : sb;
    const int n = first ? ca.n : cb.n;
    uint32_t* hr = reinterpret_cast<uint32_t*>(hi + r * pitch);
    uint32_t* lr = reinterpret_cast<uint32_t*>(lo + r * pitch);
    for (int c = 2 * lane; c < n; c += 64) {
      const float v0 = src[sc[c]], v1 = (c + 1 < n) ? src[sc[c + 1]] : 0.f;
      const uint32_t hp = pack_bf16x2(v0, v1);
      hr[c >> 1] = hp;
      lr[c >> 1] = pack_bf16x2(v0 - __uint_as_float(hp << 16), v1 - __uint_as_float(hp & 0xffff0000u));
    }
  }
}

__global__ void scatter_cols_list_add_kernel(const float* __restrict__ go, int64_t go_rs, float* __restrict__ gi,
                                             int64_t gi_rs, ColList cols, int64_t rows) {
  __shared__ int sc[GANTTS_MAX_COLS];
  for (int i = threadIdx.x; i < cols.n; i += blockDim.x) sc[i] = cols.c[i];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t r = warp; r < rows; r += nwarps)
    for (int j = lane; j < cols.n; j += 32) gi[r * gi_rs + sc[j]] += go[r * go_rs + j];
}

// inv_frames <= 0: derive the normaliser on the device, 1 / sum_b min(len_b, T) (= mask.sum() of train.py:258,286) --
// single-process use; a data-parallel caller passes 1 / (GLOBAL number of valid frames).
__global__ void set_scales_kernel(float* scal, float inv_frames, float adv_w, float mge_w, float mse_w,
                                  int zero_norms, const int64_t* __restrict__ lengths, int B, int T) {
  pdl_entry();
  if (threadIdx.x == 0) {
    if (zero_norms) scal[S_DSUMSQ] = scal[S_GSUMSQ] = 0.f;
    if (!(inv_frames > 0.f)) {
      int64_t n = 0;
      for (int b = 0; b < B; ++b) {
        const int64_t l = lengths[b];
        n += l < 0 ? 0 : (l > T ? T : l);
      }
      inv_frames = n > 0 ? 1.f / (float)n : 0.f;
    }
    scal[S_INV_T] = inv_frames;
    scal[S_ADV_SCALE] = adv_w * inv_frames;
    scal[S_MGE_SCALE] = mge_w * inv_frames;
    scal[S_MSE_SCALE] = mse_w * inv_frames;
  }
}

// Deferred reductions: every loss kernel of the step leaves per-block partial sums in its own slot; the single
// finalize kernel at the end of the step reduces all of them (deterministic: fixed block order) -- no per-loss
// "finish" launch on the way.
enum RedSlot { R_REAL = 0, R_FAKE = 1, R_ADV = 2, R_MGE = 3, R_MSE = 4, R_COUNT = 5 };

struct RedCounts {
  int n[R_COUNT];      // blocks that wrote partials into slot i (0 = slot unused this step)
};

// Adversarial BCE terms of train.py:262-270,307-308 for one or two halves of a stacked discriminator output, forward
// sums AND the gradient w.r.t. D in one pass: half 0 = rows [0, M) with kind0, half 1 = rows [M, 2M) with kind1
// (kind 0: -log(D + eps) * m, correct = D > 0.5; kind 1: -log(1 - D + eps) * m, correct = D < 0.5).  mask is [M] for
// both halves.  Blocks [0, nbh) serve half 0 and write ws0, blocks [nbh, 2 nbh) serve half 1 and write ws1.
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
  const float s = scale[0];
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

// MaskedMSELoss forward sums (gantts/seqloss.py:41-43) AND its gradient 2 * scale * (a m - b m) * m in one pass
// (ga == nullptr: forward only).  The gradient is STORED (not accumulated): this launch initialises the buffer.
// bmap.n > 0: column d of the target is column bmap.c[d] of `b` (the static features are read straight out of y:
// get_static_features of multistream.py:56-79 without materialising y_static).
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

// clip_grad_norm_ + Adagrad with the sum of squares taken from the per-block partials of sumsq_partial_kernel:
// every block re-reduces the (<= 592) partials itself in the same fixed order, which removes the finish launch.
__global__ void __launch_bounds__(OPT_THREADS)
clip_adagrad_partials_kernel(TensorList tl, const float* __restrict__ partial, int npartial, float* __restrict__ sumsq_out,
                             float max_norm, float lr, float wd, float eps) {
  pdl_entry();
  __shared__ float sm[32];
  __shared__ float total_s;
  float v[1] = {0.f};
  for (int i = threadIdx.x; i < npartial; i += OPT_THREADS) v[0] += partial[i];
  block_sum<1>(v, sm);
  if (threadIdx.x == 0) {
    total_s = v[0];
    if (blockIdx.x == 0) sumsq_out[0] = v[0];
  }
  __syncthreads();
  const float total_norm = sqrtf(total_s);
  float coef = max_norm / (total_norm + 1e-6f);
  coef = coef < 1.f ? coef : 1.f;
  const int64_t total = tl.off[tl.n];
  for (int64_t i = (int64_t)blockIdx.x * OPT_THREADS + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * OPT_THREADS) {
    int k = find_tensor(tl, i);
    int64_t j = i - tl.off[k];
    float g = tl.g[k][j] * coef;
    tl.g[k][j] = g;
    float p = tl.p[k][j];
    g = fmaf(wd, p, g);
    float s = fmaf(g, g, tl.s[k][j]);
    tl.s[k][j] = s;
    tl.p[k][j] = p - lr * g / (sqrtf(s) + eps);
  }
}

// The same with torch.optim.Adam (amsgrad off; reference hparams.py:125-130): tl.s = exp_avg, tl.s2 = exp_avg_sq;
// step_size = lr / (1 - beta1^t), inv_sqrt_bc2 = 1 / sqrt(1 - beta2^t) come from the host.
__global__ void __launch_bounds__(OPT_THREADS)
clip_adam_partials_kernel(TensorList tl, const float* __restrict__ partial, int npartial, float* __restrict__ sumsq_out,
                          float max_norm, float b1, float b2, float wd, float eps, float step_size, float inv_sqrt_bc2) {
  pdl_entry();
  __shared__ float sm[32];
  __shared__ float total_s;
  float v[1] = {0.f};
  for (int i = threadIdx.x; i < npartial; i += OPT_THREADS) v[0] += partial[i];
  block_sum<1>(v, sm);
  if (threadIdx.x == 0) {
    total_s = v[0];
    if (blockIdx.x == 0) sumsq_out[0] = v[0];
  }
  __syncthreads();
  const float total_norm = sqrtf(total_s);
  float coef = max_norm / (total_norm + 1e-6f);
  coef = coef < 1.f ? coef : 1.f;
  const int64_t total = tl.off[tl.n];
  for (int64_t i = (int64_t)blockIdx.x * OPT_THREADS + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * OPT_THREADS) {
    int k = find_tensor(tl, i);
    int64_t j = i - tl.off[k];
    float g = tl.g[k][j] * coef;
    tl.g[k][j] = g;
    const float p = tl.p[k][j];
    g = fmaf(wd, p, g);
    const float m = b1 * tl.s[k][j] + (1.f - b1) * g;
    const float q = b2 * tl.s2[k][j] + (1.f - b2) * g * g;
    tl.s[k][j] = m;
    tl.s2[k][j] = q;
    tl.p[k][j] = p - step_size * m / (sqrtf(q) * inv_sqrt_bc2 + eps);
  }
}

// losses[0..11] = loss_d, loss_fake_d, loss_real_d, loss_mse, loss_mge, loss_adv, loss_g,
//                 real_correct, fake_correct, frames(local sum of mask), d_grad_norm, g_grad_norm
__global__ void __launch_bounds__(RED_THREADS)
finalize_losses_kernel(const float* scal, float* losses, const RedWs* red, RedCounts cnt, float adv_w, float mge_w,
                       float mse_w, int has_d) {
  pdl_entry();
  __shared__ float sm[RED_NV * 32];
  __shared__ float tot[R_COUNT][RED_NV];
  for (int sl = 0; sl < R_COUNT; ++sl) {
    float v[RED_NV] = {0.f, 0.f, 0.f, 0.f};
    for (int i = threadIdx.x; i < cnt.n[sl]; i += RED_THREADS) {
#pragma unroll
      for (int k = 0; k < RED_NV; ++k) v[k] += red[sl].partial[i][k];
    }
    block_sum<RED_NV>(v, sm);
    if (threadIdx.x == 0) {
#pragma unroll
      for (int k = 0; k < RED_NV; ++k) tot[sl][k] = v[k];
    }
    __syncthreads();
  }
  if (threadIdx.x != 0) return;
  const float invT = scal[S_INV_T];
  const float real = has_d ? tot[R_REAL][0] * invT : 0.f, fake = has_d ? tot[R_FAKE][0] * invT : 0.f;
  const float adv = (has_d && adv_w > 0.f) ? tot[R_ADV][0] * invT : 0.f;
  const float mge = tot[R_MGE][0] * invT, mse = tot[R_MSE][0] * invT;
  losses[0] = real + fake;
  losses[1] = fake;
  losses[2] = real;
  losses[3] = mse;
  losses[4] = mge;
  losses[5] = adv;
  losses[6] = (mse_w * mse + mge_w * mge) + adv_w * adv;
  losses[7] = has_d ? tot[R_REAL][1] : 0.f;
  losses[8] = has_d ? tot[R_FAKE][1] : 0.f;
  losses[9] = tot[R_MGE][1];
  losses[10] = has_d ? sqrtf(scal[S_DSUMSQ]) : 0.f;
  losses[11] = sqrtf(scal[S_GSUMSQ]);
}

static inline int blocks_1d(int64_t work, int per_block) {
  int64_t b = (work + per_block - 1) / per_block;
  if (b < 1) b = 1;
  if (b > 132 * 8) b = 132 * 8;
  return (int)b;
}

// + the highway gate's weight and bias, or the SRU stack's weights and biases (the two are mutually exclusive); an
// LSTM generator (gate, 8 tensors per layer, hidden2out) fits in the same count and in one TensorList of the clip kernels
constexpr int MAX_PARAMS = 2 * GANTTS_MAX_LAYERS + 2 * GANTTS_MAX_SRU_LAYERS;
static_assert(2 + 8 * GANTTS_MAX_LSTM_LAYERS + 2 <= MAX_PARAMS && 2 + 8 * GANTTS_MAX_LSTM_LAYERS + 2 <= OPT_MAX_TENSORS,
              "the LSTM generator's tensors must fit one TensorList");

struct ParamList {
  int n;
  float* p[MAX_PARAMS];
  float* g[MAX_PARAMS];
  float* s[MAX_PARAMS];
  float* s2[MAX_PARAMS];                                // Adam: exp_avg_sq (null for Adagrad)
  int64_t sizes[MAX_PARAMS];
  float* gW[GANTTS_MAX_LAYERS];
  float* gb[GANTTS_MAX_LAYERS];
  float* sgW[GANTTS_MAX_SRU_LAYERS];                    // SRU stack: gradient of W[l] / b[l] in the flat buffer
  float* sgb[GANTTS_MAX_SRU_LAYERS];
  float* lgW_ih[GANTTS_MAX_LSTM_LAYERS][2];             // LSTM stack: gradients of layer l, direction d in the flat buffer
  float* lgW_hh[GANTTS_MAX_LSTM_LAYERS][2];
  float* lgb_ih[GANTTS_MAX_LSTM_LAYERS][2];
  float* lgb_hh[GANTTS_MAX_LSTM_LAYERS][2];
  int64_t total;
};

static inline size_t al256(size_t v) { return (v + 255) / 256 * 256; }

struct StepLayout {
  float* scal;
  float* mask;            // [M]
  float* d_in;            // [2M][dD]  rows 0..M-1 real, M..2M-1 fake
  float* d_out;           // [2M]
  float* g_dout;          // [2M]
  float* g_din;           // [2M][dD]
  float* y_static;        // [M][n_static]
  float* g_static;        // [M][n_static]
  float* g_yhat;          // [M][d_out]
  float* g_grads;         // flat generator gradients
  float* d_grads;         // flat discriminator gradients
  char* g_tape;
  size_t g_tape_bytes;
  char* d_tape;
  size_t d_tape_bytes;
  char* mlp_ws;
  size_t mlp_ws_bytes;
  RedWs* red;             // [R_COUNT] deferred loss partials
  float* opt_partial;     // [OPT_MAX_BLOCKS] sum-of-squares partials of the model being stepped
  // highway generator only (zero bytes otherwise, so the plain MLP layout is unchanged)
  float* hw_tx;           // [M][S] gate sigmoid(x_s W_T^T + b_T)
  float* hw_gx;           // [M][S] MLPG output Gx
  char* hw_w;             // planes of W_T [S][S]
  char* hw_dz;            // planes of dz [M][S]
  float* hw_partial;      // split-K partials of dW_T / db_T
  // SRU generator only (zero bytes otherwise, so the MLP and highway layouts are unchanged); per layer l:
  char* sru_in[GANTTS_MAX_SRU_LAYERS];    // planes of the masked GEMM input [M][n_in] (layer l > 0: written by scan l-1)
  float* sru_u[GANTTS_MAX_SRU_LAYERS];    // U = planes(x * mask_x) W  [M][ncols * k]
  float* sru_c[GANTTS_MAX_SRU_LAYERS];    // cell states [M][ncols]
  float* sru_h[GANTTS_MAX_SRU_LAYERS];    // fp32 h [M][ncols] below the top layer (the next layer's highway input)
  char* sru_w[GANTTS_MAX_SRU_LAYERS];     // planes of W [n_in][ncols * k], then of W^T [ncols * k][n_in]
  float* sru_partial[GANTTS_MAX_SRU_LAYERS];   // split-K partials of dW
  char* sru_du;           // planes of dU [M][ncols * k] (one layer at a time)
  float* sru_dx;          // [M][ncols] dL/dh of the top layer, then dX = dU W of each layer for the one below
  float* sru_dxp;         // [M][ncols] highway gradient (k = 3) for the layer below
  float* sru_bpart;       // [B][2 * ncols] bias-gradient partials
  // LSTM generator only (zero bytes otherwise, so every other layout is unchanged); per layer l:
  char* lstm_in[GANTTS_MAX_LSTM_LAYERS];      // planes of the GEMM input [M][n_in]: x (l = 0), else h_{l-1} * mask_{l-1}
  char* lstm_w[GANTTS_MAX_LSTM_LAYERS];       // planes of W_ih of both directions [ndir 4H][n_in], then [n_in][ndir 4H]
  float* lstm_bias[GANTTS_MAX_LSTM_LAYERS];   // b_ih + b_hh [ndir 4H]
  float* lstm_h[GANTTS_MAX_LSTM_LAYERS];      // h [M][ndir H]
  float* lstm_gates[GANTTS_MAX_LSTM_LAYERS];  // [ndir][M][4H]
  float* lstm_cells[GANTTS_MAX_LSTM_LAYERS];  // [ndir][M][H]
  float* lstm_xproj;      // [M][ndir 4H] xproj of one layer; in the backward, dgates of one layer
  float* lstm_out;        // [M][d_out] hidden2out's output, the MLPG's input
  float* lstm_dh;         // [M][ndir H] dL/dh of the top layer, then mask * dX of each layer for the one below
  char* lstm_dg;          // planes of dgates [M][ndir 4H]
  char* lstm_hp;          // planes of hprev [M][H]
  float* lstm_part[2][2]; // split-K partials per direction: [d][0] dW_ih | db_ih, [d][1] dW_hh (one layer at a time)
  unsigned int* lstm_bar; // grid-barrier counters of the recurrence
  size_t total;
};

static inline int sru_ncols(const gantts_sru_stack_t& s) { return s.hidden * (s.bidirectional ? 2 : 1); }
static inline int sru_nin(const gantts_sru_stack_t& s, int l) { return l == 0 ? s.in_dim : sru_ncols(s); }
static inline int sru_k(const gantts_sru_stack_t& s, int l) { return sru_nin(s, l) != sru_ncols(s) ? 4 : 3; }
static inline int lstm_ndir(const gantts_lstm_stack_t& s) { return s.bidirectional ? 2 : 1; }
static inline int lstm_nin(const gantts_lstm_stack_t& s, int l) { return l == 0 ? s.in_dim : lstm_ndir(s) * s.hidden; }

// width of x: the SRU or LSTM stack's input, else the generator MLP's
static inline int gen_in_width(const gantts_gan_step_t* c) {
  return c->sru.num_layers > 0 ? c->sru.in_dim : (c->lstm.num_layers > 0 ? c->lstm.in_dim : c->g.dims[0]);
}

static int64_t mlp_param_count(const gantts_mlp_t& m) {
  int64_t n = 0;
  for (int l = 0; l < m.num_layers; ++l) n += (int64_t)m.dims[l + 1] * m.dims[l] + m.dims[l + 1];
  return n;
}

// elements of the highway gate's parameters, which lead the generator's flat gradient buffer
static int64_t gate_param_count(const gantts_gan_step_t* c) {
  const int64_t S = c->highway.static_dim;
  return S * S + S;
}

// elements of the SRU stack's parameters, which lead the generator's flat gradient buffer
static int64_t sru_param_count(const gantts_gan_step_t* c) {
  const gantts_sru_stack_t& s = c->sru;
  int64_t n = 0;
  for (int l = 0; l < s.num_layers; ++l) n += (int64_t)sru_nin(s, l) * sru_ncols(s) * sru_k(s, l) + 2 * sru_ncols(s);
  return n;
}

// elements of the LSTM stack's parameters, which follow the gate in the generator's flat gradient buffer
static int64_t lstm_param_count(const gantts_gan_step_t* c) {
  const gantts_lstm_stack_t& s = c->lstm;
  const int64_t G4 = 4 * (int64_t)s.hidden;
  int64_t n = 0;
  for (int l = 0; l < s.num_layers; ++l) n += lstm_ndir(s) * (G4 * lstm_nin(s, l) + G4 * s.hidden + 2 * G4);
  return n;
}

static int64_t g_param_count(const gantts_gan_step_t* c) {
  return gate_param_count(c) + sru_param_count(c) + lstm_param_count(c) + mlp_param_count(c->g);
}

static void layout(const gantts_gan_step_t* c, char* base, StepLayout* L) {
  const int64_t M = (int64_t)c->B * c->T;
  const int dD = c->d.dims[0];
  char* cur = base;
  auto take = [&](size_t bytes) { char* p = cur; cur += al256(bytes); return p; };
  L->scal = (float*)take(S_COUNT * sizeof(float));
  L->mask = (float*)take(M * sizeof(float));
  L->d_in = (float*)take((size_t)2 * M * dD * sizeof(float));
  L->d_out = (float*)take((size_t)2 * M * sizeof(float));
  L->g_dout = (float*)take((size_t)2 * M * sizeof(float));
  L->g_din = (float*)take((size_t)2 * M * dD * sizeof(float));
  L->y_static = (float*)take((size_t)M * c->n_static * sizeof(float));
  L->g_static = (float*)take((size_t)M * c->n_static * sizeof(float));
  L->g_yhat = (float*)take((size_t)M * c->g.dims[c->g.num_layers] * sizeof(float));
  L->g_grads = (float*)take(g_param_count(c) * sizeof(float));
  L->d_grads = (float*)take(mlp_param_count(c->d) * sizeof(float));
  L->g_tape_bytes = gantts_mlp_tape_bytes(&c->g, M);
  L->g_tape = take(L->g_tape_bytes);
  L->d_tape_bytes = gantts_mlp_tape_bytes(&c->d, 2 * M);
  L->d_tape = take(L->d_tape_bytes);
  size_t a = gantts_mlp_workspace_bytes(&c->g, M), b = gantts_mlp_workspace_bytes(&c->d, 2 * M);
  L->mlp_ws_bytes = a > b ? a : b;
  L->mlp_ws = take(L->mlp_ws_bytes);
  L->red = (RedWs*)take(R_COUNT * sizeof(RedWs));
  L->opt_partial = (float*)take(OPT_MAX_BLOCKS * sizeof(float));
  const int S = c->highway.static_dim;
  const bool hw = S > 0;
  L->hw_tx = (float*)take(hw ? (size_t)M * S * sizeof(float) : 0);
  L->hw_gx = (float*)take(hw ? (size_t)M * S * sizeof(float) : 0);
  L->hw_w = take(hw ? 2 * plane_bytes(S, S) : 0);
  L->hw_dz = take(hw ? 2 * plane_bytes(M, S) : 0);
  L->hw_partial = (float*)take(hw ? mn_partial_bytes(M, S, S, nullptr, nullptr) : 0);
  const gantts_sru_stack_t& s = c->sru;
  const int nl = s.num_layers, nc = nl > 0 ? sru_ncols(s) : 0;
  int maxku = 0;
  for (int l = 0; l < GANTTS_MAX_SRU_LAYERS; ++l) {
    L->sru_in[l] = L->sru_w[l] = nullptr;
    L->sru_u[l] = L->sru_c[l] = L->sru_h[l] = L->sru_partial[l] = nullptr;
    if (l >= nl) continue;
    const int ni = sru_nin(s, l), ku = nc * sru_k(s, l);
    maxku = ku > maxku ? ku : maxku;
    L->sru_in[l] = take(2 * plane_bytes(M, ni));
    L->sru_u[l] = (float*)take((size_t)M * ku * sizeof(float));
    L->sru_c[l] = (float*)take((size_t)M * nc * sizeof(float));
    if (l < nl - 1) L->sru_h[l] = (float*)take((size_t)M * nc * sizeof(float));
    L->sru_w[l] = take(2 * plane_bytes(ni, ku) + 2 * plane_bytes(ku, ni));
    L->sru_partial[l] = (float*)take(mn_partial_bytes(M, ni, ku, nullptr, nullptr));
  }
  L->sru_du = take(nl > 0 ? 2 * plane_bytes(M, maxku) : 0);
  L->sru_dx = (float*)take((size_t)M * nc * sizeof(float));
  L->sru_dxp = (float*)take((size_t)M * nc * sizeof(float));
  L->sru_bpart = (float*)take((size_t)c->B * 2 * nc * sizeof(float));
  const gantts_lstm_stack_t& ls = c->lstm;
  const int lnl = ls.num_layers, H = lnl > 0 ? ls.hidden : 0, nd = lstm_ndir(ls), n4 = nd * 4 * H;
  size_t part_ih = 0, part_hh = 0;
  for (int l = 0; l < GANTTS_MAX_LSTM_LAYERS; ++l) {
    L->lstm_in[l] = L->lstm_w[l] = nullptr;
    L->lstm_bias[l] = L->lstm_h[l] = L->lstm_gates[l] = L->lstm_cells[l] = nullptr;
    if (l >= lnl) continue;
    const int ni = lstm_nin(ls, l);
    L->lstm_in[l] = take(2 * plane_bytes(M, ni));
    L->lstm_w[l] = take(2 * plane_bytes(n4, ni) + 2 * plane_bytes(ni, n4));
    L->lstm_bias[l] = (float*)take((size_t)n4 * sizeof(float));
    L->lstm_h[l] = (float*)take((size_t)M * nd * H * sizeof(float));
    L->lstm_gates[l] = (float*)take((size_t)M * n4 * sizeof(float));
    L->lstm_cells[l] = (float*)take((size_t)M * nd * H * sizeof(float));
    const size_t pi = mn_partial_bytes(M, 4 * H, ni, nullptr, nullptr), ph = mn_partial_bytes(M, 4 * H, H, nullptr, nullptr);
    part_ih = pi > part_ih ? pi : part_ih;
    part_hh = ph > part_hh ? ph : part_hh;
  }
  const bool lstm = lnl > 0;
  L->lstm_xproj = (float*)take((size_t)M * n4 * sizeof(float));
  L->lstm_out = (float*)take(lstm ? (size_t)M * c->g.dims[c->g.num_layers] * sizeof(float) : 0);
  L->lstm_dh = (float*)take((size_t)M * nd * H * sizeof(float));
  L->lstm_dg = take(lstm ? 2 * plane_bytes(M, n4) : 0);
  L->lstm_hp = take(lstm ? 2 * plane_bytes(M, H) : 0);
  for (int d = 0; d < 2; ++d) {
    L->lstm_part[d][0] = (float*)take(d < nd ? part_ih : 0);
    L->lstm_part[d][1] = (float*)take(d < nd ? part_hh : 0);
  }
  L->lstm_bar = (unsigned int*)take(lstm ? 256 : 0);
  L->total = (size_t)(cur - base) + 256;
}

// appends the layers of m; `flat` is where their gradients start in the model's flat buffer
static void param_list(const gantts_mlp_t& m, float* const* sumW, float* const* sumb, float* const* sqW, float* const* sqb,
                       float* flat, ParamList* pl) {
  float* cur = flat;
  for (int l = 0; l < m.num_layers; ++l) {
    const int64_t nw = (int64_t)m.dims[l + 1] * m.dims[l], nb = m.dims[l + 1];
    pl->gW[l] = cur;
    pl->p[pl->n] = const_cast<float*>(m.W[l]);
    pl->g[pl->n] = cur;
    pl->s[pl->n] = sumW[l];
    pl->s2[pl->n] = sqW[l];
    pl->sizes[pl->n++] = nw;
    cur += nw;
    pl->gb[l] = cur;
    pl->p[pl->n] = const_cast<float*>(m.b[l]);
    pl->g[pl->n] = cur;
    pl->s[pl->n] = sumb[l];
    pl->s2[pl->n] = sqb[l];
    pl->sizes[pl->n++] = nb;
    cur += nb;
  }
  pl->total += cur - flat;
}

// generator parameters in model.parameters() order: [T.weight, T.bias] of a highway generator, or [W, b] of every layer
// of an SRU stack; then [W_ih, W_hh, b_ih, b_hh] of every layer and direction of an LSTM stack; then the MLP layers
static void g_param_list(const gantts_gan_step_t* c, float* flat, ParamList* pl) {
  pl->n = 0;
  pl->total = 0;
  const gantts_highway_t& h = c->highway;
  const gantts_sru_stack_t& s = c->sru;
  for (int l = 0; l < s.num_layers; ++l) {
    const int64_t sizes[2] = {(int64_t)sru_nin(s, l) * sru_ncols(s) * sru_k(s, l), 2 * (int64_t)sru_ncols(s)};
    float* const ps[2] = {const_cast<float*>(s.W[l]), const_cast<float*>(s.b[l])};
    float* const ss[2] = {s.sumW[l], s.sumb[l]};
    float* const qs[2] = {s.sqW[l], s.sqb[l]};
    pl->sgW[l] = flat + pl->total;
    pl->sgb[l] = flat + pl->total + sizes[0];
    for (int i = 0; i < 2; ++i) {
      pl->p[pl->n] = ps[i];
      pl->g[pl->n] = flat + pl->total;
      pl->s[pl->n] = ss[i];
      pl->s2[pl->n] = qs[i];
      pl->sizes[pl->n++] = sizes[i];
      pl->total += sizes[i];
    }
  }
  if (h.static_dim > 0) {
    const int64_t S = h.static_dim;
    const int64_t sizes[2] = {S * S, S};
    float* const ps[2] = {const_cast<float*>(h.W), const_cast<float*>(h.b)};
    float* const ss[2] = {h.sumW, h.sumb};
    float* const qs[2] = {h.sqW, h.sqb};
    for (int i = 0; i < 2; ++i) {
      pl->p[pl->n] = ps[i];
      pl->g[pl->n] = flat + pl->total;
      pl->s[pl->n] = ss[i];
      pl->s2[pl->n] = qs[i];
      pl->sizes[pl->n++] = sizes[i];
      pl->total += sizes[i];
    }
  }
  const gantts_lstm_stack_t& ls = c->lstm;
  for (int l = 0; l < ls.num_layers; ++l)
    for (int d = 0; d < lstm_ndir(ls); ++d) {
      const int64_t G4 = 4 * (int64_t)ls.hidden;
      const int64_t sizes[4] = {G4 * lstm_nin(ls, l), G4 * ls.hidden, G4, G4};
      float* const ps[4] = {const_cast<float*>(ls.W_ih[l][d]), const_cast<float*>(ls.W_hh[l][d]),
                            const_cast<float*>(ls.b_ih[l][d]), const_cast<float*>(ls.b_hh[l][d])};
      float* const ss[4] = {ls.sumW_ih[l][d], ls.sumW_hh[l][d], ls.sumb_ih[l][d], ls.sumb_hh[l][d]};
      float* const qs[4] = {ls.sqW_ih[l][d], ls.sqW_hh[l][d], ls.sqb_ih[l][d], ls.sqb_hh[l][d]};
      float** const gs[4] = {&pl->lgW_ih[l][d], &pl->lgW_hh[l][d], &pl->lgb_ih[l][d], &pl->lgb_hh[l][d]};
      for (int i = 0; i < 4; ++i) {
        *gs[i] = flat + pl->total;
        pl->p[pl->n] = ps[i];
        pl->g[pl->n] = flat + pl->total;
        pl->s[pl->n] = ss[i];
        pl->s2[pl->n] = qs[i];
        pl->sizes[pl->n++] = sizes[i];
        pl->total += sizes[i];
      }
    }
  param_list(c->g, c->g_sumW, c->g_sumb, c->g_sqW, c->g_sqb, flat + pl->total, pl);
}

static inline int bce_blocks(int64_t rows) { return grid_for(rows, RED_THREADS); }
static inline int sse_blocks(int64_t rows, int D) { return grid_for(rows * D, RED_THREADS * 4); }

// BCE of a stacked discriminator output: halves = 2 -> rows [0,M) kind0 into slot0 and rows [M,2M) kind1 into slot1
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

// clip_grad_norm_ + optimiser step over one model's parameter list: two launches (partials, update), no finish kernel
static int clip_opt_model(const gantts_gan_step_t* c, const ParamList& pl, float* partial, float* sumsq_out, float lr, float wd,
                          cudaStream_t st) {
  TensorList tl;
  const bool adam = c->optimizer == GANTTS_OPT_ADAM;
  int rc = fill(tl, pl.p, pl.g, pl.s, adam ? pl.s2 : nullptr, pl.sizes, 0, pl.n);
  if (rc) return rc;
  const int nb = blocks_for(tl.off[tl.n], OPT_MAX_BLOCKS);
  GANTTS_PDL_LAUNCH((sumsq_partial_kernel), nb, OPT_THREADS, 0, st, tl, partial);
  GANTTS_LAUNCH_CHECK("sumsq_partial_kernel");
  if (adam) {
    for (int i = 0; i < pl.n; ++i) GANTTS_CHECK_ARG(pl.s[i] && pl.s2[i], "gan_step: Adam needs exp_avg and exp_avg_sq for every tensor");
    GANTTS_CHECK_ARG(c->opt_step >= 1, "gan_step: Adam needs opt_step >= 1 (the number of the step being taken)");
    const double t = (double)c->opt_step;
    const float step_size = (float)((double)lr / (1.0 - pow((double)c->beta1, t)));
    const float inv_sqrt_bc2 = (float)(1.0 / sqrt(1.0 - pow((double)c->beta2, t)));
    GANTTS_PDL_LAUNCH((clip_adam_partials_kernel), nb, OPT_THREADS, 0, st, tl, partial, nb, sumsq_out, c->max_norm, c->beta1, c->beta2,
                      wd, c->eps, step_size, inv_sqrt_bc2);
    GANTTS_LAUNCH_CHECK("clip_adam_partials_kernel");
  } else {
    GANTTS_PDL_LAUNCH((clip_adagrad_partials_kernel), nb, OPT_THREADS, 0, st, tl, partial, nb, sumsq_out, c->max_norm, lr, wd, c->eps);
    GANTTS_LAUNCH_CHECK("clip_adagrad_partials_kernel");
  }
  return GANTTS_OK;
}

static int check_step(const gantts_gan_step_t* c) {
  GANTTS_CHECK_ARG(c, "gan_step: null config");
  GANTTS_CHECK_ARG(c->B >= 1 && c->T >= 1, "gan_step: bad batch shape");
  GANTTS_CHECK_ARG(c->optimizer == GANTTS_OPT_ADAGRAD || c->optimizer == GANTTS_OPT_ADAM, "gan_step: unknown optimizer %d", c->optimizer);
  if (c->optimizer == GANTTS_OPT_ADAM)
    GANTTS_CHECK_ARG(c->beta1 >= 0.f && c->beta1 < 1.f && c->beta2 >= 0.f && c->beta2 < 1.f, "gan_step: Adam betas out of range");
  GANTTS_CHECK_ARG(c->g.num_layers >= 1 && c->g.num_layers <= GANTTS_MAX_LAYERS, "gan_step: bad generator");
  GANTTS_CHECK_ARG(c->n_static >= 1 && c->n_static <= GANTTS_MAX_COLS, "gan_step: bad n_static");
  GANTTS_CHECK_ARG(c->n_static_cols == c->n_static, "gan_step: static column list must have n_static entries");
  const gantts_lstm_stack_t& ls = c->lstm;
  GANTTS_CHECK_ARG(ls.num_layers >= 0 && ls.num_layers <= GANTTS_MAX_LSTM_LAYERS,
                   "gan_step: LSTM layer count %d not in [0, %d] (train larger stacks with GanTrainer)", ls.num_layers,
                   GANTTS_MAX_LSTM_LAYERS);
  if (ls.num_layers > 0) {
    // In2OutRNNHighwayNet (models.py:72-118): the gate, the LSTM stack, then hidden2out as a one-layer MLP
    GANTTS_CHECK_ARG(c->highway.static_dim > 0,
                     "gan_step: an LSTM stack runs only with the highway gate (In2OutRNNHighwayNet); LSTMRNN and GRURNN "
                     "train with GanTrainer");
    GANTTS_CHECK_ARG(c->sru.num_layers == 0, "gan_step: the LSTM stack and the SRU stack are mutually exclusive");
    GANTTS_CHECK_ARG(ls.in_dim >= 1 && (ls.bidirectional == 0 || ls.bidirectional == 1),
                     "gan_step: bad LSTM shape (in_dim %d, bidirectional %d)", ls.in_dim, ls.bidirectional);
    GANTTS_CHECK_ARG(ls.hidden >= 4 && ls.hidden % 4 == 0, "gan_step: LSTM hidden size %d is not a positive multiple of 4",
                     ls.hidden);
    GANTTS_CHECK_ARG(c->B <= LSTM_MAX_B, "gan_step: an LSTM stack runs at most LSTM_MAX_B = %d sequences (B = %d)",
                     LSTM_MAX_B, c->B);
    GANTTS_CHECK_ARG(ls.dropout >= 0.f && ls.dropout < 1.f, "gan_step: LSTM dropout out of [0, 1)");
    const int nh = lstm_ndir(ls) * ls.hidden;
    GANTTS_CHECK_ARG(c->g.num_layers == 1 && c->g.dims[0] == nh,
                     "gan_step: with an LSTM stack g is hidden2out alone: 1 layer of input width %d (got %d layer(s), "
                     "input width %d)", nh, c->g.num_layers, c->g.dims[0]);
    GANTTS_CHECK_ARG(ls.in_dim == c->g.dims[1],
                     "gan_step: LSTM in_dim %d != hidden2out output width %d (the model returns its input as y_hat)",
                     ls.in_dim, c->g.dims[1]);
    for (int l = 0; l < ls.num_layers; ++l)
      for (int d = 0; d < lstm_ndir(ls); ++d) {
        GANTTS_CHECK_ARG(ls.W_ih[l][d] && ls.W_hh[l][d] && ls.b_ih[l][d] && ls.b_hh[l][d],
                         "gan_step: null LSTM weight/bias of layer %d direction %d", l, d);
        GANTTS_CHECK_ARG(ls.sumW_ih[l][d] && ls.sumW_hh[l][d] && ls.sumb_ih[l][d] && ls.sumb_hh[l][d],
                         "gan_step: null LSTM optimiser state of layer %d direction %d", l, d);
        if (c->optimizer == GANTTS_OPT_ADAM)
          GANTTS_CHECK_ARG(ls.sqW_ih[l][d] && ls.sqW_hh[l][d] && ls.sqb_ih[l][d] && ls.sqb_hh[l][d],
                           "gan_step: Adam needs exp_avg_sq for LSTM layer %d direction %d", l, d);
      }
  }
  const gantts_sru_stack_t& s = c->sru;
  GANTTS_CHECK_ARG(s.num_layers >= 0 && s.num_layers <= GANTTS_MAX_SRU_LAYERS, "gan_step: SRU layer count %d not in [0, %d]",
                   s.num_layers, GANTTS_MAX_SRU_LAYERS);
  if (s.num_layers > 0) {
    // SRURNN (models.py:144-167): the SRU stack, then hidden2out as a one-layer MLP
    GANTTS_CHECK_ARG(c->highway.static_dim == 0, "gan_step: the SRU stack and the highway gate are mutually exclusive");
    GANTTS_CHECK_ARG(s.in_dim >= 1 && s.hidden >= 1 && (s.bidirectional == 0 || s.bidirectional == 1),
                     "gan_step: bad SRU shape (in_dim %d, hidden %d, bidirectional %d)", s.in_dim, s.hidden, s.bidirectional);
    GANTTS_CHECK_ARG(s.act >= 0 && s.act <= 2, "gan_step: SRU activation %d not in 0..2", s.act);
    GANTTS_CHECK_ARG(s.dropout >= 0.f && s.dropout < 1.f && s.rnn_dropout >= 0.f && s.rnn_dropout < 1.f,
                     "gan_step: SRU dropout / rnn_dropout out of [0, 1)");
    const int nc = sru_ncols(s);
    GANTTS_CHECK_ARG(c->g.num_layers == 1 && c->g.dims[0] == nc,
                     "gan_step: with an SRU stack g is hidden2out alone: 1 layer of input width %d (got %d layer(s), input "
                     "width %d)", nc, c->g.num_layers, c->g.dims[0]);
    for (int l = 0; l < s.num_layers; ++l) {
      GANTTS_CHECK_ARG(s.W[l] && s.b[l], "gan_step: null SRU weight/bias of layer %d", l);
      GANTTS_CHECK_ARG(s.sumW[l] && s.sumb[l], "gan_step: null SRU optimiser state of layer %d", l);
      if (c->optimizer == GANTTS_OPT_ADAM)
        GANTTS_CHECK_ARG(s.sqW[l] && s.sqb[l], "gan_step: Adam needs exp_avg_sq for SRU layer %d", l);
    }
  }
  if (c->w_d > 0.f) {
    GANTTS_CHECK_ARG(c->d.num_layers >= 1 && c->d.num_layers <= GANTTS_MAX_LAYERS, "gan_step: bad discriminator");
    const int cond_w = c->d_conditioned ? gen_in_width(c) : 0;
    GANTTS_CHECK_ARG(c->n_adv >= 1 && c->n_adv <= GANTTS_MAX_COLS && c->d.dims[0] == cond_w + c->n_adv,
                     "gan_step: discriminator input width %d != %d conditioning + %d adversarial columns",
                     c->d.dims[0], cond_w, c->n_adv);
    GANTTS_CHECK_ARG(c->d.dims[c->d.num_layers] == 1 && c->d.last_act == GANTTS_ACT_SIGMOID,
                     "gan_step: discriminator must end in a single sigmoid output");
  }
  GANTTS_CHECK_ARG(c->g.last_act == GANTTS_ACT_NONE, "gan_step: generator must have a linear output");
  GANTTS_CHECK_ARG(c->mlpg_table, "gan_step: null MLPG table");
  const gantts_highway_t& h = c->highway;
  GANTTS_CHECK_ARG(h.static_dim >= 0, "gan_step: negative highway static_dim");
  if (h.static_dim > 0) {
    // the arithmetic of In2OutHighwayNet (models.py:54-69): x_s and y_hat_static are the same S columns, and the
    // generator's output is the S static columns of one dynamic stream followed by their delta windows
    const int S = h.static_dim, nw = c->windows.n, Lg = c->g.num_layers;
    const gantts_streams_t& st = c->streams;
    GANTTS_CHECK_ARG(st.n == 1 && st.dyn[0] && st.in_start[0] == 0 && st.out_start[0] == 0 && st.sd[0] == S,
                     "gan_step: a highway generator needs exactly one dynamic stream with in_start = out_start = 0 and "
                     "sd = static_dim = %d (got %d stream(s), first sd %d)", S, st.n, st.sd[0]);
    GANTTS_CHECK_ARG(c->n_static == S, "gan_step: highway static_dim %d != n_static %d", S, c->n_static);
    GANTTS_CHECK_ARG(gen_in_width(c) >= S, "gan_step: highway generator input width %d < static_dim %d", gen_in_width(c),
                     S);
    GANTTS_CHECK_ARG(c->g.dims[Lg] == nw * S, "gan_step: highway generator output width %d != %d windows x static_dim %d",
                     c->g.dims[Lg], nw, S);
    GANTTS_CHECK_ARG(h.W && h.b, "gan_step: null highway gate weight/bias");
    GANTTS_CHECK_ARG((reinterpret_cast<uintptr_t>(h.b) & 15) == 0, "gan_step: highway gate bias must be 16-byte aligned");
    GANTTS_CHECK_ARG(h.sumW && h.sumb, "gan_step: null highway gate optimiser state");
    if (c->optimizer == GANTTS_OPT_ADAM)
      GANTTS_CHECK_ARG(h.sqW && h.sqb, "gan_step: Adam needs exp_avg_sq for the highway gate");
  }
  return GANTTS_OK;
}

// LSTM layer l's workspace: planes of its GEMM input, and of W_ih of both directions [ndir 4H][n_in] then transposed
static Planes lstm_in_planes(const gantts_gan_step_t* c, const StepLayout& L, int l, int64_t M) {
  char* cur = L.lstm_in[l];
  return carve_planes(cur, M, lstm_nin(c->lstm, l));
}
static void lstm_w_planes(const gantts_gan_step_t* c, const StepLayout& L, int l, Planes* w, Planes* wt) {
  const int ni = lstm_nin(c->lstm, l), n4 = lstm_ndir(c->lstm) * 4 * c->lstm.hidden;
  char* cur = L.lstm_w[l];
  *w = carve_planes(cur, n4, ni);
  *wt = carve_planes(cur, ni, n4);
}

// x_s: the first S columns of x's operand planes -- the generator MLP's tape input, or the LSTM stack's layer-0 input
// (written by the generator's forward), so x is not converted twice.
static int gate_input_planes(const gantts_gan_step_t* c, const gantts_mlp_t& g, const StepLayout& L, int64_t M,
                             Planes* xs) {
  if (c->lstm.num_layers > 0) {
    *xs = lstm_in_planes(c, L, 0, M);
  } else {
    int rc = mlp_tape_input_planes(&g, M, L.g_tape, L.g_tape_bytes, xs);
    if (rc) return rc;
  }
  xs->cols = c->highway.static_dim;
  return GANTTS_OK;
}

// Tx = sigmoid(x_s W_T^T + b_T)
static int highway_gate_fwd(const gantts_gan_step_t* c, const gantts_mlp_t& g, const StepLayout& L, int64_t M,
                            cudaStream_t st) {
  const int S = c->highway.static_dim;
  Planes xs;
  int rc = gate_input_planes(c, g, L, M, &xs);
  if (rc) return rc;
  char* cur = L.hw_w;
  const Planes w = carve_planes(cur, S, S);
  if ((rc = launch_split(c->highway.W, S, S, S, w, 0, st))) return rc;
  EpiArgs e;
  e.epi = EPI_F32;
  e.C = L.hw_tx;
  e.ldc = S;
  e.bias = c->highway.b;
  e.act = GANTTS_ACT_SIGMOID;
  return launch_gemm_kk(xs, w, e, st);
}

// dW_T = dz^T x_s and db_T = colsum(dz) (ones-tile MMA) into the first S * S + S entries of the generator's buffer
static int highway_gate_bwd(const gantts_gan_step_t* c, const gantts_mlp_t& g, const StepLayout& L, int64_t M,
                            cudaStream_t st) {
  const int S = c->highway.static_dim;
  Planes xs;
  int rc = gate_input_planes(c, g, L, M, &xs);
  if (rc) return rc;
  char* cur = L.hw_dz;
  const Planes dz = carve_planes(cur, M, S);
  ReduceList rl;
  if ((rc = launch_gemm_mn(dz, xs, L.g_grads, L.g_grads + (int64_t)S * S, 0, L.hw_partial, st, &rl))) return rc;
  return flush_reduce(rl, 0, st);
}

// SRU layer l's workspace: planes of its masked input, and of W [n_in][ncols k] then W^T [ncols k][n_in]
static Planes sru_in_planes(const gantts_gan_step_t* c, const StepLayout& L, int l, int64_t M) {
  char* cur = L.sru_in[l];
  return carve_planes(cur, M, sru_nin(c->sru, l));
}
static void sru_w_planes(const gantts_gan_step_t* c, const StepLayout& L, int l, Planes* w, Planes* wt) {
  const int ni = sru_nin(c->sru, l), ku = sru_ncols(c->sru) * sru_k(c->sru, l);
  char* cur = L.sru_w[l];
  *w = carve_planes(cur, ni, ku);
  *wt = carve_planes(cur, ku, ni);
}

// SRU stack forward (rnn.SRUCell per layer): the last layer's h goes unmasked into hidden2out's tape input planes, so
// the caller runs hidden2out with mlp_fwd_impl(..., input_ready = true).  train = false: no masks.
static int sru_stack_fwd(const gantts_gan_step_t* c, const gantts_mlp_t& g, const StepLayout& L, const float* x, int64_t M,
                         uint64_t seed, bool train, cudaStream_t st) {
  const gantts_sru_stack_t& s = c->sru;
  const int nl = s.num_layers, nc = sru_ncols(s);
  const float p_h = train ? s.dropout : 0.f, p_x = train ? s.rnn_dropout : 0.f;
  int rc;
  {
    // every layer's weight -> planes as stored (operand of dX = dU W^T) and transposed (operand of U = x W), one launch
    WeightSplitList wl;
    wl.n = nl;
    wl.off[0] = 0;
    for (int l = 0; l < nl; ++l) {
      Planes w, wt;
      sru_w_planes(c, L, l, &w, &wt);
      wl.W[l] = s.W[l];
      wl.N[l] = (int)w.rows;
      wl.K[l] = (int)w.cols;
      wl.hi[l] = w.hi;
      wl.lo[l] = w.lo;
      wl.pitch[l] = w.pitch;
      wl.thi[l] = wt.hi;
      wl.tlo[l] = wt.lo;
      wl.tpitch[l] = wt.pitch;
      wl.off[l + 1] = wl.off[l] + (int64_t)((w.rows + 31) / 32) * ((w.cols + 31) / 32);
    }
    int nb = (int)(wl.off[nl] < num_sms() * 8 ? wl.off[nl] : num_sms() * 8);
    GANTTS_PDL_LAUNCH((split_weights_kernel), nb < 1 ? 1 : nb, 256, 0, st, wl);
    GANTTS_LAUNCH_CHECK("split_weights_kernel(sru)");
  }
  const Planes in0 = sru_in_planes(c, L, 0, M);
  if (p_x > 0.f) {
    GANTTS_PDL_LAUNCH((sru_mask_split_kernel), blocks_1d(M * s.in_dim, 1024), 256, 0, st, x, (int64_t)s.in_dim, M, s.in_dim,
                      c->T, sru_mask(gantts_sru_mask_seed(seed, 0, 0), p_x), in0.hi, in0.lo, in0.pitch);
    GANTTS_LAUNCH_CHECK("sru_mask_split_kernel");
  } else if ((rc = launch_split(x, s.in_dim, M, s.in_dim, in0, 0, st))) {
    return rc;
  }
  Planes top;
  if ((rc = mlp_tape_input_planes(&g, M, L.g_tape, L.g_tape_bytes, &top))) return rc;
  for (int l = 0; l < nl; ++l) {
    const int k = sru_k(s, l);
    const bool last = l == nl - 1;
    Planes w, wt;
    sru_w_planes(c, L, l, &w, &wt);
    EpiArgs e;
    e.epi = EPI_F32;
    e.C = L.sru_u[l];
    e.ldc = (int64_t)nc * k;
    if ((rc = launch_gemm_kk(sru_in_planes(c, L, l, M), wt, e, st))) return rc;
    const Planes out = last ? top : sru_in_planes(c, L, l + 1, M);
    SruStepFwd p{};
    p.u = L.sru_u[l];
    p.xh = k == 3 ? (l == 0 ? x : L.sru_h[l - 1]) : nullptr;
    p.xh_rs = l == 0 ? s.in_dim : nc;
    p.bias = s.b[l];
    p.c = L.sru_c[l];
    p.h = L.sru_h[l];
    p.hi = out.hi;
    p.lo = out.lo;
    p.pitch = out.pitch;
    p.mh = sru_mask(gantts_sru_mask_seed(seed, l, 1), last ? 0.f : p_h);      // SRU(): no output dropout on the last layer
    p.mx = sru_mask(gantts_sru_mask_seed(seed, l + 1, 0), last ? 0.f : p_x);
    p.B = c->B;
    p.T = c->T;
    p.d = s.hidden;
    p.bidir = s.bidirectional;
    p.act = s.act;
    if ((rc = launch_sru_step_fwd(p, k, st))) return rc;
  }
  return GANTTS_OK;
}

// SRU stack backward from dL/dh of the top layer in L.sru_dx (hidden2out's input gradient), top layer first:
//   scan backward -> dU planes, highway gradient dx' (k = 3), bias partials -> bias gradient (fixed order over B)
//   dW = (x * mask_x)^T dU  (MN-major, lands in the [n_in][ncols k] parameter layout)
//   dX = dU W^T             (K-major on W as stored; not for layer 0)
// The layer below's dh = mask_x * dX + dx' is formed on load by its scan backward.
static int sru_stack_bwd(const gantts_gan_step_t* c, const StepLayout& L, const ParamList& pg, const float* x, int64_t M,
                         uint64_t seed, cudaStream_t st) {
  const gantts_sru_stack_t& s = c->sru;
  const int nl = s.num_layers, nc = sru_ncols(s);
  int rc;
  ReduceList rl;
  for (int l = nl - 1; l >= 0; --l) {
    const int k = sru_k(s, l);
    const bool top = l == nl - 1;
    char* cur = L.sru_du;
    const Planes du = carve_planes(cur, M, (int64_t)nc * k);
    SruStepBwd p{};
    p.u = L.sru_u[l];
    p.xh = k == 3 ? (l == 0 ? x : L.sru_h[l - 1]) : nullptr;
    p.xh_rs = l == 0 ? s.in_dim : nc;
    p.bias = s.b[l];
    p.c = L.sru_c[l];
    p.dx = L.sru_dx;
    p.dxp_in = top ? nullptr : L.sru_dxp;
    p.mxu = sru_mask(gantts_sru_mask_seed(seed, l + 1, 0), top ? 0.f : s.rnn_dropout);
    p.mh = sru_mask(gantts_sru_mask_seed(seed, l, 1), top ? 0.f : s.dropout);
    p.du_hi = du.hi;
    p.du_lo = du.lo;
    p.du_pitch = du.pitch;
    p.dxp_out = (k == 3 && l > 0) ? L.sru_dxp : nullptr;
    p.dbias_part = L.sru_bpart;
    p.B = c->B;
    p.T = c->T;
    p.d = s.hidden;
    p.bidir = s.bidirectional;
    p.act = s.act;
    if ((rc = launch_sru_step_bwd(p, k, st))) return rc;
    GANTTS_PDL_LAUNCH((sru_bias_reduce_kernel), (2 * nc + 255) / 256, 256, 0, st, L.sru_bpart, c->B, 2 * nc, pg.sgb[l]);
    GANTTS_LAUNCH_CHECK("sru_bias_reduce_kernel");
    if ((rc = launch_gemm_mn(sru_in_planes(c, L, l, M), du, pg.sgW[l], nullptr, 0, L.sru_partial[l], st, &rl))) return rc;
    if (l > 0) {
      Planes w, wt;
      sru_w_planes(c, L, l, &w, &wt);
      EpiArgs e;
      e.epi = EPI_F32;
      e.C = L.sru_dx;
      e.ldc = nc;
      if ((rc = launch_gemm_kk(du, w, e, st))) return rc;
    }
  }
  return flush_reduce(rl, 0, st);
}

static LstmParams lstm_layer_params(const gantts_gan_step_t* c, const StepLayout& L, int l, const int64_t* lengths) {
  const gantts_lstm_stack_t& s = c->lstm;
  LstmParams p{};
  p.W_hh = s.W_hh[l][0];
  if (s.bidirectional)      // the two directions' tensors are 4-byte aligned: their distance is a whole number of floats
    p.W_hh_dir = ((int64_t)reinterpret_cast<uintptr_t>(s.W_hh[l][1]) - (int64_t)reinterpret_cast<uintptr_t>(s.W_hh[l][0])) /
                 (int64_t)sizeof(float);
  p.lengths = lengths;
  p.h_out = L.lstm_h[l];
  p.gates = L.lstm_gates[l];
  p.cells = L.lstm_cells[l];
  p.bar = L.lstm_bar;
  p.B = c->B;
  p.T = c->T;
  p.H = s.hidden;
  p.ndir = lstm_ndir(s);
  return p;
}

// LSTM stack forward (nn.LSTM on packed sequences, per-element dropout between layers): per layer one xproj GEMM over
// both directions, the cooperative recurrence, and one kernel that writes the next GEMM's operand planes of h * mask --
// on the top layer the unmasked h into hidden2out's tape input planes, so the caller runs hidden2out with
// mlp_fwd_impl(..., input_ready = true).  train = false: no masks.
static int lstm_stack_fwd(const gantts_gan_step_t* c, const gantts_mlp_t& g, const StepLayout& L, const float* x,
                          const int64_t* lengths, int64_t M, uint64_t seed, bool train, cudaStream_t st) {
  const gantts_lstm_stack_t& s = c->lstm;
  const int nl = s.num_layers, H = s.hidden, nd = lstm_ndir(s), G4 = 4 * H, nh = nd * H;
  const float p_drop = train ? s.dropout : 0.f;
  int rc;
  {
    // every W_ih -> planes as stored (rows d * 4H.. of the direction-stacked operand of xproj) and transposed (columns
    // d * 4H.. of the operand of dX = dgates W_ih), one launch; and b_ih + b_hh of every layer and direction, one launch
    WeightSplitList wl;
    LstmBiasList bl;
    wl.n = bl.n = nl * nd;
    wl.off[0] = 0;
    bl.len = G4;
    for (int l = 0; l < nl; ++l) {
      Planes w, wt;
      lstm_w_planes(c, L, l, &w, &wt);
      for (int d = 0; d < nd; ++d) {
        const int i = l * nd + d;
        wl.W[i] = s.W_ih[l][d];
        wl.N[i] = G4;
        wl.K[i] = lstm_nin(s, l);
        wl.hi[i] = w.hi + (int64_t)d * G4 * w.pitch;
        wl.lo[i] = w.lo + (int64_t)d * G4 * w.pitch;
        wl.pitch[i] = w.pitch;
        wl.thi[i] = wt.hi + (int64_t)d * G4;
        wl.tlo[i] = wt.lo + (int64_t)d * G4;
        wl.tpitch[i] = wt.pitch;
        wl.off[i + 1] = wl.off[i] + (int64_t)((G4 + 31) / 32) * ((wl.K[i] + 31) / 32);
        bl.a[i] = s.b_ih[l][d];
        bl.b[i] = s.b_hh[l][d];
        bl.out[i] = L.lstm_bias[l] + (int64_t)d * G4;
      }
    }
    const int nb = (int)(wl.off[wl.n] < num_sms() * 8 ? wl.off[wl.n] : num_sms() * 8);
    GANTTS_PDL_LAUNCH((split_weights_kernel), nb < 1 ? 1 : nb, 256, 0, st, wl);
    GANTTS_LAUNCH_CHECK("split_weights_kernel(lstm)");
    GANTTS_PDL_LAUNCH((lstm_bias_sum_kernel), (bl.n * G4 + 255) / 256, 256, 0, st, bl);
    GANTTS_LAUNCH_CHECK("lstm_bias_sum_kernel");
  }
  if ((rc = launch_split(x, s.in_dim, M, s.in_dim, lstm_in_planes(c, L, 0, M), 0, st))) return rc;
  Planes top;
  if ((rc = mlp_tape_input_planes(&g, M, L.g_tape, L.g_tape_bytes, &top))) return rc;
  for (int l = 0; l < nl; ++l) {
    const bool last = l == nl - 1;
    Planes w, wt;
    lstm_w_planes(c, L, l, &w, &wt);
    EpiArgs e;
    e.epi = EPI_F32;
    e.C = L.lstm_xproj;
    e.ldc = (int64_t)nd * G4;
    e.bias = L.lstm_bias[l];
    if ((rc = launch_gemm_kk(lstm_in_planes(c, L, l, M), w, e, st))) return rc;
    LstmParams p = lstm_layer_params(c, L, l, lengths);
    p.xproj = L.lstm_xproj;
    if ((rc = lstm_run(false, p, st))) return rc;
    const Planes out = last ? top : lstm_in_planes(c, L, l + 1, M);
    const float pl = last ? 0.f : p_drop;             // nn.LSTM: no dropout on the last layer's output
    GANTTS_PDL_LAUNCH((lstm_planes_kernel), blocks_1d(M * nh, 1024), 256, 0, st, L.lstm_h[l], M, nh,
                      gantts_lstm_mask_seed(seed, l), pl > 0.f ? (uint32_t)(pl * 65536.f + 0.5f) : 0u,
                      pl > 0.f ? 1.f / (1.f - pl) : 1.f, out.hi, out.lo, out.pitch);
    GANTTS_LAUNCH_CHECK("lstm_planes_kernel");
  }
  return GANTTS_OK;
}

// LSTM stack backward from dL/dh of the top layer in L.lstm_dh (hidden2out's input gradient), top layer first:
//   recurrence backward -> dgates (fp32, in the xproj buffer) -> dgates planes
//   per direction: dW_ih and db_ih = dgates_d^T in (MN-major, ones-tile bias), dW_hh = dgates_d^T hprev_d (MN-major)
//   dX = dgates W_ih, times the mask of the layer below in the GEMM epilogue (not for layer 0)
//   db_hh = db_ih (b_ih and b_hh enter xproj as one sum)
// Each layer's split-K reductions go through one flush_reduce.
static int lstm_stack_bwd(const gantts_gan_step_t* c, const StepLayout& L, const ParamList& pg, const int64_t* lengths,
                          int64_t M, uint64_t seed, cudaStream_t st) {
  const gantts_lstm_stack_t& s = c->lstm;
  const int nl = s.num_layers, H = s.hidden, nd = lstm_ndir(s), G4 = 4 * H, nh = nd * H;
  int rc;
  char* cur = L.lstm_dg;
  const Planes dg = carve_planes(cur, M, (int64_t)nd * G4);
  cur = L.lstm_hp;
  const Planes hp = carve_planes(cur, M, H);
  ReduceList rl;
  for (int l = nl - 1; l >= 0; --l) {
    LstmParams p = lstm_layer_params(c, L, l, lengths);
    p.dh_out = L.lstm_dh;
    p.dxproj = L.lstm_xproj;
    if ((rc = lstm_run(true, p, st))) return rc;
    if ((rc = launch_split(L.lstm_xproj, (int64_t)nd * G4, M, nd * G4, dg, 0, st))) return rc;
    const Planes in = lstm_in_planes(c, L, l, M);
    for (int d = 0; d < nd; ++d) {
      Planes dgd = dg;
      dgd.hi += (int64_t)d * G4;
      dgd.lo += (int64_t)d * G4;
      dgd.cols = G4;
      if ((rc = launch_gemm_mn(dgd, in, pg.lgW_ih[l][d], pg.lgb_ih[l][d], 0, L.lstm_part[d][0], st, &rl))) return rc;
      GANTTS_PDL_LAUNCH((lstm_hprev_planes_kernel), blocks_1d(M * H, 1024), 256, 0, st, L.lstm_h[l], lengths, c->B, c->T, H, nd,
                        d, hp.hi, hp.lo, hp.pitch);
      GANTTS_LAUNCH_CHECK("lstm_hprev_planes_kernel");
      if ((rc = launch_gemm_mn(dgd, hp, pg.lgW_hh[l][d], nullptr, 0, L.lstm_part[d][1], st, &rl))) return rc;
    }
    if (l > 0) {
      Planes w, wt;
      lstm_w_planes(c, L, l, &w, &wt);
      EpiArgs e;
      e.epi = EPI_F32;
      e.C = L.lstm_dh;
      e.ldc = nh;
      if (s.dropout > 0.f) {      // dh_{l-1} = mask_{l-1} * dX: LeakyReLU with slope 1 is the identity, then the mask
        e.act = GANTTS_ACT_LEAKY_DROPOUT;
        e.slope = 1.f;
        e.p = s.dropout;
        e.seed = gantts_lstm_mask_seed(seed, l - 1);
      }
      if ((rc = launch_gemm_kk(dg, wt, e, st))) return rc;
    }
    if ((rc = flush_reduce(rl, 0, st))) return rc;
    for (int d = 0; d < nd; ++d)
      GANTTS_CUDA(cudaMemcpyAsync(pg.lgb_hh[l][d], pg.lgb_ih[l][d], (size_t)G4 * sizeof(float), cudaMemcpyDeviceToDevice, st));
  }
  return GANTTS_OK;
}

// Generator forward: the MLP from x into y_hat; or the SRU stack and then hidden2out on the planes it left in the tape,
// into y_hat; or the LSTM stack and then hidden2out into L.lstm_out, with y_hat a copy of x (models.py:118).
static int generator_fwd(const gantts_gan_step_t* c, const gantts_mlp_t& g, const StepLayout& L, const float* x, int x_rs,
                         const int64_t* lengths, int64_t M, float* y_hat, int d_out, uint64_t seed, bool train,
                         cudaStream_t st) {
  int rc;
  if (c->lstm.num_layers > 0) {
    if ((rc = lstm_stack_fwd(c, g, L, x, lengths, M, seed, train, st))) return rc;
    if ((rc = mlp_fwd_impl(&g, nullptr, 0, M, L.lstm_out, d_out, L.g_tape, L.g_tape_bytes, st, true))) return rc;
    GANTTS_CUDA(cudaMemcpyAsync(y_hat, x, (size_t)M * x_rs * sizeof(float), cudaMemcpyDeviceToDevice, st));
    return GANTTS_OK;
  }
  if (c->sru.num_layers == 0) return gantts_mlp_fwd(&g, x, x_rs, M, y_hat, d_out, L.g_tape, L.g_tape_bytes, st);
  if ((rc = sru_stack_fwd(c, g, L, x, M, seed, train, st))) return rc;
  return mlp_fwd_impl(&g, nullptr, 0, M, y_hat, d_out, L.g_tape, L.g_tape_bytes, st, true);
}

}  // namespace gantts

using namespace gantts;

extern "C" uint64_t gantts_gan_step_seed(uint64_t seed, int which) { return seed * 4 + (uint64_t)which; }

extern "C" uint64_t gantts_sru_mask_seed(uint64_t seed, int layer, int which) {
  return gantts_mlp_layer_seed(gantts_gan_step_seed(seed, 3), 2 * layer + which);
}

// after every SRU index 2 * layer + which < 2 * GANTTS_MAX_SRU_LAYERS of the same stream
extern "C" uint64_t gantts_lstm_mask_seed(uint64_t seed, int layer) {
  return gantts_mlp_layer_seed(gantts_gan_step_seed(seed, 3), 2 * GANTTS_MAX_SRU_LAYERS + layer);
}

extern "C" size_t gantts_gan_step_workspace_bytes(const gantts_gan_step_t* c) {
  if (check_step(c)) return 0;
  StepLayout L;
  layout(c, nullptr, &L);
  return L.total + 256;
}

extern "C" int gantts_gan_step_grad_buffer(const gantts_gan_step_t* c, void* workspace, int which, float** ptr,
                                           int64_t* count) {
  int rc = check_step(c);
  if (rc) return rc;
  GANTTS_CHECK_ARG(workspace && ptr && count, "gan_step_grad_buffer: null pointer");
  StepLayout L;
  layout(c, reinterpret_cast<char*>(al256(reinterpret_cast<uintptr_t>(workspace))), &L);
  *ptr = which == 0 ? L.g_grads : L.d_grads;
  *count = which == 0 ? g_param_count(c) : mlp_param_count(c->d);
  return GANTTS_OK;
}

extern "C" int gantts_gan_step(const gantts_gan_step_t* c, int phases, const float* x, const float* y,
                               const int64_t* lengths_dev, float inv_frames, uint64_t seed, float* y_hat,
                               float* y_hat_static, float* losses_dev, void* workspace, size_t workspace_bytes,
                               void* stream) {
  int rc = check_step(c);
  if (rc) return rc;
  GANTTS_CHECK_ARG(x && y && lengths_dev && y_hat && y_hat_static && losses_dev, "gan_step: null pointer");
  size_t need = gantts_gan_step_workspace_bytes(c);
  if (!workspace || workspace_bytes < need) {
    set_error("gan_step: workspace too small (%zu < %zu)", workspace_bytes, need);
    return GANTTS_E_WORKSPACE;
  }
  cudaStream_t st = as_stream(stream);
  StepLayout L;
  layout(c, reinterpret_cast<char*>(al256(reinterpret_cast<uintptr_t>(workspace))), &L);
  const int64_t M = (int64_t)c->B * c->T;
  // d_in: the width (and row stride) of x -- the SRU stack's input width when there is one
  const int Lg = c->g.num_layers, d_in = gen_in_width(c), d_out = c->g.dims[Lg];
  const int dD = c->d.dims[0], nS = c->n_static;
  const bool has_d = c->w_d > 0.f;
  const bool has_adv = has_d && c->adv_w > 0.f;
  // discriminator_linguistic_condition (train.py:254-256,302-303): D sees cat((x, y_adv), -1); the first
  // cond_w columns of both halves of d_in are copies of x, the gradient w.r.t. them is discarded.
  const int cond_w = (has_d && c->d_conditioned) ? d_in : 0;
  const int nA = dD - cond_w;
  ParamList pg, pd;
  g_param_list(c, L.g_grads, &pg);
  pd.n = 0;
  pd.total = 0;
  if (has_d) param_list(c->d, c->d_sumW, c->d_sumb, c->d_sqW, c->d_sqb, L.d_grads, &pd);
  // In2OutHighwayNet: gate + combine around the MLPG (x_s = the first S columns of x)
  const bool hw = c->highway.static_dim > 0;
  HighwayArgs hwa{};
  if (hw) {
    char* cur = L.hw_dz;
    const Planes dz = carve_planes(cur, M, nS);
    hwa.x = x;
    hwa.x_rs = d_in;
    hwa.tx = L.hw_tx;
    hwa.gx = L.hw_gx;
    hwa.dz_hi = dz.hi;
    hwa.dz_lo = dz.lo;
    hwa.dz_pitch = dz.pitch;
    hwa.S = nS;
  }
  const HighwayArgs* hwp = hw ? &hwa : nullptr;
  ColList static_cols, adv_cols;
  static_cols.n = c->n_static_cols;
  for (int i = 0; i < c->n_static_cols; ++i) static_cols.c[i] = c->static_cols[i];
  adv_cols.n = has_d ? c->n_adv : 0;
  for (int i = 0; i < adv_cols.n; ++i) adv_cols.c[i] = c->adv_cols[i];
  // the adversarial columns are one contiguous window of y_hat_static (mgc with the first coefficients masked, the
  // hparams case): the discriminator's input gradient can be accumulated in place
  bool adv_window = has_d && !cond_w && adv_cols.n >= 1;
  for (int i = 1; i < adv_cols.n; ++i) adv_window = adv_window && adv_cols.c[i] == adv_cols.c[0] + i;
  ColList real_cols;          // adversarial columns taken from y directly: static_cols o adv_cols
  real_cols.n = adv_cols.n;
  for (int i = 0; i < adv_cols.n; ++i) {
    GANTTS_CHECK_ARG(adv_cols.c[i] >= 0 && adv_cols.c[i] < c->n_static_cols, "gan_step: adversarial column out of range");
    real_cols.c[i] = static_cols.c[adv_cols.c[i]];
  }
  gantts_mlp_t g = c->g, d = c->d;
  g.seed = gantts_gan_step_seed(seed, 0);
  // In2OutRNNHighwayNet: hidden2out's output feeds the MLPG, y_hat is x, and loss_mse sends no gradient into G
  const bool lstm = c->lstm.num_layers > 0;
  const float* gen_out = lstm ? L.lstm_out : y_hat;
  const bool mse_grad = c->mse_w != 0.f && !lstm;

  RedCounts cnt{};
  if (phases & GANTTS_STEP_EVAL) {
    NvtxRange r_eval("gantts_gan_step/eval");
    // ---- "test" phase of train.py:481-486 (model.eval(), phase != "train" at :273,:315): forwards and losses only
    GANTTS_CHECK_ARG(phases == GANTTS_STEP_EVAL, "gan_step: GANTTS_STEP_EVAL cannot be combined with training phases");
    g.dropout_p = 0.f;
    d.dropout_p = 0.f;
    if ((rc = gantts_sequence_mask(lengths_dev, L.mask, c->B, c->T, stream))) return rc;
    GANTTS_PDL_LAUNCH((set_scales_kernel), 1, 32, 0, st, L.scal, inv_frames, has_adv ? c->adv_w : 0.f, c->mge_w, c->mse_w, 1, lengths_dev, c->B, c->T);
    GANTTS_LAUNCH_CHECK("set_scales_kernel");
    if (has_d) {      // (the eval path keeps the two-step gather of the discriminator input)
      gather_cols_list_kernel<<<blocks_1d(M * nS, 1024), 256, 0, st>>>(y, d_out, L.y_static, nS, static_cols, M);
      GANTTS_LAUNCH_CHECK("gather_cols_list_kernel(y_static)");
    }
    if ((rc = generator_fwd(c, g, L, x, d_in, lengths_dev, M, y_hat, d_out, seed, false, st))) return rc;
    if (hw && (rc = highway_gate_fwd(c, g, L, M, st))) return rc;
    if ((rc = mlpg_fwd_impl(gen_out, (int64_t)c->T * d_out, d_out, y_hat_static, (int64_t)c->T * nS, nS,
                            c->mlpg_table, &c->streams, &c->windows, c->B, c->T, stream, hwp)))
      return rc;
    if (has_d) {
      gather_cols_list_kernel<<<blocks_1d(M * nA, 1024), 256, 0, st>>>(L.y_static, nS, L.d_in + cond_w, dD, adv_cols,
                                                                       M);
      GANTTS_LAUNCH_CHECK("gather_cols_list_kernel(real)");
      gather_cols_list_kernel<<<blocks_1d(M * nA, 1024), 256, 0, st>>>(y_hat_static, nS, L.d_in + M * dD + cond_w, dD,
                                                                       adv_cols, M);
      GANTTS_LAUNCH_CHECK("gather_cols_list_kernel(fake)");
      if (cond_w) {
        GANTTS_CUDA(cudaMemcpy2DAsync(L.d_in, (size_t)dD * sizeof(float), x, (size_t)d_in * sizeof(float),
                                      (size_t)cond_w * sizeof(float), (size_t)M, cudaMemcpyDeviceToDevice, st));
        GANTTS_CUDA(cudaMemcpy2DAsync(L.d_in + M * dD, (size_t)dD * sizeof(float), x, (size_t)d_in * sizeof(float),
                                      (size_t)cond_w * sizeof(float), (size_t)M, cudaMemcpyDeviceToDevice, st));
      }
      if ((rc = gantts_mlp_fwd(&d, L.d_in, dD, 2 * M, L.d_out, 1, L.d_tape, L.d_tape_bytes, stream))) return rc;
      if ((rc = launch_bce(L.d_out, L.mask, M, 2, 0, 1, L.scal + S_INV_T, nullptr, &L.red[R_REAL], &L.red[R_FAKE], st)))
        return rc;
      cnt.n[R_REAL] = cnt.n[R_FAKE] = bce_blocks(M);
      if (has_adv) {
        if ((rc = launch_bce(L.d_out + M, L.mask, M, 1, 0, 0, L.scal + S_INV_T, nullptr, &L.red[R_ADV], nullptr, st)))
          return rc;
        cnt.n[R_ADV] = bce_blocks(M);
      }
    }
    if ((rc = launch_sse(y_hat_static, nS, y, d_out, L.mask, M, nS, L.scal + S_MGE_SCALE, nullptr, 0, &L.red[R_MGE], st,
                         &static_cols)))
      return rc;
    if ((rc = launch_sse(y_hat, d_out, y, d_out, L.mask, M, d_out, L.scal + S_MSE_SCALE, nullptr, 0, &L.red[R_MSE], st)))
      return rc;
    cnt.n[R_MGE] = sse_blocks(M, nS);
    cnt.n[R_MSE] = sse_blocks(M, d_out);
    GANTTS_PDL_LAUNCH((finalize_losses_kernel), 1, RED_THREADS, 0, st, L.scal, losses_dev, L.red, cnt, has_adv ? c->adv_w : 0.f, c->mge_w,
                                                      c->mse_w, has_d ? 1 : 0);
    GANTTS_LAUNCH_CHECK("finalize_losses_kernel");
    return GANTTS_OK;
  }

  if (phases & 1) {
    NvtxRange r1("gantts_gan_step/phase1: G fwd, MLPG, MGE, D fwd+bwd");
    // ---- prologue: mask, scales, y_static (train.py:528-535)
    if ((rc = gantts_sequence_mask(lengths_dev, L.mask, c->B, c->T, stream))) return rc;
    GANTTS_PDL_LAUNCH((set_scales_kernel), 1, 32, 0, st, L.scal, inv_frames, has_adv ? c->adv_w : 0.f, c->mge_w, c->mse_w, 0, lengths_dev, c->B, c->T);
    GANTTS_LAUNCH_CHECK("set_scales_kernel");
    if (has_d && cond_w) {      // only the conditioned-discriminator fallback still gathers from y_static
      gather_cols_list_kernel<<<blocks_1d(M * nS, 1024), 256, 0, st>>>(y, d_out, L.y_static, nS, static_cols, M);
      GANTTS_LAUNCH_CHECK("gather_cols_list_kernel(y_static)");
    }
    // ---- apply_generator (train.py:336-355): G forward + MLPG
    if ((rc = generator_fwd(c, g, L, x, d_in, lengths_dev, M, y_hat, d_out, seed, true, st))) return rc;
    if (hw && (rc = highway_gate_fwd(c, g, L, M, st))) return rc;
    if ((rc = mlpg_fwd_impl(gen_out, (int64_t)c->T * d_out, d_out, y_hat_static, (int64_t)c->T * nS, nS,
                            c->mlpg_table, &c->streams, &c->windows, c->B, c->T, stream, hwp)))
      return rc;
    // MGE loss (train.py:291) and its gradient in one pass; the gradient INITIALISES g_static, the two discriminator
    // passes then accumulate their input gradients on top of it
    if ((rc = launch_sse(y_hat_static, nS, y, d_out, L.mask, M, nS, L.scal + S_MGE_SCALE, L.g_static, nS,
                         &L.red[R_MGE], st, &static_cols)))
      return rc;
    if (has_d) {
      // ---- update_discriminator (train.py:245-279): stacked real | fake batch of 2M rows
      d.seed = gantts_gan_step_seed(seed, 1);
      if (!cond_w) {
        // selected columns of y (real) and y_hat_static (fake) straight into the discriminator's input planes
        Planes din;
        if ((rc = mlp_tape_input_planes(&d, 2 * M, L.d_tape, L.d_tape_bytes, &din))) return rc;
        GANTTS_PDL_LAUNCH((gather_planes_kernel), blocks_1d(2 * M * nA, 1024), 256, 0, st, y, d_out, real_cols, M, y_hat_static, nS,
                                                                          adv_cols, M, din.hi, din.lo, din.pitch);
        GANTTS_LAUNCH_CHECK("gather_planes_kernel(real|fake)");
        if ((rc = mlp_fwd_impl(&d, nullptr, 0, 2 * M, L.d_out, 1, L.d_tape, L.d_tape_bytes, stream, true))) return rc;
      } else {
        gather_cols_list_kernel<<<blocks_1d(M * nA, 1024), 256, 0, st>>>(L.y_static, nS, L.d_in + cond_w, dD, adv_cols,
                                                                         M);
        GANTTS_LAUNCH_CHECK("gather_cols_list_kernel(real)");
        gather_cols_list_kernel<<<blocks_1d(M * nA, 1024), 256, 0, st>>>(y_hat_static, nS, L.d_in + M * dD + cond_w, dD,
                                                                         adv_cols, M);
        GANTTS_LAUNCH_CHECK("gather_cols_list_kernel(fake)");
        GANTTS_CUDA(cudaMemcpy2DAsync(L.d_in, (size_t)dD * sizeof(float), x, (size_t)d_in * sizeof(float),
                                      (size_t)cond_w * sizeof(float), (size_t)M, cudaMemcpyDeviceToDevice, st));
        GANTTS_CUDA(cudaMemcpy2DAsync(L.d_in + M * dD, (size_t)dD * sizeof(float), x, (size_t)d_in * sizeof(float),
                                      (size_t)cond_w * sizeof(float), (size_t)M, cudaMemcpyDeviceToDevice, st));
        if ((rc = gantts_mlp_fwd(&d, L.d_in, dD, 2 * M, L.d_out, 1, L.d_tape, L.d_tape_bytes, stream))) return rc;
      }
      // real and fake BCE terms, counts and dL/dD of both halves (train.py:262-270) in one launch
      if ((rc = launch_bce(L.d_out, L.mask, M, 2, 0, 1, L.scal + S_INV_T, L.g_dout, &L.red[R_REAL], &L.red[R_FAKE], st)))
        return rc;
      // loss_d.backward(): D parameter gradients + gradient w.r.t. the (fake) D input (rows M..2M-1 only).  When the
      // adversarial columns form one window of y_hat_static the last GEMM adds its result straight into g_static
      // (the scatter of the column gather's backward); otherwise it goes to g_din and a scatter kernel follows.
      if (adv_window) {
        float* win = L.g_static + adv_cols.c[0] - M * (int64_t)nS;      // row r of the stacked batch -> g_static[r - M]
        if ((rc = mlp_bwd_impl(&d, L.g_dout, 1, L.d_out, 1, 2 * M, L.d_tape, L.d_tape_bytes, win, nS, M, pd.gW, pd.gb, 0,
                               L.mlp_ws, L.mlp_ws_bytes, stream, 1)))
          return rc;
      } else {
        if ((rc = mlp_bwd_impl(&d, L.g_dout, 1, L.d_out, 1, 2 * M, L.d_tape, L.d_tape_bytes, L.g_din, dD, M, pd.gW,
                               pd.gb, 0, L.mlp_ws, L.mlp_ws_bytes, stream)))
          return rc;
        scatter_cols_list_add_kernel<<<blocks_1d(M * nA, 1024), 256, 0, st>>>(L.g_din + M * dD + cond_w, dD, L.g_static,
                                                                              nS, adv_cols, M);
        GANTTS_LAUNCH_CHECK("scatter_cols_list_add_kernel(fake)");
      }
    }
  }
  if (phases & 2) {
    NvtxRange r2("gantts_gan_step/phase2: D step, adv D fwd+bwd, MLPG bwd, G bwd");
    if (has_d) {
      // ---- clip_grad_norm_ + Adagrad on D (train.py:275-276)
      if ((rc = clip_opt_model(c, pd, L.opt_partial, L.scal + S_DSUMSQ, c->lr_d, c->wd_d, st)))
        return rc;
    }
    // ---- update_generator (train.py:282-320); the MGE term was evaluated in phase 1
    if (has_adv) {
      // third D forward: updated weights, fresh dropout mask (train.py:307)
      d.seed = gantts_gan_step_seed(seed, 2);
      if (!cond_w) {
        Planes din;
        if ((rc = mlp_tape_input_planes(&d, M, L.d_tape, L.d_tape_bytes, &din))) return rc;
        ColList none;
        none.n = 0;
        GANTTS_PDL_LAUNCH((gather_planes_kernel), blocks_1d(M * nA, 1024), 256, 0, st, y_hat_static, nS, adv_cols, M, nullptr, 0, none, 0,
                                                                      din.hi, din.lo, din.pitch);
        GANTTS_LAUNCH_CHECK("gather_planes_kernel(adv)");
        if ((rc = mlp_fwd_impl(&d, nullptr, 0, M, L.d_out, 1, L.d_tape, L.d_tape_bytes, stream, true))) return rc;
      } else if ((rc = gantts_mlp_fwd(&d, L.d_in + M * dD, dD, M, L.d_out, 1, L.d_tape, L.d_tape_bytes, stream))) {
        return rc;
      }
      if ((rc = launch_bce(L.d_out, L.mask, M, 1, 0, 0, L.scal + S_ADV_SCALE, L.g_dout, &L.red[R_ADV], nullptr, st)))
        return rc;
      if (adv_window) {
        if ((rc = mlp_bwd_impl(&d, L.g_dout, 1, L.d_out, 1, M, L.d_tape, L.d_tape_bytes, L.g_static + adv_cols.c[0], nS, 0,
                               nullptr, nullptr, 0, L.mlp_ws, L.mlp_ws_bytes, stream, 1)))
          return rc;
      } else {
        if ((rc = gantts_mlp_bwd(&d, L.g_dout, 1, L.d_out, 1, M, L.d_tape, L.d_tape_bytes, L.g_din, dD, nullptr,
                                 nullptr, 0, L.mlp_ws, L.mlp_ws_bytes, stream)))
          return rc;
        scatter_cols_list_add_kernel<<<blocks_1d(M * nA, 1024), 256, 0, st>>>(L.g_din + cond_w, dD, L.g_static, nS,
                                                                              adv_cols, M);
        GANTTS_LAUNCH_CHECK("scatter_cols_list_add_kernel(adv)");
      }
    }
    // ---- loss_g.backward(): MSE term (train.py:294) + MLPG backward + generator backward on the summed gradient.
    // With mse_w != 0 the MSE pass stores its gradient into g_yhat and the MLPG backward accumulates on top of it.
    if ((rc = launch_sse(y_hat, d_out, y, d_out, L.mask, M, d_out, L.scal + S_MSE_SCALE, mse_grad ? L.g_yhat : nullptr,
                         d_out, &L.red[R_MSE], st)))
      return rc;
    // no MSE gradient (mse_w == 0, the CLI default, train.py:15; or y_hat = x): nothing else adds to dL/dy_hat, so the
    // MLPG backward writes the operand planes of the generator's backward GEMMs directly (no fp32 matrix, no conversion)
    bool direct = false;
    if (!mse_grad) {
      Planes gp;
      if ((rc = mlp_bwd_gy_planes(&g, M, L.mlp_ws, L.mlp_ws_bytes, &gp))) return rc;
      rc = mlpg_bwd_planes(L.g_static, (int64_t)c->T * nS, nS, gp.hi, gp.lo, gp.pitch, c->mlpg_table, &c->streams,
                           &c->windows, c->B, c->T, stream, hwp);
      if (rc == GANTTS_OK) direct = true;
      else if (rc != GANTTS_E_UNSUPPORTED) return rc;
    }
    // (highway: the adjoint solves with Tx * g_static and leaves dz for the gate's weight gradient)
    if (!direct &&
        (rc = mlpg_bwd_impl(L.g_static, (int64_t)c->T * nS, nS, L.g_yhat, (int64_t)c->T * d_out, d_out, c->mlpg_table,
                            &c->streams, &c->windows, c->B, c->T, mse_grad ? 1 : 0, stream, hwp)))
      return rc;
    if (hw && (rc = highway_gate_bwd(c, g, L, M, st))) return rc;
    // (SRU or LSTM stack: hidden2out's input gradient is dL/dh of the stack's top layer)
    const bool sru = c->sru.num_layers > 0;
    float* gx = sru ? L.sru_dx : (lstm ? L.lstm_dh : nullptr);
    const int gx_rs = sru ? sru_ncols(c->sru) : (lstm ? lstm_ndir(c->lstm) * c->lstm.hidden : 0);
    if ((rc = mlp_bwd_impl(&g, direct ? nullptr : L.g_yhat, d_out, nullptr, 0, M, L.g_tape, L.g_tape_bytes, gx, gx_rs, 0,
                           pg.gW, pg.gb, 0, L.mlp_ws, L.mlp_ws_bytes, stream, -1, direct)))
      return rc;
    if (sru && (rc = sru_stack_bwd(c, L, pg, x, M, seed, st))) return rc;
    if (lstm && (rc = lstm_stack_bwd(c, L, pg, lengths_dev, M, seed, st))) return rc;
  }
  if (phases & 4) {
    NvtxRange r4("gantts_gan_step/phase4: G step, losses");
    // ---- clip_grad_norm_ + Adagrad on G (train.py:317-318), then the loss scalars
    if ((rc = clip_opt_model(c, pg, L.opt_partial, L.scal + S_GSUMSQ, c->lr_g, c->wd_g, st)))
      return rc;
    if (has_d) cnt.n[R_REAL] = cnt.n[R_FAKE] = bce_blocks(M);
    if (has_adv) cnt.n[R_ADV] = bce_blocks(M);
    cnt.n[R_MGE] = sse_blocks(M, nS);
    cnt.n[R_MSE] = sse_blocks(M, d_out);
    GANTTS_PDL_LAUNCH((finalize_losses_kernel), 1, RED_THREADS, 0, st, L.scal, losses_dev, L.red, cnt, has_adv ? c->adv_w : 0.f, c->mge_w,
                                                      c->mse_w, has_d ? 1 : 0);
    GANTTS_LAUNCH_CHECK("finalize_losses_kernel");
  }
  return GANTTS_OK;
}
