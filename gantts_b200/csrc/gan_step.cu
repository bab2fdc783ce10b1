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

// Spoofing-rate count of reference train.py:549-558: sum over valid frames of [D_ref > 0.5], row r = b * T + t valid
// when t < lengths[b].  One block in a fixed order; every partial sum is an integer below 2^24, so the float is exact.
// The count is STORED (count[0] = n), not accumulated.
__global__ void __launch_bounds__(RED_THREADS)
spoof_count_kernel(const float* __restrict__ Dv, const int64_t* __restrict__ lengths, int B, int T, float* __restrict__ count) {
  pdl_entry();
  __shared__ float sm[32];
  float v[1] = {0.f};
  const int64_t rows = (int64_t)B * T;
  for (int64_t r = threadIdx.x; r < rows; r += RED_THREADS) {
    const int64_t t = r % T;
    if (t < lengths[r / T] && Dv[r] > 0.5f) v[0] += 1.f;
  }
  block_sum<1>(v, sm);
  if (threadIdx.x == 0) count[0] = v[0];
}

// Deferred reductions: every loss kernel of the step leaves per-block partial sums in its own slot; the single
// finalize kernel at the end of the step reduces all of them (deterministic: fixed block order) -- no per-loss
// "finish" launch on the way.
enum RedSlot { R_REAL = 0, R_FAKE = 1, R_ADV = 2, R_MGE = 3, R_MSE = 4, R_COUNT = 5 };

struct RedCounts {
  int n[R_COUNT];      // blocks that wrote partials into slot i (0 = slot unused this step)
};

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

static_assert(GANTTS_MAX_STEP_TENSORS == OPT_MAX_TENSORS, "one model's tensor table is one TensorList of the clip kernels");
static_assert(2 + 2 * GANTTS_MAX_LAYERS <= GANTTS_MAX_STEP_TENSORS && 2 * GANTTS_MAX_SRU_LAYERS + 2 <= GANTTS_MAX_STEP_TENSORS &&
                  2 + 8 * GANTTS_MAX_LSTM_LAYERS + 2 <= GANTTS_MAX_STEP_TENSORS,
              "every generator the step accepts fits one tensor table");

struct Bound {
  float* p;               // parameter (updated in place)
  float* g;               // its gradient in the model's flat buffer
};
enum { WEIGHT = 0, BIAS = 1 };
enum { W_IH = 0, W_HH = 1, B_IH = 2, B_HH = 3 };     // nn.LSTM's tensors of one layer and direction

// One model's tensor table bound to its stages (g_param_list / d_param_list): the lists of the clip + optimiser kernels,
// and the pointers each stage uses.  The MLP layers' parameters go into the step's local gantts_mlp_t.
struct ParamList {
  int n;
  float* p[GANTTS_MAX_STEP_TENSORS];
  float* g[GANTTS_MAX_STEP_TENSORS];
  float* s[GANTTS_MAX_STEP_TENSORS];
  float* s2[GANTTS_MAX_STEP_TENSORS];                   // Adam: exp_avg_sq
  int64_t sizes[GANTTS_MAX_STEP_TENSORS];
  int64_t total;
  Bound gate[2];                                        // T.weight, T.bias
  Bound sru[GANTTS_MAX_SRU_LAYERS][2];                  // weight, bias per SRU layer
  Bound lstm[GANTTS_MAX_LSTM_LAYERS][2][4];             // [layer][direction] W_ih, W_hh, b_ih, b_hh
  float* gW[GANTTS_MAX_LAYERS];                         // gradients of the MLP layers
  float* gb[GANTTS_MAX_LAYERS];
};

static inline size_t al256(size_t v) { return (v + 255) / 256 * 256; }

// The step's workspace, carved front to back; every buffer starts on a 256-byte boundary (base nullptr: sizes only).
struct Arena {
  char* cur;
  char* take(size_t bytes) {
    char* p = cur;
    cur += al256(bytes);
    return p;
  }
  float* f32(size_t n) { return reinterpret_cast<float*>(take(n * sizeof(float))); }
};

// highway generator (zero bytes otherwise)
struct HighwayWs {
  float* tx;              // [M][S] gate sigmoid(x_s W_T^T + b_T)
  float* gx;              // [M][S] MLPG output Gx
  char* w;                // planes of W_T [S][S]
  char* dz;               // planes of dz [M][S]
  float* partial;         // split-K partials of dW_T / db_T
};

// SRU generator (zero bytes otherwise); per layer l:
struct SruWs {
  char* in[GANTTS_MAX_SRU_LAYERS];       // planes of the masked GEMM input [M][n_in] (layer l > 0: written by scan l-1)
  float* u[GANTTS_MAX_SRU_LAYERS];       // U = planes(x * mask_x) W  [M][ncols * k]
  float* c[GANTTS_MAX_SRU_LAYERS];       // cell states [M][ncols]
  float* h[GANTTS_MAX_SRU_LAYERS];       // fp32 h [M][ncols] below the top layer (the next layer's highway input)
  char* w[GANTTS_MAX_SRU_LAYERS];        // planes of W [n_in][ncols * k], then of W^T [ncols * k][n_in]
  float* partial[GANTTS_MAX_SRU_LAYERS]; // split-K partials of dW
  char* du;               // planes of dU [M][ncols * k] (one layer at a time)
  float* dx;              // [M][ncols] dL/dh of the top layer, then dX = dU W of each layer for the one below
  float* dxp;             // [M][ncols] highway gradient (k = 3) for the layer below
  float* bpart;           // [B][2 * ncols] bias-gradient partials
};

// LSTM stack of the generator, or of the discriminator at 2M rows (zero bytes otherwise); per layer l:
struct LstmWs {
  char* in[GANTTS_MAX_LSTM_LAYERS];      // planes of the GEMM input [M][n_in]: x (l = 0), else h_{l-1} * mask_{l-1}
  char* w[GANTTS_MAX_LSTM_LAYERS];       // planes of W_ih of both directions [ndir 4H][n_in], then [n_in][ndir 4H]
  float* bias[GANTTS_MAX_LSTM_LAYERS];   // b_ih + b_hh [ndir 4H]
  float* h[GANTTS_MAX_LSTM_LAYERS];      // h [M][ndir H]
  float* gates[GANTTS_MAX_LSTM_LAYERS];  // [ndir][M][4H]
  float* cells[GANTTS_MAX_LSTM_LAYERS];  // [ndir][M][H]
  float* xproj;           // [M][ndir 4H] xproj of one layer; in the backward, dgates of one layer
  float* out;             // [M][d_out] hidden2out's output, the MLPG's input
  float* dh;              // [M][ndir H] dL/dh of the top layer, then mask * dX of each layer for the one below
  char* dg;               // planes of dgates [M][ndir 4H]
  char* hp;               // planes of hprev [M][H]
  float* part[2][2];      // split-K partials per direction: [d][0] dW_ih | db_ih, [d][1] dW_hh (one layer at a time)
  unsigned int* bar;      // grid-barrier counters of the recurrence
  int64_t* lengths;       // discriminator: [2B] lengths of the stacked [real | fake] batch, the call's lengths twice
};

struct StepLayout {
  float* scal;
  float* mask;            // [M]
  float* d_in;            // [2M][dD]  rows 0..M-1 real, M..2M-1 fake (conditioned discriminator)
  float* d_out;           // [2M]
  float* g_dout;          // [2M]
  float* g_din;           // [2M][dD]
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
  HighwayWs hw;
  SruWs sru;
  LstmWs lstm;
  LstmWs d_lstm;
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

// width of the discriminator's input: the LSTM stack's, else the MLP's
static inline int d_in_width(const gantts_gan_step_t* c) {
  return c->d_lstm.num_layers > 0 ? c->d_lstm.in_dim : c->d.dims[0];
}

// tensor pl->n of table t: the next `size` elements of the model's flat gradient buffer (flat nullptr: counts only)
static Bound take_tensor(const gantts_step_tensors_t& t, int64_t size, float* flat, ParamList* pl) {
  const int i = pl->n++;
  const Bound b{t.param[i], flat ? flat + pl->total : nullptr};
  pl->p[i] = b.p;
  pl->g[i] = b.g;
  pl->s[i] = t.state[i];
  pl->s2[i] = t.state2[i];
  pl->sizes[i] = size;
  pl->total += size;
  return b;
}

// the layers of m in order [W, b] each: parameters into m->W / m->b, gradients into pl->gW / pl->gb
static void bind_mlp(const gantts_step_tensors_t& t, gantts_mlp_t* m, float* flat, ParamList* pl) {
  for (int l = 0; l < m->num_layers; ++l) {
    const Bound w = take_tensor(t, (int64_t)m->dims[l + 1] * m->dims[l], flat, pl);
    const Bound b = take_tensor(t, m->dims[l + 1], flat, pl);
    m->W[l] = w.p;
    m->b[l] = b.p;
    pl->gW[l] = w.g;
    pl->gb[l] = b.g;
  }
}

// [W_ih, W_hh, b_ih, b_hh] of every layer and direction of an LSTM stack into pl->lstm (none when ls.num_layers = 0)
static void bind_lstm(const gantts_step_tensors_t& t, const gantts_lstm_stack_t& ls, float* flat, ParamList* pl) {
  const int64_t G4 = 4 * (int64_t)ls.hidden;
  for (int l = 0; l < ls.num_layers; ++l)
    for (int d = 0; d < lstm_ndir(ls); ++d) {
      const int64_t sizes[4] = {G4 * lstm_nin(ls, l), G4 * ls.hidden, G4, G4};
      for (int i = 0; i < 4; ++i) pl->lstm[l][d][i] = take_tensor(t, sizes[i], flat, pl);
    }
}

// The generator's table bound from the shapes, in model.parameters() order: [weight, bias] of every SRU layer, or
// [T.weight, T.bias] of the highway gate and then [W_ih, W_hh, b_ih, b_hh] of every LSTM layer and direction; then the
// MLP layers (hidden2out alone after a stack).  pl->n is the tensor count the shapes give, pl->total the elements.
static void g_param_list(const gantts_gan_step_t* c, gantts_mlp_t* g, float* flat, ParamList* pl) {
  pl->n = 0;
  pl->total = 0;
  const gantts_step_tensors_t& t = c->g_tensors;
  const gantts_sru_stack_t& s = c->sru;
  for (int l = 0; l < s.num_layers; ++l) {
    pl->sru[l][WEIGHT] = take_tensor(t, (int64_t)sru_nin(s, l) * sru_ncols(s) * sru_k(s, l), flat, pl);
    pl->sru[l][BIAS] = take_tensor(t, 2 * (int64_t)sru_ncols(s), flat, pl);
  }
  const int64_t S = c->highway.static_dim;
  if (S > 0) {
    pl->gate[WEIGHT] = take_tensor(t, S * S, flat, pl);
    pl->gate[BIAS] = take_tensor(t, S, flat, pl);
  }
  bind_lstm(t, c->lstm, flat, pl);
  bind_mlp(t, g, flat, pl);
}

// The discriminator's table: [W_ih, W_hh, b_ih, b_hh] of every LSTM layer and direction (LSTMRNN / GRURNN), then the MLP
// layers (hidden2out alone after a stack).
static void d_param_list(const gantts_gan_step_t* c, gantts_mlp_t* d, float* flat, ParamList* pl) {
  pl->n = 0;
  pl->total = 0;
  bind_lstm(c->d_tensors, c->d_lstm, flat, pl);
  bind_mlp(c->d_tensors, d, flat, pl);
}

static int64_t d_param_count(const gantts_gan_step_t* c) {
  ParamList pl;
  gantts_mlp_t d = c->d;
  d_param_list(c, &d, nullptr, &pl);
  return pl.total;
}

static int64_t g_param_count(const gantts_gan_step_t* c) {
  ParamList pl;
  gantts_mlp_t g = c->g;
  g_param_list(c, &g, nullptr, &pl);
  return pl.total;
}

// One model's optimiser: the step's top-level fields for the generator, d_opt for the discriminator when it has its own
struct OptSpec {
  int kind;
  float beta1, beta2, eps;
  int64_t step;
};
static OptSpec g_opt_spec(const gantts_gan_step_t* c) { return {c->optimizer, c->beta1, c->beta2, c->eps, c->opt_step}; }
static OptSpec d_opt_spec(const gantts_gan_step_t* c) {
  const gantts_optimizer_t& o = c->d_opt;
  return o.own ? OptSpec{o.optimizer, o.beta1, o.beta2, o.eps, o.opt_step} : g_opt_spec(c);
}

// clip_grad_norm_ + optimiser step over one model's parameter list: two launches (partials, update), no finish kernel
static int clip_opt_model(const gantts_gan_step_t* c, const OptSpec& o, const ParamList& pl, float* partial, float* sumsq_out,
                          float lr, float wd, cudaStream_t st) {
  TensorList tl;
  const bool adam = o.kind == GANTTS_OPT_ADAM;
  int rc = fill(tl, pl.p, pl.g, pl.s, adam ? pl.s2 : nullptr, pl.sizes, 0, pl.n);
  if (rc) return rc;
  const int nb = blocks_for(tl.off[tl.n], OPT_MAX_BLOCKS);
  GANTTS_PDL_LAUNCH((sumsq_partial_kernel), nb, OPT_THREADS, 0, st, tl, partial);
  GANTTS_LAUNCH_CHECK("sumsq_partial_kernel");
  if (adam) {
    GANTTS_CHECK_ARG(o.step >= 1, "gan_step: Adam needs opt_step >= 1 (the number of the step being taken)");
    const AdamScales a = adam_scales(lr, o.beta1, o.beta2, o.step);
    GANTTS_PDL_LAUNCH((clip_adam_partials_kernel), nb, OPT_THREADS, 0, st, tl, partial, nb, sumsq_out, c->max_norm, o.beta1, o.beta2,
                      wd, o.eps, a.step_size, a.inv_sqrt_bc2);
    GANTTS_LAUNCH_CHECK("clip_adam_partials_kernel");
  } else {
    GANTTS_PDL_LAUNCH((clip_adagrad_partials_kernel), nb, OPT_THREADS, 0, st, tl, partial, nb, sumsq_out, c->max_norm, lr, wd, o.eps);
    GANTTS_LAUNCH_CHECK("clip_adagrad_partials_kernel");
  }
  return GANTTS_OK;
}

// a model's table: the tensor count its shapes give, every tensor and its optimiser state non-null (exp_avg_sq too when
// that model's optimiser is Adam)
static int check_table(const gantts_step_tensors_t& t, int want, int kind, const char* model) {
  GANTTS_CHECK_ARG(t.n == want, "gan_step: the %s table has %d tensors, its shapes give %d", model, t.n, want);
  for (int i = 0; i < t.n; ++i) {
    GANTTS_CHECK_ARG(t.param[i], "gan_step: null %s tensor %d", model, i);
    GANTTS_CHECK_ARG(t.state[i], "gan_step: null %s optimiser state of tensor %d", model, i);
    if (kind == GANTTS_OPT_ADAM)
      GANTTS_CHECK_ARG(t.state2[i], "gan_step: Adam needs exp_avg_sq for %s tensor %d", model, i);
  }
  return GANTTS_OK;
}

static int check_step(const gantts_gan_step_t* c) {
  GANTTS_CHECK_ARG(c, "gan_step: null config");
  GANTTS_CHECK_ARG(c->B >= 1 && c->T >= 1, "gan_step: bad batch shape");
  GANTTS_CHECK_ARG(c->optimizer == GANTTS_OPT_ADAGRAD || c->optimizer == GANTTS_OPT_ADAM, "gan_step: unknown optimizer %d", c->optimizer);
  if (c->optimizer == GANTTS_OPT_ADAM)
    GANTTS_CHECK_ARG(c->beta1 >= 0.f && c->beta1 < 1.f && c->beta2 >= 0.f && c->beta2 < 1.f, "gan_step: Adam betas out of range");
  const gantts_optimizer_t& dopt = c->d_opt;
  GANTTS_CHECK_ARG(dopt.own == 0 || dopt.own == 1, "gan_step: d_opt.own must be 0 (follow the step's optimiser) or 1 (got %d)",
                   dopt.own);
  if (dopt.own) {
    GANTTS_CHECK_ARG(dopt.optimizer == GANTTS_OPT_ADAGRAD || dopt.optimizer == GANTTS_OPT_ADAM,
                     "gan_step: unknown discriminator optimizer %d (d_opt.optimizer)", dopt.optimizer);
    if (dopt.optimizer == GANTTS_OPT_ADAM) {
      GANTTS_CHECK_ARG(dopt.beta1 >= 0.f && dopt.beta1 < 1.f && dopt.beta2 >= 0.f && dopt.beta2 < 1.f,
                       "gan_step: discriminator Adam betas out of range (d_opt.beta1 %g, d_opt.beta2 %g: each in [0, 1))",
                       (double)dopt.beta1, (double)dopt.beta2);
      GANTTS_CHECK_ARG(dopt.opt_step >= 1,
                       "gan_step: discriminator Adam needs d_opt.opt_step >= 1 (the number of the step being taken; got %lld)",
                       (long long)dopt.opt_step);
    }
  }
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
    // refused here rather than by the first backward, after a forward has run
    if (int rc = lstm_check_trainable(ls.hidden, lstm_ndir(ls))) return rc;
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
  }
  const gantts_lstm_stack_t& dl = c->d_lstm;
  GANTTS_CHECK_ARG(dl.num_layers >= 0 && dl.num_layers <= GANTTS_MAX_LSTM_LAYERS,
                   "gan_step: discriminator LSTM layer count %d not in [0, %d] (train larger stacks with GanTrainer)",
                   dl.num_layers, GANTTS_MAX_LSTM_LAYERS);
  if (c->w_d > 0.f) {
    GANTTS_CHECK_ARG(c->d.num_layers >= 1 && c->d.num_layers <= GANTTS_MAX_LAYERS, "gan_step: bad discriminator");
    if (dl.num_layers > 0) {
      // LSTMRNN / GRURNN with last_sigmoid (models.py:170-213): the LSTM stack, then hidden2out as a one-layer MLP
      GANTTS_CHECK_ARG(dl.bidirectional == 0 || dl.bidirectional == 1, "gan_step: bad discriminator LSTM bidirectional %d",
                       dl.bidirectional);
      GANTTS_CHECK_ARG(dl.hidden >= 4 && dl.hidden % 4 == 0,
                       "gan_step: discriminator LSTM hidden size %d is not a positive multiple of 4 (train it with GanTrainer)",
                       dl.hidden);
      GANTTS_CHECK_ARG(2 * c->B <= LSTM_MAX_B,
                       "gan_step: a recurrent discriminator runs the stacked [real | fake] batch of 2B sequences, at most "
                       "LSTM_MAX_B = %d, so B <= %d (B = %d); GanTrainer runs real and fake separately", LSTM_MAX_B,
                       LSTM_MAX_B / 2, c->B);
      GANTTS_CHECK_ARG(dl.dropout >= 0.f && dl.dropout < 1.f, "gan_step: discriminator LSTM dropout out of [0, 1)");
      const int nh = lstm_ndir(dl) * dl.hidden;
      GANTTS_CHECK_ARG(c->d.num_layers == 1 && c->d.dims[0] == nh,
                       "gan_step: with a discriminator LSTM stack d is hidden2out alone: 1 layer of input width %d (got %d "
                       "layer(s), input width %d)", nh, c->d.num_layers, c->d.dims[0]);
      if (int rc = lstm_check_trainable(dl.hidden, lstm_ndir(dl))) return rc;
    }
    const int cond_w = c->d_conditioned ? gen_in_width(c) : 0;
    GANTTS_CHECK_ARG(c->n_adv >= 1 && c->n_adv <= GANTTS_MAX_COLS && d_in_width(c) == cond_w + c->n_adv,
                     "gan_step: discriminator input width %d != %d conditioning + %d adversarial columns",
                     d_in_width(c), cond_w, c->n_adv);
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
  }
  // the tensor tables, bound from the shapes checked above
  ParamList pl;
  gantts_mlp_t g = c->g;
  g_param_list(c, &g, nullptr, &pl);
  int rc = check_table(c->g_tensors, pl.n, c->optimizer, "generator");
  if (rc) return rc;
  if (h.static_dim > 0)
    GANTTS_CHECK_ARG((reinterpret_cast<uintptr_t>(pl.gate[BIAS].p) & 15) == 0,
                     "gan_step: highway gate bias must be 16-byte aligned");
  if (!(c->w_d > 0.f)) return GANTTS_OK;
  gantts_mlp_t d = c->d;
  d_param_list(c, &d, nullptr, &pl);
  return check_table(c->d_tensors, pl.n, d_opt_spec(c).kind, "discriminator");
}

// out_cols: width of the head's fp32 output kept in w->out (the generator's hidden2out); seqs: sequences whose lengths
// w->lengths holds (the discriminator's stacked batch; 0 = none).  bwd = false: a stack that only runs forward (the
// spoofing-rate count's reference discriminator) -- no dh, dgates or hprev planes and no split-K partials.
static void layout_lstm(const gantts_lstm_stack_t& ls, int64_t M, int out_cols, int64_t seqs, Arena& a, LstmWs* w,
                        bool bwd = true) {
  const int nl = ls.num_layers, H = nl > 0 ? ls.hidden : 0, nd = lstm_ndir(ls), n4 = nd * 4 * H;
  const bool on = nl > 0, on_bwd = on && bwd;
  size_t part_ih = 0, part_hh = 0;
  for (int l = 0; l < nl; ++l) {
    const int ni = lstm_nin(ls, l);
    w->in[l] = a.take(2 * plane_bytes(M, ni));
    w->w[l] = a.take(2 * plane_bytes(n4, ni) + 2 * plane_bytes(ni, n4));
    w->bias[l] = a.f32((size_t)n4);
    w->h[l] = a.f32((size_t)M * nd * H);
    w->gates[l] = a.f32((size_t)M * n4);
    w->cells[l] = a.f32((size_t)M * nd * H);
    const size_t pi = mn_partial_bytes_upto(M, 4 * H, ni), ph = mn_partial_bytes_upto(M, 4 * H, H);
    part_ih = pi > part_ih ? pi : part_ih;
    part_hh = ph > part_hh ? ph : part_hh;
  }
  w->xproj = a.f32((size_t)M * n4);
  w->out = a.f32(on ? (size_t)M * out_cols : 0);
  w->dh = a.f32(bwd ? (size_t)M * nd * H : 0);
  w->dg = a.take(on_bwd ? 2 * plane_bytes(M, n4) : 0);
  w->hp = a.take(on_bwd ? 2 * plane_bytes(M, H) : 0);
  for (int d = 0; d < 2; ++d) {
    w->part[d][0] = reinterpret_cast<float*>(a.take(bwd && d < nd ? part_ih : 0));
    w->part[d][1] = reinterpret_cast<float*>(a.take(bwd && d < nd ? part_hh : 0));
  }
  w->bar = reinterpret_cast<unsigned int*>(a.take(on ? 256 : 0));
  w->lengths = reinterpret_cast<int64_t*>(a.take(on ? (size_t)seqs * sizeof(int64_t) : 0));
}

// One LSTM stack of the step: the generator's (In2OutRNNHighwayNet) or the discriminator's (LSTMRNN / GRURNN), with its
// workspace, its tensors and the stream its inter-layer masks are drawn from.
struct LstmStack {
  const gantts_lstm_stack_t* s;
  const LstmWs* w;
  const Bound (*p)[2][4];   // ParamList::lstm: [layer][direction] W_ih, W_hh, b_ih, b_hh
  int which;                // 0: gantts_lstm_mask_seed; 1, 2: gantts_d_lstm_mask_seed(seed, which, layer)
  uint64_t mask_seed(uint64_t seed, int l) const {
    return which == 0 ? gantts_lstm_mask_seed(seed, l) : gantts_d_lstm_mask_seed(seed, which, l);
  }
};

// LSTM layer l's workspace: planes of its GEMM input, and of W_ih of both directions [ndir 4H][n_in] then transposed
static Planes lstm_in_planes(const LstmStack& k, int l, int64_t M) {
  char* cur = k.w->in[l];
  return carve_planes(cur, M, lstm_nin(*k.s, l));
}
static void lstm_w_planes(const LstmStack& k, int l, Planes* w, Planes* wt) {
  const int ni = lstm_nin(*k.s, l), n4 = lstm_ndir(*k.s) * 4 * k.s->hidden;
  char* cur = k.w->w[l];
  *w = carve_planes(cur, n4, ni);
  *wt = carve_planes(cur, ni, n4);
}

static LstmStack g_lstm(const gantts_gan_step_t* c, const StepLayout& L, const ParamList& pg) {
  return LstmStack{&c->lstm, &L.lstm, pg.lstm, 0};
}

static void layout_highway(const gantts_gan_step_t* c, int64_t M, Arena& a, HighwayWs* w) {
  const int S = c->highway.static_dim;
  const bool on = S > 0;
  w->tx = a.f32(on ? (size_t)M * S : 0);
  w->gx = a.f32(on ? (size_t)M * S : 0);
  w->w = a.take(on ? 2 * plane_bytes(S, S) : 0);
  w->dz = a.take(on ? 2 * plane_bytes(M, S) : 0);
  w->partial = reinterpret_cast<float*>(a.take(on ? mn_partial_bytes_upto(M, S, S) : 0));
}

// x_s: the first S columns of x's operand planes -- the generator MLP's tape input, or the LSTM stack's layer-0 input
// (written by the generator's forward), so x is not converted twice.
static int gate_input_planes(const gantts_gan_step_t* c, const gantts_mlp_t& g, const StepLayout& L, int64_t M,
                             Planes* xs) {
  if (c->lstm.num_layers > 0) {
    *xs = lstm_in_planes(LstmStack{&c->lstm, &L.lstm, nullptr, 0}, 0, M);
  } else {
    int rc = mlp_tape_input_planes(&g, M, L.g_tape, L.g_tape_bytes, xs);
    if (rc) return rc;
  }
  xs->cols = c->highway.static_dim;
  return GANTTS_OK;
}

// Tx = sigmoid(x_s W_T^T + b_T)
static int highway_gate_fwd(const gantts_gan_step_t* c, const gantts_mlp_t& g, const ParamList& pg, const StepLayout& L,
                            int64_t M, cudaStream_t st) {
  const int S = c->highway.static_dim;
  Planes xs;
  int rc = gate_input_planes(c, g, L, M, &xs);
  if (rc) return rc;
  char* cur = L.hw.w;
  const Planes w = carve_planes(cur, S, S);
  if ((rc = launch_split(pg.gate[WEIGHT].p, S, S, S, w, 0, st))) return rc;
  EpiArgs e;
  e.epi = EPI_F32;
  e.C = L.hw.tx;
  e.ldc = S;
  e.bias = pg.gate[BIAS].p;
  e.act = GANTTS_ACT_SIGMOID;
  return launch_gemm_kk(xs, w, e, st);
}

// dW_T = dz^T x_s and db_T = colsum(dz) (ones-tile MMA) into the first S * S + S entries of the generator's buffer
static int highway_gate_bwd(const gantts_gan_step_t* c, const gantts_mlp_t& g, const ParamList& pg, const StepLayout& L,
                            int64_t M, cudaStream_t st) {
  const int S = c->highway.static_dim;
  Planes xs;
  int rc = gate_input_planes(c, g, L, M, &xs);
  if (rc) return rc;
  char* cur = L.hw.dz;
  const Planes dz = carve_planes(cur, M, S);
  ReduceList rl;
  if ((rc = launch_gemm_mn(dz, xs, pg.gate[WEIGHT].g, pg.gate[BIAS].g, 0, L.hw.partial, st, &rl))) return rc;
  return flush_reduce(rl, 0, st);
}

static void layout_sru(const gantts_gan_step_t* c, int64_t M, Arena& a, SruWs* w) {
  const gantts_sru_stack_t& s = c->sru;
  const int nl = s.num_layers, nc = nl > 0 ? sru_ncols(s) : 0;
  int maxku = 0;
  for (int l = 0; l < nl; ++l) {
    const int ni = sru_nin(s, l), ku = nc * sru_k(s, l);
    maxku = ku > maxku ? ku : maxku;
    w->in[l] = a.take(2 * plane_bytes(M, ni));
    w->u[l] = a.f32((size_t)M * ku);
    w->c[l] = a.f32((size_t)M * nc);
    if (l < nl - 1) w->h[l] = a.f32((size_t)M * nc);
    w->w[l] = a.take(2 * plane_bytes(ni, ku) + 2 * plane_bytes(ku, ni));
    w->partial[l] = reinterpret_cast<float*>(a.take(mn_partial_bytes_upto(M, ni, ku)));
  }
  w->du = a.take(nl > 0 ? 2 * plane_bytes(M, maxku) : 0);
  w->dx = a.f32((size_t)M * nc);
  w->dxp = a.f32((size_t)M * nc);
  w->bpart = a.f32((size_t)c->B * 2 * nc);
}

// SRU layer l's workspace: planes of its masked input, and of W [n_in][ncols k] then W^T [ncols k][n_in]
static Planes sru_in_planes(const gantts_gan_step_t* c, const StepLayout& L, int l, int64_t M) {
  char* cur = L.sru.in[l];
  return carve_planes(cur, M, sru_nin(c->sru, l));
}
static void sru_w_planes(const gantts_gan_step_t* c, const StepLayout& L, int l, Planes* w, Planes* wt) {
  const int ni = sru_nin(c->sru, l), ku = sru_ncols(c->sru) * sru_k(c->sru, l);
  char* cur = L.sru.w[l];
  *w = carve_planes(cur, ni, ku);
  *wt = carve_planes(cur, ku, ni);
}

// SRU stack forward (rnn.SRUCell per layer): the last layer's h goes unmasked into hidden2out's tape input planes, so
// the caller runs hidden2out with mlp_fwd_impl(..., input_ready = true).  train = false: no masks.
static int sru_stack_fwd(const gantts_gan_step_t* c, const gantts_mlp_t& g, const ParamList& pg, const StepLayout& L,
                         const float* x, int B, int T, uint64_t seed, bool train, cudaStream_t st) {
  const int64_t M = (int64_t)B * T;
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
      wl.W[l] = pg.sru[l][WEIGHT].p;
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
                      T, sru_mask(gantts_sru_mask_seed(seed, 0, 0), p_x), in0.hi, in0.lo, in0.pitch);
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
    e.C = L.sru.u[l];
    e.ldc = (int64_t)nc * k;
    if ((rc = launch_gemm_kk(sru_in_planes(c, L, l, M), wt, e, st))) return rc;
    const Planes out = last ? top : sru_in_planes(c, L, l + 1, M);
    SruStepFwd p{};
    p.u = L.sru.u[l];
    p.xh = k == 3 ? (l == 0 ? x : L.sru.h[l - 1]) : nullptr;
    p.xh_rs = l == 0 ? s.in_dim : nc;
    p.bias = pg.sru[l][BIAS].p;
    p.c = L.sru.c[l];
    p.h = L.sru.h[l];
    p.hi = out.hi;
    p.lo = out.lo;
    p.pitch = out.pitch;
    p.mh = sru_mask(gantts_sru_mask_seed(seed, l, 1), last ? 0.f : p_h);      // SRU(): no output dropout on the last layer
    p.mx = sru_mask(gantts_sru_mask_seed(seed, l + 1, 0), last ? 0.f : p_x);
    p.B = B;
    p.T = T;
    p.d = s.hidden;
    p.bidir = s.bidirectional;
    p.act = s.act;
    if ((rc = launch_sru_step_fwd(p, k, st))) return rc;
  }
  return GANTTS_OK;
}

// SRU stack backward from dL/dh of the top layer in L.sru.dx (hidden2out's input gradient), top layer first:
//   scan backward -> dU planes, highway gradient dx' (k = 3), bias partials -> bias gradient (fixed order over B)
//   dW = (x * mask_x)^T dU  (MN-major, lands in the [n_in][ncols k] parameter layout)
//   dX = dU W^T             (K-major on W as stored; not for layer 0)
// The layer below's dh = mask_x * dX + dx' is formed on load by its scan backward.
static int sru_stack_bwd(const gantts_gan_step_t* c, const StepLayout& L, const ParamList& pg, const float* x, int B, int T,
                         uint64_t seed, cudaStream_t st) {
  const int64_t M = (int64_t)B * T;
  const gantts_sru_stack_t& s = c->sru;
  const int nl = s.num_layers, nc = sru_ncols(s);
  int rc;
  ReduceList rl;
  for (int l = nl - 1; l >= 0; --l) {
    const int k = sru_k(s, l);
    const bool top = l == nl - 1;
    char* cur = L.sru.du;
    const Planes du = carve_planes(cur, M, (int64_t)nc * k);
    SruStepBwd p{};
    p.u = L.sru.u[l];
    p.xh = k == 3 ? (l == 0 ? x : L.sru.h[l - 1]) : nullptr;
    p.xh_rs = l == 0 ? s.in_dim : nc;
    p.bias = pg.sru[l][BIAS].p;
    p.c = L.sru.c[l];
    p.dx = L.sru.dx;
    p.dxp_in = top ? nullptr : L.sru.dxp;
    p.mxu = sru_mask(gantts_sru_mask_seed(seed, l + 1, 0), top ? 0.f : s.rnn_dropout);
    p.mh = sru_mask(gantts_sru_mask_seed(seed, l, 1), top ? 0.f : s.dropout);
    p.du_hi = du.hi;
    p.du_lo = du.lo;
    p.du_pitch = du.pitch;
    p.dxp_out = (k == 3 && l > 0) ? L.sru.dxp : nullptr;
    p.dbias_part = L.sru.bpart;
    p.B = B;
    p.T = T;
    p.d = s.hidden;
    p.bidir = s.bidirectional;
    p.act = s.act;
    if ((rc = launch_sru_step_bwd(p, k, st))) return rc;
    GANTTS_PDL_LAUNCH((sru_bias_reduce_kernel), (2 * nc + 255) / 256, 256, 0, st, L.sru.bpart, B, 2 * nc, pg.sru[l][BIAS].g);
    GANTTS_LAUNCH_CHECK("sru_bias_reduce_kernel");
    if ((rc = launch_gemm_mn(sru_in_planes(c, L, l, M), du, pg.sru[l][WEIGHT].g, nullptr, 0, L.sru.partial[l], st, &rl))) return rc;
    if (l > 0) {
      Planes w, wt;
      sru_w_planes(c, L, l, &w, &wt);
      EpiArgs e;
      e.epi = EPI_F32;
      e.C = L.sru.dx;
      e.ldc = nc;
      if ((rc = launch_gemm_kk(du, w, e, st))) return rc;
    }
  }
  return flush_reduce(rl, 0, st);
}

static LstmParams lstm_layer_params(const LstmStack& k, int l, const int64_t* lengths, int B, int T) {
  const gantts_lstm_stack_t& s = *k.s;
  LstmParams p{};
  p.W_hh = k.p[l][0][W_HH].p;
  if (s.bidirectional)      // the two directions' tensors are 4-byte aligned: their distance is a whole number of floats
    p.W_hh_dir = ((int64_t)reinterpret_cast<uintptr_t>(k.p[l][1][W_HH].p) - (int64_t)reinterpret_cast<uintptr_t>(k.p[l][0][W_HH].p)) /
                 (int64_t)sizeof(float);
  p.lengths = lengths;
  p.h_out = k.w->h[l];
  p.gates = k.w->gates[l];
  p.cells = k.w->cells[l];
  p.bar = k.w->bar;
  p.B = B;
  p.T = T;
  p.H = s.hidden;
  p.ndir = lstm_ndir(s);
  return p;
}

// LSTM stack forward (nn.LSTM on packed sequences, per-element dropout between layers) over B sequences of T steps: per
// layer one xproj GEMM over both directions, the cooperative recurrence, and one kernel that writes the next GEMM's operand
// planes of h * mask -- on the top layer the unmasked h into `top`, the head's tape input planes, so the caller runs the
// head with mlp_fwd_impl(..., input_ready = true).  x (row stride x_rs) is split into layer 0's input planes here; x =
// nullptr: the caller has written them.  train = false: no masks.
static int lstm_stack_fwd(const LstmStack& k, const float* x, int64_t x_rs, const Planes& top, const int64_t* lengths,
                          int B, int T, uint64_t seed, bool train, cudaStream_t st) {
  const int64_t M = (int64_t)B * T;
  const gantts_lstm_stack_t& s = *k.s;
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
      lstm_w_planes(k, l, &w, &wt);
      for (int d = 0; d < nd; ++d) {
        const int i = l * nd + d;
        wl.W[i] = k.p[l][d][W_IH].p;
        wl.N[i] = G4;
        wl.K[i] = lstm_nin(s, l);
        wl.hi[i] = w.hi + (int64_t)d * G4 * w.pitch;
        wl.lo[i] = w.lo + (int64_t)d * G4 * w.pitch;
        wl.pitch[i] = w.pitch;
        wl.thi[i] = wt.hi + (int64_t)d * G4;
        wl.tlo[i] = wt.lo + (int64_t)d * G4;
        wl.tpitch[i] = wt.pitch;
        wl.off[i + 1] = wl.off[i] + (int64_t)((G4 + 31) / 32) * ((wl.K[i] + 31) / 32);
        bl.a[i] = k.p[l][d][B_IH].p;
        bl.b[i] = k.p[l][d][B_HH].p;
        bl.out[i] = k.w->bias[l] + (int64_t)d * G4;
      }
    }
    const int nb = (int)(wl.off[wl.n] < num_sms() * 8 ? wl.off[wl.n] : num_sms() * 8);
    GANTTS_PDL_LAUNCH((split_weights_kernel), nb < 1 ? 1 : nb, 256, 0, st, wl);
    GANTTS_LAUNCH_CHECK("split_weights_kernel(lstm)");
    GANTTS_PDL_LAUNCH((lstm_bias_sum_kernel), (bl.n * G4 + 255) / 256, 256, 0, st, bl);
    GANTTS_LAUNCH_CHECK("lstm_bias_sum_kernel");
  }
  if (x && (rc = launch_split(x, x_rs, M, s.in_dim, lstm_in_planes(k, 0, M), 0, st))) return rc;
  for (int l = 0; l < nl; ++l) {
    const bool last = l == nl - 1;
    Planes w, wt;
    lstm_w_planes(k, l, &w, &wt);
    EpiArgs e;
    e.epi = EPI_F32;
    e.C = k.w->xproj;
    e.ldc = (int64_t)nd * G4;
    e.bias = k.w->bias[l];
    if ((rc = launch_gemm_kk(lstm_in_planes(k, l, M), w, e, st))) return rc;
    LstmParams p = lstm_layer_params(k, l, lengths, B, T);
    p.xproj = k.w->xproj;
    if ((rc = lstm_run(false, p, st))) return rc;
    const Planes out = last ? top : lstm_in_planes(k, l + 1, M);
    const float pl = last ? 0.f : p_drop;             // nn.LSTM: no dropout on the last layer's output
    GANTTS_PDL_LAUNCH((lstm_planes_kernel), blocks_1d(M * nh, 1024), 256, 0, st, k.w->h[l], M, nh,
                      k.mask_seed(seed, l), pl > 0.f ? (uint32_t)(pl * 65536.f + 0.5f) : 0u,
                      pl > 0.f ? 1.f / (1.f - pl) : 1.f, out.hi, out.lo, out.pitch);
    GANTTS_LAUNCH_CHECK("lstm_planes_kernel");
  }
  return GANTTS_OK;
}

// Layer 0's input gradient of a stack backward: columns [col0, col0 + cols) of dX_0 = dgates W_ih for the rows
// [row0, rows) into C (row r -> C + (r - row0) * ldc), stored or added (the discriminator's adversarial input columns of
// the fake rows, into g_static or g_din).
struct LstmInGrad {
  int64_t row0;
  int col0, cols;
  float* C;
  int64_t ldc;
  int accumulate;
};

// LSTM stack backward from dL/dh of the top layer in k.w->dh (the head's input gradient), top layer first:
//   recurrence backward -> dgates (fp32, in the xproj buffer) -> dgates planes
//   per direction: dW_ih and db_ih = dgates_d^T in (MN-major, ones-tile bias), dW_hh = dgates_d^T hprev_d (MN-major)
//   dX = dgates W_ih, times the mask of the layer below in the GEMM epilogue (not for layer 0)
//   db_hh = db_ih (b_ih and b_hh enter xproj as one sum)
// Each layer's split-K reductions go through one flush_reduce.  param_grads = false: the input gradients alone (the
// discriminator's adversarial pass); din: layer 0's input gradient, or none.
static int lstm_stack_bwd(const LstmStack& k, const int64_t* lengths, int B, int T, uint64_t seed, bool param_grads,
                          const LstmInGrad* din, cudaStream_t st) {
  const int64_t M = (int64_t)B * T;
  const gantts_lstm_stack_t& s = *k.s;
  const int nl = s.num_layers, H = s.hidden, nd = lstm_ndir(s), G4 = 4 * H, nh = nd * H;
  int rc;
  char* cur = k.w->dg;
  const Planes dg = carve_planes(cur, M, (int64_t)nd * G4);
  cur = k.w->hp;
  const Planes hp = carve_planes(cur, M, H);
  ReduceList rl;
  for (int l = nl - 1; l >= 0; --l) {
    LstmParams p = lstm_layer_params(k, l, lengths, B, T);
    p.dh_out = k.w->dh;
    p.dxproj = k.w->xproj;
    if ((rc = lstm_run(true, p, st))) return rc;
    if ((rc = launch_split(k.w->xproj, (int64_t)nd * G4, M, nd * G4, dg, 0, st))) return rc;
    const Planes in = lstm_in_planes(k, l, M);
    for (int d = 0; d < nd && param_grads; ++d) {
      Planes dgd = dg;
      dgd.hi += (int64_t)d * G4;
      dgd.lo += (int64_t)d * G4;
      dgd.cols = G4;
      if ((rc = launch_gemm_mn(dgd, in, k.p[l][d][W_IH].g, k.p[l][d][B_IH].g, 0, k.w->part[d][0], st, &rl))) return rc;
      GANTTS_PDL_LAUNCH((lstm_hprev_planes_kernel), blocks_1d(M * H, 1024), 256, 0, st, k.w->h[l], lengths, B, T, H, nd,
                        d, hp.hi, hp.lo, hp.pitch);
      GANTTS_LAUNCH_CHECK("lstm_hprev_planes_kernel");
      if ((rc = launch_gemm_mn(dgd, hp, k.p[l][d][W_HH].g, nullptr, 0, k.w->part[d][1], st, &rl))) return rc;
    }
    if (l > 0) {
      Planes w, wt;
      lstm_w_planes(k, l, &w, &wt);
      EpiArgs e;
      e.epi = EPI_F32;
      e.C = k.w->dh;
      e.ldc = nh;
      if (s.dropout > 0.f) {      // dh_{l-1} = mask_{l-1} * dX: LeakyReLU with slope 1 is the identity, then the mask
        e.act = GANTTS_ACT_LEAKY_DROPOUT;
        e.slope = 1.f;
        e.p = s.dropout;
        e.seed = k.mask_seed(seed, l - 1);
      }
      if ((rc = launch_gemm_kk(dg, wt, e, st))) return rc;
    } else if (din) {
      // the rows [row0, M) of dgates against the rows [col0, col0 + cols) of W_ih^T's planes
      Planes w, wt;
      lstm_w_planes(k, 0, &w, &wt);
      Planes a = dg;
      a.hi += din->row0 * dg.pitch;
      a.lo += din->row0 * dg.pitch;
      a.rows = M - din->row0;
      wt.hi += (int64_t)din->col0 * wt.pitch;
      wt.lo += (int64_t)din->col0 * wt.pitch;
      wt.rows = din->cols;
      EpiArgs e;
      e.epi = EPI_F32;
      e.C = din->C;
      e.ldc = din->ldc;
      e.accumulate = din->accumulate;
      if ((rc = launch_gemm_kk(a, wt, e, st))) return rc;
    }
    if (!param_grads) continue;
    if ((rc = flush_reduce(rl, 0, st))) return rc;
    for (int d = 0; d < nd; ++d)
      GANTTS_CUDA(cudaMemcpyAsync(k.p[l][d][B_HH].g, k.p[l][d][B_IH].g, (size_t)G4 * sizeof(float), cudaMemcpyDeviceToDevice, st));
  }
  return GANTTS_OK;
}

// The MLP stacks' backward passes run their weight gradients on the side stream (mlp_bwd_impl), beside the input-gradient
// chain; an SRU or LSTM generator's head and a recurrent discriminator's head stay on one stream (DESIGN.md section 5).
static bool g_side_bwd(const gantts_gan_step_t* c) { return c->sru.num_layers == 0 && c->lstm.num_layers == 0; }
static bool d_side_bwd(const gantts_gan_step_t* c) { return c->d_lstm.num_layers == 0; }
// Phase 1 runs the real half of the stacked discriminator pass on the branch stream, beside the generator's forward,
// when both stacks run their weight gradients on the side stream (DESIGN.md section 5).
static bool d_real_branch(const gantts_gan_step_t* c) { return g_side_bwd(c) && d_side_bwd(c); }

// The workspace is laid out once for the configured (B, T), the capacity: a call of shape (b, t) uses the first
// M = b * t rows of every per-row buffer, and the split-K partials are sized for every M up to the capacity.  So the flat
// gradient buffers (gantts_gan_step_grad_buffer) and every buffer one call leaves for the next (phases 1|2 then 4) sit at
// the same offsets whatever the call's shape.
static void layout(const gantts_gan_step_t* c, char* base, StepLayout* L) {
  const int64_t M = (int64_t)c->B * c->T;
  const int dD = d_in_width(c);
  *L = StepLayout{};      // the buffers of absent layers stay null
  Arena a{base};
  L->scal = a.f32(S_COUNT);
  L->mask = a.f32((size_t)M);
  L->d_in = a.f32((size_t)2 * M * dD);
  L->d_out = a.f32((size_t)2 * M);
  L->g_dout = a.f32((size_t)2 * M);
  L->g_din = a.f32((size_t)2 * M * dD);
  L->g_static = a.f32((size_t)M * c->n_static);
  L->g_yhat = a.f32((size_t)M * c->g.dims[c->g.num_layers]);
  L->g_grads = a.f32(g_param_count(c));
  L->d_grads = a.f32(d_param_count(c));
  L->g_tape_bytes = gantts_mlp_tape_bytes(&c->g, M);
  L->g_tape = a.take(L->g_tape_bytes);
  L->d_tape_bytes = gantts_mlp_tape_bytes(&c->d, 2 * M);
  L->d_tape = a.take(L->d_tape_bytes);
  const size_t gb = mlp_workspace_bytes(&c->g, M, true, g_side_bwd(c));
  const size_t db = mlp_workspace_bytes(&c->d, 2 * M, true, d_side_bwd(c));
  L->mlp_ws_bytes = gb > db ? gb : db;
  L->mlp_ws = a.take(L->mlp_ws_bytes);
  L->red = reinterpret_cast<RedWs*>(a.take(R_COUNT * sizeof(RedWs)));
  L->opt_partial = a.f32(OPT_MAX_BLOCKS);
  layout_highway(c, M, a, &L->hw);
  layout_sru(c, M, a, &L->sru);
  layout_lstm(c->lstm, M, c->g.dims[c->g.num_layers], 0, a, &L->lstm);
  layout_lstm(c->d_lstm, 2 * M, 0, 2 * (int64_t)c->B, a, &L->d_lstm);
  L->total = (size_t)(a.cur - base) + 256;
}

// Everything one gantts_gan_step call works with: the config, its workspace, the bound tables and the batch.
struct Step {
  const gantts_gan_step_t* c;
  StepLayout L;
  int B, T;                 // the call's shape (<= the configured capacity c->B, c->T), M = B * T
  const float* table;       // MLPG table of the call's T
  gantts_mlp_t g, d;      // local copies: parameters from the tables, per-forward dropout and seed
  ParamList pg, pd;
  const float *x, *y;
  const int64_t* lengths;
  float *y_hat, *y_hat_static;
  int64_t M;
  int d_in, d_out, dD, nS;  // d_in: the width (and row stride) of x -- the SRU or LSTM stack's input width when there is one
  int cond_w, nA;           // conditioning columns of D's input (copies of x), adversarial columns
  bool has_d, has_adv;
  bool train;               // dropout on (every call but the eval phase)
  bool adv_window;          // the adversarial columns are one contiguous window of y_hat_static
  HighwayArgs hwa;
  ColList static_cols, adv_cols, real_cols;
  uint64_t seed;
  void* stream;
  cudaStream_t st;
  cudaStream_t side;        // the library's side stream (nullptr when no pass of the configuration uses it)
  cudaStream_t branch;      // the library's branch stream (nullptr unless phase 1 runs D's real half on it)
  const HighwayArgs* hw() const { return c->highway.static_dim > 0 ? &hwa : nullptr; }
  bool d_rnn() const { return c->d_lstm.num_layers > 0; }
  // the discriminator's LSTM stack in forward `which` (1 stacked, 2 adversarial)
  LstmStack d_lstm(int which) const { return LstmStack{&c->d_lstm, &L.d_lstm, pd.lstm, which}; }
};

// batch prologue (train.py:528-535): sequence mask and loss scales.  zero_norms: a step that steps neither model (eval)
// or only D (D_ONLY) reports 0 for the gradient norm it does not compute, never an earlier step's value.
static int step_prologue(const Step& s, float inv_frames, bool zero_norms) {
  const gantts_gan_step_t* c = s.c;
  int rc = gantts_sequence_mask(s.lengths, s.L.mask, s.B, s.T, s.stream);
  if (rc) return rc;
  GANTTS_PDL_LAUNCH((set_scales_kernel), 1, 32, 0, s.st, s.L.scal, inv_frames, s.has_adv ? c->adv_w : 0.f, c->mge_w, c->mse_w,
                    zero_norms ? 1 : 0, s.lengths, s.B, s.T);
  GANTTS_LAUNCH_CHECK("set_scales_kernel");
  return GANTTS_OK;
}

// the loss scalars from every deferred partial the step wrote
static int step_finalize(const Step& s, float* losses_dev) {
  const gantts_gan_step_t* c = s.c;
  RedCounts cnt{};
  if (s.has_d) cnt.n[R_REAL] = cnt.n[R_FAKE] = bce_blocks(s.M);
  if (s.has_adv) cnt.n[R_ADV] = bce_blocks(s.M);
  cnt.n[R_MGE] = sse_blocks(s.M, s.nS);
  cnt.n[R_MSE] = sse_blocks(s.M, s.d_out);
  GANTTS_PDL_LAUNCH((finalize_losses_kernel), 1, RED_THREADS, 0, s.st, s.L.scal, losses_dev, s.L.red, cnt,
                    s.has_adv ? c->adv_w : 0.f, c->mge_w, c->mse_w, s.has_d ? 1 : 0);
  GANTTS_LAUNCH_CHECK("finalize_losses_kernel");
  return GANTTS_OK;
}

// Generator forward (apply_generator, train.py:336-355) into y_hat and y_hat_static: the MLP from x; or the SRU stack and
// then hidden2out on the planes it left in the tape; or the LSTM stack and then hidden2out into L.lstm.out, with y_hat a
// copy of x (models.py:118).  Then the highway gate, and the MLPG (with the highway combine) on the generator's output.
// train = false: no SRU / LSTM masks (the caller sets g.dropout_p).
static int generator_fwd(Step& s, bool train) {
  const gantts_gan_step_t* c = s.c;
  const StepLayout& L = s.L;
  const int64_t M = s.M;
  const float* gen_out = s.y_hat;
  int rc;
  if (c->lstm.num_layers > 0) {
    Planes top;
    if ((rc = mlp_tape_input_planes(&s.g, M, L.g_tape, L.g_tape_bytes, &top))) return rc;
    if ((rc = lstm_stack_fwd(g_lstm(c, L, s.pg), s.x, s.d_in, top, s.lengths, s.B, s.T, s.seed, train, s.st))) return rc;
    if ((rc = mlp_fwd_impl(&s.g, nullptr, 0, M, L.lstm.out, s.d_out, L.g_tape, L.g_tape_bytes, s.st, true))) return rc;
    GANTTS_CUDA(cudaMemcpyAsync(s.y_hat, s.x, (size_t)M * s.d_in * sizeof(float), cudaMemcpyDeviceToDevice, s.st));
    gen_out = L.lstm.out;
  } else if (c->sru.num_layers > 0) {
    if ((rc = sru_stack_fwd(c, s.g, s.pg, L, s.x, s.B, s.T, s.seed, train, s.st))) return rc;
    if ((rc = mlp_fwd_impl(&s.g, nullptr, 0, M, s.y_hat, s.d_out, L.g_tape, L.g_tape_bytes, s.st, true))) return rc;
  } else if ((rc = gantts_mlp_fwd(&s.g, s.x, s.d_in, M, s.y_hat, s.d_out, L.g_tape, L.g_tape_bytes, s.st))) {
    return rc;
  }
  if (c->highway.static_dim > 0 && (rc = highway_gate_fwd(c, s.g, s.pg, L, M, s.st))) return rc;
  return mlpg_fwd_impl(gen_out, (int64_t)s.T * s.d_out, s.d_out, s.y_hat_static, (int64_t)s.T * s.nS, s.nS, s.table,
                       &c->streams, &c->windows, s.B, s.T, s.stream, s.hw());
}

// Generator backward (loss_g.backward(), train.py:294-318) on dL/dy_hat_static summed in g_static, in order:
//   the MSE term (train.py:294), whose pass stores its gradient into g_yhat when it sends one (not when y_hat = x);
//   the MLPG adjoint: with no MSE gradient (mse_w == 0, the CLI default, train.py:15) nothing else adds to dL/dy_hat, so
//     it writes the operand planes of the head's backward GEMMs directly; otherwise it accumulates onto g_yhat in fp32
//     (highway: it solves with Tx * g_static and leaves dz for the gate's weight gradient);
//   the gate's backward; the head (g) backward, whose input gradient is dL/dh of the SRU / LSTM stack's top layer;
//   the stack's backward.
static int generator_bwd(Step& s) {
  const gantts_gan_step_t* c = s.c;
  const StepLayout& L = s.L;
  const int64_t M = s.M;
  const int d_out = s.d_out, nS = s.nS;
  const bool sru = c->sru.num_layers > 0, lstm = c->lstm.num_layers > 0;
  const bool mse_grad = c->mse_w != 0.f && !lstm;
  const cudaStream_t side = g_side_bwd(c) ? s.side : nullptr;
  int rc;
  // without a gradient the MSE pass writes its loss partials alone: it runs on the side stream, which the head's backward
  // joins back before it returns
  const cudaStream_t mse_st = side && !mse_grad ? side : s.st;
  if (mse_st != s.st && (rc = stream_wait(mse_st, s.st))) return rc;
  if ((rc = launch_sse(s.y_hat, d_out, s.y, d_out, L.mask, M, d_out, L.scal + S_MSE_SCALE, mse_grad ? L.g_yhat : nullptr,
                       d_out, &L.red[R_MSE], mse_st)))
    return rc;
  bool direct = false;
  if (!mse_grad) {
    Planes gp;
    if ((rc = mlp_bwd_gy_planes(&s.g, M, L.mlp_ws, L.mlp_ws_bytes, &gp))) return rc;
    rc = mlpg_bwd_planes(L.g_static, (int64_t)s.T * nS, nS, gp.hi, gp.lo, gp.pitch, s.table, &c->streams,
                         &c->windows, s.B, s.T, s.stream, s.hw());
    if (rc == GANTTS_OK) direct = true;
    else if (rc != GANTTS_E_UNSUPPORTED) return rc;
  }
  if (!direct &&
      (rc = mlpg_bwd_impl(L.g_static, (int64_t)s.T * nS, nS, L.g_yhat, (int64_t)s.T * d_out, d_out, s.table,
                          &c->streams, &c->windows, s.B, s.T, mse_grad ? 1 : 0, s.stream, s.hw())))
    return rc;
  if (c->highway.static_dim > 0 && (rc = highway_gate_bwd(c, s.g, s.pg, L, M, s.st))) return rc;
  float* gx = sru ? L.sru.dx : (lstm ? L.lstm.dh : nullptr);
  const int gx_rs = sru ? sru_ncols(c->sru) : (lstm ? lstm_ndir(c->lstm) * c->lstm.hidden : 0);
  if ((rc = mlp_bwd_impl(&s.g, direct ? nullptr : L.g_yhat, d_out, nullptr, 0, M, L.g_tape, L.g_tape_bytes, gx, gx_rs, 0,
                         s.pg.gW, s.pg.gb, 0, L.mlp_ws, L.mlp_ws_bytes, s.stream, -1, direct, side)))
    return rc;
  if (sru) return sru_stack_bwd(c, L, s.pg, s.x, s.B, s.T, s.seed, s.st);
  if (lstm) return lstm_stack_bwd(g_lstm(c, L, s.pg), s.lengths, s.B, s.T, s.seed, true, nullptr, s.st);
  return GANTTS_OK;
}

// A recurrent discriminator's LSTM stack on the stacked batch (2B sequences: the lengths twice) or the adversarial one,
// from x (the conditioned input d_in, row stride dD) or from input planes the caller gathered (x = nullptr), up to the
// top h in hidden2out's tape input planes.
static int discriminator_stack_fwd(Step& s, bool stacked, const float* x, const Planes& top) {
  const int64_t* lengths = s.lengths;
  if (stacked) {
    lengths = s.L.d_lstm.lengths;
    for (int half = 0; half < 2; ++half)
      GANTTS_CUDA(cudaMemcpyAsync(s.L.d_lstm.lengths + half * s.B, s.lengths, (size_t)s.B * sizeof(int64_t),
                                  cudaMemcpyDeviceToDevice, s.st));
  }
  return lstm_stack_fwd(s.d_lstm(stacked ? 1 : 2), x, s.dD, top, lengths, stacked ? 2 * s.B : s.B, s.T, s.seed, s.train,
                        s.st);
}

// Discriminator forward into L.d_out.  stacked: the [real | fake] batch of 2M rows (train.py:261,265), real = the
// adversarial columns of y's static features (real_cols), fake = those of y_hat_static; otherwise the fake rows alone
// (the adversarial forward, train.py:307).  Unconditioned, the columns go straight into the operand planes of D's tape;
// conditioned (train.py:254-256), D's input cat((x, columns), -1) is assembled in fp32 d_in, and the adversarial forward
// re-uses the fake half the stacked one assembled.  half (stacked, with the weight planes already split by
// mlp_split_weights): 0 = the real rows [0, M) alone, 1 = the fake rows [M, 2M) alone; -1 = the whole pass.
static int discriminator_fwd(Step& s, bool stacked, int half = -1) {
  const StepLayout& L = s.L;
  const int64_t M = s.M, rows = stacked ? 2 * M : M;
  const int64_t r0 = half == 1 ? M : 0, r1 = half == 0 ? M : rows;
  int rc;
  Planes tape_in;
  if ((rc = mlp_tape_input_planes(&s.d, rows, L.d_tape, L.d_tape_bytes, &tape_in))) return rc;
  // a recurrent D (LSTMRNN / GRURNN): its stack reads the input planes, hidden2out the stack's top h in the tape
  const Planes din = s.d_rnn() ? lstm_in_planes(s.d_lstm(stacked ? 1 : 2), 0, rows) : tape_in;
  ColList none;
  none.n = 0;
  if (!s.cond_w) {
    if (stacked && half < 0) {
      GANTTS_PDL_LAUNCH((gather_planes_kernel), blocks_1d(2 * M * s.nA, 1024), 256, 0, s.st, s.y, s.d_out, s.real_cols, M,
                        s.y_hat_static, s.nS, s.adv_cols, M, din.hi, din.lo, din.pitch);
      GANTTS_LAUNCH_CHECK("gather_planes_kernel(real|fake)");
    } else if (half == 0) {
      GANTTS_PDL_LAUNCH((gather_planes_kernel), blocks_1d(M * s.nA, 1024), 256, 0, s.st, s.y, s.d_out, s.real_cols, M,
                        nullptr, 0, none, 0, din.hi, din.lo, din.pitch);
      GANTTS_LAUNCH_CHECK("gather_planes_kernel(real)");
    } else {
      // the fake rows: the adversarial forward's batch, or the stacked one's second half
      const Planes fk = plane_rows(din, r0, r0 + M);
      GANTTS_PDL_LAUNCH((gather_planes_kernel), blocks_1d(M * s.nA, 1024), 256, 0, s.st, s.y_hat_static, s.nS, s.adv_cols, M,
                        nullptr, 0, none, 0, fk.hi, fk.lo, fk.pitch);
      GANTTS_LAUNCH_CHECK("gather_planes_kernel(fake)");
    }
    if (s.d_rnn() && (rc = discriminator_stack_fwd(s, stacked, nullptr, tape_in))) return rc;
    if (half >= 0) return mlp_fwd_rows(&s.d, nullptr, 0, rows, r0, r1, L.d_out, 1, L.d_tape, L.d_tape_bytes, s.st);
    return mlp_fwd_impl(&s.d, nullptr, 0, rows, L.d_out, 1, L.d_tape, L.d_tape_bytes, s.stream, true);
  }
  const int dD = s.dD;
  if (stacked) {
    if (half != 1) {
      gather_cols_list_kernel<<<blocks_1d(M * s.nA, 1024), 256, 0, s.st>>>(s.y, s.d_out, L.d_in + s.cond_w, dD, s.real_cols, M);
      GANTTS_LAUNCH_CHECK("gather_cols_list_kernel(real)");
    }
    if (half != 0) {
      gather_cols_list_kernel<<<blocks_1d(M * s.nA, 1024), 256, 0, s.st>>>(s.y_hat_static, s.nS, L.d_in + M * dD + s.cond_w,
                                                                            dD, s.adv_cols, M);
      GANTTS_LAUNCH_CHECK("gather_cols_list_kernel(fake)");
    }
    for (int64_t h = r0 / M; h < r1 / M; ++h)
      GANTTS_CUDA(cudaMemcpy2DAsync(L.d_in + h * M * dD, (size_t)dD * sizeof(float), s.x, (size_t)s.d_in * sizeof(float),
                                    (size_t)s.cond_w * sizeof(float), (size_t)M, cudaMemcpyDeviceToDevice, s.st));
    if (half >= 0) return mlp_fwd_rows(&s.d, L.d_in, dD, rows, r0, r1, L.d_out, 1, L.d_tape, L.d_tape_bytes, s.st);
  }
  if (s.d_rnn()) {
    if ((rc = discriminator_stack_fwd(s, stacked, L.d_in + (stacked ? 0 : M * dD), tape_in))) return rc;
    return mlp_fwd_impl(&s.d, nullptr, 0, rows, L.d_out, 1, L.d_tape, L.d_tape_bytes, s.stream, true);
  }
  return gantts_mlp_fwd(&s.d, L.d_in + (stacked ? 0 : M * dD), dD, rows, L.d_out, 1, L.d_tape, L.d_tape_bytes, s.stream);
}

// Discriminator backward from dL/dD in g_dout, adding the gradient w.r.t. the fake rows' adversarial columns into
// g_static.  stacked: loss_d.backward() on the [real | fake] batch, with D's parameter gradients; otherwise the
// adversarial batch, input gradient only.  When the adversarial columns form one window of y_hat_static the last GEMM
// adds its result straight into g_static (the scatter of the column gather's backward); otherwise it goes to g_din and a
// scatter kernel follows.  input_grad = false (the D-only step, where nothing consumes dL/dy_hat_static): parameter
// gradients alone.  fake_chain (stacked): the real rows' input-gradient chain already ran (discriminator_real_half), the
// chain covers the fake rows.
static int discriminator_bwd(Step& s, bool stacked, bool input_grad = true, bool fake_chain = false) {
  const StepLayout& L = s.L;
  const int64_t M = s.M, skip = stacked ? M : 0;      // the real rows' input gradient is not needed
  float* const* gW = stacked ? s.pd.gW : nullptr;
  float* const* gb = stacked ? s.pd.gb : nullptr;
  // in place: row r of the batch -> g_static[r - skip]
  float* gx = !input_grad ? nullptr : (s.adv_window ? L.g_static + s.adv_cols.c[0] - skip * (int64_t)s.nS : L.g_din);
  int rc;
  if (s.d_rnn()) {
    // hidden2out's backward gives dL/dh of the stack's top layer; the stack's backward computes the parameter gradients
    // on the stacked pass only, and the input gradient w.r.t. the adversarial columns of the fake rows alone
    const LstmStack k = s.d_lstm(stacked ? 1 : 2);
    const int nh = lstm_ndir(s.c->d_lstm) * s.c->d_lstm.hidden;
    if ((rc = mlp_bwd_impl(&s.d, L.g_dout, 1, L.d_out, 1, skip + M, L.d_tape, L.d_tape_bytes, k.w->dh, nh, 0, gW, gb, 0,
                           L.mlp_ws, L.mlp_ws_bytes, s.stream, 0)))
      return rc;
    // row r of the batch -> row r - skip of g_static's adversarial window (in place), else of g_din's adversarial columns
    LstmInGrad din{};
    if (input_grad) {
      const int64_t rs = s.adv_window ? s.nS : s.dD;
      din = LstmInGrad{skip, s.cond_w, s.nA, (s.adv_window ? gx : gx + s.cond_w) + skip * rs, rs, s.adv_window ? 1 : 0};
    }
    if ((rc = lstm_stack_bwd(k, stacked ? L.d_lstm.lengths : s.lengths, stacked ? 2 * s.B : s.B, s.T, s.seed, stacked,
                             input_grad ? &din : nullptr, s.st)))
      return rc;
  } else {
    // the weight gradients on the side stream read both halves' gradient planes: it waits for the real half's branch
    if (fake_chain && (rc = stream_wait(s.side, s.branch))) return rc;
    if ((rc = mlp_bwd_impl(&s.d, L.g_dout, 1, L.d_out, 1, skip + M, L.d_tape, L.d_tape_bytes, gx, s.adv_window ? s.nS : s.dD,
                           skip, gW, gb, 0, L.mlp_ws, L.mlp_ws_bytes, s.stream, s.adv_window ? 1 : -1, false,
                           stacked ? s.side : nullptr, fake_chain ? M : 0)))
      return rc;
  }
  if (s.adv_window || !input_grad) return GANTTS_OK;
  scatter_cols_list_add_kernel<<<blocks_1d(M * s.nA, 1024), 256, 0, s.st>>>(L.g_din + skip * s.dD + s.cond_w, s.dD,
                                                                             L.g_static, s.nS, s.adv_cols, M);
  GANTTS_LAUNCH_CHECK("scatter_cols_list_add_kernel");
  return GANTTS_OK;
}

// The real half of phase 1's stacked discriminator pass, on the branch stream from the end of the prologue: the real
// rows' input gathered into D's tape, their forward, their BCE terms and dL/dD, and their input-gradient chain.  None
// of it reads what the generator writes, so it runs beside the generator's forward, the MGE pass and the fake half's
// forward.  D's weight planes are split on the caller's stream first, for both halves.  The stacked backward
// (discriminator_bwd with fake_chain) makes the side stream wait for the branch before D's weight gradients, which read
// both halves' gradient planes, and its closing join brings both back into the caller's stream.
static int discriminator_real_half(Step& s) {
  const StepLayout& L = s.L;
  int rc;
  if ((rc = mlp_split_weights(&s.d, 2 * s.M, L.d_tape, L.d_tape_bytes, s.st))) return rc;
  if ((rc = stream_wait(s.branch, s.st))) return rc;
  Step b = s;            // the same step, enqueued on the branch stream
  b.st = s.branch;
  b.stream = s.branch;
  if ((rc = discriminator_fwd(b, true, 0))) return rc;
  if ((rc = launch_bce(L.d_out, L.mask, s.M, 1, 0, 0, L.scal + S_INV_T, L.g_dout, &L.red[R_REAL], nullptr, b.st)))
    return rc;
  return mlp_bwd_impl(&s.d, L.g_dout, 1, L.d_out, 1, 2 * s.M, L.d_tape, L.d_tape_bytes, nullptr, 0, 0, nullptr, nullptr,
                      0, L.mlp_ws, L.mlp_ws_bytes, b.stream, -1, false, nullptr, 0, s.M);
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

// after every generator LSTM index 2 * GANTTS_MAX_SRU_LAYERS + layer of the same stream
extern "C" uint64_t gantts_d_lstm_mask_seed(uint64_t seed, int which, int layer) {
  return gantts_mlp_layer_seed(gantts_gan_step_seed(seed, 3),
                               2 * GANTTS_MAX_SRU_LAYERS + GANTTS_MAX_LSTM_LAYERS * which + layer);
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
  *count = which == 0 ? g_param_count(c) : d_param_count(c);
  return GANTTS_OK;
}

extern "C" int gantts_gan_step(const gantts_gan_step_t* c, int phases, const float* x, const float* y,
                               const int64_t* lengths_dev, float inv_frames, uint64_t seed, float* y_hat,
                               float* y_hat_static, float* losses_dev, void* workspace, size_t workspace_bytes,
                               void* stream) {
  GANTTS_CHECK_ARG(c, "gan_step: null config");
  return gantts_gan_step_shaped(c, c->B, c->T, c->mlpg_table, phases, x, y, lengths_dev, inv_frames, seed, y_hat,
                                y_hat_static, losses_dev, workspace, workspace_bytes, stream);
}

extern "C" int gantts_gan_step_shaped(const gantts_gan_step_t* c, int B, int T, const float* mlpg_table, int phases,
                                      const float* x, const float* y, const int64_t* lengths_dev, float inv_frames,
                                      uint64_t seed, float* y_hat, float* y_hat_static, float* losses_dev, void* workspace,
                                      size_t workspace_bytes, void* stream) {
  int rc = check_step(c);
  if (rc) return rc;
  // the call's shape is at most the configured one, the capacity the workspace was laid out for
  GANTTS_CHECK_ARG(B >= 1 && B <= c->B, "gan_step_shaped: batch size B = %d must be in [1, configured B = %d]", B, c->B);
  GANTTS_CHECK_ARG(T >= 1 && T <= c->T, "gan_step_shaped: padded length T = %d must be in [1, configured T = %d]", T, c->T);
  GANTTS_CHECK_ARG(mlpg_table, "gan_step_shaped: null MLPG table (it must be gantts_mlpg_table(windows, T) of the call's T)");
  // the discriminator warm-up (train.py --discriminator-warmup, :696 update_g = False): D steps, G is left alone
  const bool d_only = (phases & GANTTS_STEP_D_ONLY) != 0;
  if (d_only) {
    GANTTS_CHECK_ARG(!(phases & GANTTS_STEP_EVAL),
                     "gan_step: GANTTS_STEP_D_ONLY cannot be combined with GANTTS_STEP_EVAL (the test phase updates nothing)");
    GANTTS_CHECK_ARG(c->w_d > 0.f, "gan_step: GANTTS_STEP_D_ONLY trains the discriminator and needs w_d > 0 (got %g)",
                     (double)c->w_d);
  }
  GANTTS_CHECK_ARG(x && y && lengths_dev && y_hat && y_hat_static && losses_dev, "gan_step: null pointer");
  size_t need = gantts_gan_step_workspace_bytes(c);
  if (!workspace || workspace_bytes < need) {
    set_error("gan_step: workspace too small (%zu < %zu)", workspace_bytes, need);
    return GANTTS_E_WORKSPACE;
  }
  Step s;
  s.c = c;
  s.B = B;
  s.T = T;
  s.table = mlpg_table;
  s.stream = stream;
  s.st = as_stream(stream);
  s.side = nullptr;
  s.branch = nullptr;
  if ((g_side_bwd(c) || d_side_bwd(c)) && (rc = side_stream(&s.side))) return rc;
  if (d_real_branch(c) && (rc = branch_stream(&s.branch))) return rc;
  layout(c, reinterpret_cast<char*>(al256(reinterpret_cast<uintptr_t>(workspace))), &s.L);
  const StepLayout& L = s.L;
  const int64_t M = s.M = (int64_t)B * T;
  s.x = x;
  s.y = y;
  s.lengths = lengths_dev;
  s.y_hat = y_hat;
  s.y_hat_static = y_hat_static;
  s.seed = seed;
  s.train = !(phases & GANTTS_STEP_EVAL);
  s.d_in = gen_in_width(c);
  s.d_out = c->g.dims[c->g.num_layers];
  s.dD = d_in_width(c);
  const int nS = s.nS = c->n_static;
  s.has_d = c->w_d > 0.f;
  s.has_adv = s.has_d && c->adv_w > 0.f && !d_only;
  // discriminator_linguistic_condition (train.py:254-256,302-303): D sees cat((x, y_adv), -1); the first cond_w columns
  // of both halves of d_in are copies of x, the gradient w.r.t. them is discarded.
  s.cond_w = (s.has_d && c->d_conditioned) ? s.d_in : 0;
  s.nA = s.dD - s.cond_w;
  s.g = c->g;
  s.d = c->d;
  g_param_list(c, &s.g, L.g_grads, &s.pg);
  s.pd.n = 0;
  s.pd.total = 0;
  if (s.has_d) d_param_list(c, &s.d, L.d_grads, &s.pd);
  // In2OutHighwayNet: gate + combine around the MLPG (x_s = the first S columns of x)
  s.hwa = HighwayArgs{};
  if (c->highway.static_dim > 0) {
    char* cur = L.hw.dz;
    const Planes dz = carve_planes(cur, M, nS);
    s.hwa = HighwayArgs{x, s.d_in, L.hw.tx, L.hw.gx, dz.hi, dz.lo, dz.pitch, nS};
  }
  s.static_cols.n = c->n_static_cols;
  for (int i = 0; i < c->n_static_cols; ++i) s.static_cols.c[i] = c->static_cols[i];
  s.adv_cols.n = s.has_d ? c->n_adv : 0;
  for (int i = 0; i < s.adv_cols.n; ++i) s.adv_cols.c[i] = c->adv_cols[i];
  // the adversarial columns are one contiguous window of y_hat_static (mgc with the first coefficients masked, the
  // hparams case): the discriminator's input gradient can be accumulated in place
  s.adv_window = s.has_d && !s.cond_w && s.adv_cols.n >= 1;
  for (int i = 1; i < s.adv_cols.n; ++i) s.adv_window = s.adv_window && s.adv_cols.c[i] == s.adv_cols.c[0] + i;
  s.real_cols.n = s.adv_cols.n;          // adversarial columns taken from y directly: static_cols o adv_cols
  for (int i = 0; i < s.adv_cols.n; ++i) {
    GANTTS_CHECK_ARG(s.adv_cols.c[i] >= 0 && s.adv_cols.c[i] < c->n_static_cols, "gan_step: adversarial column out of range");
    s.real_cols.c[i] = s.static_cols.c[s.adv_cols.c[i]];
  }
  s.g.seed = gantts_gan_step_seed(seed, 0);
  const cudaStream_t st = s.st;

  if (phases & GANTTS_STEP_EVAL) {
    NvtxRange r_eval("gantts_gan_step/eval");
    // ---- "test" phase of train.py:481-486 (model.eval(), phase != "train" at :273,:315): forwards and losses only
    GANTTS_CHECK_ARG(phases == GANTTS_STEP_EVAL, "gan_step: GANTTS_STEP_EVAL cannot be combined with training phases");
    s.g.dropout_p = 0.f;
    s.d.dropout_p = 0.f;
    if ((rc = step_prologue(s, inv_frames, true))) return rc;
    if ((rc = generator_fwd(s, false))) return rc;
    if (s.has_d) {
      if ((rc = discriminator_fwd(s, true))) return rc;
      if ((rc = launch_bce(L.d_out, L.mask, M, 2, 0, 1, L.scal + S_INV_T, nullptr, &L.red[R_REAL], &L.red[R_FAKE], st)))
        return rc;
      // the adversarial loss re-uses the fake half: no dropout and no D step in between
      if (s.has_adv &&
          (rc = launch_bce(L.d_out + M, L.mask, M, 1, 0, 0, L.scal + S_INV_T, nullptr, &L.red[R_ADV], nullptr, st)))
        return rc;
    }
    if ((rc = launch_sse(y_hat_static, nS, y, s.d_out, L.mask, M, nS, L.scal + S_MGE_SCALE, nullptr, 0, &L.red[R_MGE], st,
                         &s.static_cols)))
      return rc;
    if ((rc = launch_sse(y_hat, s.d_out, y, s.d_out, L.mask, M, s.d_out, L.scal + S_MSE_SCALE, nullptr, 0, &L.red[R_MSE],
                         st)))
      return rc;
    return step_finalize(s, losses_dev);
  }

  if (phases & 1) {
    NvtxRange r1("gantts_gan_step/phase1: G fwd, MLPG, MGE, D fwd+bwd");
    if ((rc = step_prologue(s, inv_frames, d_only))) return rc;
    const bool branch = s.has_d && d_real_branch(c);
    if (branch) {
      s.d.seed = gantts_gan_step_seed(seed, 1);
      if ((rc = discriminator_real_half(s))) return rc;
    }
    if ((rc = generator_fwd(s, true))) return rc;
    // MGE loss (train.py:291) and its gradient in one pass; the gradient INITIALISES g_static, the two discriminator
    // passes then accumulate their input gradients on top of it.  D-only: forward values of MGE and MSE alone (the
    // generator backward that would evaluate MSE does not run).
    if ((rc = launch_sse(y_hat_static, nS, y, s.d_out, L.mask, M, nS, L.scal + S_MGE_SCALE, d_only ? nullptr : L.g_static, nS,
                         &L.red[R_MGE], st, &s.static_cols)))
      return rc;
    if (d_only && (rc = launch_sse(y_hat, s.d_out, y, s.d_out, L.mask, M, s.d_out, L.scal + S_MSE_SCALE, nullptr, 0,
                                   &L.red[R_MSE], st)))
      return rc;
    if (s.has_d) {
      // ---- update_discriminator (train.py:245-279)
      s.d.seed = gantts_gan_step_seed(seed, 1);
      if (branch) {
        // the fake half; the real half runs on the branch stream (discriminator_real_half), with the same launches per
        // half, so both halves' terms, partials and gradients are those of the whole pass, bit for bit
        if ((rc = discriminator_fwd(s, true, 1))) return rc;
        if ((rc = launch_bce(L.d_out + M, L.mask, M, 1, 1, 0, L.scal + S_INV_T, L.g_dout + M, &L.red[R_FAKE], nullptr,
                             st)))
          return rc;
      } else {
        if ((rc = discriminator_fwd(s, true))) return rc;
        // real and fake BCE terms, counts and dL/dD of both halves (train.py:262-270) in one launch
        if ((rc = launch_bce(L.d_out, L.mask, M, 2, 0, 1, L.scal + S_INV_T, L.g_dout, &L.red[R_REAL], &L.red[R_FAKE], st)))
          return rc;
      }
      if ((rc = discriminator_bwd(s, true, !d_only, branch))) return rc;
    }
  }
  if (d_only) {
    // ---- update_generator is not called (train.py:562-566 with update_g = False): D's clip + optimiser step, then the
    // loss scalars; no third D forward, no MLPG adjoint, no generator backward or step
    if (phases & 2) {
      NvtxRange r2("gantts_gan_step/phase2 (D only): D step");
      if ((rc = clip_opt_model(c, d_opt_spec(c), s.pd, L.opt_partial, L.scal + S_DSUMSQ, c->lr_d, c->wd_d, st))) return rc;
    }
    if (phases & 4) {
      NvtxRange r4("gantts_gan_step/phase4 (D only): losses");
      return step_finalize(s, losses_dev);
    }
    return GANTTS_OK;
  }
  if (phases & 2) {
    NvtxRange r2("gantts_gan_step/phase2: D step, adv D fwd+bwd, MLPG bwd, G bwd");
    // ---- clip_grad_norm_ + Adagrad on D (train.py:275-276)
    if (s.has_d && (rc = clip_opt_model(c, d_opt_spec(c), s.pd, L.opt_partial, L.scal + S_DSUMSQ, c->lr_d, c->wd_d, st)))
      return rc;
    // ---- update_generator (train.py:282-320); the MGE term was evaluated in phase 1
    if (s.has_adv) {
      // third D forward: updated weights, fresh dropout mask (train.py:307)
      s.d.seed = gantts_gan_step_seed(seed, 2);
      if ((rc = discriminator_fwd(s, false))) return rc;
      if ((rc = launch_bce(L.d_out, L.mask, M, 1, 0, 0, L.scal + S_ADV_SCALE, L.g_dout, &L.red[R_ADV], nullptr, st)))
        return rc;
      if ((rc = discriminator_bwd(s, false))) return rc;
    }
    if ((rc = generator_bwd(s))) return rc;
  }
  if (phases & 4) {
    NvtxRange r4("gantts_gan_step/phase4: G step, losses");
    // ---- clip_grad_norm_ + Adagrad on G (train.py:317-318), then the loss scalars
    if ((rc = clip_opt_model(c, g_opt_spec(c), s.pg, L.opt_partial, L.scal + S_GSUMSQ, c->lr_g, c->wd_g, st))) return rc;
    return step_finalize(s, losses_dev);
  }
  return GANTTS_OK;
}

// ---- spoofing-rate count (train.py:549-558): D_ref on the adversarial columns of y_hat_static, dropout off
// (train.py:445), no conditioning (train.py:554-555), no gradient.  Workspace: D_ref's tape, then its output [rows].
static int check_spoof_d(const gantts_mlp_t* d, int64_t rows) {
  GANTTS_CHECK_ARG(d, "spoof_count: null reference discriminator");
  GANTTS_CHECK_ARG(d->num_layers >= 1 && d->num_layers <= GANTTS_MAX_LAYERS, "spoof_count: bad layer count %d", d->num_layers);
  GANTTS_CHECK_ARG(d->dims[d->num_layers] == 1 && d->last_act == GANTTS_ACT_SIGMOID,
                   "spoof_count: the reference discriminator must end in a single sigmoid output");
  GANTTS_CHECK_ARG(rows >= 1 && rows < (1 << 24),
                   "spoof_count: B * T = %lld frames, the float count is exact below 2^24", (long long)rows);
  return GANTTS_OK;
}

// The adversarial columns of y_hat_static the reference discriminator reads: n_adv of them, as many as its input width
static int spoof_cols(const char* who, const int* adv_cols, int n_adv, int n_static, int d_width, ColList* cols) {
  GANTTS_CHECK_ARG(n_adv >= 1 && n_adv <= GANTTS_MAX_COLS && n_adv == d_width,
                   "%s: %d adversarial columns != reference discriminator input width %d (it gets no "
                   "linguistic conditioning, train.py:554-555)", who, n_adv, d_width);
  GANTTS_CHECK_ARG(n_static >= 1, "%s: bad n_static", who);
  cols->n = n_adv;
  for (int i = 0; i < n_adv; ++i) {
    GANTTS_CHECK_ARG(adv_cols[i] >= 0 && adv_cols[i] < n_static, "%s: adversarial column %d out of range", who,
                     adv_cols[i]);
    cols->c[i] = adv_cols[i];
  }
  return GANTTS_OK;
}

// those columns of y_hat_static's `rows` frames into the operand planes of the discriminator's first layer
static int spoof_gather(const float* y_hat_static, int n_static, const ColList& cols, int64_t rows, const Planes& in,
                        cudaStream_t st) {
  ColList none;
  none.n = 0;
  GANTTS_PDL_LAUNCH((gather_planes_kernel), blocks_1d(rows * cols.n, 1024), 256, 0, st, y_hat_static, (int64_t)n_static, cols,
                    rows, nullptr, 0, none, 0, in.hi, in.lo, in.pitch);
  GANTTS_LAUNCH_CHECK("gather_planes_kernel(spoof)");
  return GANTTS_OK;
}

// the threshold count over the discriminator's output dout [B * T]
static int spoof_threshold(const float* dout, const int64_t* lengths_dev, int B, int T, float* count_dev, cudaStream_t st) {
  GANTTS_PDL_LAUNCH((spoof_count_kernel), 1, RED_THREADS, 0, st, dout, lengths_dev, B, T, count_dev);
  GANTTS_LAUNCH_CHECK("spoof_count_kernel");
  return GANTTS_OK;
}

extern "C" size_t gantts_spoof_count_workspace_bytes(const gantts_mlp_t* d, int64_t rows) {
  if (check_spoof_d(d, rows)) return 0;
  return al256(gantts_mlp_tape_bytes(d, rows)) + al256((size_t)rows * sizeof(float)) + 256;
}

extern "C" int gantts_spoof_count(const gantts_mlp_t* d, const float* y_hat_static, int n_static, const int* adv_cols,
                                  int n_adv, const int64_t* lengths_dev, int B, int T, float* count_dev, void* ws,
                                  size_t ws_bytes, void* stream) {
  GANTTS_CHECK_ARG(B >= 1 && T >= 1, "spoof_count: bad batch shape");
  const int64_t rows = (int64_t)B * T;
  int rc = check_spoof_d(d, rows);
  if (rc) return rc;
  GANTTS_CHECK_ARG(y_hat_static && adv_cols && lengths_dev && count_dev, "spoof_count: null pointer");
  ColList cols;
  if ((rc = spoof_cols("spoof_count", adv_cols, n_adv, n_static, d->dims[0], &cols))) return rc;
  const size_t need = gantts_spoof_count_workspace_bytes(d, rows);
  if (!ws || ws_bytes < need) {
    set_error("spoof_count: workspace too small (%zu < %zu)", ws_bytes, need);
    return GANTTS_E_WORKSPACE;
  }
  gantts_mlp_t m = *d;
  m.dropout_p = 0.f;
  char* base = reinterpret_cast<char*>(al256(reinterpret_cast<uintptr_t>(ws)));
  const size_t tape_bytes = gantts_mlp_tape_bytes(&m, rows);
  char* tape = base;
  float* dout = reinterpret_cast<float*>(base + al256(tape_bytes));
  const cudaStream_t st = as_stream(stream);
  Planes din;
  if ((rc = mlp_tape_input_planes(&m, rows, tape, tape_bytes, &din))) return rc;
  if ((rc = spoof_gather(y_hat_static, n_static, cols, rows, din, st))) return rc;
  if ((rc = mlp_fwd_impl(&m, nullptr, 0, rows, dout, 1, tape, tape_bytes, stream, true))) return rc;
  return spoof_threshold(dout, lengths_dev, B, T, count_dev, st);
}

// ---- the same count with a recurrent reference discriminator (LSTMRNN / GRURNN with last_sigmoid, train.py:779-781
// builds it from hp.discriminator like D): the adversarial columns go into layer 0's input planes, the LSTM stack runs
// forward with dropout off over the B packed sequences, its top h goes into hidden2out's tape input planes, and the
// one-output sigmoid head and the threshold count follow.  Workspace, laid out at the call's B * T rows: the stack's
// forward buffers (layout_lstm without the backward ones), hidden2out's tape, its output [rows].
struct SpoofLstmLayout {
  LstmWs lstm;
  char* tape;
  size_t tape_bytes;
  float* dout;
  size_t total;
};

static void layout_spoof_lstm(const gantts_lstm_stack_t& ls, const gantts_mlp_t& head, int64_t rows, char* base,
                              SpoofLstmLayout* L) {
  *L = SpoofLstmLayout{};
  Arena a{base};
  layout_lstm(ls, rows, 0, 0, a, &L->lstm, false);
  L->tape_bytes = gantts_mlp_tape_bytes(&head, rows);
  L->tape = a.take(L->tape_bytes);
  L->dout = a.f32((size_t)rows);
  L->total = (size_t)(a.cur - base);
}

static int check_spoof_lstm(const gantts_lstm_stack_t* ls, const gantts_mlp_t* head, int B, int T) {
  GANTTS_CHECK_ARG(ls && head, "spoof_count_lstm: null reference discriminator");
  GANTTS_CHECK_ARG(ls->num_layers >= 1 && ls->num_layers <= GANTTS_MAX_LSTM_LAYERS,
                   "spoof_count_lstm: LSTM layer count %d not in [1, %d] (count with GanTrainer)", ls->num_layers,
                   GANTTS_MAX_LSTM_LAYERS);
  GANTTS_CHECK_ARG(ls->hidden >= 4 && ls->hidden % 4 == 0,
                   "spoof_count_lstm: LSTM hidden size %d is not a positive multiple of 4", ls->hidden);
  GANTTS_CHECK_ARG(ls->bidirectional == 0 || ls->bidirectional == 1, "spoof_count_lstm: bad LSTM bidirectional %d",
                   ls->bidirectional);
  GANTTS_CHECK_ARG(ls->in_dim >= 1, "spoof_count_lstm: bad LSTM in_dim %d", ls->in_dim);
  GANTTS_CHECK_ARG(B >= 1 && T >= 1, "spoof_count_lstm: bad batch shape");
  GANTTS_CHECK_ARG(B <= LSTM_MAX_B, "spoof_count_lstm: an LSTM stack runs at most LSTM_MAX_B = %d sequences (B = %d)",
                   LSTM_MAX_B, B);
  GANTTS_CHECK_ARG((int64_t)B * T < (1 << 24), "spoof_count_lstm: B * T = %lld frames, the float count is exact below 2^24",
                   (long long)B * T);
  const int nh = lstm_ndir(*ls) * ls->hidden;
  GANTTS_CHECK_ARG(head->num_layers == 1 && head->dims[0] == nh && head->dims[1] == 1 && head->last_act == GANTTS_ACT_SIGMOID,
                   "spoof_count_lstm: the head must be hidden2out alone, 1 layer of %d -> 1 with a sigmoid (got %d "
                   "layer(s), input width %d)", nh, head->num_layers, head->dims[0]);
  return GANTTS_OK;
}

extern "C" size_t gantts_spoof_count_lstm_workspace_bytes(const gantts_lstm_stack_t* ls, const gantts_mlp_t* head, int B,
                                                          int T) {
  if (check_spoof_lstm(ls, head, B, T)) return 0;
  SpoofLstmLayout L;
  layout_spoof_lstm(*ls, *head, (int64_t)B * T, nullptr, &L);
  return L.total + 256;
}

extern "C" int gantts_spoof_count_lstm(const gantts_lstm_stack_t* ls, const float* const* lstm_tensors, int n_tensors,
                                       const gantts_mlp_t* head, const float* y_hat_static, int n_static,
                                       const int* adv_cols, int n_adv, const int64_t* lengths_dev, int B, int T,
                                       float* count_dev, void* ws, size_t ws_bytes, void* stream) {
  int rc = check_spoof_lstm(ls, head, B, T);
  if (rc) return rc;
  GANTTS_CHECK_ARG(lstm_tensors && y_hat_static && adv_cols && lengths_dev && count_dev && head->W[0] && head->b[0],
                   "spoof_count_lstm: null pointer");
  const int want = 4 * lstm_ndir(*ls) * ls->num_layers;
  GANTTS_CHECK_ARG(n_tensors == want,
                   "spoof_count_lstm: %d LSTM tensors, the stack has %d (W_ih, W_hh, b_ih, b_hh per layer and direction)",
                   n_tensors, want);
  for (int i = 0; i < n_tensors; ++i) GANTTS_CHECK_ARG(lstm_tensors[i], "spoof_count_lstm: null pointer (LSTM tensor %d)", i);
  ColList cols;
  if ((rc = spoof_cols("spoof_count_lstm", adv_cols, n_adv, n_static, ls->in_dim, &cols))) return rc;
  const size_t need = gantts_spoof_count_lstm_workspace_bytes(ls, head, B, T);
  if (!ws || ws_bytes < need) {
    set_error("spoof_count_lstm: workspace too small (%zu < %zu)", ws_bytes, need);
    return GANTTS_E_WORKSPACE;
  }
  const int64_t rows = (int64_t)B * T;
  SpoofLstmLayout L;
  layout_spoof_lstm(*ls, *head, rows, reinterpret_cast<char*>(al256(reinterpret_cast<uintptr_t>(ws))), &L);
  // the stack's tensors in model.parameters() order, bound like a step's tables (no gradients, no optimiser state)
  gantts_step_tensors_t t{};
  t.n = n_tensors;
  for (int i = 0; i < n_tensors; ++i) t.param[i] = const_cast<float*>(lstm_tensors[i]);
  ParamList pl;
  pl.n = 0;
  pl.total = 0;
  bind_lstm(t, *ls, nullptr, &pl);
  const LstmStack k{ls, &L.lstm, pl.lstm, 0};     // eval mode: the mask stream is never drawn
  gantts_mlp_t m = *head;
  m.dropout_p = 0.f;
  const cudaStream_t st = as_stream(stream);
  if ((rc = spoof_gather(y_hat_static, n_static, cols, rows, lstm_in_planes(k, 0, rows), st))) return rc;
  Planes top;
  if ((rc = mlp_tape_input_planes(&m, rows, L.tape, L.tape_bytes, &top))) return rc;
  if ((rc = lstm_stack_fwd(k, nullptr, 0, top, lengths_dev, B, T, 0, false, st))) return rc;
  if ((rc = mlp_fwd_impl(&m, nullptr, 0, rows, L.dout, 1, L.tape, L.tape_bytes, stream, true))) return rc;
  return spoof_threshold(L.dout, lengths_dev, B, T, count_dev, st);
}
