/*
 * gantts_b200.h -- C ABI of libgantts_b200.so: the H100 (sm_90a) GAN-step hot path of r9y9/gantts.
 *
 * Every entry point takes plain device/host pointers and sizes; no torch types.  All work is
 * enqueued on the caller's `stream` (a cudaStream_t passed as void*), nothing synchronises
 * internally unless stated.  The fused GAN step also runs some branches on a side stream the library
 * owns (one per device); it forks them from `stream` and joins them back into it through events before
 * it returns, so everything it writes is ordered on `stream` like the rest.  Return value: 0 on success, otherwise a GANTTS_E_* code; the message
 * for the calling thread's last failure is available from gantts_last_error_string().  The library
 * owns no device memory: every buffer, including workspaces, is the caller's.
 *
 * Each declaration cites the reference interface (r9y9/gantts @ fb1e75f, file:line) it replaces.
 * The reference-side binding is shown in INTEGRATION.md (ctypes, since the reference is Python).
 */
#ifndef GANTTS_B200_H_
#define GANTTS_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GANTTS_OK 0
#define GANTTS_E_BADARG 1   /* shape / pointer / enum out of contract */
#define GANTTS_E_CUDA 2     /* a CUDA runtime or driver call failed */
#define GANTTS_E_UNSUPPORTED 3
#define GANTTS_E_WORKSPACE 4 /* caller workspace too small */

#define GANTTS_MAX_STREAMS 8
#define GANTTS_MAX_WINDOWS 4
#define GANTTS_MAX_WINDOW_TAPS 5 /* l, u <= 2 */
#define GANTTS_MLPG_HALF_TAPS 24 /* FIR half width K: P^-1 decays to 2.6e-10 at lag 24 */
/* floats per row of the MLPG coefficient table: [0, 2K+1) rows of P^-1 (FIR form), [52, 56) = {1/L_tt, L[t][t-1], L[t][t-2], 0}
 * and [56, 60) = {L[t+1][t], L[t+2][t], 0, 0}: rows of the banded Cholesky factor of P for the substitution kernels */
#define GANTTS_MLPG_TABLE_COLS 60
#define GANTTS_MAX_LAYERS 8
#define GANTTS_MAX_COLS 256 /* static / adversarial column lists of the fused step */

int gantts_version(void);                       /* 100 * major + minor */
const char* gantts_last_error_string(void);     /* thread-local, never NULL */
/* 1 when the current device is compute capability 9.0 (the kernels are sm_90a only). */
int gantts_device_supported(void);
/* Number of kernels this library has launched in this process (bench.py's gpu_launches). */
long long gantts_launch_count(void);
/* Measurement hooks: when enabled, the tensor-core GEMM, MLPG, LSTM and WORLD synthesis launches are bracketed by CUDA
 * events on the launching stream.  gantts_profile_collect synchronises those events and ADDS, per
 * kind (0 = GEMM K-major, 1 = GEMM MN-major, 2 = MLPG fwd, 3 = MLPG bwd, 4 / 5 = LSTM fwd / bwd, 6 = WORLD pulse
 * responses, 7 = WORLD overlap-add), the elapsed milliseconds, the work (flops for GEMMs, bytes for MLPG, pulses for
 * kind 6, output samples for kind 7) and the launch count into arrays of 8. */
int gantts_profile_enable(int on);
int gantts_profile_collect(double* ms, double* work, long long* launches);

/* ---------------------------------------------------------------------------------------------
 * Feature-stream layout (reference hparams.py:196-206: stream_sizes / has_dynamic_features).
 * Stream s occupies input columns [in_start, in_start + width) laid out window-major
 * [static sd | delta sd | delta-delta sd] when dyn != 0 (width = num_windows * sd), or sd plain
 * columns when dyn == 0; its static part lands in output columns [out_start, out_start + sd).
 * Disabled streams are simply left out of the table.
 */
typedef struct {
  int n;
  int in_start[GANTTS_MAX_STREAMS];
  int sd[GANTTS_MAX_STREAMS];
  int dyn[GANTTS_MAX_STREAMS];
  int out_start[GANTTS_MAX_STREAMS];
} gantts_streams_t;

/* Delta windows (reference hparams.py:22-26,183-187): window w has taps coef[w][0..l+u]. */
typedef struct {
  int n;
  int l[GANTTS_MAX_WINDOWS];
  int u[GANTTS_MAX_WINDOWS];
  float coef[GANTTS_MAX_WINDOWS][GANTTS_MAX_WINDOW_TAPS];
} gantts_windows_t;

/* ---------------------------------------------------------------------------------------------
 * MLPG (replaces nnmnkwii.paramgen.unit_variance_mlpg_matrix + nnmnkwii.autograd.unit_variance_mlpg
 * as called at reference train.py:510-513, gantts/multistream.py:82-123, gantts/models.py:66,115).
 *
 * The reference multiplies by the dense (T x nw*T) matrix R = (W^T W)^-1 W^T.  Here
 *   y = P^-1 (sum_w W_w^T mu_w),  P = sum_w W_w^T W_w (banded SPD),
 * is evaluated as a 3-tap stencil followed by a (2K+1)-tap row-variant FIR with the rows of P^-1
 * (K = GANTTS_MLPG_HALF_TAPS), over the PADDED length T for every batch row, exactly like the
 * reference (SURVEY.md 8a note iv).
 *
 * gantts_mlpg_table: HOST function.  Fills table_host[T * GANTTS_MLPG_TABLE_COLS] (row stride GANTTS_MLPG_TABLE_COLS) with
 *   table[t][j] = (P^-1)[t, t + j - K]   (0 outside [0,T)), computed in float64 by banded Cholesky,
 * stored as float32.  The caller uploads it once per (windows, T) and passes the device copy below.
 * Returns GANTTS_E_UNSUPPORTED when P^-1 has not decayed below 1e-8 of its diagonal at lag K.
 */
int gantts_mlpg_table(const gantts_windows_t* windows, int T, float* table_host);

/* The same table built on the device and enqueued on `stream` (no host synchronisation, no host copy): table_dev[T *
 * GANTTS_MLPG_TABLE_COLS] is bit for bit what gantts_mlpg_table writes -- one thread factors the band in the host's
 * operation order, then one thread per row t solves P x = e_t, all in float64 without FMA contraction.  Scratch memory is
 * allocated stream-ordered and freed on the stream.  The windows are checked like gantts_mlpg_table's; the two numerical
 * conditions it reports (P positive definite, P^-1 decayed at lag K) are properties of the windows that the host builder
 * verifies -- validate a window set once with it. */
int gantts_mlpg_table_device(const gantts_windows_t* windows, int T, float* table_dev, void* stream);

/* out[b,t,out_col] = MLPG(in[b,:,stream cols]) for dynamic streams, copy for static ones.
 * in:  float32 [B][T][*] with element strides (in_bstride, in_tstride), unit column stride.
 * out: float32 [B][T][*] with element strides (out_bstride, out_tstride). */
int gantts_mlpg_fwd(const float* in, int64_t in_bstride, int64_t in_tstride,
                    float* out, int64_t out_bstride, int64_t out_tstride,
                    const float* table_dev, const gantts_streams_t* streams,
                    const gantts_windows_t* windows, int B, int T, void* stream);

/* grad_in[b,t,stream cols] (+)= W_w P^-1 grad_out (backward of the above; reference backward is
 * R^T g).  Columns of grad_in belonging to no listed stream are NOT written.  accumulate != 0
 * adds into grad_in instead of overwriting. */
int gantts_mlpg_bwd(const float* grad_out, int64_t go_bstride, int64_t go_tstride,
                    float* grad_in, int64_t gi_bstride, int64_t gi_tstride,
                    const float* table_dev, const gantts_streams_t* streams,
                    const gantts_windows_t* windows, int B, int T, int accumulate, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Stream column gathers (reference gantts/multistream.py:33-43 select_streams, :56-79
 * get_static_features, train.py:232-242 get_selected_static_stream).  Pure copies => bit-exact.
 * out[r, j] = in[r, cols[j]] for r < rows.  cols_dev: int32[ncols] on the device.
 */
int gantts_gather_cols(const float* in, int64_t in_rstride, float* out, int64_t out_rstride,
                       const int32_t* cols_dev, int ncols, int64_t rows, void* stream);
/* Scatter-add of the backward: gin[r, cols[j]] += gout[r, j]. */
int gantts_scatter_cols_add(const float* gout, int64_t go_rstride, float* gin, int64_t gi_rstride,
                            const int32_t* cols_dev, int ncols, int64_t rows, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Sequence mask + masked MSE (reference gantts/seqloss.py:9-20 sequence_mask, :27-43
 * MaskedMSELoss.forward).
 */
/* mask[b,t] = (t < lengths[b]) ? 1.f : 0.f ; lengths_dev int64[B]. */
int gantts_sequence_mask(const int64_t* lengths_dev, float* mask, int B, int T, void* stream);

/* sums_dev[0] = sum_{b,t,d} ((a - b) * m[b,t])^2 ; sums_dev[1] = sum_{b,t} m[b,t].
 * a, b: float32 [rows][D] with row strides; mask: float32[rows].  Deterministic two-pass reduction;
 * workspace must hold gantts_masked_sse_workspace_bytes() bytes. The loss is sums[0] / sums[1]. */
size_t gantts_masked_sse_workspace_bytes(void);
int gantts_masked_sse_fwd(const float* a, int64_t a_rstride, const float* b, int64_t b_rstride,
                          const float* mask, int64_t rows, int D, float* sums_dev,
                          void* workspace, size_t workspace_bytes, void* stream);
/* grad_a[r,d] (+)= scale_dev[0] * 2 * (a - b) * m^2 ; scale is read on the device
 * (= upstream_grad / sum(mask)), so no host sync is needed. */
int gantts_masked_sse_bwd(const float* a, int64_t a_rstride, const float* b, int64_t b_rstride,
                          const float* mask, int64_t rows, int D, const float* scale_dev,
                          float* grad_a, int64_t ga_rstride, int accumulate, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Masked adversarial BCE terms (written inline in reference train.py:258-271,286,307-310):
 *   kind 0 ("real"/"adv"):  -(log(D + 1e-20) * m).sum()      count: sum((D > 0.5) * m)
 *   kind 1 ("fake"):        -(log(1 - D + 1e-20) * m).sum()   count: sum((D < 0.5) * m)
 * D: float32[rows] discriminator outputs (after sigmoid).  out_dev[0] = un-normalised loss sum,
 * out_dev[1] = count, out_dev[2] = sum(mask).  Same workspace contract as masked_sse.
 */
int gantts_masked_bce_fwd(const float* D, const float* mask, int64_t rows, int kind,
                          float* out_dev, void* workspace, size_t workspace_bytes, void* stream);
/* grad_D[r] = scale_dev[0] * d/dD of the un-normalised sum above. */
int gantts_masked_bce_bwd(const float* D, const float* mask, int64_t rows, int kind,
                          const float* scale_dev, float* grad_D, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Fused Linear -> LeakyReLU(0.01) -> Dropout layer (reference gantts/models.py:137-141 MLP.forward,
 * :63-65 In2OutHighwayNet.forward; NOTE the reference order is Linear -> LeakyReLU -> Dropout).
 *
 * act: 0 = none (last_linear), 1 = LeakyReLU(slope) then dropout(p), 2 = sigmoid.
 * Dropout keeps an element with probability 1-p and scales it by 1/(1-p); the keep decision is a
 * counter-based hash of (seed, row * N + col), so no mask is stored: the backward recovers
 * "dropped" / "negative" from the saved OUTPUT y (y == 0 <=> dropped, sign(y) = sign(pre-act)).
 *
 * engine: GANTTS_ENGINE_SIMT  = exact fp32 FFMA tiles (validation / odd shapes),
 *         GANTTS_ENGINE_TC    = wgmma tensor cores, bf16x3 split operands with fp32 accumulation
 *                               in registers (a_hi*b_hi + a_hi*b_lo + a_lo*b_hi, ~2^-16 per product).
 */
#define GANTTS_ENGINE_SIMT 0
#define GANTTS_ENGINE_TC 1
#define GANTTS_ACT_NONE 0
#define GANTTS_ACT_LEAKY_DROPOUT 1
#define GANTTS_ACT_SIGMOID 2

/* y[M][N] = act(x[M][K] W[N][K]^T + bias[N]); x, y row-major with row strides; W row-major [N][K]
 * (the nn.Linear state_dict layout). */
int gantts_linear_fwd(const float* x, int64_t x_rstride, const float* W, const float* bias,
                      float* y, int64_t y_rstride, int64_t M, int N, int K, int act, float slope,
                      float p, uint64_t seed, int engine, void* workspace, size_t workspace_bytes,
                      void* stream);
size_t gantts_linear_workspace_bytes(int64_t M, int N, int K, int engine);

/* Backward of the fused layer.  gy: upstream gradient w.r.t. the layer OUTPUT y [M][N].
 * Computes gz = gy * act'(y) (in place into gz_scratch [M][N], may alias gy when gy is dead),
 *   gx[M][K]  (=) gz W          (skipped when gx == NULL),
 *   gW[N][K] (+)= gz^T x,  gb[N] (+)= column sums of gz   (accumulate != 0 adds; skipped if NULL).
 */
int gantts_linear_bwd(const float* gy, int64_t gy_rstride, const float* y, int64_t y_rstride,
                      const float* x, int64_t x_rstride, const float* W,
                      float* gz_scratch, float* gx, int64_t gx_rstride, float* gW, float* gb,
                      int64_t M, int N, int K, int act, float slope, float p, int accumulate,
                      int engine, void* workspace, size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Whole MLP on the tensor-core engine (reference gantts/models.py:121-141 MLP, used as generator and
 * discriminator): hidden layers Linear -> LeakyReLU(slope) -> Dropout(p), then last_linear with
 * last_act (NONE or SIGMOID).  Activations stay resident as bf16 hi/lo planes between layers; the
 * caller-owned `tape` keeps them (plus the split weights) for the backward.  dropout_p = 0 in eval
 * mode; hidden layer l draws its mask from seed + golden-ratio * (l+1).
 */
typedef struct {
  int num_layers;                     /* linear layers including last_linear, 1..GANTTS_MAX_LAYERS */
  int dims[GANTTS_MAX_LAYERS + 1];    /* dims[0] = in ... dims[num_layers] = out */
  const float* W[GANTTS_MAX_LAYERS];  /* W[l]: [dims[l+1]][dims[l]] row-major (nn.Linear layout) */
  const float* b[GANTTS_MAX_LAYERS];  /* b[l]: [dims[l+1]], 16-byte aligned */
  float slope;
  float dropout_p;
  int last_act;
  uint64_t seed;
} gantts_mlp_t;

size_t gantts_mlp_tape_bytes(const gantts_mlp_t* mlp, int64_t M);
size_t gantts_mlp_workspace_bytes(const gantts_mlp_t* mlp, int64_t M);
/* y[M][dims[L]] = MLP(x[M][dims[0]]); fills `tape`. */
int gantts_mlp_fwd(const gantts_mlp_t* mlp, const float* x, int64_t x_rstride, int64_t M, float* y,
                   int64_t y_rstride, void* tape, size_t tape_bytes, void* stream);
/* Backward from gy = dL/dy.  y is the forward output (needed for SIGMOID, may be NULL otherwise).
 * gW[l] / gb[l] (host arrays of device pointers, entries may be NULL) receive (+= when accumulate)
 * the parameter gradients; gx (may be NULL) receives dL/dx. */
int gantts_mlp_bwd(const gantts_mlp_t* mlp, const float* gy, int64_t gy_rstride, const float* y,
                   int64_t y_rstride, int64_t M, const void* tape, size_t tape_bytes, float* gx,
                   int64_t gx_rstride, float* const* gW, float* const* gb, int accumulate,
                   void* workspace, size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Gradient clipping + Adagrad (torch.nn.utils.clip_grad_norm_ + torch.optim.Adagrad as used at
 * reference train.py:275-276,317-318 with hparams.py:223-227,240-244).  Operates on a list of
 * parameter tensors given as device pointer arrays.
 */
/* Tensor lists are HOST arrays of device pointers (any count: lists longer than 32 tensors are processed in
 * chunks of 32 that share the same sum of squares); sizes are element counts.
 * sumsq_dev[0] = sum over all tensors of g^2 (deterministic two-stage reduction). */
size_t gantts_optim_workspace_bytes(void);
int gantts_grad_sumsq(float* const* grads, const int64_t* sizes_host, int ntensors, float* sumsq_dev,
                      void* workspace, size_t workspace_bytes, void* stream);
/* coef = min(1, max_norm / (sqrt(sumsq) + 1e-6)); g *= coef (in place, like clip_grad_norm_);
 * g' = g + wd * p; s += g'*g'; p -= lr * g' / (sqrt(s) + eps).  sumsq_dev is read on the device. */
int gantts_clip_adagrad_step(float* const* params, float* const* grads, float* const* state_sums,
                             const int64_t* sizes_host, int ntensors, const float* sumsq_dev,
                             float max_norm, float lr, float weight_decay, float eps, void* stream);
/* clip_grad_norm_ + torch.optim.Adam.step() (reference hparams.py:125-130: the duration model's optimiser,
 * lr 1e-3, betas (0.5, 0.9), weight_decay 0, eps 1e-8, amsgrad off):  g *= coef; g' = g + wd * p;
 * m = b1 m + (1-b1) g'; v = b2 v + (1-b2) g'^2; p -= lr / (1 - b1^t) * m / (sqrt(v) / sqrt(1 - b2^t) + eps),
 * t = step (1 for the first call). */
int gantts_clip_adam_step(float* const* params, float* const* grads, float* const* exp_avg,
                          float* const* exp_avg_sq, const int64_t* sizes_host, int ntensors,
                          const float* sumsq_dev, float max_norm, float lr, float beta1, float beta2,
                          float weight_decay, float eps, int64_t step, void* stream);

/* ---------------------------------------------------------------------------------------------
 * LSTM layer with packed-sequence semantics (reference gantts/models.py:84-85 In2OutRNNHighwayNet,
 * :175-176 GRURNN -- an nn.LSTM --, :198-199 LSTMRNN; pack_padded_sequence / pad_packed_sequence at
 * :101-112,182-187,205-210).  Gate order i,f,g,o and weight layout of torch.nn.LSTM.
 *
 * xproj  [B][T][ndir*4H] = x W_ih^T + b_ih + b_hh for every time step (one tensor-core GEMM, e.g.
 *        gantts_linear_fwd with the direction-stacked W_ih), direction-major columns.
 * W_hh   [ndir][4H][H].   lengths_dev int64[B] (any order).   ndir = 1 or 2 (bidirectional).
 * h_out  [B][T][ndir*H]: hidden states, ZERO for t >= lengths[b]; the reverse direction starts at
 *        t = lengths[b]-1.   gates [ndir][B][T][4H] / cells [ndir][B][T][H]: saved for the backward.
 * One cooperative launch runs all T steps of both directions (persistent CTAs, W_hh slices resident in
 * shared memory, one grid barrier per step).  workspace: gantts_lstm_workspace_bytes() bytes.
 */
size_t gantts_lstm_workspace_bytes(void);
/* GANTTS_OK when the current device runs the forward of a layer of hidden size H and ndir directions and, with train != 0,
 * its backward too; otherwise GANTTS_E_UNSUPPORTED and the error string names the limit (one wave of CTAs, or the
 * shared memory per CTA).  The kernel, and so the limit, depends on H, ndir and the device's SM count. */
int gantts_lstm_layer_supported(int H, int ndir, int train);
int gantts_lstm_layer_fwd(const float* xproj, const float* W_hh, const int64_t* lengths_dev, float* h_out,
                          float* gates, float* cells, int B, int T, int H, int ndir, void* workspace,
                          size_t workspace_bytes, void* stream);
/* dxproj [B][T][ndir*4H] = dL/d(xproj) by back-propagation through time from dh_out = dL/dh_out. */
int gantts_lstm_layer_bwd(const float* dh_out, const float* W_hh, const int64_t* lengths_dev,
                          const float* gates, const float* cells, float* dxproj, int B, int T, int H,
                          int ndir, void* workspace, size_t workspace_bytes, void* stream);
/* hprev[b][t][:] = h_out[b][t-1 (dir 0) | t+1 (dir 1)][dir*H:(dir+1)*H], zero at the first step of each
 * sequence and beyond its length: the right operand of dW_hh[dir] = dxproj_dir^T hprev. */
int gantts_lstm_hprev(const float* h_out, const int64_t* lengths_dev, float* hprev, int B, int T, int H,
                      int ndir, int dir, void* stream);
/* y = keep ? x/(1-p) : 0 with the counter-hash mask (inter-layer dropout of nn.LSTM(dropout=p)); applying
 * the same call to the gradient is the backward. */
int gantts_dropout(const float* x, float* y, int64_t rows, int cols, float p, uint64_t seed, void* stream);

/* ---------------------------------------------------------------------------------------------
 * SRU v1 scan (third-party cuda_functional.SRU imported by reference gantts/models.py:144-167 SRURNN;
 * github.com/taolei87/sru is not vendored and untested by the reference: parity unpinned).
 * u [B][T][ncols*k] = x W (tensor-core GEMM by the caller), ncols = d * (bidir ? 2 : 1), k = 3 or 4 values per
 * column (k fastest): candidate, forget pre-activation, reset pre-activation[, highway input];
 * x [B][T][ncols] is the highway input when k == 3; bias [2*ncols] = forget | reset; mask_h [B][ncols]
 * optional (already scaled) output dropout mask shared over time; act: 0 identity, 1 tanh, 2 relu.
 * Outputs h, c [B][T][ncols].  Backward: du [B][T][ncols*k], dx += (k == 3), dbias_part [B][2*ncols]
 * (sum over B gives the bias gradient).  Rules, checked before any device work: B, T, d >= 1, k = 3 or 4,
 * B * ncols <= 2^30.
 */
int gantts_sru_fwd(const float* u, const float* x, const float* bias, const float* mask_h, float* h, float* c,
                   int B, int T, int d, int k, int bidir, int act, void* stream);
int gantts_sru_bwd(const float* u, const float* x, const float* bias, const float* mask_h, const float* c,
                   const float* dh, float* du, float* dx, float* dbias_part, int B, int T, int d, int k,
                   int bidir, int act, void* stream);
/* Length-exact SRU forward of generation (replaces the SRU stack of reference gantts/models.py:162-165 SRURNN.forward as
 * evaluation_tts.py:167,221 run it: one utterance at B = 1 and T = its own length).  gantts_sru_fwd in eval mode (no
 * dropout mask, no cell states kept) except that sequence b runs over its own L = lengths_dev[b] frames (int64[B], clamped
 * to [0, T]): the reverse direction starts at frame L - 1 with a zero cell, and h is 0 at and beyond L.  So each row
 * equals gantts_sru_fwd of that sequence alone at T = L, and nothing in it depends on the padding.  With every length
 * equal to T the output is bit for bit gantts_sru_fwd's h.  gantts_sru_fwd keeps the reference's padded semantics
 * (training).  Rules, checked before any device work: lengths_dev non-null, 1 <= T <= 2^24, B, d >= 1. */
int gantts_sru_fwd_lengths(const float* u, const float* x, const float* bias, const int64_t* lengths_dev, float* h,
                           int B, int T, int d, int k, int bidir, int act, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Fused GAN training step: one call enqueues the whole mini-batch of reference train.py:528-580
 * (batch prologue :528-535, apply_generator :336-355, update_discriminator :245-279,
 * update_generator :282-320, both clip_grad_norm_ + Adagrad steps) on `stream`, no host sync.
 *
 * MLP generator (g, linear output) and MLP discriminator (d, one sigmoid output, input = the
 * `adv_cols` columns of the static features).  The tensors of g_tensors / d_tensors and their
 * optimiser state are updated IN PLACE.  phases is a bit mask so that a data-parallel caller can
 * all-reduce the gradient buffers (gantts_gan_step_grad_buffer) between the pieces:
 *   1 = prologue, G forward, MLPG, D forward on [real | fake], loss_d backward  -> D gradients ready
 *   2 = D clip+Adagrad, MGE/MSE/ADV losses, third D forward, loss_g backward    -> G gradients ready
 *   4 = G clip+Adagrad, loss scalars
 * inv_frames = 1 / (GLOBAL number of valid frames) (reference normaliser T = mask.sum()); a value <= 0 makes the
 * step derive it on the device from lengths_dev (single-process use).
 * losses_dev[12] = loss_d, loss_fake_d, loss_real_d, loss_mse, loss_mge, loss_adv, loss_g,
 *                  real_correct, fake_correct, local frames, d_grad_norm, g_grad_norm.
 *
 * In2OutHighwayNet generator (reference gantts/models.py:21-69, hparams.py `vc`): highway.static_dim = S > 0.  Then g is
 * the network's H stack + last_linear and the step computes, with x_s = x[:, :, :S] and h = g(x) (= y_hat),
 *   Tx = sigmoid(x_s T.weight^T + T.bias),   Gx = MLPG(h),   y_hat_static = x_s + Tx * Gx,
 * and in the backward, from g = dL/dy_hat_static:  dGx = Tx * g (into the MLPG adjoint and the stack's backward),
 * dz = g * Gx * Tx * (1 - Tx),  dT.weight = dz^T x_s,  dT.bias = sum over rows of dz (no gradient w.r.t. x).
 * Accepted layout: exactly one stream, dynamic, in_start = out_start = 0, sd = S; n_static = S; g.dims[0] >= S;
 * g.dims[L] = windows.n * S; a 16-byte aligned T.bias.  The gate is part of the generator everywhere: its two
 * tensors come FIRST in the flat gradient buffer (model.parameters() order: T.weight, T.bias, then g's layers), in the
 * clip norm and in the optimiser step.  The eval phase runs the same forward and leaves the gate and its state untouched.
 */
typedef struct {
  int static_dim;                          /* 0 = plain MLP generator; S > 0 = In2OutHighwayNet with S static columns */
} gantts_highway_t;

/* SRURNN generator (reference gantts/models.py:144-167, hparams.py `tts_acoustic` / `tts_duration`): num_layers > 0.
 * Then g is hidden2out alone (g.num_layers == 1, g.dims[0] = ncols = hidden * (bidirectional ? 2 : 1)) and the step
 * runs the SRU stack of gantts_sru_fwd in front of it.  Layer l has n_in = in_dim (l = 0) or ncols, k = 4 when
 * n_in != ncols else 3, weight [n_in][ncols * k] and bias [2 * ncols] = forget | reset (the SRUCell layout).
 * In training, layer l multiplies its GEMM input (only: the highway term keeps the unmasked input) by the variational
 * mask gantts_dropout(ones[B][n_in], rnn_dropout, gantts_sru_mask_seed(seed, l, 0)) and, for every layer but the last,
 * g(c_t) by gantts_dropout(ones[B][ncols], dropout, gantts_sru_mask_seed(seed, l, 1)); both are shared over time.
 * The reverse direction starts at the padded frame T - 1: the generator ignores `lengths` like the reference's SRURNN.
 * The stack's tensors come FIRST in model.parameters() order (gru.rnn_lst.0.weight, .0.bias, ..., then hidden2out)
 * in the flat gradient buffer, the clip norm, and the optimiser step.  A conditioned D has d.dims[0] = in_dim + n_adv.
 * Mutually exclusive with the highway block. */
#define GANTTS_MAX_SRU_LAYERS 8
typedef struct {
  int num_layers;                          /* 0 = no SRU stack (all other generators) */
  int in_dim, hidden, bidirectional;
  int act;                                 /* 0 identity, 1 tanh, 2 relu */
  float dropout, rnn_dropout;              /* each in [0, 1) */
} gantts_sru_stack_t;

/* In2OutRNNHighwayNet generator (reference gantts/models.py:72-118, the RNN VC model of hparams.py): num_layers > 0,
 * together with the highway block (static_dim = S).  Then g is hidden2out alone (g.num_layers == 1, g.dims[0] =
 * ndir * hidden, g.dims[1] = in_dim) and the step computes, with x_s = x[:, :, :S],
 *   h = nn.LSTM(in_dim, hidden, num_layers, bidirectional, dropout)(x) with the packed-sequence semantics of
 *       gantts_lstm_layer_fwd (sequence b runs for t < lengths[b], outputs beyond are zero),
 *   Tx = sigmoid(x_s T.weight^T + T.bias),   Gx = MLPG(hidden2out(h)),   y_hat_static = x_s + Tx * Gx,   y_hat = x.
 * Like the reference the model returns its INPUT as y_hat (models.py:118), so loss_mse = MaskedMSE(x, y) is reported
 * but sends no gradient into the generator.  In training the output of every layer but the last is multiplied by
 * gantts_dropout(ones[B * T][ndir * hidden], dropout, gantts_lstm_mask_seed(seed, layer)) (nn.LSTM's per-element
 * inter-layer dropout).  Layer l has n_in = in_dim (l = 0) or ndir * hidden and, per direction d (0 forward, 1 reverse),
 * the torch.nn.LSTM tensors W_ih [4H][n_in], W_hh [4H][H], b_ih, b_hh [4H] (gates i, f, g, o).
 * In model.parameters() order the gate's two tensors come first, then per layer and direction W_ih, W_hh, b_ih, b_hh,
 * then hidden2out, in the flat gradient buffer, the clip norm and the optimiser step; b_ih and b_hh get the same
 * gradient and keep separate optimiser state.  B <= 128, hidden a multiple of 4.  LSTMRNN / GRURNN (an LSTM stack
 * without the gate) and stacks of more than GANTTS_MAX_LSTM_LAYERS layers train with the modular path.  Mutually
 * exclusive with the SRU block. */
#define GANTTS_MAX_LSTM_LAYERS 3
typedef struct {
  int num_layers;                          /* 0 = no LSTM stack (all other generators) */
  int in_dim, hidden, bidirectional;
  float dropout;                           /* in [0, 1) */
} gantts_lstm_stack_t;

/* One model's tensors in model.parameters() order: what the step updates in place, and their optimiser state.  One table
 * is one TensorList of the clip + optimiser kernels, so GANTTS_MAX_STEP_TENSORS is their tensor limit. */
#define GANTTS_MAX_STEP_TENSORS 32
typedef struct {
  int n;
  float* param[GANTTS_MAX_STEP_TENSORS];
  float* state[GANTTS_MAX_STEP_TENSORS];   /* Adagrad state_sum | Adam exp_avg */
  float* state2[GANTTS_MAX_STEP_TENSORS];  /* Adam exp_avg_sq (unused by Adagrad) */
} gantts_step_tensors_t;

/* The discriminator's own optimiser (reference train.py:796-799 builds optimizer_d from hp.optimizer_d and
 * hp.optimizer_d_params, apart from optimizer_g).  own = 0 (a zero-filled block): the discriminator follows the step's
 * optimizer, beta1, beta2, eps and opt_step like the generator.  own = 1: it steps with the kind, betas, eps and step
 * number below (opt_step = number of D's step being taken, 1 for the first; read under Adam only), and the step's
 * top-level fields are the generator's alone.  Its lr and weight decay are lr_d / wd_d either way. */
typedef struct {
  int own;                                 /* 0: follow the step's optimiser fields; 1: the fields below */
  int optimizer;                           /* GANTTS_OPT_ADAGRAD | GANTTS_OPT_ADAM */
  float beta1, beta2, eps;
  int64_t opt_step;
} gantts_optimizer_t;

/* The shape blocks (g, highway, sru, lstm, d) describe the two models; their tensors come from g_tensors and d_tensors
 * alone: the W / b pointers of g and d are not read.  The step binds the tables to the stages from the shapes and
 * rejects a table whose n differs from the count the shapes give, or with a null param or state (state2 where that
 * model's optimiser is Adam). */
typedef struct {
  int B, T;
  gantts_mlp_t g;                          /* generator: dims[0] = linguistic width, dims[L] = acoustic width */
  gantts_highway_t highway;                /* static_dim = 0: no highway gate */
  gantts_sru_stack_t sru;                  /* num_layers = 0: no SRU stack */
  gantts_lstm_stack_t lstm;                /* num_layers = 0: no LSTM stack */
  gantts_mlp_t d;                          /* discriminator: dims[0] = n_adv, dims[L] = 1, last_act = SIGMOID */
  gantts_step_tensors_t g_tensors;         /* generator tensors, model_g.parameters() order */
  gantts_step_tensors_t d_tensors;         /* discriminator tensors, model_d.parameters() order (read when w_d > 0) */
  gantts_streams_t streams;                /* MLPG stream layout of the generator output */
  gantts_windows_t windows;
  const float* mlpg_table;                 /* device copy of gantts_mlpg_table(windows, T) */
  int n_static;                            /* width of y_hat_static */
  int n_static_cols;                       /* == n_static */
  int static_cols[GANTTS_MAX_COLS];        /* columns of y forming y_static (get_static_features) */
  int n_adv;
  int adv_cols[GANTTS_MAX_COLS];           /* columns of y_(hat_)static fed to D (select + mask_nth) */
  int d_conditioned;                       /* hp.discriminator_linguistic_condition (train.py:254-256): D input =
                                              cat((x, y_adv), -1), d.dims[0] = g.dims[0] + n_adv */
  float lr_g, lr_d, wd_g, wd_d, eps, max_norm;
  float w_d, mse_w, mge_w, adv_w;
  /* Optimiser of the generator, and of the discriminator unless d_opt.own (reference train.py:796-799
   * getattr(optim, hp.optimizer_g)(...)): 0 = Adagrad (hparams.py:201-206; state = state_sum), 1 = Adam
   * (hparams.py:125-130, the duration model: lr 1e-3, betas (0.5, 0.9), weight_decay 0, eps 1e-8, amsgrad off; state =
   * exp_avg, state2 = exp_avg_sq, opt_step = number of the step being taken, 1 for the first -- the bias corrections
   * are computed on the host).  With d_opt.own = 0, opt_step is the discriminator's number under GANTTS_STEP_D_ONLY. */
  int optimizer;
  float beta1, beta2;
  gantts_optimizer_t d_opt;                /* zero-filled: the discriminator shares the fields around it */
  int64_t opt_step;
  /* Recurrent discriminator (reference LSTMRNN models.py:193-213, or GRURNN :170-190 -- also an nn.LSTM -- with
   * last_sigmoid=True; train.py:774 builds the class hp.discriminator names): num_layers > 0.  num_layers = 0 (a zero-filled
   * block) is the MLP discriminator above.  Then d is hidden2out alone (d.num_layers == 1, d.dims[0] = ndir * hidden,
   * d.dims[1] = 1, last_act = SIGMOID), in_dim = the discriminator's input width (n_adv, plus the conditioning columns when
   * d_conditioned), and every discriminator forward runs the stack with the packed-sequence semantics of
   * gantts_lstm_layer_fwd on lengths_dev (train.py:261,265,307 pass `lengths`).  The stacked [real | fake] forward runs 2B
   * sequences, so the configured B is at most 64 (LSTM_MAX_B / 2).  In training the output of every layer but the last is
   * multiplied by gantts_dropout(ones[rows][ndir * hidden], dropout, gantts_d_lstm_mask_seed(seed, which, layer)), rows = 2B
   * T on the stacked forward (which = 1) and B T on the adversarial one (which = 2).  The d_tensors table is
   * model_d.parameters(): per layer and direction W_ih, W_hh, b_ih, b_hh, then hidden2out's weight and bias; b_ih and b_hh
   * get the same gradient.  Only the adversarial columns of the fake rows receive an input gradient. */
  gantts_lstm_stack_t d_lstm;
} gantts_gan_step_t;
#define GANTTS_OPT_ADAGRAD 0
#define GANTTS_OPT_ADAM 1

/* Phase bits of gantts_gan_step.  GANTTS_STEP_EVAL = the "test" phase of reference train.py:481-486,
 * :273,:315 (model.eval(), phase != "train"): forwards and losses only -- dropout off, no backward, no
 * optimiser step, parameters and Adagrad state untouched; the adversarial loss re-uses the fake half of the
 * discriminator forward (with dropout off and no discriminator step in between, the reference's third forward
 * returns exactly those values). */
#define GANTTS_STEP_D 1
#define GANTTS_STEP_G 2
#define GANTTS_STEP_FINISH 4
#define GANTTS_STEP_EVAL 8
/* Modifier of the training phases: the discriminator warm-up step (reference train.py --discriminator-warmup, :696
 * update_g = False; train_loop :541-566 without update_generator).  With it the phases are
 *   1 = prologue, G forward (train mode: its dropout is on), MLPG, MGE and MSE forward values, D forward on
 *       [real | fake], BCE, D backward for its parameter gradients only (no gradient w.r.t. its input)
 *   2 = D clip + optimiser step (no third D forward, no MLPG adjoint, no generator backward)
 *   4 = loss scalars (no G clip / step: G's tensors and optimiser state are untouched)
 * and the loss slots mean what they mean in the full step, except loss_adv = 0, loss_g = mse_w loss_mse + mge_w loss_mge
 * and g_grad_norm = 0.  A data-parallel caller all-reduces the discriminator's buffer between 1 and 2 only.  Needs
 * w_d > 0; cannot be combined with GANTTS_STEP_EVAL.  D's Adam step number is d_opt.opt_step, or opt_step when
 * d_opt.own = 0. */
#define GANTTS_STEP_D_ONLY 16

/* Dropout seeds of the fused step, so a test can regenerate every keep mask with gantts_dropout():
 * forward `which` (0 generator, 1 stacked real|fake discriminator batch, 2 adversarial discriminator forward)
 * of a step called with `seed` runs its MLP with gantts_gan_step_seed(seed, which); hidden layer l of an MLP
 * run with seed s draws its mask as gantts_dropout(ones[rows][dims[l+1]], p, gantts_mlp_layer_seed(s, l)). */
uint64_t gantts_gan_step_seed(uint64_t seed, int which);
uint64_t gantts_mlp_layer_seed(uint64_t seed, int layer);
/* Seed of SRU layer `layer`'s masks in a step called with `seed`: which = 0 the variational input mask [B][n_in],
 * 1 the output mask [B][ncols].  A stream of its own (gantts_mlp_layer_seed(gantts_gan_step_seed(seed, 3), 2 layer +
 * which)), apart from the three MLP forwards above. */
uint64_t gantts_sru_mask_seed(uint64_t seed, int layer, int which);
/* Seed of the inter-layer dropout mask on the output of LSTM layer `layer` in a step called with `seed`: a stream of its
 * own, apart from the three MLP forwards and every SRU mask. */
uint64_t gantts_lstm_mask_seed(uint64_t seed, int layer);
/* Seed of the inter-layer dropout mask on the output of the recurrent discriminator's layer `layer` in forward `which`
 * (1 stacked real|fake batch, 2 adversarial forward) of a step called with `seed`: a stream of its own, apart from every
 * seed above. */
uint64_t gantts_d_lstm_mask_seed(uint64_t seed, int which, int layer);

size_t gantts_gan_step_workspace_bytes(const gantts_gan_step_t* cfg);
/* Flat gradient buffer inside `workspace` (which: 0 = generator, 1 = discriminator). */
int gantts_gan_step_grad_buffer(const gantts_gan_step_t* cfg, void* workspace, int which, float** ptr,
                                int64_t* count);
int gantts_gan_step(const gantts_gan_step_t* cfg, int phases, const float* x, const float* y,
                    const int64_t* lengths_dev, float inv_frames, uint64_t seed, float* y_hat,
                    float* y_hat_static, float* losses_dev, void* workspace, size_t workspace_bytes,
                    void* stream);
/* The same step on a mini-batch of its own shape (B, T), 1 <= B <= cfg->B and 1 <= T <= cfg->T: the configured (B, T) is
 * the capacity the workspace is laid out for, and gantts_gan_step is this call with (cfg->B, cfg->T, cfg->mlpg_table).
 * x [B][T][*], y, y_hat, y_hat_static [B][T][*] and lengths_dev [B] are contiguous at the call's shape; mlpg_table is the
 * device table of the call's T (gantts_mlpg_table or gantts_mlpg_table_device).  The arithmetic is exactly that of a step
 * configured for (B, T): dropout masks and split-K plans follow the call's rows M = B * T, and the MLPG solves over T.
 * The flat gradient buffers and whatever one call leaves for the next (phases 1|2 then 4 of the same shape) sit at the
 * same offsets for every shape, so gantts_gan_step_grad_buffer holds for all of them.  The shape and the table are
 * checked before any device work. */
int gantts_gan_step_shaped(const gantts_gan_step_t* cfg, int B, int T, const float* mlpg_table, int phases,
                           const float* x, const float* y, const int64_t* lengths_dev, float inv_frames, uint64_t seed,
                           float* y_hat, float* y_hat_static, float* losses_dev, void* workspace,
                           size_t workspace_bytes, void* stream);

/* Spoofing-rate count of reference train.py:549-558 (the adversarial stage's metric, logged as
 * regard_fake_as_natural / total_num_frames): count_dev[0] = sum over b, t < lengths_dev[b] of [D_ref(x) > 0.5] with
 * x = columns adv_cols[0..n_adv) of y_hat_static [B][T][n_static].  d is the frozen reference discriminator (its W / b
 * are read, dropout_p is ignored: it runs in eval mode as train.py:445 puts it); it gets no linguistic conditioning
 * (train.py:554-555), so d->dims[0] must equal n_adv, and it must end in one sigmoid output.  The count is stored, not
 * accumulated, and is exact while B * T < 2^24 (checked).  Workspace: gantts_spoof_count_workspace_bytes(d, B * T)
 * (0 = the descriptor is rejected). */
size_t gantts_spoof_count_workspace_bytes(const gantts_mlp_t* d, int64_t rows);
int gantts_spoof_count(const gantts_mlp_t* d, const float* y_hat_static, int n_static, const int* adv_cols, int n_adv,
                       const int64_t* lengths_dev, int B, int T, float* count_dev, void* ws, size_t ws_bytes,
                       void* stream);
/* The same count with a recurrent reference discriminator: LSTMRNN, or GRURNN (also an nn.LSTM), with last_sigmoid=True
 * -- train.py:779-781 builds it from hp.discriminator like D, so with a recurrent D it is recurrent too.  ls is its nn.LSTM
 * (1..GANTTS_MAX_LSTM_LAYERS layers, hidden a multiple of 4; dropout is ignored: eval mode), lstm_tensors its n_tensors =
 * 4 ndir num_layers tensors in model.parameters() order (per layer and direction W_ih, W_hh, b_ih, b_hh), head its
 * hidden2out (1 layer of ndir hidden -> 1, last_act = SIGMOID, W[0] / b[0] read).  The stack runs with the packed-sequence
 * semantics of gantts_lstm_layer_fwd on lengths_dev (train.py:554-555 passes the lengths), so frames at or beyond a sequence's
 * length have h = 0; the count masks them out.  ls->in_dim must equal n_adv (no linguistic conditioning), B <= 128 and
 * B * T < 2^24.  Workspace: gantts_spoof_count_lstm_workspace_bytes(ls, head, B, T) of the call's shape, or of any larger
 * one (0 = the descriptor is rejected); it is separate from the step's. */
size_t gantts_spoof_count_lstm_workspace_bytes(const gantts_lstm_stack_t* ls, const gantts_mlp_t* head, int B, int T);
int gantts_spoof_count_lstm(const gantts_lstm_stack_t* ls, const float* const* lstm_tensors, int n_tensors,
                            const gantts_mlp_t* head, const float* y_hat_static, int n_static, const int* adv_cols,
                            int n_adv, const int64_t* lengths_dev, int B, int T, float* count_dev, void* ws,
                            size_t ws_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Inference-time MLPG with real variances (replaces nnmnkwii.paramgen.mlpg as called by reference
 * evaluation_tts.py:70-72,92-94):  solves, per static dimension d and batch row b,
 *   (sum_w W_w^T diag(1/var_w) W_w) y = sum_w W_w^T diag(1/var_w) mean_w
 * by banded Cholesky in float64.  mean/var: float32 [B][T][nw*sd], window-major feature blocks
 * ([static sd, delta sd, delta-delta sd]), element strides (bstride, tstride); a time-invariant variance
 * vector (the reference's use) is passed with v_tstride = 0 (and v_bstride = 0).  out: float32 [B][T][sd].
 */
size_t gantts_mlpg_var_workspace_bytes(const gantts_windows_t* windows, int B, int T, int sd);
int gantts_mlpg_var(const float* mean, int64_t m_bstride, int64_t m_tstride, const float* var,
                    int64_t v_bstride, int64_t v_tstride, float* out, int64_t o_bstride, int64_t o_tstride,
                    const gantts_windows_t* windows, int B, int T, int sd, void* workspace,
                    size_t workspace_bytes, void* stream);

/* Length-exact multi-stream MLPG of generation (replaces, per utterance, the parameter generation of reference
 * evaluation_vc.py:70,74-89 -- unit_variance_mlpg_matrix(hp.windows, T) with multi_stream_mlpg, then inv_scale -- and
 * evaluation_tts.py:62-98 gen_parameters, both branches).  Row b is solved over its own L = lengths_dev[b] frames
 * (int64[B], clamped to [0, T]) by the banded Cholesky of gantts_mlpg_var: W^T P W has its end boundary at L, so the row
 * equals the evaluation scripts' solve of that utterance alone at T = L.  Frames at or beyond L are written as 0.
 *   in  float32 [B][T][*], element strides (in_bstride, in_tstride); the stream table gives the columns as for
 *       gantts_mlpg_fwd.  Dynamic streams are solved; static-only streams (dyn = 0, e.g. vuv) are passed through.
 *   var [input columns]: time-invariant variance per input column (evaluation_tts.py:95-98 Y_var = Y_std**2), or NULL for
 *       unit variance (:71-74, evaluation_vc.py:70).
 *   in_scale / in_shift [input columns], or both NULL: x * in_scale + in_shift as each mean is read, BEFORE the solve
 *       (the non-MGE branch's inv_scale, evaluation_tts.py:86).
 *   out_scale / out_shift [output columns], or both NULL: y * out_scale + out_shift as each frame is stored, AFTER the
 *       solve (the MGE branch's inv_scale, evaluation_tts.py:77-83; evaluation_vc.py:88-89).
 *   out float32 [B][T][*], strides (out_bstride, out_tstride): stream s's static part in [out_start, out_start + sd).
 * The affine maps and the solve run in double.  Workspace: gantts_mlpg_ragged_workspace_bytes (0 = rejected, the error
 * string names the rule): lengths_dev non-null, B >= 1, 1 <= T <= 2^24, 1..GANTTS_MAX_STREAMS streams of static width
 * sd in [1, GANTTS_MAX_COLS], 1..GANTTS_MAX_WINDOWS windows of at most GANTTS_MAX_WINDOW_TAPS taps. */
size_t gantts_mlpg_ragged_workspace_bytes(const gantts_streams_t* streams, const gantts_windows_t* windows,
                                          const int64_t* lengths_dev, int B, int T);
int gantts_mlpg_ragged(const float* in, int64_t in_bstride, int64_t in_tstride, const float* var, const float* in_scale,
                       const float* in_shift, float* out, int64_t out_bstride, int64_t out_tstride,
                       const float* out_scale, const float* out_shift, const gantts_streams_t* streams,
                       const gantts_windows_t* windows, const int64_t* lengths_dev, int B, int T, void* workspace,
                       size_t workspace_bytes, void* stream);

/* Spectral post-processing of generated mel-cepstra (replaces, per utterance, reference evaluation_tts.py:112-115:
 * nnmnkwii.postfilters.merlin_post_filter(mgc, alpha, coef=coef) and pysptk.mc2sp(mgc, fftlen, alpha)).  Up to the final
 * exp both are linear in the frame, so each is one K x (M+1) fp64 matrix (K = fftlen/2 + 1 bins, M the order) whose row k
 * maps a frame to its log power at bin k:
 *   GANTTS_MCEP_R0  cosine transform of freqt(., fftlen/2 - 1, -alpha): the merlin_post_filter energy r0 =
 *                   c2acr(freqt(mc, 511, -alpha), 0, 1024) = sum_k w_k exp(row_k . mc) / fftlen, w = 1, 2, ..., 2, 1;
 *   GANTTS_MCEP_SP  cosine transform of freqt(., fftlen/2, -alpha) with c0 doubled and the Nyquist term counted once:
 *                   mc2sp(mc)[k] = exp(row_k . mc).
 * gantts_mcep_operator builds either matrix on the host in double by running SPTK's freqt recursion on unit vectors; it
 * writes out[k * (M+1) + m].  Rules: |alpha| < 1, 1 <= M+1 <= 128, fftlen a power of two in [64, 4096], kind 0 or 1,
 * out non-null.  No device work.
 * gantts_sp2mc_operator is the other way (pysptk.sp2mc(sp, order, alpha), Test VC.ipynb / Test RNN VC.ipynb
 * compute_static_features, Test TTS.ipynb compute_mgc_from_waveform): the K x (M+1) matrix, built by the same freqt
 * recursion, of freqt(., M, alpha) of the inverse real FFT of the log power with c0 halved, so that
 * sp2mc(sp)[m] = sum_k out[k * (M+1) + m] log sp[k].  Same rules but kind, no device work. */
#define GANTTS_MCEP_R0 0
#define GANTTS_MCEP_SP 1
int gantts_mcep_operator(double alpha, int order, int fftlen, int kind, double* out);
int gantts_sp2mc_operator(double alpha, int order, int fftlen, double* out);
/* Merlin's post filter on every valid frame of a padded batch: mc float32 [B][T][M+1] (element strides mc_bstride,
 * mc_tstride; unit column stride), op_r the GANTTS_MCEP_R0 matrix on the device at fftlen = 2 (K - 1) (the reference's
 * defaults are fftlen 1024, minimum-phase order 511).  Writes w*mc with c0 shifted by log(r0(mc) / r0(w*mc)) / 2,
 * w = coef except w[0] = w[1] = 1: what mc2b(w*mc), b[0] += that shift, b2mc computes in closed form.  out [B][T][M+1]
 * (strides out_bstride, out_tstride). */
int gantts_mcep_postfilter(const float* mc, int64_t mc_bstride, int64_t mc_tstride, float* out, int64_t out_bstride,
                           int64_t out_tstride, const double* op_r, double coef, const int64_t* lengths_dev, int B,
                           int T, int M, int K, void* stream);
/* pysptk.mc2sp on every valid frame of a padded batch: sp float32 [B][T][K] (strides sp_bstride, sp_tstride; unit bin
 * stride) = exp(op_s . mc), op_s the GANTTS_MCEP_SP matrix on the device.
 * Both kernels: row b is processed over its own L = lengths_dev[b] frames (int64[B], clamped to [0, T]); frames at or
 * beyond L are written as 0, and a row equals that utterance alone at B = 1, T = L, bit for bit.  They compute in double
 * and store float32.  Rules, checked before any device work (the error string names the one that failed): lengths_dev
 * non-null, 1 <= B <= 65535, 1 <= T <= 2^24, 1 <= M+1 <= 128, fftlen = 2 (K - 1) a power of two in [64, 4096], non-null
 * buffers, and for the post filter a finite coef. */
int gantts_mcep_to_sp(const float* mc, int64_t mc_bstride, int64_t mc_tstride, float* sp, int64_t sp_bstride,
                      int64_t sp_tstride, const double* op_s, const int64_t* lengths_dev, int B, int T, int M, int K,
                      void* stream);

/* Objective measures of generated features (the reference notebooks' vis_gv and mean_modspec), per feature column of
 * every row of a padded batch x float32 [B][T][D] (element strides x_bstride, x_tstride; unit column stride), over
 * the row's own L = lengths_dev[b] frames (int64[B], clamped to [0, T]).  Frames at or beyond L are never read.
 * gantts_modspec: out[b][k][d] = log(|rfft(x[b, :L, d], n)[k]|^2) in fp64, k = 0 .. n/2 (nnmnkwii.preprocessing.modspec
 *   followed by np.log; frames beyond n are cropped, shorter columns zero-padded, a zero power gives -inf).  out is
 *   contiguous fp64 [B][n/2+1][D].  sum_dev: NULL, or a contiguous fp64 [n/2+1][D] to which out[0], out[1], ... are
 *   added in that order after the spectra are written.
 * gantts_global_variance: out[b][d] = np.var(x[b, :L, d]) in fp64 (two passes, ddof 0; L = 0 gives NaN); out is
 *   contiguous fp64 [B][D].
 * Both compute in fp64, and a column's result depends on nothing but its valid frames: the same bits at any batch
 * position, padded length or padding contents, whatever the other columns hold.  Rules, checked before any device work
 * (the error string names the one that failed): lengths_dev non-null, 1 <= B <= 65535, 1 <= T <= 2^24,
 * 1 <= D <= 65535, strides >= 0, non-null x and out, and for gantts_modspec n a power of two in [64, 8192]. */
int gantts_modspec(const float* x, int64_t x_bstride, int64_t x_tstride, const int64_t* lengths_dev, int B, int T,
                   int D, int n, double* out, double* sum_dev, void* stream);
int gantts_global_variance(const float* x, int64_t x_bstride, int64_t x_tstride, const int64_t* lengths_dev, int B,
                           int T, int D, double* out, void* stream);

/* Acoustic-model inputs from phone-level rows and predicted state durations (replaces, per utterance, the frame
 * expansion of reference evaluation_tts.py:200-212: fe.linguistic_features(labels with the durations set,
 * add_frame_features=True, subphone_features="full"), silence frames removed, P.minmax_scale).  Phone p of row b has
 * state durations d_1..d_S (dur float32 [B][P][S], element strides dur_bstride, dur_pstride, unit state stride),
 * N = sum d_s frames and base_s = sum_{r<s} d_r.  Frame i (0-based) of state s (1-based) is the phone's L linguistic
 * columns followed by GANTTS_SUBPHONE_FEATURES columns (Merlin's "full" block):
 *   L+0 (i+1)/d_s   L+1 (d_s-i)/d_s   L+2 d_s   L+3 s   L+4 S+1-s   L+5 N   L+6 d_s/N   L+7 (N-i-base_s)/N
 *   L+8 (base_s+i+1)/N
 * each computed in double and rounded to float.
 * gantts_state_frame_offsets: offsets int64 [B][P+1], offsets[b][p] the first frame of phone p (an exact prefix sum of
 *   the phones' N; phones at or beyond the row's length phone_lengths_dev[b] (int64[B], clamped to [0, P]) count 0
 *   frames and are never read), frame_lengths int64 [B] = offsets[b][P].  *status_dev (int64) is zeroed and then gets
 *   GANTTS_FRAMES_BAD_DURATION when a duration read is not a finite integer in [1, 2^24] (it is counted as 1) and
 *   GANTTS_FRAMES_TOO_LONG when a row has more than 2^24 frames.  No host synchronisation: the caller reads the status.
 * gantts_expand_state_frames: out contiguous float32 [B][T][L+9], frame t of row b = fl(fl(v * scale_dev[c]) +
 *   min_dev[c]) per column c (two float32 roundings, no FMA: generate.normalize_input's arithmetic on float32
 *   statistics; scale 1 and min 0 give the raw features), v the raw value.  phone_x float32 [B][P][L] (element strides
 *   x_bstride, x_pstride, unit column stride); offsets and frame_lengths as gantts_state_frame_offsets wrote them.
 *   Frames at and beyond min(frame_lengths[b], T) are written as 0, frames >= T never.  A row's bits depend only on
 *   its own valid phones and durations.
 * Rules, checked before any device work (the error string names the one that failed): non-null pointers,
 * 1 <= B <= 65535, P >= 1, 1 <= S <= 16, strides >= 0, and for the expansion 1 <= L <= 65535, 1 <= T <= 2^24. */
#define GANTTS_SUBPHONE_FEATURES 9
#define GANTTS_FRAMES_BAD_DURATION 1
#define GANTTS_FRAMES_TOO_LONG 2
int gantts_state_frame_offsets(const float* dur, int64_t dur_bstride, int64_t dur_pstride,
                               const int64_t* phone_lengths_dev, int B, int P, int S, int64_t* offsets,
                               int64_t* frame_lengths, int64_t* status_dev, void* stream);
int gantts_expand_state_frames(const float* phone_x, int64_t x_bstride, int64_t x_pstride, const float* dur,
                               int64_t dur_bstride, int64_t dur_pstride, const int64_t* offsets,
                               const int64_t* frame_lengths, const float* scale_dev, const float* min_dev, int B,
                               int P, int L, int S, int T, float* out, void* stream);

/* Mini-batches of the training loop gathered from a split held on the device (replaces, per batch, reference
 * train.py:145-159 collate_fn and the sort of :494-501 on the host, and the batch's host-to-device copy).  The split's
 * normalised utterances are packed frame after frame: X float32 [N][Dx] and Y float32 [N][Dy], contiguous.  Row r of
 * the batch is the utterance at frames [offsets_dev[r], offsets_dev[r] + lengths_dev[r]) of the pack (int64[b] each,
 * on the device; the caller lists the rows in sorted order).  Outputs, contiguous float32: x_out [b][t][Dx] and
 * y_out [b][t][Dy], where row r's first lengths_dev[r] frames are the utterance's frames and frames at or beyond its
 * length are written as 0.  One launch writes both outputs; it only copies, so a row's bits are its utterance's bits
 * and depend on nothing else.  A row with offsets_dev[r] < 0, lengths_dev[r] < 0, lengths_dev[r] > t or
 * offsets_dev[r] + lengths_dev[r] > N is written as all 0 and, when status_dev is non-null, GANTTS_CORPUS_BAD_ROW is
 * OR-ed into *status_dev (never cleared here: the caller zeroes it and reads it when it chooses).  No host
 * synchronisation.  Rules, checked before any device work (the error string names the one that failed): non-null
 * X, Y, offsets_dev, lengths_dev, x_out and y_out, N >= 1, 1 <= Dx, Dy <= 65535, 1 <= b <= 65535, 1 <= t <= 2^24. */
#define GANTTS_CORPUS_BAD_ROW 1
int gantts_corpus_gather(const float* X, const float* Y, int64_t N, int Dx, int Dy, const int64_t* offsets_dev,
                         const int64_t* lengths_dev, int b, int t, float* x_out, float* y_out, int64_t* status_dev,
                         void* stream);

/* Waveforms from generated TTS features: WORLD's decode_aperiodicity and Synthesis (replaces, per utterance, reference
 * evaluation_tts.py:116-122: pyworld.decode_aperiodicity(bap, fs, fftlen) and pyworld.synthesize(f0, sp, ap, fs,
 * frame_period)), in fp64.  Row b is processed over its own F = lengths_dev[b] frames (int64[B], clamped to [0, T]), and
 * its results depend only on that row: the same bits at any batch position, padded length or padding contents.
 * gantts_world_band_count: WORLD's number of coded aperiodicity bands, floor(min(15000, fs/2 - 3000) / 3000) (0 below
 *   fs = 12000).  gantts_world_y_length: int(frames * frame_period * fs / 1000), the samples pyworld.synthesize makes.
 * gantts_world_decode_aperiodicity: bap float32 [B][T][nb] (element strides bap_bstride, bap_tstride) -> ap contiguous
 *   fp64 [B][T][fftlen/2 + 1].  A frame whose mean coded value is above -0.5 is 1 - 1e-12 in every bin; any other
 *   interpolates linearly in dB over bin frequency k fs / fftlen through (0 Hz, -60), (3000 j Hz, bap[j-1]) for
 *   j = 1..nb and (fs/2, -1e-12), then ap = 10^(dB/20).  Frames at or beyond F are written as 0.
 * gantts_world_time_base: f0 float32 [B][T] (strides f0_bstride, f0_tstride) -> the pulses of each row: pulse_index int32
 *   [B][cap] (the sample of each pulse, ascending), pulse_shift fp64 [B][cap] (its fractional shift in seconds),
 *   pulse_vuv uint8 [B][cap] (the interpolated V/UV at its sample), and info_dev int64 [2B + 1]: the pulse count of each
 *   row, its y_length, then a status word, zeroed here, that gets GANTTS_WORLD_BAD_F0 when a valid frame's f0 is not
 *   finite and GANTTS_WORLD_SHORT when a row has fewer than 2 frames (its count is 0).  cap >= gantts_world_y_length(T).
 *   The accumulated phase is one sequential fp64 chain in sample order per row, as WORLD's loop runs it, and the time
 *   base is computed without FMA contraction, so the pulses are those of the C loop.  No host synchronisation: the caller
 *   reads info_dev to size gantts_world_synthesize.
 * gantts_world_randn: out fp64 [count] = draws 0 .. count-1 of WORLD's randn after randn_reseed (xorshift128 seeded
 *   123456789, 362436069, 521288629, 88675123; a draw is the uint32 sum of w >> 4 over 12 outputs, / 2^28 - 6), bit for
 *   bit, made in parallel by GF(2) jump-ahead.  Workspace: gantts_world_randn_workspace_bytes(count).
 * gantts_world_synthesize: y contiguous fp64 [B][y_max], row b WORLD's Synthesis of its F frames of f0 (through the pulses
 *   of gantts_world_time_base and its info_dev), sp float32 [B][T][fftlen/2 + 1] and ap fp64 [B][T][fftlen/2 + 1]
 *   (element strides given, unit bin stride), with 0 beyond its y_length.  noise: gantts_world_randn of at least y_max
 *   draws (Synthesis reseeds per utterance, so every row reads the same stream from draw 0).  total_pulses = the sum of the
 *   pulse counts.  Each pulse's response is computed on its own; y[s] then adds the responses covering s in ascending
 *   pulse order (no atomics), in chunks of as many pulses as the workspace holds, processed in order:
 *   gantts_world_synthesize_workspace_bytes(B, fftlen, chunk_pulses) holds chunk_pulses.  A pulse whose noise segment is
 *   longer than fftlen keeps its first fftlen zero-mean samples (WORLD writes past its FFT buffer there).
 * Rules, checked before any device work (the error string names the one that failed): non-null pointers,
 * 1 <= B <= 65535, 1 <= T <= 2^24, fs >= 1, frame_period finite and > 0, fftlen a power of two in [64, 4096],
 * 1 <= gantts_world_y_length(T) <= 2^31 - 1, strides >= 0, cap >= gantts_world_y_length(T), 1 <= y_max <= that, and for
 * the decoder nb == gantts_world_band_count(fs) >= 1. */
#define GANTTS_WORLD_BAD_F0 1
#define GANTTS_WORLD_SHORT 2
int gantts_world_band_count(int fs);
int64_t gantts_world_y_length(int64_t frames, int fs, double frame_period);
int gantts_world_decode_aperiodicity(const float* bap, int64_t bap_bstride, int64_t bap_tstride,
                                     const int64_t* lengths_dev, int B, int T, int nb, int fs, int fftlen, double* ap,
                                     void* stream);
int gantts_world_time_base(const float* f0, int64_t f0_bstride, int64_t f0_tstride, const int64_t* lengths_dev, int B,
                           int T, int fs, double frame_period, int fftlen, int cap, int32_t* pulse_index,
                           double* pulse_shift, uint8_t* pulse_vuv, int64_t* info_dev, void* stream);
size_t gantts_world_randn_workspace_bytes(int64_t count);
int gantts_world_randn(int64_t count, double* out, void* workspace, size_t workspace_bytes, void* stream);
size_t gantts_world_synthesize_workspace_bytes(int B, int fftlen, int64_t chunk_pulses);
int gantts_world_synthesize(const float* sp, int64_t sp_bstride, int64_t sp_tstride, const double* ap,
                            int64_t ap_bstride, int64_t ap_tstride, const int64_t* lengths_dev, const int32_t* pulse_index,
                            const double* pulse_shift, const uint8_t* pulse_vuv, const int64_t* info_dev, int cap,
                            int64_t total_pulses, const double* noise, int B, int T, int fs, double frame_period,
                            int fftlen, int y_max, double* y, void* workspace, size_t workspace_bytes, void* stream);

/* Analysis of natural waveforms: WORLD's DIO, StoneMask and CheapTrick with pyworld's defaults, pysptk.sp2mc and
 * nnmnkwii.preprocessing.modspec_smoothing (replace, per utterance, the notebooks' compute_static_features in Test VC.ipynb
 * and Test RNN VC.ipynb, and compute_mgc_from_waveform in Test TTS.ipynb: pyworld.dio(x, fs, frame_period=hp.frame_period),
 * pyworld.stonemask(x, f0, timeaxis, fs), pyworld.cheaptrick(x, f0, timeaxis, fs), pysptk.sp2mc(sp, order, alpha) and,
 * for TTS, P.modspec_smoothing(mc, modfs, cutoff=50)), in fp64.  x is fp64 [B][S] (row stride x_bstride >= S); row b is
 * processed over its own L = lengths_dev[b] samples (int64[B], clamped to [0, S]) and its results depend only on that row:
 * the same bits at any batch position, padded length or padding contents.  Frame j of a row is at j frame_period / 1000 s.
 * gantts_world_dio_frames: WORLD's GetSamplesForDIO, int(1000 samples / fs / frame_period) + 1.
 * gantts_world_dio: f0 fp64 [B][T], T = gantts_world_dio_frames(S), pyworld.dio with f0_floor 71, f0_ceil 800,
 *   channels_in_octave 2, speed 1, allowed_range 0.1; 0 beyond a row's frames.  info_dev int64 [B + 1]: each row's frame
 *   count, then the status word, zeroed here: GANTTS_ANALYSIS_BAD_INPUT when a sample within a row's length is not
 *   finite, GANTTS_ANALYSIS_SHORT when a row has no more frames than FixF0Contour's window (WORLD leaves its f0 unset;
 *   7 frames at 5 ms), whose f0 is then written as 0.  The mean removed is a fixed-order sum, and both filters are direct
 *   FIR sums.  Workspace: gantts_world_dio_workspace_bytes(B, S, fs, frame_period).
 * gantts_world_stonemask: out fp64 [B][T] = pyworld.stonemask of f0 [B][T] (DIO's) over the frames_dev[b] frames of each
 *   row (DIO's info_dev).  An f0 whose window needs an FFT over 4096 points sets GANTTS_ANALYSIS_FFT in status_dev (DIO's
 *   info_dev + B) and is written as 0; a non-finite one sets GANTTS_ANALYSIS_BAD_INPUT.
 * gantts_world_cheaptrick: sp fp64 [B][T][fftlen/2 + 1] = pyworld.cheaptrick(x, f0, timeaxis, fs, q1=-0.15,
 *   f0_floor=71, fft_size=fftlen).  noise: gantts_world_randn's draws, at least gantts_world_cheaptrick_draws(T, fs,
 *   fftlen) of them (WORLD reseeds randn per utterance, so every row reads the same stream); offsets int64 [B][T] is
 *   scratch for each frame's first draw.  An f0 that is not finite, or above what fftlen can analyse (2 + f0 fftlen / fs
 *   beyond fftlen / 2), sets GANTTS_ANALYSIS_BAD_INPUT and its frame is written as 0.
 * gantts_sp2mc: mc fp64 [B][T][M+1] = sp2mc(sp[b][t], M, alpha) through op, gantts_sp2mc_operator's matrix on the device,
 *   for t < frames_dev[b], 0 beyond; sp fp64 [B][T][K] contiguous.
 * gantts_modspec_smoothing: out fp64 [B][T][D] = modspec_smoothing of x fp64 [B][T][D] (contiguous) over each row's
 *   lengths_dev[b] frames, 0 beyond: every column's n-point real FFT along time, bins cutoff_bin .. n/2 set to 0 (the
 *   notebooks' cut-off bin is int(n cutoff / modfs)), the inverse real FFT, its first L frames.  Defined for L <= n only,
 *   so T <= n is a rule.
 * Rules, checked before any device work (the error string names the one that failed): non-null pointers,
 * 1 <= B <= 65535, 1 <= S <= 2^28, 4000 <= fs <= 96000, 1 <= frame_period <= 100 ms, 1 <= T <= 2^24, fftlen and n powers
 * of two in [64, 4096], 1 <= M+1 <= 128, 2 (K - 1) a power of two in [64, 4096], 1 <= D <= 65535, cutoff_bin >= 0. */
#define GANTTS_ANALYSIS_BAD_INPUT 1
#define GANTTS_ANALYSIS_SHORT 2
#define GANTTS_ANALYSIS_FFT 4
int64_t gantts_world_dio_frames(int64_t samples, int fs, double frame_period);
size_t gantts_world_dio_workspace_bytes(int B, int S, int fs, double frame_period);
int gantts_world_dio(const double* x, int64_t x_bstride, const int64_t* lengths_dev, int B, int S, int fs,
                     double frame_period, double* f0, int64_t* info_dev, void* workspace, size_t workspace_bytes,
                     void* stream);
int gantts_world_stonemask(const double* x, int64_t x_bstride, const int64_t* lengths_dev, const double* f0,
                           const int64_t* frames_dev, int B, int S, int T, int fs, double frame_period, double* out,
                           int64_t* status_dev, void* stream);
int64_t gantts_world_cheaptrick_draws(int T, int fs, int fftlen);
int gantts_world_cheaptrick(const double* x, int64_t x_bstride, const int64_t* lengths_dev, const double* f0,
                            const int64_t* frames_dev, int B, int S, int T, int fs, double frame_period, int fftlen,
                            const double* noise, int64_t noise_count, int64_t* offsets, double* sp, int64_t* status_dev,
                            void* stream);
int gantts_sp2mc(const double* sp, const double* op, const int64_t* frames_dev, int B, int T, int M, int K, double* mc,
                 void* stream);
int gantts_modspec_smoothing(const double* x, const int64_t* lengths_dev, int B, int T, int D, int n, int cutoff_bin,
                             double* out, void* stream);

/* Voice conversion with the difference MLSA filter (reference evaluation_vc.py:40-110, test_vc_from_path with
 * diffvc=True), over each row's own frames or samples; every row gives the same bits at any batch position, padded length
 * or padding contents.
 * gantts_vc_inputs (evaluation_vc.py:61-71): for t < lengths_dev[b], stat float32 [B][T][D] = float32(window 0 of mc) and
 *   xin float32 [B][T][n_windows D] = float32((float32(delta_features(mc)) - mean) / std), mean and std fp64 device vectors
 *   of n_windows D.  mc is fp64 with strides (mc_bstride, mc_tstride) and unit column stride.  Window k spans l[k] frames
 *   back and u[k] ahead; coef holds the l[k] + u[k] + 1 taps of each window in turn (host memory).  Each window runs over
 *   the row's own frames, 0 outside them (nnmnkwii's correlate, mode "same"), summing tap products in tap order in fp64.
 *   Both outputs are 0 beyond each row's length.
 * gantts_mc2b (:95-98): b fp64 [B][T][M+1] = pysptk.mc2b([0, pred - src], alpha) for t < lengths_dev[b], 0 beyond: the
 *   difference in fp64, then b[M] = mc[M], b[m] = mc[m] - alpha b[m+1], rounded as written.  pred and src float32
 *   [..][..][M] with the given strides and unit column stride.
 * gantts_mlsa_filter (:99-101): y fp64 [B][S] = Synthesizer(MLSADF(order=M, alpha=alpha), hopsize=hop).synthesis(x, b) of
 *   each row's lengths_dev[b] samples of x (fp64, row stride x_bstride) with the frames_dev[b] frames of b (fp64
 *   [B][T][M+1], gantts_mc2b's): SPTK's mlsadf at Pade order 5, without the gain exp(b[0]).  Hop t covers samples
 *   [t hop, min((t+1) hop, L)); its coefficients start at frame max(t-1, 0) and after each sample add
 *   (b[t] - b[max(t-1, 0)]) / (the hop's sample count).  Samples at or beyond min(L, frames hop) are 0.
 * Rules, checked before any device work: non-null pointers, 1 <= B <= 65535 (mlsa_filter: 4 x 65535), 1 <= T <= 2^24,
 * 1 <= D <= 65535, 1 to 4 windows of at most 5 taps, 1 <= M <= 65535 (mlsa_filter: M <= 63), |alpha| < 1,
 * 1 <= S <= 2^28, hop >= 1. */
int gantts_vc_inputs(const double* mc, int64_t mc_bstride, int64_t mc_tstride, const int64_t* lengths_dev, int B, int T,
                     int D, int n_windows, const int* l, const int* u, const double* coef, const double* mean,
                     const double* std, float* xin, float* stat, void* stream);
int gantts_mc2b(const float* pred, int64_t pred_bstride, int64_t pred_tstride, const float* src, int64_t src_bstride,
                int64_t src_tstride, const int64_t* lengths_dev, int B, int T, int M, double alpha, double* b,
                void* stream);
int gantts_mlsa_filter(const double* x, int64_t x_bstride, const int64_t* lengths_dev, const double* b,
                       const int64_t* frames_dev, int B, int S, int T, int M, double alpha, int hop, double* y,
                       void* stream);

/* ---------------------------------------------------------------------------------------------
 * Objective distortions of the training loop (reference train.py:399-432 compute_distortions, :383-396
 * split_streams, :358-380 inv_scale; nnmnkwii.metrics.{melcd, lf0_mean_squared_error, vuv_error,
 * mean_squared_error}).  y, y_hat: float32 [B][T][D] static-domain features (normalised); mean_dev /
 * std_dev: float32[D] de-normalisation per static column (the caller maps the reference's
 * static+dynamic-domain indices).  Column groups (count 0 / col -1 disables a term):
 *   mcd  : [mcd_start, +mcd_count)   sum over valid frames of ||delta||_2   (reference passes mgc[:, :, 1:])
 *   bap  : [bap_start, +bap_count)   the same for band aperiodicity
 *   lf0_col, vuv_col: F0 squared error (after exp when lf0_linear) over frames voiced in both; V/UV is
 *          binarised at 0.5 after de-normalisation (train.py:374-377)
 *   mse  : [mse_start, +mse_count)   plain squared error sum (duration model / VC)
 * out8_dev: { sum ||d mcd||, sum ||d bap||, sum f0 err^2, #frames voiced in both, #V/UV mismatches,
 *             #valid frames, sum sq err of the mse group, 0 }.  One device-to-host read of 32 bytes
 * gives every metric: mcd = 10/ln10*sqrt(2) * out[0]/out[5], f0_rmse = sqrt(out[2]/out[3]), ...
 */
typedef struct {
  int mcd_start, mcd_count;
  int bap_start, bap_count;
  int lf0_col, vuv_col;
  int lf0_linear;
  int mse_start, mse_count;
} gantts_distortion_cols_t;

size_t gantts_distortions_workspace_bytes(void);
int gantts_distortions(const float* y, int64_t y_bstride, int64_t y_tstride, const float* y_hat,
                       int64_t yh_bstride, int64_t yh_tstride, const int64_t* lengths_dev, int B, int T, int D,
                       const float* mean_dev, const float* std_dev, const gantts_distortion_cols_t* cols,
                       float* out8_dev, void* workspace, size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Epoch log of the training loop (reference train.py:531-595 per batch, :597-637 per phase): gantts_epoch_log_add,
 * called once after each step, folds that step's results into a per-phase record of GANTTS_LOG_SLOTS doubles in device
 * memory.  Nothing is read back; the caller reads the record once at the end of the phase.  Enqueue-only: no allocation,
 * no host synchronisation, every argument checked before the first launch.
 *
 * Record (fp64, like train.py's Python-float sums of fp32 .item() values):
 *   [GANTTS_LOG_N]        batches added                                       (train.py:490, N)
 *   [GANTTS_LOG_FRAMES]   sum of lengths_dev over the batches                 (:532, total_num_frames)
 *   [GANTTS_LOG_LOSSES+i] sum of losses_dev[i], the 12 scalars of gantts_gan_step (loss_d, loss_fake_d, loss_real_d,
 *                         loss_mse, loss_mge, loss_adv, loss_g, real_correct, fake_correct, frames, d_grad_norm,
 *                         g_grad_norm): D's (0-2, 7, 8, 10) under LOG_UPDATE_D (:562-571), G's (3-6, 11) under
 *                         LOG_UPDATE_G (:574-585), frames (9) always
 *   [GANTTS_LOG_SPOOFED]  sum of spoof_dev[0] under LOG_SPOOF                 (:549-558, regard_fake_as_natural)
 *   [GANTTS_LOG_METRICS+k] under LOG_UPDATE_G the batch's distortions (:587-595): k = 0 mcd, 1 bap_mcd, 2 f0_rmse,
 *                         3 vuv_err, 4 dur_rmse; the metric kind says which are written
 * The batch's distortions are those of compute_distortions (:399-432) with gantts_b200/metrics.py's formulas in fp64 on
 * the eight sums of gantts_distortions (same pass, same reduction): mcd = 10/ln10 sqrt2 s0/frames, bap_mcd = the same of
 * s1 / 10, f0_rmse = sqrt(s2/s3) or NaN when no frame is voiced in both (the reference maps ZeroDivisionError to NaN and
 * the NaN stays in the epoch sum), vuv_err = s4/frames, dur_rmse = sqrt(s6/frames).
 *
 * The target is read from the step's input y [B][T][y_cols] (static + dynamic columns) through static_cols, the
 * static-column map of gantts_gan_step_t (multistream.static_feature_columns), so y_static is never built; y_hat_static
 * [B][T][n_static] is read with its own strides.  mean_dev / std_dev: float32[n_static], the de-normalisation of each
 * static column (train.py:358-380 indexes the static+dynamic-domain statistics: Y_data_mean[static_cols]).
 * Workspace: gantts_epoch_log_workspace_bytes(cfg) (0 = the config is rejected; the message names the rule).
 * gantts_epoch_log_reset zeroes a record on the stream.  y, y_hat_static, mean_dev and std_dev are only read under
 * LOG_UPDATE_G and may be NULL otherwise; spoof_dev only under LOG_SPOOF.
 */
#define GANTTS_METRIC_ACOUSTIC 0 /* hp.name "acoustic": mcd, bap_mcd, f0_rmse, vuv_err */
#define GANTTS_METRIC_DURATION 1 /* "duration": dur_rmse */
#define GANTTS_METRIC_VC 2       /* "vc": mcd */

#define GANTTS_LOG_UPDATE_D 1
#define GANTTS_LOG_UPDATE_G 2
#define GANTTS_LOG_SPOOF 4

#define GANTTS_LOG_NUM_LOSSES 12
#define GANTTS_LOG_N 0
#define GANTTS_LOG_FRAMES 1
#define GANTTS_LOG_LOSSES 2
#define GANTTS_LOG_SPOOFED 14
#define GANTTS_LOG_METRICS 15
#define GANTTS_LOG_SLOTS 20

typedef struct {
  int kind;                             /* GANTTS_METRIC_* */
  int n_static;                         /* columns of y_hat_static */
  int static_cols[GANTTS_MAX_COLS];     /* y column of each static column */
  gantts_distortion_cols_t cols;        /* column groups, in static columns (train.py:383-396, 412-428) */
} gantts_epoch_log_t;

size_t gantts_epoch_log_workspace_bytes(const gantts_epoch_log_t* cfg);
int gantts_epoch_log_reset(double* record_dev, void* stream);
int gantts_epoch_log_add(const gantts_epoch_log_t* cfg, int flags, const float* losses_dev, const float* spoof_dev,
                         const float* y, int64_t y_bstride, int64_t y_tstride, int y_cols, const float* y_hat_static,
                         int64_t yh_bstride, int64_t yh_tstride, const int64_t* lengths_dev, int B, int T,
                         const float* mean_dev, const float* std_dev, double* record_dev, void* workspace,
                         size_t workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* GANTTS_B200_H_ */
