// clip_grad_norm_ + Adagrad / Adam over a list of parameter tensors (include/gantts_b200.h).
// Reference: torch.nn.utils.clip_grad_norm_(params, 1.0) then torch.optim.Adagrad.step(), as called at
// train.py:275-276,317-318 with lr 0.01, weight_decay 1e-7 (hparams.py:223-227,240-244); Adam for the duration
// model (hparams.py:125-130).  Lists of any length: the kernels take 32 tensors per launch, longer lists (a
// 4-layer bidirectional LSTM has 34) are processed in chunks that share one sum of squares.  The clip + optimiser
// kernels here are the library's only ones: the fused step (gan_step.cu) hands them sumsq_partial_kernel's per-block
// partials, the modular steps the finished sum of gantts_grad_sumsq as a single partial.
#include "common.cuh"

namespace gantts {

constexpr int OPT_MAX_TENSORS = 32;
constexpr int OPT_THREADS = 256;
constexpr int OPT_MAX_BLOCKS = 132 * 4;

struct TensorList {
  int n;
  float* p[OPT_MAX_TENSORS];
  float* g[OPT_MAX_TENSORS];
  float* s[OPT_MAX_TENSORS];
  float* s2[OPT_MAX_TENSORS];
  int64_t off[OPT_MAX_TENSORS + 1];   // prefix sums of sizes
};

__device__ __forceinline__ int find_tensor(const TensorList& tl, int64_t i) {
  int k = 0;
  while (k + 1 < tl.n && i >= tl.off[k + 1]) ++k;
  return k;
}

__global__ void __launch_bounds__(OPT_THREADS)
sumsq_partial_kernel(TensorList tl, float* partial) {
  pdl_entry();
  __shared__ float sm[32];
  float v[1] = {0.f};
  const int64_t total = tl.off[tl.n];
  for (int64_t i = (int64_t)blockIdx.x * OPT_THREADS + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * OPT_THREADS) {
    int k = find_tensor(tl, i);
    float g = tl.g[k][i - tl.off[k]];
    v[0] = fmaf(g, g, v[0]);
  }
  block_sum<1>(v, sm);
  if (threadIdx.x == 0) partial[blockIdx.x] = v[0];
}

__global__ void __launch_bounds__(OPT_THREADS)
sumsq_finish_kernel(const float* partial, int n, float* out) {
  __shared__ float sm[32];
  float v[1] = {0.f};
  for (int i = threadIdx.x; i < n; i += OPT_THREADS) v[0] += partial[i];
  block_sum<1>(v, sm);
  if (threadIdx.x == 0) out[0] = v[0];
}

// clip_grad_norm_'s coefficient min(1, max_norm / (norm + 1e-6)) with the sum of squares taken from the per-block partials
// of sumsq_partial_kernel: every block re-reduces the (<= 592) partials itself in the same fixed order, which removes the
// finish launch; block 0 stores the sum of squares when sumsq_out is set.  The modular steps pass the finished sum as
// one partial, which the reduction returns bit for bit.
__device__ __forceinline__ float clip_coef(const float* __restrict__ partial, int npartial, float* __restrict__ sumsq_out,
                                           float max_norm) {
  __shared__ float sm[32];
  __shared__ float total_s;
  float v[1] = {0.f};
  for (int i = threadIdx.x; i < npartial; i += OPT_THREADS) v[0] += partial[i];
  block_sum<1>(v, sm);
  if (threadIdx.x == 0) {
    total_s = v[0];
    if (blockIdx.x == 0 && sumsq_out) sumsq_out[0] = v[0];
  }
  __syncthreads();
  const float total_norm = sqrtf(total_s);
  const float coef = max_norm / (total_norm + 1e-6f);
  return coef < 1.f ? coef : 1.f;
}

// clip_grad_norm_ + Adagrad
__global__ void __launch_bounds__(OPT_THREADS)
clip_adagrad_partials_kernel(TensorList tl, const float* __restrict__ partial, int npartial, float* __restrict__ sumsq_out,
                             float max_norm, float lr, float wd, float eps) {
  pdl_entry();
  const float coef = clip_coef(partial, npartial, sumsq_out, max_norm);
  const int64_t total = tl.off[tl.n];
  for (int64_t i = (int64_t)blockIdx.x * OPT_THREADS + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * OPT_THREADS) {
    int k = find_tensor(tl, i);
    int64_t j = i - tl.off[k];
    float g = tl.g[k][j] * coef;
    tl.g[k][j] = g;                       // clip_grad_norm_ scales .grad in place
    float p = tl.p[k][j];
    g = fmaf(wd, p, g);
    float s = fmaf(g, g, tl.s[k][j]);
    tl.s[k][j] = s;
    tl.p[k][j] = p - lr * g / (sqrtf(s) + eps);
  }
}

// The same with torch.optim.Adam (amsgrad off; reference hparams.py:125-130): tl.s = exp_avg, tl.s2 = exp_avg_sq;
// denom = sqrt(v) / sqrt(bias_correction2) + eps, with step_size and inv_sqrt_bc2 from adam_scales on the host.
__global__ void __launch_bounds__(OPT_THREADS)
clip_adam_partials_kernel(TensorList tl, const float* __restrict__ partial, int npartial, float* __restrict__ sumsq_out,
                          float max_norm, float b1, float b2, float wd, float eps, float step_size, float inv_sqrt_bc2) {
  pdl_entry();
  const float coef = clip_coef(partial, npartial, sumsq_out, max_norm);
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

// Adam's bias corrections of step t (>= 1): step_size = lr / (1 - beta1^t), inv_sqrt_bc2 = 1 / sqrt(1 - beta2^t), in fp64
struct AdamScales {
  float step_size, inv_sqrt_bc2;
};
static AdamScales adam_scales(float lr, float beta1, float beta2, int64_t step) {
  const double bc1 = 1.0 - pow((double)beta1, (double)step), bc2 = 1.0 - pow((double)beta2, (double)step);
  return {(float)((double)lr / bc1), (float)(1.0 / sqrt(bc2))};
}

static int fill(TensorList& tl, float* const* params, float* const* grads, float* const* sums,
                float* const* sums2, const int64_t* sizes, int first, int n) {
  tl.n = n;
  tl.off[0] = 0;
  for (int i = 0; i < n; ++i) {
    const int q = first + i;
    GANTTS_CHECK_ARG(sizes[q] >= 1 && grads[q], "optim: bad tensor %d", q);
    tl.p[i] = params ? params[q] : nullptr;
    tl.g[i] = grads[q];
    tl.s[i] = sums ? sums[q] : nullptr;
    tl.s2[i] = sums2 ? sums2[q] : nullptr;
    tl.off[i + 1] = tl.off[i] + sizes[q];
  }
  return GANTTS_OK;
}

static int blocks_for(int64_t total, int cap) {
  int64_t b = (total + OPT_THREADS * 4 - 1) / (OPT_THREADS * 4);
  if (b < 1) b = 1;
  if (b > cap) b = cap;
  return (int)b;
}

}  // namespace gantts

using namespace gantts;

extern "C" size_t gantts_optim_workspace_bytes(void) { return OPT_MAX_BLOCKS * sizeof(float); }

extern "C" int gantts_grad_sumsq(float* const* grads, const int64_t* sizes_host, int ntensors,
                                 float* sumsq_dev, void* workspace, size_t workspace_bytes, void* stream) {
  GANTTS_CHECK_ARG(grads && sizes_host && sumsq_dev && ntensors >= 1, "grad_sumsq: bad arguments");
  if (!workspace || workspace_bytes < OPT_MAX_BLOCKS * sizeof(float)) {
    set_error("grad_sumsq: workspace too small");
    return GANTTS_E_WORKSPACE;
  }
  const int chunks = (ntensors + OPT_MAX_TENSORS - 1) / OPT_MAX_TENSORS;
  GANTTS_CHECK_ARG(chunks <= OPT_MAX_BLOCKS, "grad_sumsq: too many tensors (%d)", ntensors);
  const int cap = OPT_MAX_BLOCKS / chunks;
  float* partial = static_cast<float*>(workspace);
  int used = 0;
  for (int c = 0; c < chunks; ++c) {
    TensorList tl;
    const int first = c * OPT_MAX_TENSORS;
    const int n = ntensors - first < OPT_MAX_TENSORS ? ntensors - first : OPT_MAX_TENSORS;
    int rc = fill(tl, nullptr, grads, nullptr, nullptr, sizes_host, first, n);
    if (rc) return rc;
    const int nb = blocks_for(tl.off[tl.n], cap);
    sumsq_partial_kernel<<<nb, OPT_THREADS, 0, as_stream(stream)>>>(tl, partial + used);
    GANTTS_LAUNCH_CHECK("sumsq_partial_kernel");
    used += nb;
  }
  sumsq_finish_kernel<<<1, OPT_THREADS, 0, as_stream(stream)>>>(partial, used, sumsq_dev);
  GANTTS_LAUNCH_CHECK("sumsq_finish_kernel");
  return GANTTS_OK;
}

extern "C" int gantts_clip_adagrad_step(float* const* params, float* const* grads, float* const* state_sums,
                                        const int64_t* sizes_host, int ntensors, const float* sumsq_dev,
                                        float max_norm, float lr, float weight_decay, float eps,
                                        void* stream) {
  GANTTS_CHECK_ARG(params && grads && state_sums && sizes_host && sumsq_dev && ntensors >= 1,
                   "clip_adagrad_step: null pointer");
  for (int first = 0; first < ntensors; first += OPT_MAX_TENSORS) {
    TensorList tl;
    const int n = ntensors - first < OPT_MAX_TENSORS ? ntensors - first : OPT_MAX_TENSORS;
    int rc = fill(tl, params, grads, state_sums, nullptr, sizes_host, first, n);
    if (rc) return rc;
    for (int i = 0; i < n; ++i) GANTTS_CHECK_ARG(tl.p[i] && tl.s[i], "clip_adagrad_step: null tensor %d", first + i);
    const int nb = blocks_for(tl.off[tl.n], OPT_MAX_BLOCKS);
    clip_adagrad_partials_kernel<<<nb, OPT_THREADS, 0, as_stream(stream)>>>(tl, sumsq_dev, 1, nullptr, max_norm, lr,
                                                                            weight_decay, eps);
    GANTTS_LAUNCH_CHECK("clip_adagrad_partials_kernel");
  }
  return GANTTS_OK;
}

extern "C" int gantts_clip_adam_step(float* const* params, float* const* grads, float* const* exp_avg,
                                     float* const* exp_avg_sq, const int64_t* sizes_host, int ntensors,
                                     const float* sumsq_dev, float max_norm, float lr, float beta1, float beta2,
                                     float weight_decay, float eps, int64_t step, void* stream) {
  GANTTS_CHECK_ARG(params && grads && exp_avg && exp_avg_sq && sizes_host && sumsq_dev && ntensors >= 1 && step >= 1,
                   "clip_adam_step: bad arguments");
  const AdamScales a = adam_scales(lr, beta1, beta2, step);
  for (int first = 0; first < ntensors; first += OPT_MAX_TENSORS) {
    TensorList tl;
    const int n = ntensors - first < OPT_MAX_TENSORS ? ntensors - first : OPT_MAX_TENSORS;
    int rc = fill(tl, params, grads, exp_avg, exp_avg_sq, sizes_host, first, n);
    if (rc) return rc;
    for (int i = 0; i < n; ++i)
      GANTTS_CHECK_ARG(tl.p[i] && tl.s[i] && tl.s2[i], "clip_adam_step: null tensor %d", first + i);
    const int nb = blocks_for(tl.off[tl.n], OPT_MAX_BLOCKS);
    clip_adam_partials_kernel<<<nb, OPT_THREADS, 0, as_stream(stream)>>>(tl, sumsq_dev, 1, nullptr, max_norm, beta1, beta2,
                                                                         weight_decay, eps, a.step_size, a.inv_sqrt_bc2);
    GANTTS_LAUNCH_CHECK("clip_adam_partials_kernel");
  }
  return GANTTS_OK;
}
