// Epoch log of the training loop (reference train.py:531-595 per batch, :597-637 per phase): every batch's losses,
// correct counts, spoof count, frame count and objective distortions are folded into a per-phase fp64 record in device
// memory, so a phase ends with one read instead of ~10 host reads per batch plus two (B, T, D) copies for
// compute_distortions.
//
// The distortion pass is metrics.cu's distortions_partial_kernel on the same grid, and the fold kernel finishes its sums
// with the same distortions_totals, so a batch's eight sums are bitwise those of gantts_distortions.  The kernel reads the
// target from the step's input y (static + dynamic columns) through the static-column map: the fused step never
// materialises y_static (get_static_features, train.py:528), and the map keeps it that way.  The fold kernel turns the
// sums into the batch's metrics with the formulas of gantts_b200/metrics.py in fp64 and adds them, with the flagged
// losses, to the record.
#include "common.cuh"

namespace gantts {

constexpr int ELOG_FLAGS = GANTTS_LOG_UPDATE_D | GANTTS_LOG_UPDATE_G | GANTTS_LOG_SPOOF;
// 10 / ln(10) * sqrt(2) rounded to double: nnmnkwii.metrics.melcd's constant, as gantts_b200/metrics.py computes it
constexpr double ELOG_LOGDB = 6.141851463713754;

// One block: the batch's eight sums (distortions_totals, rounded to fp32 like distortions_finish_kernel's output), the
// batch's metrics, and the fold into the record.  nblocks = 0 when the batch logs no distortions.
__global__ void __launch_bounds__(MET_THREADS)
epoch_log_fold_kernel(const MetWs* ws, int nblocks, int kind, int flags, const float* __restrict__ losses,
                      const float* __restrict__ spoof, const int64_t* __restrict__ lengths, int B, double* rec) {
  const double* tot = distortions_totals(ws, nblocks);
  if (threadIdx.x != 0) return;
  double s[MET_NV];
  for (int k = 0; k < MET_NV; ++k) s[k] = (double)(float)tot[k];
  int64_t frames = 0;
  for (int b = 0; b < B; ++b) frames += lengths[b];
  rec[GANTTS_LOG_N] += 1.0;
  rec[GANTTS_LOG_FRAMES] += (double)frames;
  // LOSS_NAMES: loss_d, loss_fake_d, loss_real_d, loss_mse, loss_mge, loss_adv, loss_g, real_correct, fake_correct,
  // frames, d_grad_norm, g_grad_norm
  constexpr unsigned D_LOSSES = (1u << 0) | (1u << 1) | (1u << 2) | (1u << 7) | (1u << 8) | (1u << 10);
  constexpr unsigned G_LOSSES = (1u << 3) | (1u << 4) | (1u << 5) | (1u << 6) | (1u << 11);
  const unsigned take = (1u << 9) | ((flags & GANTTS_LOG_UPDATE_D) ? D_LOSSES : 0u) |
                        ((flags & GANTTS_LOG_UPDATE_G) ? G_LOSSES : 0u);
  for (int i = 0; i < GANTTS_LOG_NUM_LOSSES; ++i)
    if (take & (1u << i)) rec[GANTTS_LOG_LOSSES + i] += (double)losses[i];
  if (flags & GANTTS_LOG_SPOOF) rec[GANTTS_LOG_SPOOFED] += (double)spoof[0];
  if (!(flags & GANTTS_LOG_UPDATE_G)) return;
  double* m = rec + GANTTS_LOG_METRICS;
  const double n = s[5];
  if (kind == GANTTS_METRIC_ACOUSTIC) {
    m[0] += ELOG_LOGDB * s[0] / n;
    m[1] += ELOG_LOGDB * s[1] / n / 10.0;
    m[2] += s[3] > 0 ? sqrt(s[2] / s[3]) : (double)NAN;        // ZeroDivisionError -> nan, kept in the sum
    m[3] += s[4] / n;
  } else if (kind == GANTTS_METRIC_DURATION) {
    m[4] += sqrt(s[6] / n);
  } else {
    m[0] += ELOG_LOGDB * s[0] / n;
  }
}

static int epoch_log_check(const gantts_epoch_log_t* cfg) {
  GANTTS_CHECK_ARG(cfg, "epoch_log: null config");
  const gantts_epoch_log_t& e = *cfg;
  GANTTS_CHECK_ARG(e.kind == GANTTS_METRIC_ACOUSTIC || e.kind == GANTTS_METRIC_DURATION || e.kind == GANTTS_METRIC_VC,
                   "epoch_log: unknown metric kind %d (acoustic 0, duration 1, vc 2)", e.kind);
  GANTTS_CHECK_ARG(e.n_static >= 1 && e.n_static <= GANTTS_MAX_COLS, "epoch_log: n_static %d outside [1, %d]",
                   e.n_static, GANTTS_MAX_COLS);
  for (int i = 0; i < e.n_static; ++i)
    GANTTS_CHECK_ARG(e.static_cols[i] >= 0, "epoch_log: static column %d maps to y column %d < 0", i,
                     e.static_cols[i]);
  const gantts_distortion_cols_t& c = e.cols;
  const int D = e.n_static;
  GANTTS_CHECK_ARG(c.mcd_start >= 0 && c.mcd_count >= 0 && c.mcd_start + c.mcd_count <= D && c.bap_start >= 0 &&
                       c.bap_count >= 0 && c.bap_start + c.bap_count <= D && c.mse_start >= 0 && c.mse_count >= 0 &&
                       c.mse_start + c.mse_count <= D && c.lf0_col >= -1 && c.lf0_col < D && c.vuv_col >= -1 &&
                       c.vuv_col < D,
                   "epoch_log: column groups outside [0, n_static)");
  if (e.kind == GANTTS_METRIC_ACOUSTIC)
    GANTTS_CHECK_ARG(c.mcd_count > 0 && c.bap_count > 0 && c.lf0_col >= 0 && c.vuv_col >= 0 && c.mse_count == 0,
                     "epoch_log: the acoustic metrics need the mcd and bap groups, lf0_col and vuv_col (and no mse "
                     "group)");
  else if (e.kind == GANTTS_METRIC_DURATION)
    GANTTS_CHECK_ARG(c.mse_count > 0 && c.mcd_count == 0 && c.bap_count == 0 && c.vuv_col < 0,
                     "epoch_log: the duration metric needs the mse group alone");
  else
    GANTTS_CHECK_ARG(c.mcd_count > 0 && c.bap_count == 0 && c.mse_count == 0 && c.vuv_col < 0,
                     "epoch_log: the vc metric needs the mcd group alone");
  return GANTTS_OK;
}

}  // namespace gantts

using namespace gantts;

extern "C" size_t gantts_epoch_log_workspace_bytes(const gantts_epoch_log_t* cfg) {
  return epoch_log_check(cfg) == GANTTS_OK ? sizeof(MetWs) : 0;
}

extern "C" int gantts_epoch_log_reset(double* record_dev, void* stream) {
  GANTTS_CHECK_ARG(record_dev, "epoch_log_reset: null record");
  GANTTS_CUDA(cudaMemsetAsync(record_dev, 0, GANTTS_LOG_SLOTS * sizeof(double), as_stream(stream)));
  return GANTTS_OK;
}

extern "C" int gantts_epoch_log_add(const gantts_epoch_log_t* cfg, int flags, const float* losses_dev,
                                    const float* spoof_dev, const float* y, int64_t y_bstride, int64_t y_tstride,
                                    int y_cols, const float* y_hat_static, int64_t yh_bstride, int64_t yh_tstride,
                                    const int64_t* lengths_dev, int B, int T, const float* mean_dev,
                                    const float* std_dev, double* record_dev, void* workspace, size_t workspace_bytes,
                                    void* stream) {
  const int rc = epoch_log_check(cfg);
  if (rc != GANTTS_OK) return rc;
  const gantts_epoch_log_t& e = *cfg;
  GANTTS_CHECK_ARG((flags & ~ELOG_FLAGS) == 0, "epoch_log_add: unknown flags 0x%x", flags);
  GANTTS_CHECK_ARG(losses_dev && lengths_dev && record_dev, "epoch_log_add: null losses, lengths or record");
  GANTTS_CHECK_ARG(!(flags & GANTTS_LOG_SPOOF) || spoof_dev, "epoch_log_add: LOG_SPOOF needs the spoof count");
  GANTTS_CHECK_ARG(B >= 1 && T >= 1, "epoch_log_add: bad batch shape (%d, %d)", B, T);
  const bool dist = (flags & GANTTS_LOG_UPDATE_G) != 0;
  if (dist) {
    GANTTS_CHECK_ARG(y && y_hat_static && mean_dev && std_dev,
                     "epoch_log_add: LOG_UPDATE_G needs y, y_hat_static, mean and std");
    for (int i = 0; i < e.n_static; ++i)
      GANTTS_CHECK_ARG(e.static_cols[i] < y_cols, "epoch_log_add: static column %d maps to y column %d outside [0, %d)",
                       i, e.static_cols[i], y_cols);
    GANTTS_CHECK_ARG(y_bstride >= 0 && y_tstride >= 0 && yh_bstride >= 0 && yh_tstride >= 0,
                     "epoch_log_add: negative strides");
  }
  if (!workspace || workspace_bytes < sizeof(MetWs)) {
    set_error("epoch_log_add: workspace too small (%zu < %zu)", workspace_bytes, sizeof(MetWs));
    return GANTTS_E_WORKSPACE;
  }
  MetWs* ws = static_cast<MetWs*>(workspace);
  cudaStream_t st = as_stream(stream);
  int nb = 0;
  if (dist) {
    ColList ymap;
    ymap.n = e.n_static;
    for (int i = 0; i < e.n_static; ++i) ymap.c[i] = e.static_cols[i];
    nb = distortions_blocks(B, T);
    distortions_partial_kernel<<<nb, MET_THREADS, 0, st>>>(y, y_bstride, y_tstride, y_hat_static, yh_bstride, yh_tstride,
                                                           lengths_dev, B, T, mean_dev, std_dev, e.cols, ymap, ws);
    GANTTS_LAUNCH_CHECK("distortions_partial_kernel");
  }
  epoch_log_fold_kernel<<<1, MET_THREADS, 0, st>>>(ws, nb, e.kind, flags, losses_dev, spoof_dev, lengths_dev, B,
                                                   record_dev);
  GANTTS_LAUNCH_CHECK("epoch_log_fold_kernel");
  return GANTTS_OK;
}
