// Voice conversion of source waveforms with the difference MLSA filter (reference evaluation_vc.py:40-110,
// test_vc_from_path with diffvc=True): the generator's inputs from the analysed mel-cepstra (P.delta_features, P.scale),
// the filter coefficients of the converted-minus-source difference (pysptk.mc2b) and the MLSA filtering of the source
// samples (pysptk.synthesis.Synthesizer(MLSADF(order, alpha), hopsize).synthesis(x, b)).
//
// The filter is SPTK's mlsadf at Pade order 5: mlsadf1 (five first-order sections on b[1]) feeding mlsadf2 (five cascaded
// mlsafir stages, each an order-M all-pass chain weighted by b[2..M]).  Every stage reads the previous sample's output of
// the stage before it, so the five stages of a sample are independent of each other.  One warp filters one utterance:
// lane l holds taps 2l+1 and 2l+2 of every stage (M <= 63).  A stage's new taps follow d[1] = (1-a^2) u + a d_old[1],
// d[j] = d_old[j] + a (d_old[j+1] - d[j-1]); after the delay line's shift d_old[j] is the previous sample's d[j-1], so
// d[j] = e[j] - a d[j-1] with e[j] = dp[j-1] + a dp[j] from the previous sample's taps dp alone.  That first-order
// recurrence over j runs as a log-step warp scan, and it is affine in the stage's input u: d = c + g u with c the scan at
// u = 0 and g[j] = (1-a^2)(-a)^(j-1).  The stage output sum_{j>=2} b[j] d[j] is then C + G u, two warp sums that do not
// wait for u; only the five FMAs of the outputs and the Pade combination wait for the previous sample's feedback.  The
// scan itself is carried from sample to sample through the taps: its log2(64) shuffle steps bound the per-sample time.
#include "common.cuh"

#include <algorithm>

namespace gantts {

constexpr int VC_MAX_WINDOWS = 4;
constexpr int VC_MAX_TAPS = 5;
constexpr int VC_MAX_D = 65535;
constexpr int VC_MAX_T = 1 << 24;
constexpr int MLSA_PD = 5;
constexpr int MLSA_MAX_M = 63;          // taps 1..M held two per lane
constexpr int MLSA_WARPS = 4;           // utterances per block

// SPTK's Pade coefficients at order 5 (mlsadf.c, pade[15..20]); index 0 is unused by the filter
__constant__ double MLSA_PADE[MLSA_PD + 1] = {1.0, 0.4999391, 0.1107098, 0.01369984, 0.0009564853, 0.00003041721};

struct VcWindows {
  int n, l[VC_MAX_WINDOWS], u[VC_MAX_WINDOWS];
  double coef[VC_MAX_WINDOWS][VC_MAX_TAPS];
};

static __device__ __forceinline__ int clamp_len(int64_t v, int hi) { return v < 0 ? 0 : (v > hi ? hi : (int)v); }

// One thread per (row, frame, column): every window over the row's own frames, then the float32 rounding and the scaling.
// The sum runs over the taps in order with separate multiply and add roundings, as the delta_features loop does.
__global__ void vc_inputs_kernel(const double* mc, int64_t m_bs, int64_t m_ts, const int64_t* lengths, int B, int T, int D,
                                 const VcWindows w, const double* mean, const double* std, float* xin, float* stat) {
  const int64_t total = (int64_t)B * T * D;
  const int W = w.n * D;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int d = (int)(i % D);
    const int64_t bt = i / D;
    const int t = (int)(bt % T), b = (int)(bt / T);
    const int L = clamp_len(lengths[b], T);
    float* xo = xin + bt * W;
    if (t >= L) {
      for (int k = 0; k < w.n; ++k) xo[k * D + d] = 0.f;
      stat[bt * D + d] = 0.f;
      continue;
    }
    const double* col = mc + (int64_t)b * m_bs + d;
    for (int k = 0; k < w.n; ++k) {
      double acc = 0.0;
      for (int j = -w.l[k]; j <= w.u[k]; ++j) {
        const int s = t + j;
        if (s >= 0 && s < L) acc = __dadd_rn(acc, __dmul_rn(w.coef[k][j + w.l[k]], col[(int64_t)s * m_ts]));
      }
      const float v = (float)acc;
      if (k == 0) stat[bt * D + d] = v;
      const int c = k * D + d;
      xo[c] = (float)__ddiv_rn(__dsub_rn((double)v, mean[c]), std[c]);
    }
  }
}

// b = mc2b([0, pred - src], alpha) per valid frame, 0 beyond: b[M] = mc[M], b[m] = mc[m] - alpha b[m+1].
__global__ void vc_mc2b_kernel(const float* pred, int64_t p_bs, int64_t p_ts, const float* src, int64_t s_bs,
                               int64_t s_ts, const int64_t* lengths, int B, int T, int M, double alpha, double* out) {
  const int64_t total = (int64_t)B * T;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int t = (int)(i % T), b = (int)(i / T);
    double* o = out + i * (M + 1);
    if (t >= clamp_len(lengths[b], T)) {
      for (int m = 0; m <= M; ++m) o[m] = 0.0;
      continue;
    }
    const float* p = pred + (int64_t)b * p_bs + (int64_t)t * p_ts;
    const float* s = src + (int64_t)b * s_bs + (int64_t)t * s_ts;
    double next = __dsub_rn((double)p[M - 1], (double)s[M - 1]);
    o[M] = next;
    for (int m = M - 1; m >= 0; --m) {
      const double mc = m == 0 ? 0.0 : __dsub_rn((double)p[m - 1], (double)s[m - 1]);
      next = __dsub_rn(mc, __dmul_rn(alpha, next));
      o[m] = next;
    }
  }
}

static __device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);   // the same bits in every lane
  return v;
}

struct MlsaParams {
  const double* x;
  int64_t x_bs;
  const int64_t* lengths;       // samples per row
  const double* b;              // [B][T][M+1]
  const int64_t* frames;        // frames per row
  int B, S, T, M, hop;
  double alpha;
  double* y;                    // [B][S]
};

// One warp per row.  Scalars (mlsadf1, the Pade combination, b[1]) are computed redundantly and identically in every lane.
__global__ void __launch_bounds__(32 * MLSA_WARPS) mlsa_filter_kernel(const MlsaParams p) {
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * MLSA_WARPS + (threadIdx.x >> 5);
  if (row >= p.B) return;
  const int M = p.M, hop = p.hop;
  const double a = p.alpha, aa = 1.0 - a * a;
  const int L = clamp_len(p.lengths[row], p.S);
  const int F = clamp_len(p.frames[row], p.T);
  const int end = (int)min((int64_t)L, (int64_t)F * hop);
  const double* x = p.x + (int64_t)row * p.x_bs;
  double* y = p.y + (int64_t)row * p.S;
  const double* brow = p.b + (int64_t)row * p.T * (M + 1);

  const int j_lo = 2 * lane + 1, j_hi = 2 * lane + 2;            // the taps this lane holds
  const bool v_lo = j_lo <= M, v_hi = j_hi <= M;
  // g[j] = (1-a^2)(-a)^(j-1), the taps' response to the stage input; 0 outside 2..M where the output sum reads them
  double g_lo = aa;
  for (int j = 1; j < j_lo; ++j) g_lo *= -a;
  double g_hi = g_lo * -a;
  const double gs_lo = (v_lo && j_lo >= 2) ? g_lo : 0.0, gs_hi = v_hi ? g_hi : 0.0;
  if (!v_lo) g_lo = 0.0;
  if (!v_hi) g_hi = 0.0;
  double pw[5];                                                   // a^(2d) for the scan offsets d = 1, 2, 4, 8, 16
  pw[0] = a * a;
#pragma unroll
  for (int k = 1; k < 5; ++k) pw[k] = pw[k - 1] * pw[k - 1];

  double d1[MLSA_PD + 1], pt1[MLSA_PD + 1], pt2[MLSA_PD + 1];     // mlsadf1's sections, both feedback vectors
  double t_lo[MLSA_PD + 1], t_hi[MLSA_PD + 1];                    // each stage's taps 2l+1, 2l+2 of the last sample
#pragma unroll
  for (int i = 0; i <= MLSA_PD; ++i) d1[i] = pt1[i] = pt2[i] = t_lo[i] = t_hi[i] = 0.0;

  double b1 = 0.0, i1 = 0.0, b_lo = 0.0, b_hi = 0.0, i_lo = 0.0, i_hi = 0.0;
  int t = -1, hop_end = 0;
  for (int s0 = 0; s0 < end; s0 += 32) {
    const double xv = s0 + lane < end ? x[s0 + lane] : 0.0;
    double yv = 0.0;
    const int n = min(32, end - s0);
    for (int k = 0; k < n; ++k) {
      const int s = s0 + k;
      if (s == hop_end) {                                         // hop t: b from frame max(t-1, 0) toward frame t
        ++t;
        hop_end = min(s + hop, L);
        const double len = (double)(hop_end - s);
        const double* bp = brow + (int64_t)max(t - 1, 0) * (M + 1);
        const double* bc = brow + (int64_t)t * (M + 1);
        b1 = bp[1];
        i1 = __ddiv_rn(__dsub_rn(bc[1], bp[1]), len);
        b_lo = v_lo ? bp[j_lo] : 0.0;
        i_lo = v_lo ? __ddiv_rn(__dsub_rn(bc[j_lo], bp[j_lo]), len) : 0.0;
        b_hi = v_hi ? bp[j_hi] : 0.0;
        i_hi = v_hi ? __ddiv_rn(__dsub_rn(bc[j_hi], bp[j_hi]), len) : 0.0;
      }
      const double xs = __shfl_sync(0xffffffffu, xv, k);

      // mlsadf1: section i reads the previous sample's pt1[i-1]
      double fb = xs, out1 = 0.0;
#pragma unroll
      for (int i = MLSA_PD; i >= 1; --i) {
        d1[i] = aa * pt1[i - 1] + a * d1[i];
        pt1[i] = d1[i] * b1;
        const double v = pt1[i] * MLSA_PADE[i];
        fb += (i & 1) ? v : -v;
        out1 += v;
      }
      pt1[0] = fb;
      out1 += fb;

      // mlsadf2: every stage's u-free taps c and output parts C, G
      const double w_lo = j_lo >= 2 ? b_lo : 0.0;
      const double G = warp_sum(w_lo * gs_lo + b_hi * gs_hi);
      double C[MLSA_PD + 1], c_lo[MLSA_PD + 1], c_hi[MLSA_PD + 1];
#pragma unroll
      for (int i = 1; i <= MLSA_PD; ++i) {
        const double prev = __shfl_up_sync(0xffffffffu, t_hi[i], 1);   // tap 2l of the last sample
        const double e_lo = lane == 0 ? a * t_lo[i] : prev + a * t_lo[i];
        const double e_hi = t_lo[i] + a * t_hi[i];
        double acc = fma(-a, e_lo, e_hi);                        // the pair's value at tap 2l+2 given 0 before it
#pragma unroll
        for (int k2 = 0; k2 < 5; ++k2) {
          const int dd = 1 << k2;
          const double from = __shfl_up_sync(0xffffffffu, acc, dd);
          if (lane >= dd) acc = fma(pw[k2], from, acc);
        }
        const double before = __shfl_up_sync(0xffffffffu, acc, 1);
        c_hi[i] = acc;
        c_lo[i] = lane == 0 ? e_lo : fma(-a, before, e_lo);
        C[i] = warp_sum(w_lo * c_lo[i] + b_hi * c_hi[i]);
      }
      // the stage outputs on the previous sample's inputs, the taps' update, the Pade combination
      double fb2 = out1, out2 = 0.0;
#pragma unroll
      for (int i = MLSA_PD; i >= 1; --i) {
        const double u = pt2[i - 1];
        t_lo[i] = v_lo ? fma(g_lo, u, c_lo[i]) : 0.0;
        t_hi[i] = v_hi ? fma(g_hi, u, c_hi[i]) : 0.0;
        pt2[i] = fma(G, u, C[i]);
        const double v = pt2[i] * MLSA_PADE[i];
        fb2 += (i & 1) ? v : -v;
        out2 += v;
      }
      pt2[0] = fb2;
      out2 += fb2;
      if (lane == k) yv = out2;
      b1 += i1;
      b_lo += i_lo;
      b_hi += i_hi;
    }
    if (lane < n) y[s0 + lane] = yv;
  }
  for (int s = end + lane; s < p.S; s += 32) y[s] = 0.0;
}

}  // namespace gantts

using namespace gantts;

extern "C" int gantts_vc_inputs(const double* mc, int64_t mc_bstride, int64_t mc_tstride, const int64_t* lengths_dev,
                                int B, int T, int D, int n_windows, const int* l, const int* u, const double* coef,
                                const double* mean, const double* std, float* xin, float* stat, void* stream) {
  GANTTS_CHECK_ARG(mc && lengths_dev && l && u && coef && mean && std && xin && stat,
                   "vc_inputs: null pointer: mc, lengths_dev, l, u, coef, mean, std, xin and stat are all required");
  GANTTS_CHECK_ARG(B >= 1 && B <= 65535, "vc_inputs: batch size B = %d must be in [1, 65535]", B);
  GANTTS_CHECK_ARG(T >= 1 && T <= VC_MAX_T, "vc_inputs: padded frames T = %d must be in [1, %d]", T, VC_MAX_T);
  GANTTS_CHECK_ARG(D >= 1 && D <= VC_MAX_D, "vc_inputs: width D = %d must be in [1, %d]", D, VC_MAX_D);
  GANTTS_CHECK_ARG(n_windows >= 1 && n_windows <= VC_MAX_WINDOWS, "vc_inputs: %d windows: between 1 and %d are supported",
                   n_windows, VC_MAX_WINDOWS);
  GANTTS_CHECK_ARG(mc_tstride >= D && mc_bstride >= (int64_t)T * mc_tstride,
                   "vc_inputs: mc strides (%lld, %lld) must hold (T, D) = (%d, %d) rows",
                   (long long)mc_bstride, (long long)mc_tstride, T, D);
  VcWindows w = {};
  w.n = n_windows;
  int off = 0;
  for (int k = 0; k < n_windows; ++k) {
    GANTTS_CHECK_ARG(l[k] >= 0 && u[k] >= 0 && l[k] + u[k] + 1 <= VC_MAX_TAPS,
                     "vc_inputs: window %d spans (%d, %d): at most %d taps", k, l[k], u[k], VC_MAX_TAPS);
    w.l[k] = l[k];
    w.u[k] = u[k];
    for (int j = 0; j <= l[k] + u[k]; ++j) w.coef[k][j] = coef[off + j];
    off += l[k] + u[k] + 1;
  }
  const int64_t total = (int64_t)B * T * D;
  const int blocks = (int)std::min<int64_t>((total + 255) / 256, 65535);
  vc_inputs_kernel<<<blocks, 256, 0, as_stream(stream)>>>(mc, mc_bstride, mc_tstride, lengths_dev, B, T, D, w, mean, std,
                                                          xin, stat);
  GANTTS_LAUNCH_CHECK("vc_inputs_kernel");
  return GANTTS_OK;
}

extern "C" int gantts_mc2b(const float* pred, int64_t pred_bstride, int64_t pred_tstride, const float* src,
                           int64_t src_bstride, int64_t src_tstride, const int64_t* lengths_dev, int B, int T, int M,
                           double alpha, double* b, void* stream) {
  GANTTS_CHECK_ARG(pred && src && lengths_dev && b, "mc2b: null pointer: pred, src, lengths_dev and b are all required");
  GANTTS_CHECK_ARG(B >= 1 && B <= 65535, "mc2b: batch size B = %d must be in [1, 65535]", B);
  GANTTS_CHECK_ARG(T >= 1 && T <= VC_MAX_T, "mc2b: padded frames T = %d must be in [1, %d]", T, VC_MAX_T);
  GANTTS_CHECK_ARG(M >= 1 && M <= VC_MAX_D, "mc2b: order M = %d must be in [1, %d]", M, VC_MAX_D);
  GANTTS_CHECK_ARG(alpha > -1.0 && alpha < 1.0, "mc2b: alpha = %g must be in (-1, 1)", alpha);
  const int64_t total = (int64_t)B * T;
  const int blocks = (int)std::min<int64_t>((total + 127) / 128, 65535);
  vc_mc2b_kernel<<<blocks, 128, 0, as_stream(stream)>>>(pred, pred_bstride, pred_tstride, src, src_bstride, src_tstride,
                                                        lengths_dev, B, T, M, alpha, b);
  GANTTS_LAUNCH_CHECK("vc_mc2b_kernel");
  return GANTTS_OK;
}

extern "C" int gantts_mlsa_filter(const double* x, int64_t x_bstride, const int64_t* lengths_dev, const double* b,
                                  const int64_t* frames_dev, int B, int S, int T, int M, double alpha, int hop, double* y,
                                  void* stream) {
  GANTTS_CHECK_ARG(x && lengths_dev && b && frames_dev && y,
                   "mlsa_filter: null pointer: x, lengths_dev, b, frames_dev and y are all required");
  GANTTS_CHECK_ARG(B >= 1 && B <= 65535 * MLSA_WARPS, "mlsa_filter: batch size B = %d must be in [1, %d]", B,
                   65535 * MLSA_WARPS);
  GANTTS_CHECK_ARG(S >= 1 && S <= (1 << 28), "mlsa_filter: padded samples S = %d must be in [1, 2^28]", S);
  GANTTS_CHECK_ARG(x_bstride >= S, "mlsa_filter: row stride %lld must be >= S = %d", (long long)x_bstride, S);
  GANTTS_CHECK_ARG(T >= 1 && T <= VC_MAX_T, "mlsa_filter: padded frames T = %d must be in [1, %d]", T, VC_MAX_T);
  GANTTS_CHECK_ARG(M >= 1 && M <= MLSA_MAX_M, "mlsa_filter: order M = %d must be in [1, %d]", M, MLSA_MAX_M);
  GANTTS_CHECK_ARG(alpha > -1.0 && alpha < 1.0, "mlsa_filter: alpha = %g must be in (-1, 1)", alpha);
  GANTTS_CHECK_ARG(hop >= 1, "mlsa_filter: hop = %d samples must be >= 1", hop);
  MlsaParams p = {x, x_bstride, lengths_dev, b, frames_dev, B, S, T, M, hop, alpha, y};
  mlsa_filter_kernel<<<(B + MLSA_WARPS - 1) / MLSA_WARPS, 32 * MLSA_WARPS, 0, as_stream(stream)>>>(p);
  GANTTS_LAUNCH_CHECK("mlsa_filter_kernel");
  return GANTTS_OK;
}
