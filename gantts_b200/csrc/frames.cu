// Frame-level acoustic inputs from phone-level rows and state durations (evaluation_tts.py:182-225, tts_from_label
// between the duration model and the acoustic model): every phone's linguistic row is repeated over its frames and
// followed by Merlin's nine "full" subphone features (nnmnkwii.frontend.merlin load_labels_with_state_alignment),
// then min-max scaled as the acoustic model's inputs are.
//
// gantts_state_frame_offsets turns the durations into each phone's first frame (an exact integer prefix sum per row);
// gantts_expand_state_frames writes the frames, each block a tile of one row's frames, each frame finding its phone by
// binary search in the offsets.  A frame's bits depend only on its phone's row and durations.
#include "common.cuh"

namespace gantts {

constexpr int FR_MAX_S = 16;
constexpr int FR_MAX_L = 65535;
constexpr int64_t FR_MAX_FRAMES = 1 << 24;       // per state and per row; float32 holds every count exactly
constexpr int FR_SUBPHONE = 9;                   // GANTTS_SUBPHONE_FEATURES
constexpr int FR_SCAN_THREADS = 256;
constexpr int FR_THREADS = 256;
constexpr int FR_TILE = 32;                      // frames per block of the expansion

// A state duration as a frame count: d itself when it is a finite integer in [1, 2^24], else 1 (and *bad set).  Both
// kernels count frames through this function, so the offsets and the expansion agree even on flagged input.
__device__ __forceinline__ int64_t state_frames(float d, bool* bad) {
  if (d >= 1.f && d <= (float)FR_MAX_FRAMES && d == truncf(d)) return (int64_t)d;
  *bad = true;
  return 1;
}

// One block per row: offsets[b][p] = sum of the frames of phones < p, for p = 0 .. P (phones at or beyond the row's
// length count 0 frames and are never read), frame_lengths[b] = offsets[b][P].  A chunk of FR_SCAN_THREADS phones at a
// time: warp inclusive scans, then the warp totals, then the carry.
__global__ void __launch_bounds__(FR_SCAN_THREADS) state_frame_offsets_kernel(
    const float* dur, int64_t d_bs, int64_t d_ps, const int64_t* phone_lengths, int P, int S, int64_t* offsets,
    int64_t* frame_lengths, unsigned long long* status) {
  __shared__ int64_t warp_tot[FR_SCAN_THREADS / 32];
  __shared__ int64_t carry_s;
  const int b = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t len = phone_lengths[b];
  const int n = len < 0 ? 0 : (len > P ? P : (int)len);
  int64_t* off = offsets + (int64_t)b * (P + 1);
  const float* row = dur + (int64_t)b * d_bs;
  bool bad = false;
  if (threadIdx.x == 0) {
    carry_s = 0;
    off[0] = 0;
  }
  __syncthreads();
  for (int base = 0; base < P; base += FR_SCAN_THREADS) {
    const int p = base + threadIdx.x;
    int64_t v = 0;
    if (p < n) {
      const float* d = row + (int64_t)p * d_ps;
      for (int s = 0; s < S; ++s) v += state_frames(d[s], &bad);
    }
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int64_t u = __shfl_up_sync(0xffffffffu, v, o);
      if (lane >= o) v += u;
    }
    if (lane == 31) warp_tot[warp] = v;
    __syncthreads();
    int64_t before = carry_s;
    for (int w = 0; w < warp; ++w) before += warp_tot[w];
    if (p < P) off[p + 1] = before + v;
    __syncthreads();                                     // every thread has read carry_s and warp_tot
    if (threadIdx.x == FR_SCAN_THREADS - 1) carry_s = before + v;
    __syncthreads();
  }
  const int64_t total = carry_s;
  if (threadIdx.x == 0) {
    frame_lengths[b] = total;
    if (total > FR_MAX_FRAMES) atomicOr(status, (unsigned long long)GANTTS_FRAMES_TOO_LONG);
  }
  if (bad) atomicOr(status, (unsigned long long)GANTTS_FRAMES_BAD_DURATION);
}

// Block (frame tile, row b).  Phase 1: one thread per frame of the tile finds its phone (the last p with
// offsets[p] <= t), its state s and frame i within the state, and writes the nine features, each computed in double and
// rounded to float as LinguisticSource stores them.  Phase 2: threads over (column, frame) write
// fl(fl(v * scale[c]) + min[c]), v the raw value, as generate.normalize_input computes it in float32; 0 at and beyond
// the row's frame length.
__global__ void __launch_bounds__(FR_THREADS) expand_state_frames_kernel(
    const float* phone_x, int64_t x_bs, int64_t x_ps, const float* dur, int64_t d_bs, int64_t d_ps,
    const int64_t* offsets, const int64_t* frame_lengths, const float* scale, const float* shift, int P, int L, int S,
    int T, int ncols_lanes, float* out) {
  __shared__ float feat[FR_TILE][FR_SUBPHONE];
  __shared__ int phone[FR_TILE];
  const int b = blockIdx.y, t0 = blockIdx.x * FR_TILE;
  const int W = L + FR_SUBPHONE;
  const int64_t* off = offsets + (int64_t)b * (P + 1);
  int64_t limit = frame_lengths[b];
  limit = min(limit, off[P]);
  limit = min(limit, (int64_t)T);
  if (threadIdx.x < FR_TILE) {
    const int64_t t = t0 + threadIdx.x;
    int p = -1;
    if (t < limit) {
      int lo = 0, hi = P - 1;                            // off[0] = 0 <= t < off[P]
      while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (off[mid] <= t) lo = mid; else hi = mid - 1;
      }
      p = lo;
      const float* d = dur + (int64_t)b * d_bs + (int64_t)p * d_ps;
      const int64_t k = t - off[p];                      // frame within the phone
      bool bad = false;
      int64_t N = 0, base = 0, ds = 1;
      int s = 0;
      for (int r = 0; r < S; ++r) {
        const int64_t dr = state_frames(d[r], &bad);
        if (s == 0 && k < N + dr) {
          s = r + 1;
          base = N;
          ds = dr;
        }
        N += dr;
      }
      if (s == 0) {                                      // offsets that disagree with the durations: the last state
        s = S;
        ds = state_frames(d[S - 1], &bad);
        base = N - ds;
      }
      const double i = (double)(k - base), dd = (double)ds, Nd = (double)N, bd = (double)base;
      float* f = feat[threadIdx.x];
      f[0] = (float)((i + 1.0) / dd);
      f[1] = (float)((dd - i) / dd);
      f[2] = (float)dd;
      f[3] = (float)s;
      f[4] = (float)(S + 1 - s);
      f[5] = (float)Nd;
      f[6] = (float)(dd / Nd);
      f[7] = (float)((Nd - i - bd) / Nd);
      f[8] = (float)((bd + i + 1.0) / Nd);
    }
    phone[threadIdx.x] = p;
  }
  __syncthreads();
  // ncols_lanes threads per frame (a multiple of 32), FR_THREADS / ncols_lanes frames at a time
  const int cx = threadIdx.x % ncols_lanes, fy = threadIdx.x / ncols_lanes, nf = FR_THREADS / ncols_lanes;
  const int nt = min(FR_TILE, T - t0);
  const float* xrow = phone_x + (int64_t)b * x_bs;
  float* orow = out + ((int64_t)b * T + t0) * W;
  for (int c = cx; c < W; c += ncols_lanes) {
    const float sc = scale[c], sh = shift[c];
    int last_p = -1;
    float xv = 0.f;
    for (int j = fy; j < nt; j += nf) {
      const int p = phone[j];
      float v = 0.f;
      if (p >= 0) {
        if (c < L) {
          if (p != last_p) {
            xv = xrow[(int64_t)p * x_ps + c];
            last_p = p;
          }
          v = xv;
        } else {
          v = feat[j][c - L];
        }
        v = __fadd_rn(__fmul_rn(v, sc), sh);
      }
      orow[(int64_t)j * W + c] = v;
    }
  }
}

}  // namespace gantts

using namespace gantts;

extern "C" int gantts_state_frame_offsets(const float* dur, int64_t dur_bstride, int64_t dur_pstride,
                                          const int64_t* phone_lengths_dev, int B, int P, int S, int64_t* offsets,
                                          int64_t* frame_lengths, int64_t* status_dev, void* stream) {
  GANTTS_CHECK_ARG(dur && phone_lengths_dev && offsets && frame_lengths && status_dev,
                   "state_frame_offsets: null pointer: dur, phone_lengths_dev, offsets, frame_lengths and status_dev "
                   "are all required");
  GANTTS_CHECK_ARG(B >= 1 && B <= 65535, "state_frame_offsets: batch size B = %d must be in [1, 65535]", B);
  GANTTS_CHECK_ARG(P >= 1, "state_frame_offsets: phones P = %d must be >= 1", P);
  GANTTS_CHECK_ARG(S >= 1 && S <= FR_MAX_S, "state_frame_offsets: states S = %d must be in [1, %d]", S, FR_MAX_S);
  GANTTS_CHECK_ARG(dur_bstride >= 0 && dur_pstride >= 0,
                   "state_frame_offsets: strides dur_bstride = %lld and dur_pstride = %lld must be >= 0",
                   (long long)dur_bstride, (long long)dur_pstride);
  cudaStream_t st = as_stream(stream);
  GANTTS_CUDA(cudaMemsetAsync(status_dev, 0, sizeof(int64_t), st));
  state_frame_offsets_kernel<<<(unsigned)B, FR_SCAN_THREADS, 0, st>>>(
      dur, dur_bstride, dur_pstride, phone_lengths_dev, P, S, offsets, frame_lengths,
      reinterpret_cast<unsigned long long*>(status_dev));
  GANTTS_LAUNCH_CHECK("state_frame_offsets_kernel");
  return GANTTS_OK;
}

extern "C" int gantts_expand_state_frames(const float* phone_x, int64_t x_bstride, int64_t x_pstride, const float* dur,
                                          int64_t dur_bstride, int64_t dur_pstride, const int64_t* offsets,
                                          const int64_t* frame_lengths, const float* scale_dev, const float* min_dev,
                                          int B, int P, int L, int S, int T, float* out, void* stream) {
  GANTTS_CHECK_ARG(phone_x && dur && offsets && frame_lengths && scale_dev && min_dev && out,
                   "expand_state_frames: null pointer: phone_x, dur, offsets, frame_lengths, scale_dev, min_dev and "
                   "out are all required");
  GANTTS_CHECK_ARG(B >= 1 && B <= 65535, "expand_state_frames: batch size B = %d must be in [1, 65535]", B);
  GANTTS_CHECK_ARG(P >= 1, "expand_state_frames: phones P = %d must be >= 1", P);
  GANTTS_CHECK_ARG(L >= 1 && L <= FR_MAX_L, "expand_state_frames: linguistic width L = %d must be in [1, %d]", L,
                   FR_MAX_L);
  GANTTS_CHECK_ARG(S >= 1 && S <= FR_MAX_S, "expand_state_frames: states S = %d must be in [1, %d]", S, FR_MAX_S);
  GANTTS_CHECK_ARG(T >= 1 && (int64_t)T <= FR_MAX_FRAMES, "expand_state_frames: padded length T = %d must be in [1, %d]",
                   T, (int)FR_MAX_FRAMES);
  GANTTS_CHECK_ARG(x_bstride >= 0 && x_pstride >= 0 && dur_bstride >= 0 && dur_pstride >= 0,
                   "expand_state_frames: strides x_bstride = %lld, x_pstride = %lld, dur_bstride = %lld and "
                   "dur_pstride = %lld must be >= 0", (long long)x_bstride, (long long)x_pstride,
                   (long long)dur_bstride, (long long)dur_pstride);
  const int W = L + FR_SUBPHONE;
  int lanes = 32;                                        // threads per frame: 32, 64, 128 or 256
  while (lanes < W && lanes < FR_THREADS) lanes <<= 1;
  const dim3 grid((unsigned)((T + FR_TILE - 1) / FR_TILE), (unsigned)B);
  expand_state_frames_kernel<<<grid, FR_THREADS, 0, as_stream(stream)>>>(
      phone_x, x_bstride, x_pstride, dur, dur_bstride, dur_pstride, offsets, frame_lengths, scale_dev, min_dev, P, L, S,
      T, lanes, out);
  GANTTS_LAUNCH_CHECK("expand_state_frames_kernel");
  return GANTTS_OK;
}
