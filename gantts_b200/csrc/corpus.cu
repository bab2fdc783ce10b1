// Mini-batches gathered from a training split held on the device (train.py:145-159 collate_fn, then :494-501's sort):
// the split's normalised utterances are packed frame after frame into X [N][Dx] and Y [N][Dy], and each batch is one
// launch that copies every row's frames into x [b][t][Dx] and y [b][t][Dy] and writes the padding as 0.
//
// A row of the output is one contiguous run of t * D floats whose first length * D come from one contiguous run of the
// corpus, so the kernel works on flat element ranges: block (chunk, row, tensor) copies float4 vectors where both the
// destination and the source are 16-byte aligned, float4 stores of scalar loads where only the destination is, and a
// scalar head and tail around them.  It only moves bits, so a row equals the host loader's row exactly.
#include "common.cuh"

namespace gantts {

constexpr int CG_THREADS = 256;
constexpr int CG_VECS = 4;                               // float4 stores per thread and block, on average
constexpr int CG_MAX_T = 1 << 24;
constexpr int CG_MAX_D = 65535;

// Element e of a row: src[e] below n_copy, else the padding 0.
__device__ __forceinline__ float corpus_elem(const float* src, int64_t e, int64_t n_copy) {
  return e < n_copy ? __ldg(src + e) : 0.f;
}

__global__ void __launch_bounds__(CG_THREADS) corpus_gather_kernel(
    const float* __restrict__ X, const float* __restrict__ Y, int64_t N, int Dx, int Dy,
    const int64_t* __restrict__ offsets, const int64_t* __restrict__ lengths, int t, float* __restrict__ x_out,
    float* __restrict__ y_out, unsigned long long* status) {
  const int r = blockIdx.y;
  const bool is_y = blockIdx.z != 0;
  const int D = is_y ? Dy : Dx;
  float* dst = (is_y ? y_out : x_out) + (int64_t)r * t * D;
  int64_t off = offsets[r], len = lengths[r];
  if (!(off >= 0 && len >= 0 && len <= t && off <= N - len)) {      // a row outside the corpus: all padding
    if (status && !is_y && blockIdx.x == 0 && threadIdx.x == 0) atomicOr(status, (unsigned long long)GANTTS_CORPUS_BAD_ROW);
    off = 0;
    len = 0;
  }
  const float* src = (is_y ? Y : X) + off * D;
  const int64_t n_copy = len * D, n_total = (int64_t)t * D;
  // elements before the first 16-byte aligned destination address, then whole float4s, then the rest
  const int64_t head = min((int64_t)((4 - ((reinterpret_cast<uintptr_t>(dst) >> 2) & 3)) & 3), n_total);
  const int64_t nvec = (n_total - head) >> 2;
  const int64_t tail0 = head + 4 * nvec;
  if (blockIdx.x == 0) {                                 // at most 3 + 3 scalars, on threads 0-2 and 32-34
    const int i = threadIdx.x;
    if (i < head) dst[i] = corpus_elem(src, i, n_copy);
    if (i >= 32 && tail0 + (i - 32) < n_total) dst[tail0 + (i - 32)] = corpus_elem(src, tail0 + (i - 32), n_copy);
  }
  float4* dst4 = reinterpret_cast<float4*>(dst + head);
  const float* s = src + head;
  const bool src_aligned = (reinterpret_cast<uintptr_t>(s) & 15) == 0;
  const int64_t full = n_copy > head ? (n_copy - head) >> 2 : 0;     // vectors wholly inside the copied frames
  for (int64_t v = (int64_t)blockIdx.x * CG_THREADS + threadIdx.x; v < nvec; v += (int64_t)gridDim.x * CG_THREADS) {
    float4 q;
    if (v < full) {
      if (src_aligned) {
        q = __ldg(reinterpret_cast<const float4*>(s) + v);
      } else {
        q = make_float4(__ldg(s + 4 * v), __ldg(s + 4 * v + 1), __ldg(s + 4 * v + 2), __ldg(s + 4 * v + 3));
      }
    } else {
      const int64_t e = head + 4 * v;
      q = make_float4(corpus_elem(src, e, n_copy), corpus_elem(src, e + 1, n_copy), corpus_elem(src, e + 2, n_copy),
                      corpus_elem(src, e + 3, n_copy));
    }
    dst4[v] = q;
  }
}

}  // namespace gantts

using namespace gantts;

extern "C" int gantts_corpus_gather(const float* X, const float* Y, int64_t N, int Dx, int Dy,
                                    const int64_t* offsets_dev, const int64_t* lengths_dev, int b, int t, float* x_out,
                                    float* y_out, int64_t* status_dev, void* stream) {
  GANTTS_CHECK_ARG(X && Y && offsets_dev && lengths_dev && x_out && y_out,
                   "corpus_gather: null pointer: X, Y, offsets_dev, lengths_dev, x_out and y_out are all required");
  GANTTS_CHECK_ARG(N >= 1, "corpus_gather: corpus frames N = %lld must be >= 1", (long long)N);
  GANTTS_CHECK_ARG(Dx >= 1 && Dx <= CG_MAX_D && Dy >= 1 && Dy <= CG_MAX_D,
                   "corpus_gather: widths Dx = %d and Dy = %d must be in [1, %d]", Dx, Dy, CG_MAX_D);
  GANTTS_CHECK_ARG(b >= 1 && b <= 65535, "corpus_gather: batch size b = %d must be in [1, 65535]", b);
  GANTTS_CHECK_ARG(t >= 1 && t <= CG_MAX_T, "corpus_gather: padded length t = %d must be in [1, %d]", t, CG_MAX_T);
  const int64_t vecs = ((int64_t)t * (Dx > Dy ? Dx : Dy) + 3) / 4;
  const int64_t chunks = (vecs + CG_THREADS * CG_VECS - 1) / (CG_THREADS * CG_VECS);
  const dim3 grid((unsigned)chunks, (unsigned)b, 2);
  corpus_gather_kernel<<<grid, CG_THREADS, 0, as_stream(stream)>>>(
      X, Y, N, Dx, Dy, offsets_dev, lengths_dev, t, x_out, y_out, reinterpret_cast<unsigned long long*>(status_dev));
  GANTTS_LAUNCH_CHECK("corpus_gather_kernel");
  return GANTTS_OK;
}
