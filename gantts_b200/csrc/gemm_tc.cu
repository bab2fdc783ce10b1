// Hopper tensor-core engine (GANTTS_ENGINE_TC): bf16x3 split GEMM on wgmma with fp32 accumulation in registers.
//
// Every fp32 operand v is carried as two bf16 planes (hi = bf16(v), lo = bf16(v - hi)); a product
// a*b is evaluated as a_hi*b_hi + a_hi*b_lo + a_lo*b_hi on the tensor cores (three wgmma per K=16 step
// into the same fp32 accumulator), which keeps ~2^-16 relative error per product -- fp32-grade parity at
// 1.5x the cost of a single TF32 pass, where plain TF32/BF16 (2e-3) would miss the 1e-4 bar.
//
// One persistent warp-specialised kernel, output tiles of 128 rows x BN columns, two operand layouts:
//   MN = false : C[M][N] = A[M][K] * B[N][K]^T   both operands K-major   (layer forward, gx = gz W)
//   MN = true  : C[N][K] = A[M][N]^T * B[M][K]   both operands MN-major  (gW = gz^T x, split over M)
// warpgroup 0: one TMA producer thread filling a smem ring of `num_stages` {A_hi, A_lo, B_hi, B_lo} tiles
// (SWIZZLE_128B, full/empty mbarriers per stage) across all of the CTA's tiles; warpgroups 1-2: every tile together,
// warpgroup w issuing one wgmma.m64n{BN}k16 per product for rows 64w .. 64w + 63.  Each warpgroup stages its
// accumulators through its warps' shared-memory buffers so that each epilogue thread owns 16 consecutive columns of one
// row (bias / LeakyReLU / dropout / sigmoid; fp32 outputs leave as 16-byte stores, bf16 hi/lo planes are restaged in
// the same buffer and leave as TMA stores that drain while the warps go on); that epilogue runs while the producer
// refills the ring for the CTA's next tile.
#include <cuda.h>
#include <cuda_bf16.h>

#include "common.cuh"
#include "tc_ptx.cuh"

namespace gantts {

constexpr int TC_WG_WARPS = 4;      // warps of one MMA + epilogue warpgroup
constexpr int TC_THREADS = 128 + 2 * 32 * TC_WG_WARPS;   // warpgroup 0 TMA, warpgroups 1-2 MMA + epilogue
constexpr int TC_BM = 128;          // output rows per tile (two wgmma m64 row blocks, one per MMA warpgroup)
constexpr int TC_WARP_PITCH = 20;   // floats per row of a warp's epilogue buffer (float4-aligned, conflict-free reads)
constexpr int TC_WARP_BUF_FLOATS = 32 * TC_WARP_PITCH;   // one 32-row x 16-column chunk (>= the 2 KB fp32 scratch)
constexpr int TC_MAX_BN = 128;      // output columns per tile
constexpr int TC_KK_BK = 64;        // reduction elements per stage, K-major (one 128-byte swizzled row)
constexpr int TC_MN_BK = 32;        // reduction rows per stage of the weight-gradient GEMM
constexpr int TC_MAX_STAGES = 8;
constexpr int TC_PRODUCER_REGS = 40;    // setmaxnreg: the TMA warpgroup gives registers to the MMA warpgroups
constexpr int TC_CONSUMER_REGS = 232;   // 128 x 40 + 256 x 232 <= 64 K registers
constexpr uint32_t TC_SMEM_MAX = 227 * 1024;         // opt-in shared memory per block on sm_90
constexpr uint32_t TC_BIAS_SMEM = 4096;              // staged bias vector (<= 1024 columns)
constexpr uint32_t TC_ONES_SMEM = 1024;              // all-ones bf16 tile (MN-major bias gradient)

// Epilogue flavours (template parameter of the kernel).
constexpr int EPI_F32 = 0;          // bias + {none | leaky+dropout | sigmoid} -> fp32 C (optionally +=)
constexpr int EPI_PLANES_FWD = 1;   // bias + leaky + dropout -> bf16 hi/lo planes (next layer's operand)
constexpr int EPI_PLANES_BWD = 2;   // acc * act'(saved output hi plane) -> bf16 hi/lo planes (gz)

struct GemmParams {
  int64_t rows_a;       // output rows   (extent of A's MN dimension)
  int cols_b;           // output cols   (extent of B's MN dimension)
  int64_t red;          // reduction extent
  int64_t red_chunk;    // reduction elements per z-slice (multiple of bk)
  int num_a, num_b, num_z;
  int bn;               // output columns per tile, 64 or 128
  int num_stages;
  uint32_t stage_bytes, b_plane_bytes, tx_bytes;
  int64_t row0;         // global index of the first output row (dropout keys use global rows when a launch covers a row window)
  uint32_t a_plane;     // bytes of one A plane tile in a stage
  uint32_t atom_bytes;  // MN-major: bytes of one 64-wide atom ([bk rows][128 B])
  uint32_t epi_off;     // byte offset (from the aligned smem base) of the 8 per-warp epilogue buffers
  uint32_t bar_off;     // byte offset (from the aligned smem base) of the mbarriers
  // EPI_F32 output
  float* C;
  int64_t ldc, c_zstride;
  int vec_ok;           // C 16-byte aligned, ldc % 4 == 0, no accumulate: float4 stores from registers;
                        // 0 = through the warp's buffer as a transpose scratch (epilogue_f32_smem)
  int accumulate;
  // planes output (EPI_PLANES_*): written through the tmOh / tmOl tensor maps, [rows_a][out_pitch] bf16
  int64_t out_pitch;
  // activation-derivative code plane: 2 bits per element (bit0 = zero/dropped, bit1 = negative), one
  // uint32 per (row, 16 columns).  Written by EPI_PLANES_FWD, read by EPI_PLANES_BWD.
  uint32_t* code;
  int64_t code_pitch;   // words per row
  uint32_t bias_off;    // byte offset (from the aligned smem base) of the staged bias vector, 0 = none
  // MN-major only: column sums of A (= bias gradient) via an extra N=8 MMA against a tile of ones
  float* db;            // [num_z][rows_a] partial sums, or null
  uint32_t ones_off;    // byte offset of the all-ones bf16 tile from the aligned smem base
  // epilogue math
  const float* bias;
  int act;
  float slope, keep_scale;
  uint32_t thresh;
  uint64_t seed;
};

__device__ __forceinline__ uint32_t pack_bf16x2(float a, float b) {
  __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

// Split 8 fp32 values into packed bf16 hi/lo words (4 words each).
__device__ __forceinline__ void split8(const float* v, uint32_t* h, uint32_t* l) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float a = v[2 * i], b = v[2 * i + 1];
    const uint32_t hp = pack_bf16x2(a, b);
    const float ah = __uint_as_float(hp << 16), bh = __uint_as_float(hp & 0xffff0000u);
    h[i] = hp;
    l[i] = pack_bf16x2(a - ah, b - bh);
  }
}

// One pass of a warp's planes epilogue out to global memory: lane l's 16 split values (row l % 16 of the warp's 16,
// columns 16 (l / 16) .. + 15 of the pass) go to the warp's buffer as a dense [16][32] bf16 box per plane (hi at byte
// 0, lo at 1024), and lane 0 hands both boxes to the TMA unit as one bulk group.  The caller has read the buffer out
// (the __syncwarp below orders that) and waits with bulk_wait_read before writing it again; so does this function,
// for the store it issued last.  TMA clips the box at
// rows_a and at the pitch: every 16-column chunk that starts below cols_b is written whole, the pad columns up to the
// pitch holding the epilogue of zero-padded operands.
__device__ __forceinline__ void store_planes_pass(const CUtensorMap* mh, const CUtensorMap* ml, float* buf,
                                                  const uint32_t (&h)[8], const uint32_t (&l)[8], int lane, int col,
                                                  int64_t row0, const GemmParams& p) {
  if (lane == 0) ptx::bulk_wait_read<0>();
  __syncwarp();
  uint4* sh = reinterpret_cast<uint4*>(reinterpret_cast<uint8_t*>(buf) + (lane & 15) * 64 + (lane >> 4) * 32);
  uint4* sl = sh + 1024 / 16;
  sh[0] = make_uint4(h[0], h[1], h[2], h[3]);
  sh[1] = make_uint4(h[4], h[5], h[6], h[7]);
  sl[0] = make_uint4(l[0], l[1], l[2], l[3]);
  sl[1] = make_uint4(l[4], l[5], l[6], l[7]);
  ptx::fence_proxy_async();
  __syncwarp();
  if (lane == 0 && row0 < p.rows_a && col < p.out_pitch) {
    const uint32_t s = ptx::smem_u32(buf);
    ptx::tma_store_2d(mh, s, col, (int32_t)row0);
    ptx::tma_store_2d(ml, s + 1024, col, (int32_t)row0);
    ptx::bulk_commit();
  }
}

// Dropout of the 16 values of one row at columns [col, col+16), col % 16 == 0: v = keep ? v * scale : 0
// (common.cuh: one hash chain per four columns, one unsigned compare per element).
__device__ __forceinline__ void dropout16(float (&v)[16], uint64_t seed, uint32_t row, int n_cols, int col, uint32_t thresh,
                                          float scale) {
  const uint32_t quarter_n = (uint32_t)(n_cols + 3) >> 2, limit = drop_limit(thresh);
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const DropBits d = dropout_quad_bits(seed, row, quarter_n, ((uint32_t)col >> 2) + q);
    v[4 * q] = (d.a << 16) > limit ? v[4 * q] * scale : 0.f;
    v[4 * q + 1] = d.a > limit ? v[4 * q + 1] * scale : 0.f;
    v[4 * q + 2] = (d.b << 16) > limit ? v[4 * q + 2] * scale : 0.f;
    v[4 * q + 3] = d.b > limit ? v[4 * q + 3] * scale : 0.f;
  }
}

// EPI_F32 for every output that is not vec_ok: row strides that are not a multiple of 4 floats (y_hat: ld 187, the
// discriminator input gradient: ld 58, weight-gradient partials of 425- and 58-wide layers) and accumulating outputs.
// Straight from registers a thread could only issue 16 scalar stores per chunk and a warp store would touch 32 rows =
// 32 sectors.  Here the warp's 32 x 16 tile goes through a private 2 KB shared-memory scratch (float4 writes,
// XOR-swizzled: conflict-free) and is written back with lanes 0-15 / 16-31 covering two whole 64-byte row segments per
// store instruction.  Slot l (0-31) of the pass holds row row0 + (l % 16) and the 16 columns from col + 16 (l / 16):
// the warp's 16 rows of its warpgroup's 64-row block, two 16-column chunks per pass.
__device__ __forceinline__ void epilogue_f32_smem(const GemmParams& p, const uint32_t (&r)[16], int64_t row0,
                                                  int lane, int col, int z, const float* __restrict__ bias_s,
                                                  float* scr) {
  const int64_t row = row0 + (lane & 15);
  const int lcol = col + 16 * (lane >> 4);
  float v[16];
#pragma unroll
  for (int j = 0; j < 16; ++j) v[j] = __uint_as_float(r[j]);
  if (p.bias) {
    if (bias_s) {
#pragma unroll
      for (int j = 0; j < 16; ++j) v[j] += bias_s[lcol + j];
    } else {
#pragma unroll
      for (int j = 0; j < 16; ++j)
        if (lcol + j < p.cols_b) v[j] += __ldg(p.bias + lcol + j);
    }
  }
  if (p.act == GANTTS_ACT_LEAKY_DROPOUT) {
#pragma unroll
    for (int j = 0; j < 16; ++j) v[j] = fmaxf(v[j], v[j] * p.slope);
    if (p.thresh) dropout16(v, p.seed, (uint32_t)(row + p.row0), p.cols_b, lcol, p.thresh, p.keep_scale);
  } else if (p.act == GANTTS_ACT_SIGMOID) {
#pragma unroll
    for (int j = 0; j < 16; ++j) v[j] = 1.f / (1.f + expf(-v[j]));
  }
  const int sw = (lane >> 1) & 3;
#pragma unroll
  for (int k = 0; k < 4; ++k)
    *reinterpret_cast<float4*>(scr + lane * 16 + 4 * (k ^ sw)) = make_float4(v[4 * k], v[4 * k + 1], v[4 * k + 2], v[4 * k + 3]);
  __syncwarp();
  float* cbase = p.C + (int64_t)z * p.c_zstride;
  const int j = lane & 15, hr = lane >> 4;
  // accumulate (the discriminator's input gradient added into its window of g_static): all loads of a half are issued
  // before its first store -- interleaved `*q = *q + val` serialises load -> store round trips per warp (the compiler
  // must assume the store aliases the next load).  Slots 16h .. 16h + 15 all lie in chunk h; slot 16h + 2i + hr holds
  // row row0 + 2i + hr.  Each element's address and bounds check are computed once for its load and its store: ptxas
  // then predicates the stores instead of branching around each one and recomputing its address.
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int c = col + 16 * h + j;
    const bool col_ok = c < p.cols_b;
    float* q[8];
    bool ok[8];
    float old[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int64_t rw = row0 + 2 * i + hr;
      q[i] = cbase + c + rw * p.ldc;
      ok[i] = col_ok && rw < p.rows_a;
    }
    if (p.accumulate) {
#pragma unroll
      for (int i = 0; i < 8; ++i) old[i] = ok[i] ? __ldcg(q[i]) : 0.f;
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int rr = 2 * (8 * h + i) + hr;
      const float val = scr[rr * 16 + 4 * ((j >> 2) ^ ((rr >> 1) & 3)) + (j & 3)];
      if (ok[i]) *q[i] = p.accumulate ? old[i] + val : val;
    }
  }
  __syncwarp();
}

// One 16-column chunk of one output row: registers (fp32 accumulators) -> global (EPI_F32) or -> the split hi / lo
// words `h`, `l` (EPI_PLANES_*).  Returns the derivative code word of the chunk (EPI_PLANES_FWD); `code_in` is the
// saved word (BWD).
template <int EPI>
__device__ __forceinline__ uint32_t epilogue_chunk16(const GemmParams& p, const uint32_t (&r)[16], int64_t row,
                                                     int col, int z, const float* __restrict__ bias_s,
                                                     uint32_t code_in, uint32_t (&h)[8], uint32_t (&l)[8]) {
  uint32_t code = 0;
  float v[16];
#pragma unroll
  for (int j = 0; j < 16; ++j) v[j] = __uint_as_float(r[j]);
  if (EPI == EPI_F32) {
    float* crow = p.C + (int64_t)z * p.c_zstride + row * p.ldc;
    if (p.bias) {
      if (bias_s) {
#pragma unroll
        for (int j = 0; j < 16; ++j) v[j] += bias_s[col + j];
      } else {
#pragma unroll
        for (int j = 0; j < 16; ++j)
          if (col + j < p.cols_b) v[j] += __ldg(p.bias + col + j);
      }
    }
    if (p.act == GANTTS_ACT_LEAKY_DROPOUT) {
#pragma unroll
      for (int j = 0; j < 16; ++j) v[j] = fmaxf(v[j], v[j] * p.slope);
      if (p.thresh) dropout16(v, p.seed, (uint32_t)(row + p.row0), p.cols_b, col, p.thresh, p.keep_scale);
    } else if (p.act == GANTTS_ACT_SIGMOID) {
#pragma unroll
      for (int j = 0; j < 16; ++j) v[j] = 1.f / (1.f + expf(-v[j]));
    }
    // only vec_ok outputs get here (the others are staged): float4 stores, scalar ones for the column tail
#pragma unroll
    for (int j = 0; j < 16; j += 4) {
      const int c = col + j;
      if (c + 3 < p.cols_b) {
        *reinterpret_cast<float4*>(crow + c) = make_float4(v[j], v[j + 1], v[j + 2], v[j + 3]);
      } else {
#pragma unroll
        for (int e = 0; e < 4; ++e)
          if (c + e < p.cols_b) crow[c + e] = v[j + e];
      }
    }
  } else if (EPI == EPI_PLANES_FWD) {
    // reference gantts/models.py:137-139: Dropout(LeakyReLU(Linear(x)))
    if (bias_s) {
#pragma unroll
      for (int j = 0; j < 16; j += 4) {
        const float4 b4 = *reinterpret_cast<const float4*>(bias_s + col + j);   // broadcast LDS.128
        v[j] += b4.x; v[j + 1] += b4.y; v[j + 2] += b4.z; v[j + 3] += b4.w;
      }
    } else {
#pragma unroll
      for (int j = 0; j < 16; ++j)
        if (col + j < p.cols_b) v[j] += __ldg(p.bias + col + j);
    }
    // LeakyReLU as compare + select (torch's x > 0 ? x : x * slope), dropout keep as one unsigned compare per element
    // (common.cuh); the 2-bit derivative code (bit 0: derivative 0, bit 1: negative side) is OR-ed in under the very
    // predicates those compares produce.  With dropout on, bit 0 = "dropped"; a kept element whose pre-activation is
    // exactly 0 decodes as the positive side (measure zero).  Without dropout bit 0 = (v == 0).
    if (p.thresh) {
      const uint32_t quarter_n = (uint32_t)(p.cols_b + 3) >> 2, limit = drop_limit(p.thresh);
      const uint32_t grow = (uint32_t)(row + p.row0);
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const DropBits d = dropout_quad_bits(p.seed, grow, quarter_n, ((uint32_t)col >> 2) + q);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int j = 4 * q + e;
          const uint32_t w = e < 2 ? d.a : d.b;
          const bool keep = ((e & 1) ? w : (w << 16)) > limit;
          const bool neg = v[j] < 0.f;
          const float a = neg ? v[j] * p.slope : v[j];
          v[j] = keep ? a * p.keep_scale : 0.f;
          if (!keep) code |= 1u << (2 * j);
          if (neg) code |= 2u << (2 * j);
        }
      }
    } else {
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const bool neg = v[j] < 0.f;
        v[j] = neg ? v[j] * p.slope : v[j];
        if (v[j] == 0.f) code |= 1u << (2 * j);
        if (neg) code |= 2u << (2 * j);
      }
    }
    split8(v, h, l);
    split8(v + 8, h + 4, l + 4);
  } else {  // EPI_PLANES_BWD: gz = g * act'(h), derivative class from the saved 2-bit code
    const float dpos = p.keep_scale, dneg = p.slope * p.keep_scale;
    const float dzero = p.thresh ? 0.f : p.slope;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const uint32_t cj = (code_in >> (2 * j)) & 3u;
      v[j] *= (cj & 1u) ? dzero : ((cj & 2u) ? dneg : dpos);
    }
    split8(v, h, l);
    split8(v + 8, h + 4, l + 4);
  }
  return code;
}

// One warpgroup's share of the reduction of a 128 x BN tile: the 64-row block `blk`, for each smem stage BK/16 steps
// of hi*hi, hi*lo, lo*hi (and, with DB, the two ones-tile MMAs of the bias gradient) into `acc`, while the other
// warpgroup issues the other block from the same stages.  Stage s is released (one arrive per warp) once the wgmma
// group of stage s + 1 has been issued and stage s's group has completed (wait_group 1), so one stage's MMAs are always
// in flight.
template <bool MN, int BN, bool DB>
__device__ __forceinline__ void mma_tile(const GemmParams& p, float (&acc)[BN / 2], float (&accdb)[4], uint32_t base,
                                         uint32_t full0, uint32_t empty0, uint64_t d_ones, int nk, uint32_t& s,
                                         uint32_t& ph, int lane, int blk) {
  constexpr int BK = MN ? TC_MN_BK : TC_KK_BK;
  constexpr uint32_t kstep = MN ? 2048u : 32u;   // K = 16: 16 rows of 128 B (MN-major), 32 B inside the row (K-major)
  const uint32_t a_half = MN ? p.atom_bytes : 8192u;  // rows 64-127 of A: the next MN atom / 64 rows of 128 B
  const uint32_t a_off = (uint32_t)blk * a_half;
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
  uint32_t prev = 0;
#pragma unroll 1
  for (int kb = 0; kb < nk; ++kb) {
    ptx::mbar_wait(full0 + 8 * s, ph);
    const uint32_t sa_hi = base + s * p.stage_bytes, sa_lo = sa_hi + p.a_plane;
    const uint32_t sb_hi = sa_lo + p.a_plane, sb_lo = sb_hi + p.b_plane_bytes;
    ptx::wgmma_fence();
#pragma unroll
    for (int k = 0; k < BK / 16; ++k) {
      const uint64_t db_hi = ptx::make_smem_desc(sb_hi + k * kstep, p.atom_bytes, 1024u);
      const uint64_t db_lo = ptx::make_smem_desc(sb_lo + k * kstep, p.atom_bytes, 1024u);
      const uint64_t da_hi = ptx::make_smem_desc(sa_hi + a_off + k * kstep, p.atom_bytes, 1024u);
      const uint64_t da_lo = ptx::make_smem_desc(sa_lo + a_off + k * kstep, p.atom_bytes, 1024u);
      if constexpr (BN == 128) {
        ptx::wgmma_m64n128k16<MN ? 1 : 0, MN ? 1 : 0>(acc, da_hi, db_hi);
        ptx::wgmma_m64n128k16<MN ? 1 : 0, MN ? 1 : 0>(acc, da_hi, db_lo);
        ptx::wgmma_m64n128k16<MN ? 1 : 0, MN ? 1 : 0>(acc, da_lo, db_hi);
      } else {
        ptx::wgmma_m64n64k16<MN ? 1 : 0, MN ? 1 : 0>(acc, da_hi, db_hi);
        ptx::wgmma_m64n64k16<MN ? 1 : 0, MN ? 1 : 0>(acc, da_hi, db_lo);
        ptx::wgmma_m64n64k16<MN ? 1 : 0, MN ? 1 : 0>(acc, da_lo, db_hi);
      }
      if constexpr (DB) {
        ptx::wgmma_m64n8k16<MN ? 1 : 0>(accdb, da_hi, d_ones);
        ptx::wgmma_m64n8k16<MN ? 1 : 0>(accdb, da_lo, d_ones);
      }
    }
    ptx::wgmma_commit();
    if (kb > 0) {
      ptx::wgmma_wait<1>();
      __syncwarp();
      if (lane == 0) ptx::mbar_arrive(empty0 + 8 * prev);   // the previous stage may be refilled
    }
    prev = s;
    if (++s == (uint32_t)p.num_stages) { s = 0; ph ^= 1; }
  }
  __syncwarp();
  ptx::wgmma_wait<0>();
  ptx::fence_regs(acc);
  ptx::fence_regs(accdb);
  __syncwarp();
  if (lane == 0) ptx::mbar_arrive(empty0 + 8 * prev);
}

// Persistent kernel: CTA b walks the tiles b, b + gridDim.x, ... (numbering: z-slice of the reduction, then row tile,
// then column tile, so the column tiles of one row tile are neighbours).  Warpgroup 0: one TMA producer thread runs
// through the stage ring continuously across the CTA's tiles.  Warpgroups 1 and 2 take every tile together,
// warpgroup w issuing rows 64w .. 64w + 63 from the same ring stages, which are released when both have arrived; each
// then runs the epilogue of its 64 rows while the producer refills the ring for the next tile.  Two warpgroups issuing
// MMAs side by side keep the tensor cores busy, and each epilogue covers half a tile.
template <bool MN, int EPI, int BN>
__global__ void __launch_bounds__(TC_THREADS, 1)
gemm_bf16x3_kernel(const __grid_constant__ CUtensorMap tmAh, const __grid_constant__ CUtensorMap tmAl,
                   const __grid_constant__ CUtensorMap tmBh, const __grid_constant__ CUtensorMap tmBl,
                   const __grid_constant__ CUtensorMap tmOh, const __grid_constant__ CUtensorMap tmOl,
                   const GemmParams p) {
  constexpr int BK = MN ? TC_MN_BK : TC_KK_BK;
  constexpr bool PLANES = EPI != EPI_F32;   // output planes leave through TMA stores (tmOh / tmOl)
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = ptx::smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* const gbase = smem_raw + (base - raw);
  const uint32_t full0 = base + p.bar_off, empty0 = full0 + 8 * TC_MAX_STAGES;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles_ab = p.num_a * p.num_b;
  const int tiles = tiles_ab * p.num_z;
  auto k_blocks = [&](int z) {
    const int64_t r_beg = (int64_t)z * p.red_chunk;
    const int64_t r_end = r_beg + p.red_chunk < p.red ? r_beg + p.red_chunk : p.red;
    return (int)((r_end - r_beg + BK - 1) / BK);
  };

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.num_stages; ++s) {
      ptx::mbar_init(full0 + 8 * s, 1);
      ptx::mbar_init(empty0 + 8 * s, 2 * TC_WG_WARPS);   // one arrive per consuming warp
    }
    ptx::fence_barrier_init();
    ptx::prefetch_tensormap(&tmAh);
    ptx::prefetch_tensormap(&tmAl);
    ptx::prefetch_tensormap(&tmBh);
    ptx::prefetch_tensormap(&tmBl);
    if (PLANES) {
      ptx::prefetch_tensormap(&tmOh);
      ptx::prefetch_tensormap(&tmOl);
    }
  }
  // PDL: let the next kernel of the stream set itself up while this one drains; nothing produced by the
  // previous kernel is read before the dependency wait.
  ptx::pdl_launch_dependents();
  ptx::pdl_wait();
  const float* bias_s = nullptr;
  if (p.bias_off) {
    float* bs = reinterpret_cast<float*>(gbase + p.bias_off);
    const int nb = p.num_b * BN;                         // zero-padded to whole tiles
    for (int i = threadIdx.x; i < nb; i += TC_THREADS) bs[i] = i < p.cols_b ? p.bias[i] : 0.f;
    bias_s = bs;
  }
  if (MN && p.db != nullptr) {
    // all-ones bf16 tile (any swizzle of a constant tile is the same tile)
    uint32_t* ones = reinterpret_cast<uint32_t*>(gbase + p.ones_off);
    for (int i = threadIdx.x; i < (int)(TC_ONES_SMEM / 4); i += TC_THREADS) ones[i] = 0x3F803F80u;
    ptx::fence_proxy_async();
  }
  __syncthreads();

  if (warp < 4) {
    ptx::setmaxnreg_dec<TC_PRODUCER_REGS>();
    if (threadIdx.x == 0) {
      // ------------------------------------------------------------ TMA producer
      uint32_t s = 0, ph = 0;
      for (int t = blockIdx.x; t < tiles; t += gridDim.x) {
        const int z = t / tiles_ab, rem = t - z * tiles_ab;
        const int a0 = (rem / p.num_b) * TC_BM, b0 = (rem % p.num_b) * BN;
        const int64_t r_beg = (int64_t)z * p.red_chunk;
        const int nk = k_blocks(z);
        for (int kb = 0; kb < nk; ++kb) {
          const int64_t r0 = r_beg + (int64_t)kb * BK;
          ptx::mbar_wait(empty0 + 8 * s, ph ^ 1);
          const uint32_t fb = full0 + 8 * s;
          ptx::mbar_expect_tx(fb, p.tx_bytes);
          const uint32_t sa_hi = base + s * p.stage_bytes, sa_lo = sa_hi + p.a_plane;
          const uint32_t sb_hi = sa_lo + p.a_plane, sb_lo = sb_hi + p.b_plane_bytes;
          if (!MN) {
            ptx::tma_load_2d(sa_hi, &tmAh, fb, (int32_t)r0, a0);
            ptx::tma_load_2d(sb_hi, &tmBh, fb, (int32_t)r0, b0);
            ptx::tma_load_2d(sa_lo, &tmAl, fb, (int32_t)r0, a0);
            ptx::tma_load_2d(sb_lo, &tmBl, fb, (int32_t)r0, b0);
          } else {
            // 64-wide MN atoms, each [BK reduction rows][128 B]
            for (int j = 0; j < TC_BM / 64; ++j) {
              ptx::tma_load_2d(sa_hi + j * p.atom_bytes, &tmAh, fb, a0 + 64 * j, (int32_t)r0);
              ptx::tma_load_2d(sa_lo + j * p.atom_bytes, &tmAl, fb, a0 + 64 * j, (int32_t)r0);
            }
            for (int j = 0; j < BN / 64; ++j) {
              ptx::tma_load_2d(sb_hi + j * p.atom_bytes, &tmBh, fb, b0 + 64 * j, (int32_t)r0);
              ptx::tma_load_2d(sb_lo + j * p.atom_bytes, &tmBl, fb, b0 + 64 * j, (int32_t)r0);
            }
          }
          if (++s == (uint32_t)p.num_stages) { s = 0; ph ^= 1; }
        }
      }
    }
    return;
  }

  // ---------------------------------------------------------------- MMA + epilogue warpgroups
  ptx::setmaxnreg_inc<TC_CONSUMER_REGS>();
  const int wg = (warp >> 2) - 1;          // rows 64 wg .. 64 wg + 63 of every tile
  const int q = warp & 3;
  float* const wbuf = reinterpret_cast<float*>(gbase + p.epi_off) + (warp - 4) * TC_WARP_BUF_FLOATS;
  const uint64_t d_ones = ptx::make_smem_desc(base + p.ones_off, 0u, 1024u);
  uint32_t s = 0, ph = 0;
  for (int t = blockIdx.x; t < tiles; t += gridDim.x) {
    const int z = t / tiles_ab, rem = t - z * tiles_ab;
    const int nk = k_blocks(z);
    const int ta = rem / p.num_b, tb = rem % p.num_b;
    const int a0 = ta * TC_BM, b0 = tb * BN;
    const int64_t row0 = (int64_t)a0 + 64 * wg + 16 * q;   // first row of this warp in the tile
    const int64_t row = row0 + (lane & 15);                // the lane's row in the epilogue
    const bool row_ok = row < p.rows_a;
    // derivative code words of the lane's chunk in each pass (chunk 2k + lane / 16 of the tile), loaded before the
    // mainloop so that they arrive under the MMAs
    constexpr int PASSES = BN / 32;
    uint32_t codes[PASSES];
#pragma unroll
    for (int k = 0; k < PASSES; ++k) {
      const int c = b0 + 16 * (2 * k + (lane >> 4));
      codes[k] = 0u;
      if (EPI == EPI_PLANES_BWD && row_ok && c < p.cols_b) codes[k] = __ldg(p.code + row * p.code_pitch + (c >> 4));
    }
    float acc[BN / 2];
    float accdb[4] = {0.f, 0.f, 0.f, 0.f};
    const bool do_db = MN && p.db != nullptr && tb == 0;
    if (do_db)
      mma_tile<MN, BN, MN>(p, acc, accdb, base, full0, empty0, d_ones, nk, s, ph, lane, wg);
    else
      mma_tile<MN, BN, false>(p, acc, accdb, base, full0, empty0, d_ones, nk, s, ph, lane, wg);
    if (do_db && (lane & 3) == 0) {
      // m64n8 layout: lane holds rows lane/4 and lane/4 + 8 of its warp's 16, columns 0-1 (all columns are equal)
      const int64_t r = row0 + (lane >> 2);
      if (r < p.rows_a) p.db[(int64_t)z * p.rows_a + r] = accdb[0];
      if (r + 8 < p.rows_a) p.db[(int64_t)z * p.rows_a + r + 8] = accdb[2];
    }
    // ------------------------------------------------------------ epilogue.  Warp q holds rows 16q .. 16q + 15 of its
    // warpgroup's 64-row block; per pass of two 16-column chunks its fragments go through the warp's own shared-memory
    // buffer [32][TC_WARP_PITCH] so that lane l owns 16 consecutive columns of one row: row row0 + (l % 16), chunk
    // l / 16 of the pass.  Planes: pass k's split values wait in registers (hw, lw) until pass k + 1's fragments have
    // been read out of the buffer; the buffer then stages them for a TMA store, which reads it while pass k + 1's
    // arithmetic runs.  The last pass's store drains under the next tile's mainloop.
    uint32_t code_out[PASSES];
    uint32_t hw[8], lw[8];
#pragma unroll
    for (int k = 0; k < PASSES; ++k) {
      code_out[k] = 0u;
      if (PLANES && lane == 0) ptx::bulk_wait_read<0>(); // the buffer's last TMA store has read it
      __syncwarp();                                      // the previous pass has been read out of the buffer
      // m64nN layout: register 4j + 2g + e is row 16q + lane / 4 + 8g, column 8j + 2 (lane % 4) + e.  Slots 16h ..
      // 16h + 15 take the warp's rows of chunk 2k + h.
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int jj = 0; jj < 2; ++jj) {
          const int j = 2 * (2 * k + h) + jj;
          float* w = wbuf + (16 * h + (lane >> 2)) * TC_WARP_PITCH + 8 * jj + 2 * (lane & 3);
          *reinterpret_cast<float2*>(w) = make_float2(acc[4 * j], acc[4 * j + 1]);
          *reinterpret_cast<float2*>(w + 8 * TC_WARP_PITCH) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
        }
      __syncwarp();
      uint32_t rr[16];
      const float4* src = reinterpret_cast<const float4*>(wbuf + lane * TC_WARP_PITCH);
#pragma unroll
      for (int m = 0; m < 4; ++m) {
        const float4 f = src[m];
        rr[4 * m] = __float_as_uint(f.x); rr[4 * m + 1] = __float_as_uint(f.y);
        rr[4 * m + 2] = __float_as_uint(f.z); rr[4 * m + 3] = __float_as_uint(f.w);
      }
      const int col = b0 + 32 * k;                       // first column of the pass
      const int lcol = col + 16 * (lane >> 4);
      if (EPI == EPI_F32 && !p.vec_ok) {                 // whole warp takes part; rows beyond rows_a masked at the store
        __syncwarp();                                    // the buffer becomes the transpose scratch
        if (col < p.cols_b) epilogue_f32_smem(p, rr, row0, lane, col, z, bias_s, wbuf);
      } else if (EPI == EPI_F32) {
        if (row_ok && lcol < p.cols_b) epilogue_chunk16<EPI>(p, rr, row, lcol, z, bias_s, 0u, hw, lw);
      } else {                                           // whole warp: the TMA store clips rows and columns
        if (k > 0) store_planes_pass(&tmOh, &tmOl, wbuf, hw, lw, lane, col - 32, row0, p);
        code_out[k] = epilogue_chunk16<EPI>(p, rr, row, lcol, z, bias_s, codes[k], hw, lw);
      }
    }
    if (PLANES) store_planes_pass(&tmOh, &tmOl, wbuf, hw, lw, lane, b0 + 32 * (PASSES - 1), row0, p);
    if (EPI == EPI_PLANES_FWD && p.code != nullptr && row_ok) {
      uint32_t* cpp = p.code + row * p.code_pitch + (b0 >> 4);
#pragma unroll
      for (int k = 0; k < PASSES; ++k) {
        const int ck = 2 * k + (lane >> 4);
        if (b0 + 16 * ck < p.cols_b) cpp[ck] = code_out[k];
      }
    }
  }
  if (PLANES && lane == 0) ptx::bulk_wait<0>();          // the last stores are complete before the CTA exits
}

// ---------------------------------------------------------------------------- operand planes
// fp32 [rows][cols] (row stride rs) -> bf16 hi/lo planes [rows][pitch]; transpose: out[c][r] = in[r][c].
__global__ void split_planes_kernel(const float* __restrict__ src, int64_t rs, int64_t rows, int cols,
                                    __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo,
                                    int64_t pitch, int transpose) {
  pdl_entry();
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  if (!transpose) {
    // one warp per row, each lane converts PAIRS of columns -> 4-byte stores, 128 B per warp store
    for (int64_t r = warp; r < rows; r += nwarps) {
      const float* sr = src + r * rs;
      uint32_t* hr = reinterpret_cast<uint32_t*>(hi + r * pitch);
      uint32_t* lr = reinterpret_cast<uint32_t*>(lo + r * pitch);
#pragma unroll 2
      for (int c = 2 * lane; c < cols; c += 64) {
        const float a = sr[c], b = (c + 1 < cols) ? sr[c + 1] : 0.f;
        const uint32_t hp = pack_bf16x2(a, b);
        const float ah = __uint_as_float(hp << 16), bh = __uint_as_float(hp & 0xffff0000u);
        hr[c >> 1] = hp;
        lr[c >> 1] = pack_bf16x2(a - ah, b - bh);
      }
    }
  } else {
    for (int64_t r = warp; r < rows; r += nwarps)
      for (int c = lane; c < cols; c += 32) {
        const float v = src[r * rs + c];
        const __nv_bfloat16 h = __float2bfloat16_rn(v);
        hi[(int64_t)c * pitch + r] = h;
        lo[(int64_t)c * pitch + r] = __float2bfloat16_rn(v - __bfloat162float(h));
      }
  }
}

__global__ void splitk_reduce_kernel(const float* __restrict__ partial, int nsplit, int64_t n,
                                     float* __restrict__ out, int accumulate);

// ---------------------------------------------------------------------------- host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                  CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                  CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

// 2D bf16 tensor [rows][cols] with row pitch `pitch` elements; box = {box_cols, box_rows}, by default 64 columns (one
// 128-byte swizzled row) for the operand loads.  Out-of-range box elements are filled with zeros by loads and skipped
// by stores.
static int make_map(CUtensorMap* m, const void* ptr, int64_t rows, int64_t cols, int64_t pitch, int box_rows,
                    int box_cols = 64, CUtensorMapSwizzle swizzle = CU_TENSOR_MAP_SWIZZLE_128B) {
  EncodeTiledFn enc = get_encode();
  if (!enc) {
    set_error("tc: cuTensorMapEncodeTiled entry point unavailable");
    return GANTTS_E_CUDA;
  }
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)pitch * 2};
  cuuint32_t box[2] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("tc: cuTensorMapEncodeTiled failed (%d) rows=%lld cols=%lld pitch=%lld box_rows=%d", (int)r,
              (long long)rows, (long long)cols, (long long)pitch, box_rows);
    return GANTTS_E_CUDA;
  }
  return GANTTS_OK;
}

static int current_device() {
  int dev = -1;
  if (cudaGetDevice(&dev) != cudaSuccess) return -1;
  return dev;
}

static int num_sms() {
  static int n[64] = {};
  const int dev = current_device();
  if (dev < 0 || dev >= 64) return 132;
  if (!n[dev]) {
    cudaDeviceGetAttribute(&n[dev], cudaDevAttrMultiProcessorCount, dev);
    if (n[dev] <= 0) n[dev] = 132;
  }
  return n[dev];
}

static inline int64_t pitch_for(int64_t cols) { return (cols + 15) / 16 * 16; }   // 32-byte rows
static inline size_t plane_bytes(int64_t rows, int64_t cols) {
  return ((size_t)rows * pitch_for(cols) * 2 + 255) / 256 * 256;
}

struct Planes {
  __nv_bfloat16 *hi, *lo;
  int64_t rows, cols, pitch;
};

static Planes carve_planes(char*& cur, int64_t rows, int64_t cols) {
  Planes pl;
  pl.rows = rows;
  pl.cols = cols;
  pl.pitch = pitch_for(cols);
  pl.hi = reinterpret_cast<__nv_bfloat16*>(cur);
  cur += plane_bytes(rows, cols);
  pl.lo = reinterpret_cast<__nv_bfloat16*>(cur);
  cur += plane_bytes(rows, cols);
  return pl;
}

// rows [r0, r1) of a planes matrix, as a matrix of their own (rows stay 32-byte aligned: TMA takes them as a base)
static Planes plane_rows(Planes pl, int64_t r0, int64_t r1) {
  pl.hi += r0 * pl.pitch;
  pl.lo += r0 * pl.pitch;
  pl.rows = r1 - r0;
  return pl;
}

static int launch_split(const float* src, int64_t rs, int64_t rows, int cols, const Planes& pl, int transpose,
                        cudaStream_t st) {
  int64_t total = rows * cols;
  int nb = (int)((total + 1023) / 1024);
  if (nb > num_sms() * 8) nb = num_sms() * 8;
  if (nb < 1) nb = 1;
  GANTTS_PDL_LAUNCH((split_planes_kernel), nb, 256, 0, st, src, rs, rows, cols, pl.hi, pl.lo, pl.pitch, transpose);
  GANTTS_LAUNCH_CHECK("split_planes_kernel");
  return GANTTS_OK;
}

// Output columns per tile: 64 or 128, as few column tiles as TC_MAX_BN allows, split evenly.
static int pick_bn(int n) {
  int bn = (n + 63) / 64 * 64;
  if (bn <= TC_MAX_BN) return bn;
  int tiles = (n + TC_MAX_BN - 1) / TC_MAX_BN;
  bn = ((n + tiles - 1) / tiles + 63) / 64 * 64;
  return bn;
}

// Epilogue description filled by the callers of launch_gemm_kk.
struct EpiArgs {
  int epi = EPI_F32;
  // EPI_F32
  float* C = nullptr;
  int64_t ldc = 0;
  int accumulate = 0;
  // EPI_PLANES_*
  __nv_bfloat16 *out_hi = nullptr, *out_lo = nullptr;
  int64_t out_pitch = 0;
  uint32_t* code = nullptr;           // derivative code plane (written by PLANES_FWD, read by PLANES_BWD)
  int64_t code_pitch = 0;
  // math
  const float* bias = nullptr;
  int act = GANTTS_ACT_NONE;
  float slope = 0.f, p = 0.f;
  uint64_t seed = 0;
  int64_t row0 = 0;                   // global index of A's first row (row windows of a larger matrix)
};

static void fill_epilogue(GemmParams& p, const EpiArgs& e) {
  p.C = e.C;
  p.ldc = e.ldc;
  p.accumulate = e.accumulate;
  p.vec_ok = (!e.accumulate && e.C && (e.ldc & 3) == 0 && (reinterpret_cast<uintptr_t>(e.C) & 15) == 0) ? 1 : 0;
  p.out_pitch = e.out_pitch;
  p.code = e.code;
  p.code_pitch = e.code_pitch;
  p.bias = e.bias;
  p.act = e.act;
  p.slope = e.slope;
  p.keep_scale = e.p > 0.f ? 1.f / (1.f - e.p) : 1.f;
  p.thresh = e.p > 0.f ? (uint32_t)(e.p * 65536.f + 0.5f) : 0u;
  p.seed = e.seed;
  p.row0 = e.row0;
}

// Shared-memory plan of one launch (offsets from the 1024-aligned base): as many ring stages as fit next to the 8
// per-warp epilogue buffers (20 KB), the ones tile, the bias vector and the mbarriers.  Returns the dynamic smem bytes.
static size_t plan_smem(GemmParams& p, const EpiArgs& e) {
  const uint32_t epi = 2 * TC_WG_WARPS * TC_WARP_BUF_FLOATS * 4;
  const uint32_t fixed = 1024 + epi + TC_ONES_SMEM + TC_BIAS_SMEM + 256;
  p.num_stages = (int)((TC_SMEM_MAX - fixed) / p.stage_bytes);
  if (p.num_stages > TC_MAX_STAGES) p.num_stages = TC_MAX_STAGES;
  p.epi_off = (uint32_t)p.num_stages * p.stage_bytes;
  p.ones_off = p.epi_off + epi;
  p.bias_off = (e.bias && (size_t)p.num_b * p.bn * sizeof(float) <= TC_BIAS_SMEM) ? p.ones_off + TC_ONES_SMEM : 0u;
  p.bar_off = p.ones_off + TC_ONES_SMEM + TC_BIAS_SMEM;
  return (size_t)p.bar_off + 256 + 1024;
}

// mOh / mOl: the output planes of EPI_PLANES_* (any initialised map otherwise: the kernel does not read them).
template <bool MN, int EPI, int BN>
static int launch_kernel(const CUtensorMap& mAh, const CUtensorMap& mAl, const CUtensorMap& mBh,
                         const CUtensorMap& mBl, const CUtensorMap& mOh, const CUtensorMap& mOl, const GemmParams& p,
                         size_t smem, cudaStream_t st) {
  if (smem > TC_SMEM_MAX) {
    set_error("gemm: shared-memory plan of %zu bytes exceeds %u", smem, TC_SMEM_MAX);
    return GANTTS_E_UNSUPPORTED;
  }
  if (p.num_stages < 2) {
    // a stage is released only after the next one has been issued: one stage would never be refilled
    set_error("gemm: shared-memory plan leaves %d ring stage(s), the mainloop needs 2", p.num_stages);
    return GANTTS_E_UNSUPPORTED;
  }
  // the opt-in is per device (and context): remember it per device ordinal, not per process
  static bool attr[64] = {};
  const int dev = current_device();
  if (dev < 0 || dev >= 64 || !attr[dev]) {
    GANTTS_CUDA(cudaFuncSetAttribute(gemm_bf16x3_kernel<MN, EPI, BN>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)TC_SMEM_MAX));
    if (dev >= 0 && dev < 64) attr[dev] = true;
  }
  const int tiles = p.num_a * p.num_b * p.num_z;
  const int grid = tiles < num_sms() ? tiles : num_sms();
  prof_begin(MN ? PROF_GEMM_MN : PROF_GEMM_KK, 2.0 * (double)p.rows_a * p.cols_b * (double)p.red, st);
  GANTTS_PDL_LAUNCH((gemm_bf16x3_kernel<MN, EPI, BN>), (unsigned)grid, TC_THREADS, smem, st, mAh, mAl, mBh, mBl, mOh,
                    mOl, p);
  prof_end(st);
  GANTTS_LAUNCH_CHECK("gemm_bf16x3_kernel");
  return GANTTS_OK;
}

template <bool MN, int EPI>
static int launch_bn(const CUtensorMap& mAh, const CUtensorMap& mAl, const CUtensorMap& mBh, const CUtensorMap& mBl,
                     const CUtensorMap& mOh, const CUtensorMap& mOl, const GemmParams& p, size_t smem,
                     cudaStream_t st) {
  if (p.bn == 64) return launch_kernel<MN, EPI, 64>(mAh, mAl, mBh, mBl, mOh, mOl, p, smem, st);
  return launch_kernel<MN, EPI, 128>(mAh, mAl, mBh, mBl, mOh, mOl, p, smem, st);
}

// out[rows_a][cols_b] = epi(A * B^T)   (K-major planes A [rows_a][red], B [cols_b][red]).
static int launch_gemm_kk(const Planes& A, const Planes& B, const EpiArgs& e, cudaStream_t st) {
  GemmParams p{};
  p.rows_a = A.rows;
  p.cols_b = (int)B.rows;
  p.red = A.cols;
  if (B.cols != A.cols) {
    set_error("gemm_kk: reduction extents differ (%lld vs %lld)", (long long)A.cols, (long long)B.cols);
    return GANTTS_E_BADARG;
  }
  p.a_plane = TC_BM * 128u;
  p.red_chunk = (p.red + TC_KK_BK - 1) / TC_KK_BK * TC_KK_BK;
  p.bn = pick_bn(p.cols_b);
  p.num_a = (int)((p.rows_a + TC_BM - 1) / TC_BM);
  p.num_b = (p.cols_b + p.bn - 1) / p.bn;
  p.num_z = 1;
  p.b_plane_bytes = (uint32_t)p.bn * 128u;
  p.stage_bytes = 2 * p.a_plane + 2 * p.b_plane_bytes;
  p.tx_bytes = p.stage_bytes;
  p.c_zstride = 0;
  fill_epilogue(p, e);
  const size_t smem = plan_smem(p, e);
  CUtensorMap mAh, mAl, mBh, mBl;
  int rc;
  if ((rc = make_map(&mAh, A.hi, A.rows, A.cols, A.pitch, TC_BM))) return rc;
  if ((rc = make_map(&mAl, A.lo, A.rows, A.cols, A.pitch, TC_BM))) return rc;
  if ((rc = make_map(&mBh, B.hi, B.rows, B.cols, B.pitch, p.bn))) return rc;
  if ((rc = make_map(&mBl, B.lo, B.rows, B.cols, B.pitch, p.bn))) return rc;
  if (e.epi == EPI_F32) return launch_bn<false, EPI_F32>(mAh, mAl, mBh, mBl, mAh, mAl, p, smem, st);
  // output planes [rows_a][pitch]: one warp's pass is a 16-row x 32-column box per plane, written up to the pitch
  CUtensorMap mOh, mOl;
  if ((rc = make_map(&mOh, e.out_hi, p.rows_a, e.out_pitch, e.out_pitch, 16, 32, CU_TENSOR_MAP_SWIZZLE_NONE))) return rc;
  if ((rc = make_map(&mOl, e.out_lo, p.rows_a, e.out_pitch, e.out_pitch, 16, 32, CU_TENSOR_MAP_SWIZZLE_NONE))) return rc;
  switch (e.epi) {
    case EPI_PLANES_FWD: return launch_bn<false, EPI_PLANES_FWD>(mAh, mAl, mBh, mBl, mOh, mOl, p, smem, st);
    case EPI_PLANES_BWD: return launch_bn<false, EPI_PLANES_BWD>(mAh, mAl, mBh, mBl, mOh, mOl, p, smem, st);
  }
  set_error("gemm_kk: bad epilogue %d", e.epi);
  return GANTTS_E_BADARG;
}

// C[n][k] (+)= sum_m A[m][n] * B[m][k]  (MN-major planes A [red][rows_a], B [red][cols_b]);
// split over the reduction, partials in `partial`, reduced deterministically into C (ld = cols_b).
static size_t mn_partial_bytes(int64_t red, int rows_a, int cols_b, int* splits_out, int64_t* chunk_out) {
  int bn = pick_bn(cols_b);
  int tiles = ((rows_a + TC_BM - 1) / TC_BM) * ((cols_b + bn - 1) / bn);
  const int bk = TC_MN_BK;
  int64_t blocks = (red + bk - 1) / bk;
  int64_t splits = num_sms() / tiles;
  if (splits < 1) splits = 1;
  if (splits > blocks) splits = blocks;
  int64_t chunk = (blocks + splits - 1) / splits * bk;
  splits = (red + chunk - 1) / chunk;
  if (splits_out) *splits_out = (int)splits;
  if (chunk_out) *chunk_out = chunk;
  return ((size_t)splits * ((size_t)rows_a * cols_b + rows_a) * sizeof(float) + 255) / 256 * 256;
}

// Bytes that cover mn_partial_bytes(red, ...) for EVERY red in [1, red_max]: the split count is not monotone in red (the
// rounding of the chunk can give a shorter reduction more splits), but it never exceeds min(num_sms / tiles, blocks).
static size_t mn_partial_bytes_upto(int64_t red_max, int rows_a, int cols_b) {
  const int bn = pick_bn(cols_b);
  const int tiles = ((rows_a + TC_BM - 1) / TC_BM) * ((cols_b + bn - 1) / bn);
  const int64_t blocks = (red_max + TC_MN_BK - 1) / TC_MN_BK;
  int64_t splits = num_sms() / tiles;
  if (splits > blocks) splits = blocks;
  if (splits < 1) splits = 1;
  return ((size_t)splits * ((size_t)rows_a * cols_b + rows_a) * sizeof(float) + 255) / 256 * 256;
}

// Deferred deterministic split reductions: several (partial -> out) jobs summed by ONE launch.
constexpr int REDUCE_MAX_JOBS = 2 * GANTTS_MAX_LAYERS;
struct ReduceList {
  int n = 0;
  const float* partial[REDUCE_MAX_JOBS];
  float* out[REDUCE_MAX_JOBS];
  int splits[REDUCE_MAX_JOBS];
  int64_t len[REDUCE_MAX_JOBS];
  int64_t off[REDUCE_MAX_JOBS + 1];
};

// out[j][e] = sum_z partial[j][z][e] for a list of (partial, out) pairs: the split-K reduction of a model's weight
// gradients in one launch.  A block covers 32 float4 columns; its 8 warps take the splits z = w, w+8, ... (all loads of a
// warp independent and in flight together), the per-warp sums meet in shared memory and are added in warp order -- a fixed
// summation order, so the result is deterministic.  (The first version walked the splits sequentially per thread: a few
// percent issue utilisation on L2-resident partials.)
constexpr int MR_WARPS = 8;
__global__ void __launch_bounds__(32 * MR_WARPS) multi_reduce_kernel(ReduceList rl, int accumulate) {
  pdl_entry();
  __shared__ float4 part_s[MR_WARPS][32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int64_t total4 = rl.off[rl.n];                        // in units of 4 elements
  for (int64_t base = (int64_t)blockIdx.x * 32; base < total4; base += (int64_t)gridDim.x * 32) {
    const int64_t i = base + lane;
    int j = 0;
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
    int64_t e = 0, n = 0;
    bool vec = false;
    if (i < total4) {
      while (j + 1 < rl.n && i >= rl.off[j + 1]) ++j;
      e = (i - rl.off[j]) * 4;
      n = rl.len[j];
      vec = e + 3 < n && (n & 3) == 0;
      const float* part = rl.partial[j];
      const int splits = rl.splits[j];
      if (vec) {
#pragma unroll 4
        for (int z = w; z < splits; z += MR_WARPS) {
          const float4 v = __ldcg(reinterpret_cast<const float4*>(part + (int64_t)z * n + e));
          s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
        }
      } else {
        for (int z = w; z < splits; z += MR_WARPS) {
          const float* pz = part + (int64_t)z * n + e;
          if (e < n) s.x += pz[0];
          if (e + 1 < n) s.y += pz[1];
          if (e + 2 < n) s.z += pz[2];
          if (e + 3 < n) s.w += pz[3];
        }
      }
    }
    part_s[w][lane] = s;
    __syncthreads();
    if (w == 0 && i < total4) {
      float4 t = part_s[0][lane];
#pragma unroll
      for (int k = 1; k < MR_WARPS; ++k) {
        const float4 v = part_s[k][lane];
        t.x += v.x; t.y += v.y; t.z += v.z; t.w += v.w;
      }
      float* out = rl.out[j];
      // the flat gradient buffers need not be 16-byte aligned per tensor (a highway generator's gate shifts the
      // stack's gradients by S * S + S floats): vector stores only where the output allows them
      if (vec && (reinterpret_cast<uintptr_t>(out) & 15) == 0) {
        float4* o = reinterpret_cast<float4*>(out + e);
        if (accumulate) { const float4 c = *o; t.x += c.x; t.y += c.y; t.z += c.z; t.w += c.w; }
        *o = t;
      } else {
        const float tv[4] = {t.x, t.y, t.z, t.w};
        for (int q = 0; q < 4; ++q)
          if (e + q < n) out[e + q] = accumulate ? out[e + q] + tv[q] : tv[q];
      }
    }
    __syncthreads();
  }
}

static int flush_reduce(ReduceList& rl, int accumulate, cudaStream_t st) {
  if (rl.n == 0) return GANTTS_OK;
  rl.off[0] = 0;
  for (int j = 0; j < rl.n; ++j) rl.off[j + 1] = rl.off[j] + (rl.len[j] + 3) / 4;
  int64_t nb = (rl.off[rl.n] + 31) / 32;
  if (nb > (int64_t)num_sms() * 16) nb = (int64_t)num_sms() * 16;
  GANTTS_PDL_LAUNCH((multi_reduce_kernel), (unsigned)nb, 32 * MR_WARPS, 0, st, rl, accumulate);
  GANTTS_LAUNCH_CHECK("multi_reduce_kernel");
  rl.n = 0;
  return GANTTS_OK;
}

// gb (optional) receives the column sums of A (the bias gradient) from the same launch.  With `defer`
// the split reductions are queued (the partial buffer must then stay untouched until flush_reduce).
static int launch_gemm_mn(const Planes& A, const Planes& B, float* C, float* gb, int accumulate, float* partial,
                          cudaStream_t st, ReduceList* defer = nullptr) {
  GemmParams p{};
  p.rows_a = A.cols;
  p.cols_b = (int)B.cols;
  p.red = A.rows;
  if (B.rows != A.rows) {
    set_error("gemm_mn: reduction extents differ (%lld vs %lld)", (long long)A.rows, (long long)B.rows);
    return GANTTS_E_BADARG;
  }
  int splits;
  int64_t chunk;
  mn_partial_bytes(p.red, (int)p.rows_a, p.cols_b, &splits, &chunk);
  p.red_chunk = chunk;
  p.num_z = splits;
  p.bn = pick_bn(p.cols_b);
  p.num_a = (int)((p.rows_a + TC_BM - 1) / TC_BM);
  p.num_b = (p.cols_b + p.bn - 1) / p.bn;
  p.atom_bytes = (uint32_t)TC_MN_BK * 128;                  // [bk reduction rows][128 B of 64 MN elements]
  p.a_plane = (TC_BM / 64) * p.atom_bytes;
  p.b_plane_bytes = (uint32_t)(p.bn / 64) * p.atom_bytes;
  p.stage_bytes = 2 * p.a_plane + 2 * p.b_plane_bytes;
  p.tx_bytes = p.stage_bytes;
  const bool direct = (splits == 1 && !accumulate);
  const int64_t n = (int64_t)p.rows_a * p.cols_b;
  float* db_partial = partial + (int64_t)splits * n;
  EpiArgs e;
  e.epi = EPI_F32;
  e.C = direct ? C : partial;
  e.ldc = p.cols_b;
  fill_epilogue(p, e);
  p.c_zstride = n;
  p.db = gb ? (direct ? gb : db_partial) : nullptr;
  const size_t smem = plan_smem(p, e);
  CUtensorMap mAh, mAl, mBh, mBl;
  int rc;
  if ((rc = make_map(&mAh, A.hi, A.rows, A.cols, A.pitch, TC_MN_BK))) return rc;
  if ((rc = make_map(&mAl, A.lo, A.rows, A.cols, A.pitch, TC_MN_BK))) return rc;
  if ((rc = make_map(&mBh, B.hi, B.rows, B.cols, B.pitch, TC_MN_BK))) return rc;
  if ((rc = make_map(&mBl, B.lo, B.rows, B.cols, B.pitch, TC_MN_BK))) return rc;
  if ((rc = launch_bn<true, EPI_F32>(mAh, mAl, mBh, mBl, mAh, mAl, p, smem, st))) return rc;
  if (!direct) {
    if (defer && defer->n + 2 <= REDUCE_MAX_JOBS) {
      int j = defer->n++;
      defer->partial[j] = partial; defer->out[j] = C; defer->splits[j] = splits; defer->len[j] = n;
      if (gb) {
        j = defer->n++;
        defer->partial[j] = db_partial; defer->out[j] = gb; defer->splits[j] = splits; defer->len[j] = p.rows_a;
      }
      return GANTTS_OK;
    }
    splitk_reduce_kernel<<<(unsigned)((n + 1023) / 1024), 256, 0, st>>>(partial, splits, n, C, accumulate);
    GANTTS_LAUNCH_CHECK("splitk_reduce_kernel(tc gW)");
    if (gb) {
      splitk_reduce_kernel<<<(unsigned)((p.rows_a + 1023) / 1024), 256, 0, st>>>(db_partial, splits, p.rows_a, gb,
                                                                               accumulate);
      GANTTS_LAUNCH_CHECK("splitk_reduce_kernel(tc gb)");
    }
  }
  return GANTTS_OK;
}

size_t tc_linear_workspace_bytes(int64_t M, int N, int K) {
  // forward: x planes + W planes ; backward: gz planes + x planes + W^T planes + gW partials
  size_t fwd = 2 * plane_bytes(M, K) + 2 * plane_bytes(N, K);
  size_t bwd = 2 * plane_bytes(M, N) + 2 * plane_bytes(M, K) + 2 * plane_bytes(K, N) +
               mn_partial_bytes(M, N, K, nullptr, nullptr) + 256;
  return (fwd > bwd ? fwd : bwd) + 1024;
}

int tc_linear_fwd(const float* x, int64_t x_rs, const float* W, const float* bias, float* y, int64_t y_rs,
                  int64_t M, int N, int K, int act, float slope, float p, uint64_t seed, void* ws,
                  size_t ws_bytes, cudaStream_t st) {
  size_t need = tc_linear_workspace_bytes(M, N, K);
  if (!ws || ws_bytes < need) {
    set_error("tc_linear_fwd: workspace too small (%zu < %zu)", ws_bytes, need);
    return GANTTS_E_WORKSPACE;
  }
  char* cur = reinterpret_cast<char*>((reinterpret_cast<uintptr_t>(ws) + 255) / 256 * 256);
  Planes X = carve_planes(cur, M, K), Wp = carve_planes(cur, N, K);
  int rc;
  if ((rc = launch_split(x, x_rs, M, K, X, 0, st))) return rc;
  if ((rc = launch_split(W, K, N, K, Wp, 0, st))) return rc;
  EpiArgs e;
  e.epi = EPI_F32;
  e.C = y;
  e.ldc = y_rs;
  e.bias = bias;
  e.act = act;
  e.slope = slope;
  e.p = act == GANTTS_ACT_LEAKY_DROPOUT ? p : 0.f;
  e.seed = seed;
  return launch_gemm_kk(X, Wp, e, st);
}

int tc_linear_bwd_gemms(const float* gz, const float* x, int64_t x_rs, const float* W, float* gx,
                        int64_t gx_rs, float* gW, int64_t M, int N, int K, int accumulate, void* ws,
                        size_t ws_bytes, cudaStream_t st) {
  size_t need = tc_linear_workspace_bytes(M, N, K);
  if (!ws || ws_bytes < need) {
    set_error("tc_linear_bwd: workspace too small (%zu < %zu)", ws_bytes, need);
    return GANTTS_E_WORKSPACE;
  }
  char* cur = reinterpret_cast<char*>((reinterpret_cast<uintptr_t>(ws) + 255) / 256 * 256);
  Planes G = carve_planes(cur, M, N);
  Planes X = carve_planes(cur, M, K);
  Planes Wt = carve_planes(cur, K, N);
  float* partial = reinterpret_cast<float*>(cur);
  int rc;
  if ((rc = launch_split(gz, N, M, N, G, 0, st))) return rc;
  if (gx) {
    if ((rc = launch_split(W, K, N, K, Wt, 1, st))) return rc;      // Wt[k][n] = W[n][k]
    EpiArgs e;
    e.epi = EPI_F32;
    e.C = gx;
    e.ldc = gx_rs;
    if ((rc = launch_gemm_kk(G, Wt, e, st))) return rc;             // gx[m][k] = sum_n gz[m][n] W[n][k]
  }
  if (gW) {
    if ((rc = launch_split(x, x_rs, M, K, X, 0, st))) return rc;
    if ((rc = launch_gemm_mn(G, X, gW, nullptr, accumulate, partial, st))) return rc;
  }
  return GANTTS_OK;
}

}  // namespace gantts
