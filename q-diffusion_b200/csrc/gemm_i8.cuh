// INT8 wgmma GEMM / implicit-GEMM conv3x3 for sm_90a.
//
// Realises the reference's QuantModule.forward (qdiff/quant_layer.py:248-279) as true integer
// compute:   y[m,n] = scale[n] * (sum_k xq[m,k]*ws[n,k] - corr[cls(m)][n]) + bias[n] (+ fused adds)
// where xq are the activation codes (u8 or s8), ws = wq - zw the zero-point-free weight codes (s8),
// scale[n] = delta_x * delta_w[n] and corr = zx * sum_k ws[n,k] (per border class for padded convs,
// because the reference pads with real zeros AFTER de-quantisation, SURVEY Appendix A.3).
//
// Structure (one CTA per SM, persistent, warp-specialised):
//   warps 0-3  : producer warpgroup.  Warp 0 is the TMA producer (A tile 128 x 128 B, B tile BN x 128 B, 128B swizzle,
//                mbarrier ring); warp 1 initialises the barriers.  W4 variant: warps 2-3 and warps 12-13 unpack packed
//                4-bit weight codes staged by TMA into the swizzled s8 operand tile (four warps = one per scheduler).
//   warps 4-11 : two consumer warpgroups.  Warpgroup g issues wgmma m64nNk32 (int32 accumulators in registers) for rows
//                [64g, 64g + 64) of the tile, the N tile as 64-column sub-blocks; after the K loop both warpgroups write
//                their accumulators to a shared-memory accumulator tile.
//   warps 12-  : gemm_epi_warps(MODE) epilogue warps (4 or 8) finalise the tile from there (zero-point correction / scale
//                / bias / adds / GEGLU -> coalesced fp32 or requantised stores) while the consumers already run the next
//                work item's k-blocks: two mbarriers (acc_full, acc_empty) hand the single accumulator tile back and
//                forth, so a CTA's time per tile is the longer of main loop and epilogue rather than their sum.  Each role
//                runs under its own register budget (setmaxnreg).
//   Split-K partials (stored straight from the registers), packed INT4 weights, the bfloat16 weight-only layers and the
//   generic MODE = -1 kernel keep the serial schedule: no epilogue warps, the eight consumer warps run the epilogue after
//   each main loop.
// The producer streams the next tile's operands into the ring while the current tile is finalised.
//
// The kernel is templated on the epilogue MODE so the hot variants carry no runtime flag tests
// (a version with runtime flags was instruction-issue / I-cache bound in the epilogue).  MODE = -1 keeps every runtime
// option (ragged N, both outputs).
#pragma once
#include "ptx.cuh"
#include "quant_math.cuh"
#include <cuda_fp16.h>
#include <type_traits>

namespace qd {

constexpr int GEMM_BM = 128;
constexpr int GEMM_BK = 128;  // bytes == int8 elements per k-block (one 128B swizzle row)
// BN <= 128: the two consumer warpgroups hold 128 x BN int32 accumulators in registers (BN / 2 per thread) next to the
// epilogue's working set, and the accumulator tile in shared memory is 128 x BN x 4 bytes.  The split-K partial kernel
// (EPI_SPLITK) stores its raw accumulators straight from the registers, needs no accumulator tile and takes BN <= 256.
constexpr int GEMM_MAX_BN = 128;
constexpr int GEMM_MAX_BN_SPLITK = 256;
constexpr int GEMM_A_STAGE_BYTES = GEMM_BM * GEMM_BK;
constexpr int GEMM_MAX_STAGES = 8;
constexpr int GEMM_EPI_TILE_BYTES = 32 * 128;  // one 32 x 32 int32 chunk of the accumulator tile
// accumulator tile: 4 row quarters x ceil(BN / 32) column chunks of 32 rows x 128 B, 16-byte units XOR-swizzled by row & 7
// (conflict-free for the epilogue's row-wise and column-quad-wise reads)
__host__ __device__ inline int gemm_acc_tile_bytes(int BN, bool splitk = false) {
  return splitk ? 0 : 4 * ((BN + 31) / 32) * GEMM_EPI_TILE_BYTES;
}

// epilogue MODE bits (MODE < 0: generic)
constexpr int EPI_CORR = 1;       // subtract zero-point correction
constexpr int EPI_ROWVEC = 2;     // + per-image per-channel vector (timestep embedding)
constexpr int EPI_RESIDUAL = 4;   // + residual[m, n]
constexpr int EPI_OUT_F32 = 8;    // fp32 output
constexpr int EPI_OUT_Q = 16;     // requantised code output (row-major)
constexpr int EPI_GEGLU = 32;     // columns interleaved [4 x, 4 gate]: out_q = Q(x * gelu(gate)), N/2 columns
constexpr int EPI_TRANS = 64;     // requantised code output, transposed [img][n][token'] (V^T operand of qattention)
constexpr int EPI_CONV = 128;     // 3x3 conv (taps == 9); with EPI_CORR the correction table is indexed by border class
constexpr int EPI_RESTMA = 256;   // with EPI_RESIDUAL: residual sub-tiles arrive through the per-warp TMA ring (short-K GEMMs)
constexpr int EPI_BF16 = 512;     // weight-only layers: bfloat16 x3 activation planes x bfloat16 weight codes, fp32 accumulators
constexpr int EPI_SPLITK = 1024;  // split-K partial: raw int32 accumulators of one K slice -> ws[split][M][N] (splitk_finish_kernel applies the epilogue)
__host__ __device__ constexpr int gemm_max_bn(int MODE) { return (MODE >= 0 && (MODE & EPI_SPLITK) != 0) ? GEMM_MAX_BN_SPLITK : GEMM_MAX_BN; }

// Overlapped schedule (dedicated epilogue warps behind the consumers) for every specialised int8 epilogue.  Split-K partials
// have no tile epilogue; packed INT4 weights, the bfloat16 weight-only layers and the generic MODE = -1 kernel (whose
// run-time-flag epilogue spills hundreds of bytes as an epilogue role even at 232 registers) keep the serial schedule.
__host__ __device__ constexpr bool gemm_overlap(int MODE, bool W4 = false) {
  return MODE >= 0 && !W4 && (MODE & (EPI_SPLITK | EPI_BF16)) == 0;
}
// Epilogue warps: warp (4h + q) of them finalises rows [32q, 32q + 32) of the tile, 32-column chunks h, h + EPI_WARPS / 4,
// ...  The 3x3 convs follow main loops of 20-180 k-blocks, so their epilogue is the shorter part of a tile: 4 warps at up
// to 232 registers (border-class correction rows, per-image vectors).  The plain GEMMs' epilogues (short K: the epilogue
// is the longer part) take 8 warps at 128 registers.  Serial schedule: the 8 consumer warps.
__host__ __device__ constexpr int gemm_epi_warps(int MODE, bool W4 = false) {
  return gemm_overlap(MODE, W4) && (MODE & EPI_CONV) != 0 ? 4 : 8;
}
// Registers per thread of each role on the overlapped schedule.  setmaxnreg only moves registers between the warps of
// one CTA, so the budgets must fit the CTA's launch allocation, threads x (65,536 / threads rounded down to 8):
//   8 epilogue warps (640 threads, 96 at launch: 61,440): producer warpgroup 32, consumers 96 (64 int32 accumulators at
//     BN = 128 plus descriptors and ring state), epilogue warps 128 - 61,440;
//   4 epilogue warps (512 threads, 128 at launch: 65,536): producer 32, consumers 104, epilogue warps 232 - 60,416.
constexpr int GEMM_PRODUCER_REGS = 32;
__host__ __device__ constexpr int gemm_consumer_regs(int MODE) { return gemm_epi_warps(MODE) == 8 ? 96 : 104; }
__host__ __device__ constexpr int gemm_epi_regs(int MODE) { return gemm_epi_warps(MODE) == 8 ? 128 : 232; }
// W4 (packed INT4 weights, serial schedule): warps 12-13 behind the consumer warps join warps 2-3 as unpack warps
constexpr int GEMM_W4_WARP0 = 12;
__host__ __device__ constexpr int gemm_threads(int MODE, bool W4 = false) {
  return gemm_overlap(MODE, W4) ? (12 + gemm_epi_warps(MODE)) * 32 : (GEMM_W4_WARP0 + (W4 ? 2 : 0)) * 32;
}
__host__ __device__ constexpr int gemm_launch_regs(int MODE, bool W4 = false) { return (65536 / gemm_threads(MODE, W4)) & ~7; }
// a warpgroup's move from the launch allocation FROM to R registers per thread
template <int R, int FROM>
__device__ __forceinline__ void gemm_setmaxnreg() {
  if constexpr (R < FROM) setmaxnreg_dec<R>();
  else if constexpr (R > FROM) setmaxnreg_inc<R>();
}
// Residual operand through TMA: the plain-GEMM epilogues that add a residual (to_out / ff.net.2 / proj_out: EPI_RESIDUAL
// without EPI_CONV) are bound by the latency of their residual loads when each warp issues 4 rows of LDG.128, waits a DRAM
// round trip, stores, and issues the next 4 rows.
// Now every epilogue warp owns a ring of GEMM_RES_NBUF 4 KB buffers and keeps the residual sub-tiles of its NEXT work items
// (tile, chunk) in flight as cp.async.bulk.tensor loads while it finalises the current one.  These modes take 8 epilogue
// warps on either schedule.
constexpr int GEMM_RES_NBUF = 3;
__host__ __device__ constexpr bool gemm_res_tma(int MODE) { return MODE >= 0 && (MODE & EPI_RESIDUAL) != 0 && (MODE & EPI_RESTMA) != 0; }
__host__ __device__ constexpr int gemm_res_bytes(int MODE) {
  return gemm_res_tma(MODE) ? gemm_epi_warps(MODE) * GEMM_RES_NBUF * 4096 : 0;
}

struct GemmArgs {
  int M, N;            // logical output rows / columns (columns >= N are masked)
  int C;               // reduction length per tap (multiple of 32)
  int taps;            // 1 = plain GEMM, 9 = 3x3 conv (stride 1, pad 1)
  int kdup;            // 1, or 2: two weight segments over the same activation (8-bit weights as wa + wb, qd_gemm_desc.k_dup)
  int BN;              // N tile (multiple of 16, <= GEMM_MAX_BN)
  int tiles_m, tiles_n;
  int stages;
  // conv geometry (taps == 9): activations are NHWC, tile = bn images x bh rows x W columns = 128 pixels (W > 128: a
  // 128-pixel segment of one row)
  int H, W, bh, bn;
  int a_signed, b_signed;
  // epilogue
  float* out;          // fp32 [M, ldo] or nullptr
  long long ldo;
  int8_t* out_q;       // requantised output (codes), [M, ldq] or transposed [M/rows_per_batch][N][ldq]
  long long ldq;
  int out_q_transposed;
  int rows_per_batch;  // rows (pixels/tokens) per image: rowvec index and transposed-store geometry
  float q_delta;
  int q_zp, q_lo, q_hi;
  const float* scale;      // [N]
  const float* bias;       // [N] or nullptr
  const int32_t* corr;     // [ncls][N] or nullptr   (ncls = 9 for conv, 1 plain)
  const float* rowvec;     // [M/rows_per_batch][ld_rowvec] per-image per-channel add (timestep embedding) or nullptr
  long long ld_rowvec;
  const float* residual;   // [M, ldr] or nullptr (may alias out)
  long long ldr;
  int geglu;
  int oq_d, oq_pitch;      // > 0: per-head padded code layout for row-major out_q
  int oq_f16;              // out_q receives fp16 (code - zero_point) instead of 8-bit codes (ldq / oq_pitch in fp16 elements)
  // packed INT4 weights (K3): the B tile arrives as BN x 64 packed bytes and the four unpack warps expand it to the s8
  // 128B-swizzled operand tile in shared memory (wq - wzero[n]) before the MMA consumes the stage
  int w4;
  const int8_t* wzero;     // [w_rows]
  // requantising epilogues (specialised EPI_OUT_Q modes without GEGLU): scale / delta_q and bias / delta_q + zero_point
  const float* scale_q;
  const float* bias_q;
  // GroupNorm slab statistics of the fp32 output (qd_gemm_desc.gn_stats): float2 [M/32][ld_stats]
  float2* gn_stats;
  long long ld_stats;
  int bf16;            // weight-only layer: bfloat16 operands, fp32 accumulators (EPI_BF16 modes)
  // split-K (short-M, long-K layers: few output tiles, the K loop of a tile is shared by `splits` CTAs): work item =
  // (tile, split); split z reduces k-blocks [z * kb_per_split, (z + 1) * kb_per_split) and stores its raw accumulators to
  // ws[z][M][N]; splitk_finish_kernel sums the slices (integers: exact, order-free) and applies the epilogue
  int splits, kb_per_split;
  int32_t* ws;
};
// Specialised requantising modes take the pre-divided constants (one FFMA per element: quant_math.cuh quant_bits_pre)
__host__ __device__ constexpr bool gemm_qpre(int MODE) { return MODE >= 0 && (MODE & 16) != 0 && (MODE & 32) == 0; }

struct GemmSmemLayout {
  int stage_bytes;
  int pack_off;   // packed-INT4 B tiles, stages x BN x 64 bytes (w4 only)
  int bar_offset;
  int stage_off;  // accumulator tile (gemm_acc_tile_bytes)
  int res_off;    // residual ring (GEMM_RES_NBUF x 4 KB per epilogue warp; residual-by-TMA modes only)
  int total;
};

__host__ __device__ inline int gemm_stage_footprint(int BN, int w4) {
  return GEMM_A_STAGE_BYTES + BN * GEMM_BK + (w4 ? BN * (GEMM_BK / 2) : 0);
}

__host__ __device__ inline GemmSmemLayout gemm_smem_layout(int BN, int stages, int w4 = 0, int res_bytes = 0, bool splitk = false) {
  GemmSmemLayout l;
  l.stage_bytes = GEMM_A_STAGE_BYTES + BN * GEMM_BK;
  l.pack_off = l.stage_bytes * stages;
  l.bar_offset = l.pack_off + (w4 ? stages * BN * (GEMM_BK / 2) : 0);
  l.stage_off = l.bar_offset + 512;
  // the ring buffers are TMA targets with the 128-byte swizzle: the pattern is a function of the shared-memory ADDRESS
  // (bits 4-6 ^= bits 7-9), so they must start on a 1024-byte boundary for "chunk ^ (row & 7)" to address them
  l.res_off = (l.stage_off + gemm_acc_tile_bytes(BN, splitk) + 1023) / 1024 * 1024;
  l.total = l.res_off + res_bytes + 1024;  // + alignment slack
  return l;
}

// border class (3x3 conv zero-point correction) and image index of output row m
__device__ __forceinline__ void gemm_row_meta(const GemmArgs& p, int m, int& cls, int& img) {
  cls = 0;
  img = 0;
  if (p.rows_per_batch > 0) img = m / p.rows_per_batch;
  if (p.taps == 9) {
    const int hw = p.H * p.W;
    const int r = m % hw;
    const int h = r / p.W, w = r - h * p.W;
    const int rc = (h == 0) ? 0 : (h == p.H - 1 ? 2 : 1);
    const int cc = (w == 0) ? 0 : (w == p.W - 1 ? 2 : 1);
    cls = rc * 3 + cc;
  }
}

// The consumer's activation quantizer (qdiff/quant_layer.py:82-88) is applied with quant_math.cuh's QuantK,
// built ONCE per thread before the tile loop: building it (MUFU.RCP + Newton + slow-path test) inside the
// per-row code, where the compiler will not hoist it out of the `m < M` conditional, tripled the instruction
// count of the requantising epilogues.

// Row `row` (columns 0 .. NC-1) of a 32 x 32 chunk of the accumulator tile.
template <int NC>
__device__ __forceinline__ void gemm_acc_row(const uint8_t* chunk, int row, uint32_t (&v)[NC]) {
#pragma unroll
  for (int j = 0; j < NC / 4; ++j) {
    const uint4 u = *reinterpret_cast<const uint4*>(chunk + row * 128 + ((j ^ (row & 7)) << 4));
    v[4 * j] = u.x; v[4 * j + 1] = u.y; v[4 * j + 2] = u.z; v[4 * j + 3] = u.w;
  }
}

// Thread-per-row epilogue (used for the transposed V^T code output: consecutive lanes = consecutive
// tokens, so each per-column byte store of the warp fills one 32 B sector).
template <int NC>
__device__ __forceinline__ void gemm_epilogue_rowwise(const GemmArgs& p, const QuantK& qk, const uint32_t (&acc)[NC],
                                                      int m, int n0, int cls, int img) {
  float y[NC];
  if (((p.N & 3) == 0) && n0 + NC <= p.N && !p.rowvec) {
    // vector parameter loads (uniform across the warp): 3 x LDG.128 per 4 columns instead of 12 scalar loads
#pragma unroll
    for (int j = 0; j < NC; j += 4) {
      const int n = n0 + j;
      const float4 s4 = __ldg(reinterpret_cast<const float4*>(p.scale + n));
      float4 b4 = make_float4(0.f, 0.f, 0.f, 0.f);
      if (p.bias) b4 = __ldg(reinterpret_cast<const float4*>(p.bias + n));
      int4 c4 = make_int4(0, 0, 0, 0);
      if (p.corr) c4 = __ldg(reinterpret_cast<const int4*>(p.corr + (long long)cls * p.N + n));
      y[j] = (float)((int)acc[j] - c4.x) * s4.x + b4.x;
      y[j + 1] = (float)((int)acc[j + 1] - c4.y) * s4.y + b4.y;
      y[j + 2] = (float)((int)acc[j + 2] - c4.z) * s4.z + b4.z;
      y[j + 3] = (float)((int)acc[j + 3] - c4.w) * s4.w + b4.w;
    }
    if (p.residual) {
#pragma unroll
      for (int j = 0; j < NC; ++j) y[j] += p.residual[(long long)m * p.ldr + n0 + j];
    }
  } else {
#pragma unroll
    for (int j = 0; j < NC; ++j) {
      int n = n0 + j;
      int a = (int)acc[j];
      if (n < p.N) {
        if (p.corr) a -= __ldg(p.corr + (long long)cls * p.N + n);
        float v = (float)a * __ldg(p.scale + n);
        if (p.bias) v += __ldg(p.bias + n);
        if (p.rowvec) v += __ldg(p.rowvec + (long long)img * p.ld_rowvec + n);
        if (p.residual) v += p.residual[(long long)m * p.ldr + n];
        y[j] = v;
      } else {
        y[j] = 0.f;
      }
    }
  }
  if (p.out) {
    float* o = p.out + (long long)m * p.ldo + n0;
#pragma unroll
    for (int j = 0; j < NC; ++j)
      if (n0 + j < p.N) o[j] = y[j];
  }
  if (p.out_q) {
    // V^T layout for qattention: 16-key groups permuted (attention.cuh: att_vt_perm)
    const int t_in = m - img * p.rows_per_batch;
    const int t_pos = (t_in & ~15) | (((t_in >> 1) & 3) << 2) | (((t_in >> 3) & 1) << 1) | (t_in & 1);
    int8_t* o = p.out_q + ((long long)img * p.N + n0) * p.ldq + t_pos;
#pragma unroll
    for (int j = 0; j < NC; ++j)
      if (n0 + j < p.N) o[(long long)j * p.ldq] = (int8_t)quant_code(y[j], qk);
  }
}

// Finalise 4 consecutive columns of one row.  MODE >= 0: flags are compile-time, N % 4 == 0 and all
// leading dimensions are vector-aligned (checked on the host).  MODE < 0: everything at run time.
// `of` / `oq` point at (m, n) of the fp32 / code output, `corr4` is the row's zero-point correction (plain GEMM: per
// column; conv: the caller fetched the row's border class) except in generic conv mode, which loads it here.
template <int MODE>
__device__ __forceinline__ void gemm_finalise4(const GemmArgs& p, const QuantK& qk, const bool conv, const uint4 a4,
                                               const float (&sc)[4], const float (&bi)[4], const int4 corr4,
                                               const float4 rpre, float* of, int8_t* oq, const float* res, int n,
                                               int cls, int img, float (&gsum)[4], float (&gsq)[4]) {
  constexpr bool G = MODE < 0;
  const bool has_corr = G ? (p.corr != nullptr) : bool(MODE & EPI_CORR);
  const bool has_rowvec = G ? (p.rowvec != nullptr) : bool(MODE & EPI_ROWVEC);
  const bool has_res = G ? (p.residual != nullptr) : bool(MODE & EPI_RESIDUAL);
  const bool out_f = G ? (p.out != nullptr) : bool(MODE & EPI_OUT_F32);
  const bool out_q = G ? (p.out_q != nullptr) : bool(MODE & EPI_OUT_Q);
  const bool full = G ? (n + 3 < p.N) : true;
  int a[4] = {(int)a4.x, (int)a4.y, (int)a4.z, (int)a4.w};
  if (has_corr) {
    if (G && conv) {
      if (full) {
        const int4 c = __ldg(reinterpret_cast<const int4*>(p.corr + (long long)cls * p.N + n));
        a[0] -= c.x; a[1] -= c.y; a[2] -= c.z; a[3] -= c.w;
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (n + j < p.N) a[j] -= __ldg(p.corr + (long long)cls * p.N + n + j);
      }
    } else {
      a[0] -= corr4.x; a[1] -= corr4.y; a[2] -= corr4.z; a[3] -= corr4.w;
    }
  }
  float y[4];
  if constexpr (MODE >= 0 && (MODE & EPI_BF16) != 0) {     // fp32 accumulators (weight-only layers)
    y[0] = __uint_as_float(a4.x) * sc[0] + bi[0]; y[1] = __uint_as_float(a4.y) * sc[1] + bi[1];
    y[2] = __uint_as_float(a4.z) * sc[2] + bi[2]; y[3] = __uint_as_float(a4.w) * sc[3] + bi[3];
  } else {
#pragma unroll
    for (int j = 0; j < 4; ++j) y[j] = (float)a[j] * sc[j] + bi[j];
  }
  if (has_rowvec) {
    const float* rv = p.rowvec + (long long)img * p.ld_rowvec + n;
    if (full && (G ? ((p.ld_rowvec & 3) == 0) : true)) {
      const float4 r = __ldg(reinterpret_cast<const float4*>(rv));
      y[0] += r.x; y[1] += r.y; y[2] += r.z; y[3] += r.w;
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (n + j < p.N) y[j] += rv[j];
    }
  }
  constexpr bool QPRE = gemm_qpre(MODE);
  if (has_res && !G) {
    // specialised kernels pre-load the residual of a row group before its first store: `out` may alias
    // `residual` (in-place accumulate), so the compiler cannot hoist these loads itself and they would
    // otherwise serialise one global-memory latency per row
    if constexpr (QPRE) {     // y is in code units (pre-scaled constants): bring the residual there too
      y[0] = fmaf(rpre.x, qk.rdelta, y[0]); y[1] = fmaf(rpre.y, qk.rdelta, y[1]);
      y[2] = fmaf(rpre.z, qk.rdelta, y[2]); y[3] = fmaf(rpre.w, qk.rdelta, y[3]);
    } else {
      y[0] += rpre.x; y[1] += rpre.y; y[2] += rpre.z; y[3] += rpre.w;
    }
  } else if (has_res) {
    if (full && ((p.ldr & 3) == 0)) {
      const float4 rv = *reinterpret_cast<const float4*>(res);
      y[0] += rv.x; y[1] += rv.y; y[2] += rv.z; y[3] += rv.w;
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (n + j < p.N) y[j] += res[j];
    }
  }
  if (out_f) {
    // column sums of the values being stored (GroupNorm slab statistics; dead code unless the caller uses them)
#pragma unroll
    for (int j = 0; j < 4; ++j) { gsum[j] += y[j]; gsq[j] = fmaf(y[j], y[j], gsq[j]); }
    if (full && (G ? ((p.ldo & 3) == 0) : true)) {
      *reinterpret_cast<float4*>(of) = make_float4(y[0], y[1], y[2], y[3]);
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (n + j < p.N) of[j] = y[j];
    }
  }
  if constexpr (QPRE) {
    if (p.oq_f16) {      // centred codes as fp16: float(K + code) - (K + zero_point), exact
      const float kz = 12582912.0f + (float)p.q_zp;
      const __half2 h01 = __floats2half2_rn(__uint_as_float(quant_bits_pre(y[0], qk)) - kz, __uint_as_float(quant_bits_pre(y[1], qk)) - kz);
      const __half2 h23 = __floats2half2_rn(__uint_as_float(quant_bits_pre(y[2], qk)) - kz, __uint_as_float(quant_bits_pre(y[3], qk)) - kz);
      *reinterpret_cast<uint2*>(oq) = make_uint2(*reinterpret_cast<const uint32_t*>(&h01), *reinterpret_cast<const uint32_t*>(&h23));
    } else {
      *reinterpret_cast<uint32_t*>(oq) = pack4_low_bytes(quant_bits_pre(y[0], qk), quant_bits_pre(y[1], qk),
                                                         quant_bits_pre(y[2], qk), quant_bits_pre(y[3], qk));
    }
  } else if (out_q && p.oq_f16) {
    float cz[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) cz[j] = quant_centered(y[j], qk);
    if (full) {
      const __half2 h01 = __floats2half2_rn(cz[0], cz[1]), h23 = __floats2half2_rn(cz[2], cz[3]);
      *reinterpret_cast<uint2*>(oq) = make_uint2(*reinterpret_cast<const uint32_t*>(&h01), *reinterpret_cast<const uint32_t*>(&h23));
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (n + j < p.N) reinterpret_cast<__half*>(oq)[j] = __float2half_rn(cz[j]);
    }
  } else if (out_q) {
    const uint32_t q0 = quant_code(y[0], qk), q1 = quant_code(y[1], qk);
    const uint32_t q2 = quant_code(y[2], qk), q3 = quant_code(y[3], qk);
    if (full && (G ? ((p.ldq & 3) == 0) : true)) {
      *reinterpret_cast<uint32_t*>(oq) = q0 | (q1 << 8) | (q2 << 16) | (q3 << 24);
    } else {
      const uint32_t qq[4] = {q0, q1, q2, q3};
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (n + j < p.N) oq[j] = (int8_t)qq[j];
    }
  }
}

// One k-block (128 bytes = four 32-byte K steps of every row) of a consumer warpgroup: acc[s] (+)= A[64 rows] *
// B[rows 64s .. 64s + 63]^T for the NF full 64-column sub-blocks, and a last sub-block TAIL (0, 16, 32 or 48) columns
// wide.  All compile-time: the wgmma sequence is straight-line code (a wgmma under a run-time branch is serialised by
// ptxas).  A partial last k-block of a tap needs no special case: its A columns beyond C are zero-filled by TMA, so the
// extra K steps add exact zeros.
template <bool BF16, bool SIGNED, int NF, int TAIL, int NS, typename T>
__device__ __forceinline__ void gemm_wgmma_kblock(T (&acc)[NS][32], uint64_t da, uint64_t db, uint32_t scale_first) {
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const uint32_t sd = j ? 1u : scale_first;
    const uint64_t a = da + (uint64_t)(2 * j);       // +32 bytes inside the 128B swizzle row
#pragma unroll
    for (int s = 0; s <= NF; ++s) {
      const uint64_t b = db + (uint64_t)((s * 64 * GEMM_BK) >> 4) + (uint64_t)(2 * j);
      if (s < NF) {
        if constexpr (BF16) wgmma_bf16_n64(acc[s < NS ? s : 0], a, b, sd);
        else if constexpr (SIGNED) wgmma_s8s8_n64(acc[s < NS ? s : 0], a, b, sd);
        else wgmma_u8s8_n64(acc[s < NS ? s : 0], a, b, sd);
      } else if constexpr (TAIL != 0) {
        constexpr int t = NF < NS ? NF : 0;
        if constexpr (BF16) {
          if constexpr (TAIL == 48) wgmma_bf16_n48(acc[t], a, b, sd);
          else if constexpr (TAIL == 32) wgmma_bf16_n32(acc[t], a, b, sd);
          else wgmma_bf16_n16(acc[t], a, b, sd);
        } else if constexpr (SIGNED) {
          if constexpr (TAIL == 48) wgmma_s8s8_n48(acc[t], a, b, sd);
          else if constexpr (TAIL == 32) wgmma_s8s8_n32(acc[t], a, b, sd);
          else wgmma_s8s8_n16(acc[t], a, b, sd);
        } else {
          if constexpr (TAIL == 48) wgmma_u8s8_n48(acc[t], a, b, sd);
          else if constexpr (TAIL == 32) wgmma_u8s8_n32(acc[t], a, b, sd);
          else wgmma_u8s8_n16(acc[t], a, b, sd);
        }
      }
    }
  }
}

template <int NF_, int TAIL_, bool SIGNED_>
struct GemmNCfg {
  static constexpr int NF = NF_, TAIL = TAIL_;
  static constexpr bool SIGNED = SIGNED_;
};
// Calls f(GemmNCfg<BN / 64, BN % 64, signed>{}) for the run-time N tile BN (a multiple of 16, <= 64 * NS).
template <int NS, bool S, typename F>
__device__ __forceinline__ void gemm_dispatch_bn(int BN, F&& f) {
  switch (BN >> 4) {
    case 1: f(GemmNCfg<0, 16, S>{}); break;
    case 2: f(GemmNCfg<0, 32, S>{}); break;
    case 3: f(GemmNCfg<0, 48, S>{}); break;
    case 4: f(GemmNCfg<1, 0, S>{}); break;
    case 5: f(GemmNCfg<1, 16, S>{}); break;
    case 6: f(GemmNCfg<1, 32, S>{}); break;
    case 7: f(GemmNCfg<1, 48, S>{}); break;
    default:
      if constexpr (NS == 2) {
        f(GemmNCfg<2, 0, S>{});
      } else {
        switch (BN >> 4) {
          case 8: f(GemmNCfg<2, 0, S>{}); break;
          case 9: f(GemmNCfg<2, 16, S>{}); break;
          case 10: f(GemmNCfg<2, 32, S>{}); break;
          case 11: f(GemmNCfg<2, 48, S>{}); break;
          case 12: f(GemmNCfg<3, 0, S>{}); break;
          case 13: f(GemmNCfg<3, 16, S>{}); break;
          case 14: f(GemmNCfg<3, 32, S>{}); break;
          case 15: f(GemmNCfg<3, 48, S>{}); break;
          default: f(GemmNCfg<4, 0, S>{}); break;
        }
      }
  }
}

// W4: packed-INT4 weight variant (compile-time, so the s8 kernels carry none of the unpack role's code: with a
// run-time flag the register allocation of the epilogue changed and the default path lost 8 %).
template <int MODE, bool W4 = false>
__global__ void __launch_bounds__(gemm_threads(MODE, W4), 1)
gemm_i8_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
               const __grid_constant__ CUtensorMap tmR, const GemmArgs p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  const uint32_t pad = ((raw_addr + 1023u) & ~1023u) - raw_addr;
  uint8_t* smem = smem_raw + pad;

  constexpr bool OVL = gemm_overlap(MODE, W4);
  constexpr int EPI_WARPS = gemm_epi_warps(MODE, W4);
  constexpr int CSTEP = 32 * (EPI_WARPS / 4);   // column stride between the chunks of one epilogue warp
  constexpr bool RES_TMA = gemm_res_tma(MODE);
  constexpr bool SPLITK = MODE >= 0 && (MODE & EPI_SPLITK) != 0;
  constexpr int NS = gemm_max_bn(MODE) / 64;     // 64-column accumulator sub-blocks
  static_assert(!OVL || 128 * GEMM_PRODUCER_REGS + 256 * gemm_consumer_regs(MODE) + 32 * EPI_WARPS * gemm_epi_regs(MODE) <=
                            gemm_threads(MODE) * gemm_launch_regs(MODE), "role register budgets exceed the CTA's allocation");
  const GemmSmemLayout lay = gemm_smem_layout(p.BN, p.stages, W4 ? 1 : 0, gemm_res_bytes(MODE), SPLITK);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + lay.bar_offset);
  uint64_t* full_bar = bars;                          // [stages]
  uint64_t* empty_bar = bars + GEMM_MAX_STAGES;       // [stages] (one arrival per consumer warpgroup)
  uint64_t* ready_bar = bars + 2 * GEMM_MAX_STAGES;   // [stages] (w4: B tile unpacked, stage ready for the MMA)
  uint64_t* res_bar = bars + 3 * GEMM_MAX_STAGES;     // [EPI_WARPS][GEMM_RES_NBUF] (residual ring, RES_TMA only)
  // overlapped schedule: the accumulator tile holds the current work item (one arrival per consumer warp) / the epilogue
  // warps have finished reading it (one arrival per epilogue warp)
  uint64_t* acc_full = bars + 3 * GEMM_MAX_STAGES + 8 * GEMM_RES_NBUF;
  uint64_t* acc_empty = acc_full + 1;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int splits = p.splits > 1 ? p.splits : 1;
  const int num_tiles = p.tiles_m * p.tiles_n * splits;       // work items: (tile, K slice)
  const int kb_per_tap = (p.C + GEMM_BK - 1) / GEMM_BK;
  const int num_kb_all = kb_per_tap * p.taps * p.kdup;
  const int kb_slice = splits > 1 ? p.kb_per_split : num_kb_all;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    if constexpr (RES_TMA) tma_prefetch_desc(&tmR);
  }
  if (warp == 1 && lane == 0) {
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2);
      if constexpr (W4) mbar_init(&ready_bar[s], 4);    // one arrival per unpack warp
    }
    if constexpr (RES_TMA)
      for (int s = 0; s < EPI_WARPS * GEMM_RES_NBUF; ++s) mbar_init(&res_bar[s], 1);
    if constexpr (OVL) {
      mbar_init(acc_full, 8);
      mbar_init(acc_empty, EPI_WARPS);
    }
    fence_mbar_init();
    fence_proxy_async();
  }
  __syncthreads();

  if (warp < 4 || (W4 && warp >= GEMM_W4_WARP0)) {
    // ===================== producer warpgroup: TMA producer (warp 0), INT4 unpack (W4: warps 2-3 and 12-13) ============
    if constexpr (OVL) gemm_setmaxnreg<GEMM_PRODUCER_REGS, gemm_launch_regs(MODE)>();
    if (warp == 0) {
      if (lane == 0) {
        int stage = 0;
        uint32_t phase = 0;
        const uint32_t tx_bytes = (uint32_t)(GEMM_A_STAGE_BYTES + (W4 ? p.BN * (GEMM_BK / 2) : p.BN * GEMM_BK));
        for (int item = blockIdx.x; item < num_tiles; item += gridDim.x) {
          const int tile = item / splits;
          const int kb0 = (item - tile * splits) * kb_slice;
          const int kb1 = min(num_kb_all, kb0 + kb_slice);
          const int tm = tile / p.tiles_n;
          const int tn = tile - tm * p.tiles_n;
          const int m0 = tm * GEMM_BM;
          const int n0 = tn * p.BN;
          int b0 = 0, h0 = 0, w0 = 0;
          if (p.taps == 9) {
            const int hw = p.H * p.W;
            b0 = m0 / hw;
            h0 = (m0 - b0 * hw) / p.W;
            w0 = m0 - b0 * hw - h0 * p.W;      // != 0 only for rows wider than a tile (W > 128: the tile is a 128-pixel row segment)
          }
          int seg = kb0 / kb_per_tap, kc = kb0 - seg * kb_per_tap;
          for (int kb = kb0; kb < kb1; ++kb) {
            const int tap = seg % p.taps;            // activation geometry of this segment; the weight column offset is seg * C
            const int ky = tap / 3, kx = tap - ky * 3;
            {
              mbar_wait(&empty_bar[stage], phase ^ 1);
              uint8_t* sa = smem + (size_t)stage * lay.stage_bytes;
              uint8_t* sb = sa + GEMM_A_STAGE_BYTES;
              mbar_arrive_expect_tx(&full_bar[stage], tx_bytes);
              if (p.taps == 9)
                tma_load_4d(sa, &tmA, &full_bar[stage], kc * GEMM_BK, w0 + kx - 1, h0 + ky - 1, b0);
              else
                tma_load_4d(sa, &tmA, &full_bar[stage], kc * GEMM_BK, m0, 0, 0);
              if constexpr (W4)
                tma_load_2d(smem + lay.pack_off + (size_t)stage * p.BN * (GEMM_BK / 2), &tmB, &full_bar[stage],
                            (seg * p.C + kc * GEMM_BK) / 2, n0);
              else
                tma_load_2d(sb, &tmB, &full_bar[stage], seg * p.C + kc * GEMM_BK, n0);
              if (++stage == p.stages) { stage = 0; phase ^= 1; }
            }
            if (++kc == kb_per_tap) { kc = 0; ++seg; }
          }
        }
      }
    } else if (W4 && warp != 1) {
      // ===================== INT4 unpack (warps 2, 3 and the two warps behind the consumer warps; W4 only) ==========
      // 128 threads = 32 rows x 4 sixteen-byte pieces per pass.  A piece holds 32 codes (k = 32j .. 32j+31 of the
      // k-block) and becomes two 16-byte chunks of the row in the 128B-swizzled s8 tile the MMA descriptor expects
      // (chunk index XOR row&7, identical to what TMA SWIZZLE_128B writes on the unpacked path).
      // Nibble order (ops.pack_int4): byte j of a 4-byte word holds code k0+j in its low and code k0+4+j in its high nibble,
      // so the masked word IS four consecutive codes - no byte permutation.  code - zp per byte without borrows:
      // (code + (0x80 - zp)) ^ 0x80, the constant 0x80808080 - zp*0x01010101 kept per row.  7 integer instructions per 8
      // codes (round 1: 11, on two warps: 1.7 k cycles per k-block against 0.9 k for the main loop).
      if constexpr (W4) {
        const int t = warp < 4 ? (int)threadIdx.x - 64 : (int)threadIdx.x - GEMM_W4_WARP0 * 32 + 64;   // 0..127
        const int r32 = t >> 2, piece = t & 3;
        int stage = 0;
        uint32_t phase = 0;
        for (int item = blockIdx.x; item < num_tiles; item += gridDim.x) {
          const int tile = item / splits;
          const int kb0 = (item - tile * splits) * kb_slice;
          const int num_kb = min(num_kb_all, kb0 + kb_slice) - kb0;
          const int tn = tile % p.tiles_n;
          const int n0 = tn * p.BN;
          uint32_t kz[8];       // 0x80808080 - zero point replicated into 4 bytes, rows r32 + 32*i
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const int n = n0 + r32 + 32 * i;
            kz[i] = 0x80808080u - ((r32 + 32 * i < p.BN && n < p.N) ? 0x01010101u * (uint32_t)(uint8_t)__ldg(p.wzero + n) : 0u);
          }
          for (int kb = 0; kb < num_kb; ++kb) {
            mbar_wait(&full_bar[stage], phase);
            const uint8_t* sp = smem + lay.pack_off + (size_t)stage * p.BN * (GEMM_BK / 2);
            uint8_t* sb = smem + (size_t)stage * lay.stage_bytes + GEMM_A_STAGE_BYTES;
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              const int row = r32 + 32 * i;
              if (row < p.BN) {
                const uint4 w = *reinterpret_cast<const uint4*>(sp + row * (GEMM_BK / 2) + piece * 16);
                const uint32_t in[4] = {w.x, w.y, w.z, w.w};
                uint32_t o[8];
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                  o[2 * q] = ((in[q] & 0x0F0F0F0Fu) + kz[i]) ^ 0x80808080u;             // k = 8q+0..3
                  o[2 * q + 1] = (((in[q] >> 4) & 0x0F0F0F0Fu) + kz[i]) ^ 0x80808080u;  // k = 8q+4..7
                }
                uint8_t* dst = sb + row * GEMM_BK;
                *reinterpret_cast<uint4*>(dst + (((2 * piece) ^ (row & 7)) << 4)) = make_uint4(o[0], o[1], o[2], o[3]);
                *reinterpret_cast<uint4*>(dst + (((2 * piece + 1) ^ (row & 7)) << 4)) = make_uint4(o[4], o[5], o[6], o[7]);
              }
            }
            fence_proxy_async();     // generic-proxy smem writes -> visible to the tensor core (async proxy)
            __syncwarp();
            if (lane == 0) mbar_arrive(&ready_bar[stage]);
            if (++stage == p.stages) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
  } else {
    // ===================== consumers (warps 4-11): wgmma main loop -> accumulator tile; epilogue warps =====================
    // The accumulators leave the registers into the shared-memory accumulator tile (32 x 32 int32 chunks, 128 B rows,
    // 16 B units XOR-swizzled by row&7: conflict-free both ways); the epilogue reads each chunk in the transposed
    // mapping: 8 lanes x 16 B = one full 128 B line per row, 4 rows per instruction, per-column parameters loaded once
    // per thread per chunk.
    const int cw = warp - 4;            // consumer warp 0..7
    const int wg = cw >> 2;             // its warpgroup: accumulator rows [64 wg, 64 wg + 64)
    const bool wg_leader = (threadIdx.x & 127) == 0;
    const int nch = (p.BN + 31) >> 5;   // 32-column chunks per row quarter of the accumulator tile
    uint8_t* const acc_tile = smem + lay.stage_off;
    constexpr bool BF16 = MODE >= 0 && (MODE & EPI_BF16) != 0;
    using AccT = typename std::conditional<BF16, float, uint32_t>::type;
    int stage = 0;
    uint32_t phase = 0;

    // ---- consumer: main loop of one work item over its k-blocks [kb0, kb1); a stage returns to the producer once the
    // MMAs reading it are complete (one k-block of MMAs stays in flight).  Then the accumulators go to the accumulator
    // tile once `before_dump()` returns (the previous item's epilogue has read it), or - split-K partials - straight from
    // the registers to the workspace.  The accumulators live in this scope only.
    auto consume = [&](const int item, auto&& before_dump) {
      const int tile = item / splits;
      const int zsplit = item - tile * splits;
      AccT accr[NS][32];
#pragma unroll
      for (int s = 0; s < NS; ++s)
#pragma unroll
        for (int i = 0; i < 32; ++i) accr[s][i] = 0;
      const int kb0 = zsplit * kb_slice;
      const int kb1 = min(num_kb_all, kb0 + kb_slice);
      int prev_stage = -1;
      // the N-tile width and the operand signedness are selected once per work item; each configuration's k-loop is
      // its own straight-line wgmma sequence
      auto mainloop = [&](auto cfg) {
        using Cfg = decltype(cfg);
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait(&full_bar[stage], phase);
          if constexpr (W4) mbar_wait(&ready_bar[stage], phase);   // ... and the B tile has been unpacked
          wgmma_fence();
          const uint32_t sa = smem_u32(smem + (size_t)stage * lay.stage_bytes);
          const uint64_t da = make_smem_desc_sw128(sa + (uint32_t)(wg * 64 * GEMM_BK));
          const uint64_t db = make_smem_desc_sw128(sa + GEMM_A_STAGE_BYTES);
          gemm_wgmma_kblock<BF16, Cfg::SIGNED, Cfg::NF, Cfg::TAIL>(accr, da, db, kb > kb0 ? 1u : 0u);
          wgmma_commit();
          wgmma_wait<1>();
          if (prev_stage >= 0 && wg_leader) mbar_arrive(&empty_bar[prev_stage]);
          prev_stage = stage;
          if (++stage == p.stages) { stage = 0; phase ^= 1; }
        }
        wgmma_wait<0>();
      };
      if constexpr (BF16) gemm_dispatch_bn<NS, true>(p.BN, mainloop);
      else if (p.a_signed) gemm_dispatch_bn<NS, true>(p.BN, mainloop);
      else gemm_dispatch_bn<NS, false>(p.BN, mainloop);
#pragma unroll
      for (int s = 0; s < NS; ++s) wgmma_fence_regs(accr[s]);
      if (prev_stage >= 0 && wg_leader) mbar_arrive(&empty_bar[prev_stage]);
      const int r0 = 64 * wg + 16 * (cw & 3) + (lane >> 2);
      if constexpr (SPLITK) {
        // raw accumulators of this K slice -> ws[zsplit][M][N] straight from the registers (host: N % 4 == 0); a warp
        // store covers 8 rows x 32 contiguous bytes
        const int tm = tile / p.tiles_n;
        const int n_base = (tile - tm * p.tiles_n) * p.BN;
        int32_t* wz = p.ws + (long long)zsplit * p.M * p.N;
#pragma unroll
        for (int s = 0; s < NS; ++s)
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const int n = n_base + 64 * s + 8 * j + 2 * (lane & 3);
            if (64 * s + 8 * j < p.BN && n < p.N) {
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                const int m = tm * GEMM_BM + r0 + 8 * h;
                if (m < p.M)
                  *reinterpret_cast<uint2*>(wz + (long long)m * p.N + n) = make_uint2(accr[s][4 * j + 2 * h], accr[s][4 * j + 2 * h + 1]);
              }
            }
          }
      } else {
        before_dump();
#pragma unroll
        for (int s = 0; s < NS; ++s)
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const int col = 64 * s + 8 * j + 2 * (lane & 3);
            if (col < p.BN) {
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                const int row = r0 + 8 * h;
                uint8_t* dst = acc_tile + ((row >> 5) * nch + (col >> 5)) * GEMM_EPI_TILE_BYTES + (row & 31) * 128 +
                               ((((col & 31) >> 2) ^ (row & 7)) << 4) + (col & 3) * 4;
                uint32_t lo, hi;
                if constexpr (BF16) { lo = __float_as_uint(accr[s][4 * j + 2 * h]); hi = __float_as_uint(accr[s][4 * j + 2 * h + 1]); }
                else { lo = accr[s][4 * j + 2 * h]; hi = accr[s][4 * j + 2 * h + 1]; }
                *reinterpret_cast<uint2*>(dst) = make_uint2(lo, hi);
              }
            }
          }
      }
    };

    // ---- epilogue warp `ew` (0 .. EPI_WARPS - 1): finalises rows [32q, 32q + 32) of each work item's tile, 32-column
    // chunks half * 32, half * 32 + CSTEP, ...  `acquire(item)` returns once the item's accumulators are in the tile,
    // `release()` follows the warp's last read of it.
    auto epilogue = [&](const int ew, auto&& acquire, auto&& release) {
      const int q = ew & 3;               // row quarter [32q, 32q + 32) of the tile
      const int half = ew >> 2;           // which of the EPI_WARPS / 4 warps sharing this row quarter
      const int rsub = lane >> 3;   // row within a group of 4
      [[maybe_unused]] const int cq = lane & 7;      // column quad within the 32-column chunk
      constexpr bool QPRE = gemm_qpre(MODE);
      const QuantK qk = QPRE ? make_quantk_pre(p.q_delta, p.q_lo, p.q_hi) : make_quantk(p.q_delta, p.q_zp, p.q_lo, p.q_hi);
      const float* const ep_scale = QPRE ? p.scale_q : p.scale;      // per-column epilogue constants of this mode
      const float* const ep_bias = QPRE ? p.bias_q : p.bias;
      [[maybe_unused]] const bool conv = MODE < 0 ? (p.taps == 9) : ((MODE & EPI_CONV) != 0);
      // ---- residual ring (RES_TMA): work items of this warp = (tile, chunk) in processing order; `pf_*` is the prefetch
      // cursor, GEMM_RES_NBUF - 1 items ahead of the item being finalised
      uint8_t* rring = smem + lay.res_off + ew * (GEMM_RES_NBUF * 4096);
      uint64_t* rbar = res_bar + ew * GEMM_RES_NBUF;
      int pf_tile = blockIdx.x, pf_c = half * 32, pf_buf = 0;
      [[maybe_unused]] int rd_buf = 0;
      [[maybe_unused]] uint32_t rd_phase = 0;
      auto res_issue = [&]() {          // issue the load of the cursor's item (if any) and advance the cursor
        if (pf_tile >= num_tiles) return;
        if (lane == 0) {
          const int ptm = pf_tile / p.tiles_n, ptn = pf_tile - ptm * p.tiles_n;
          mbar_arrive_expect_tx(&rbar[pf_buf], 4096u);
          tma_load_2d(rring + pf_buf * 4096, &tmR, &rbar[pf_buf], (ptn * p.BN + pf_c) * 4, ptm * GEMM_BM + q * 32);
        }
        if (++pf_buf == GEMM_RES_NBUF) pf_buf = 0;
        pf_c += CSTEP;
        if (pf_c >= p.BN) { pf_c = half * 32; pf_tile += gridDim.x; }
      };
      if constexpr (RES_TMA) {
        if (half * 32 >= p.BN) pf_tile = num_tiles;      // this warp owns no chunk (BN narrower than its first column)
#pragma unroll 1
        for (int i = 0; i < GEMM_RES_NBUF - 1; ++i) res_issue();
      }
      for (int item = blockIdx.x; item < num_tiles; item += gridDim.x) {
        const int tile = item / splits;
        const int tm = tile / p.tiles_n;
        const int tn = tile - tm * p.tiles_n;
        const int n_base = tn * p.BN;
        const int m_warp = tm * GEMM_BM + q * 32;
        const bool transposed = (MODE < 0) && p.out_q_transposed;
        constexpr bool kTrans = MODE >= 0 && (MODE & EPI_TRANS) != 0;
        int cls8[8], img8[8];
        if (!transposed && !kTrans) {
#pragma unroll
          for (int it = 0; it < 8; ++it) gemm_row_meta(p, m_warp + it * 4 + rsub, cls8[it], img8[it]);
        }
        acquire(item);
        if constexpr (kTrans) {
          // V^T code output [img][n][token'] (token' = att_vt_perm order inside each group of 16).  The warp's
          // 32 tokens x 32 channels go through the staging tile; each lane then owns ONE channel and emits whole
          // 16-token groups as 16 B stores (the thread-per-row form below needs 32 byte stores per lane and chunk).
          // Host guarantees rows_per_batch % 32 == 0 (a warp never straddles images), ldq % 16 == 0.
          const int img = m_warp / p.rows_per_batch;
          const int tok0 = m_warp - img * p.rows_per_batch;
          for (int c = half * 32; c < p.BN; c += CSTEP) {
            const int ncols = (p.BN - c) >= 32 ? 32 : 16;
            const uint8_t* stg = acc_tile + (q * nch + (c >> 5)) * GEMM_EPI_TILE_BYTES;
            const int col = ncols == 32 ? lane : (lane & 15);
            const int n = n_base + c + col;
            if (m_warp < p.M && n < p.N) {
              const float sc1 = __ldg(ep_scale + n);
              const float bi1 = ep_bias ? __ldg(ep_bias + n) : 0.f;
              int cr = 0;
              if constexpr ((MODE & EPI_CORR) != 0) cr = __ldg(p.corr + n);
              int8_t* o = p.out_q + ((long long)img * p.N + n) * p.ldq + tok0;
              const uint8_t* src = stg + (col & 3) * 4;
              const int cj = col >> 2;
              const int g0 = ncols == 32 ? 0 : (lane >> 4), g1 = ncols == 32 ? 2 : g0 + 1;
              for (int g = g0; g < g1; ++g) {
                uint32_t w4[4];
#pragma unroll
                for (int k = 0; k < 16; ++k) {
                  const int r7 = (((k >> 1) & 1) << 3) | (((k >> 2) & 3) << 1) | (k & 1);   // token of byte k
                  const int a = *reinterpret_cast<const int*>(src + (g * 16 + r7) * 128 + ((cj ^ (r7 & 7)) << 4));
                  const uint32_t qv = QPRE ? (quant_bits_pre(fmaf((float)(a - cr), sc1, bi1), qk) & 0xFFu)
                                           : quant_code((float)(a - cr) * sc1 + bi1, qk);
                  w4[k >> 2] = (k & 3) ? (w4[k >> 2] | (qv << (8 * (k & 3)))) : qv;
                }
                *reinterpret_cast<uint4*>(o + g * 16) = make_uint4(w4[0], w4[1], w4[2], w4[3]);
              }
            }
            __syncwarp();
          }
        } else if constexpr (MODE >= 0 && (MODE & EPI_GEGLU) != 0) {
          // GEGLU projection (ldm/modules/attention.py:42-44) fused with the consumer's quantizer: a 32-column chunk
          // holds 4 x (4 x-features | 4 gate-features); lane -> (row group of 8, pair); 4 iterations cover 32 rows.
          const int r8 = lane >> 2, pq = lane & 3;
          for (int c = half * 32; c < p.BN; c += CSTEP) {
            const uint8_t* stg = acc_tile + (q * nch + (c >> 5)) * GEMM_EPI_TILE_BYTES;
            const int nx = n_base + c + 8 * pq;          // 4 x columns, then 4 gate columns
            if (nx < p.N) {
              const float4 sx = __ldg(reinterpret_cast<const float4*>(p.scale + nx));
              const float4 sg = __ldg(reinterpret_cast<const float4*>(p.scale + nx + 4));
              float4 bx = make_float4(0.f, 0.f, 0.f, 0.f), bg = bx;
              if (p.bias) {
                bx = __ldg(reinterpret_cast<const float4*>(p.bias + nx));
                bg = __ldg(reinterpret_cast<const float4*>(p.bias + nx + 4));
              }
              int4 cx = make_int4(0, 0, 0, 0), cg = cx;
              if constexpr ((MODE & EPI_CORR) != 0) {
                cx = __ldg(reinterpret_cast<const int4*>(p.corr + nx));
                cg = __ldg(reinterpret_cast<const int4*>(p.corr + nx + 4));
              }
#pragma unroll
              for (int it = 0; it < 4; ++it) {
                const int row = it * 8 + r8;
                const int m = m_warp + row;
                if (m < p.M) {
                  const uint4 ax = *reinterpret_cast<const uint4*>(stg + row * 128 + (((2 * pq) ^ (row & 7)) << 4));
                  const uint4 ag = *reinterpret_cast<const uint4*>(stg + row * 128 + (((2 * pq + 1) ^ (row & 7)) << 4));
                  const float x0 = (float)((int)ax.x - cx.x) * sx.x + bx.x, g0 = (float)((int)ag.x - cg.x) * sg.x + bg.x;
                  const float x1 = (float)((int)ax.y - cx.y) * sx.y + bx.y, g1 = (float)((int)ag.y - cg.y) * sg.y + bg.y;
                  const float x2 = (float)((int)ax.z - cx.z) * sx.z + bx.z, g2 = (float)((int)ag.z - cg.z) * sg.z + bg.z;
                  const float x3 = (float)((int)ax.w - cx.w) * sx.w + bx.w, g3 = (float)((int)ag.w - cg.w) * sg.w + bg.w;
                  const uint32_t code = quant_code_fast(x0 * gelu_fast(g0), qk) | (quant_code_fast(x1 * gelu_fast(g1), qk) << 8) |
                                        (quant_code_fast(x2 * gelu_fast(g2), qk) << 16) | (quant_code_fast(x3 * gelu_fast(g3), qk) << 24);
                  *reinterpret_cast<uint32_t*>(p.out_q + (long long)m * p.ldq + (nx >> 1)) = code;
                }
              }
            }
            __syncwarp();
          }
        } else if (transposed) {
          const int m = m_warp + lane;
          int cls, img;
          gemm_row_meta(p, m, cls, img);
          for (int c = half * 32; c < p.BN; c += CSTEP) {
            if (p.BN - c >= 32) {
              uint32_t v[32];
              gemm_acc_row(acc_tile + (q * nch + (c >> 5)) * GEMM_EPI_TILE_BYTES, lane, v);
              if (m < p.M && n_base + c < p.N) gemm_epilogue_rowwise<32>(p, qk, v, m, n_base + c, cls, img);
            } else {
              uint32_t v[16];
              gemm_acc_row(acc_tile + (q * nch + (c >> 5)) * GEMM_EPI_TILE_BYTES, lane, v);
              if (m < p.M && n_base + c < p.N) gemm_epilogue_rowwise<16>(p, qk, v, m, n_base + c, cls, img);
            }
          }
        } else {
          for (int c = half * 32; c < p.BN; c += CSTEP) {
            const int ncols = (p.BN - c) >= 32 ? 32 : 16;
            const uint8_t* stg = acc_tile + (q * nch + (c >> 5)) * GEMM_EPI_TILE_BYTES;
            [[maybe_unused]] const uint8_t* rbuf = nullptr;
            if constexpr (RES_TMA) {
              res_issue();                              // keep GEMM_RES_NBUF - 1 loads in flight
              mbar_wait(&rbar[rd_buf], rd_phase);       // this item's residual sub-tile (32 rows x 128 B, 128B-swizzled)
              rbuf = rring + rd_buf * 4096;
            }
            const int n = n_base + c + cq * 4;
            const bool col_ok = cq * 4 < ncols && n < p.N;
            const unsigned cmask = __ballot_sync(0xffffffffu, col_ok);   // lanes ^8 / ^16 share cq: partners are always both in or out
            if (col_ok) {
              float sc[4], bi[4];
              int4 corr4 = make_int4(0, 0, 0, 0);
              if (MODE >= 0 || n + 3 < p.N) {
                const float4 s4 = *reinterpret_cast<const float4*>(ep_scale + n);
                sc[0] = s4.x; sc[1] = s4.y; sc[2] = s4.z; sc[3] = s4.w;
                if (ep_bias) {
                  const float4 b4 = *reinterpret_cast<const float4*>(ep_bias + n);
                  bi[0] = b4.x; bi[1] = b4.y; bi[2] = b4.z; bi[3] = b4.w;
                } else {
                  bi[0] = bi[1] = bi[2] = bi[3] = 0.f;
                }
                if (p.corr && !conv) corr4 = *reinterpret_cast<const int4*>(p.corr + n);
              } else {
                int cc[4] = {0, 0, 0, 0};
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                  const bool ok = n + j < p.N;
                  sc[j] = ok ? __ldg(p.scale + n + j) : 0.f;
                  bi[j] = (ok && p.bias) ? __ldg(p.bias + n + j) : 0.f;
                  cc[j] = (ok && p.corr && !conv) ? __ldg(p.corr + n + j) : 0;
                }
                corr4 = make_int4(cc[0], cc[1], cc[2], cc[3]);
              }
              int nq = n;   // column of the code output (per-head padded layout: attention Q/K operands)
              if (p.oq_d > 0) { const int hq = n / p.oq_d; nq = hq * p.oq_pitch + (n - hq * p.oq_d); }
              // Rows are finalised four at a time with everything they need from global memory (residual, conv
              // border-class correction) fetched up front, and - on the full-tile path - without any per-row
              // branch: the `m < M` tests split the unrolled loop into basic blocks, and with two epilogue warps
              // per scheduler the resulting dependent-issue chains (stall_wait) bounded the small-K GEMMs.
              const long long mrow = m_warp + rsub;
              float* of0 = p.out ? p.out + mrow * p.ldo + n : nullptr;
              const int oq_es = p.oq_f16 ? 2 : 1;      // bytes per emitted code
              int8_t* oq0 = p.out_q ? p.out_q + (mrow * p.ldq + nq) * oq_es : nullptr;
              const float* res0 = p.residual ? p.residual + mrow * p.ldr + n : nullptr;
              const long long of_step = 4 * p.ldo, oq_step = 4 * p.ldq * oq_es, res_step = 4 * p.ldr;
              float gsum[4] = {0.f, 0.f, 0.f, 0.f}, gsq[4] = {0.f, 0.f, 0.f, 0.f};
              auto rows = [&](auto full_tag) {
                constexpr bool FULL = decltype(full_tag)::value;
#pragma unroll
                for (int h4 = 0; h4 < 8; h4 += 4) {
                  float4 rpre[4];
                  int4 cpre[4];
#pragma unroll
                  for (int i = 0; i < 4; ++i) {
                    const int it = h4 + i;
                    [[maybe_unused]] const int m = m_warp + it * 4 + rsub;
                    rpre[i] = make_float4(0.f, 0.f, 0.f, 0.f);
                    cpre[i] = corr4;
                    if constexpr (RES_TMA) {
                      const int row = it * 4 + rsub;    // rows beyond M were zero-filled by the TMA unit
                      rpre[i] = *reinterpret_cast<const float4*>(rbuf + row * 128 + ((cq ^ (row & 7)) << 4));
                    } else if constexpr (MODE >= 0 && (MODE & EPI_RESIDUAL) != 0) {
                      if (FULL || m < p.M) rpre[i] = *reinterpret_cast<const float4*>(res0 + it * res_step);
                    }
                    if constexpr (MODE >= 0 && (MODE & EPI_CORR) != 0 && (MODE & EPI_CONV) != 0)
                      cpre[i] = __ldg(reinterpret_cast<const int4*>(p.corr + (long long)cls8[it] * p.N + n));
                  }
#pragma unroll
                  for (int i = 0; i < 4; ++i) {
                    const int it = h4 + i;
                    const int row = it * 4 + rsub;
                    const int m = m_warp + row;
                    if (FULL || m < p.M) {
                      const uint4 a4 = *reinterpret_cast<const uint4*>(stg + row * 128 + ((cq ^ (row & 7)) << 4));
                      gemm_finalise4<MODE>(p, qk, conv, a4, sc, bi, cpre[i], rpre[i], of0 + it * of_step, oq0 + it * oq_step,
                                           res0 + it * res_step, n, cls8[it], img8[it], gsum, gsq);
                    }
                  }
                }
              };
              if (m_warp + 32 <= p.M) rows(std::true_type{}); else rows(std::false_type{});
              if ((MODE < 0 || (MODE & EPI_OUT_F32) != 0) && p.gn_stats != nullptr && m_warp < p.M) {
                // this thread holds 8 of the slab's 32 rows for 4 columns: add the other three row groups (lanes ^ 8, ^ 16),
                // lanes 0-7 then own the slab's column sums for the chunk's 32 columns.  A row quarter wholly beyond M (the
                // last tile of a ragged M) has no slab: gn_stats holds ceil(M / 32) of them.
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                  gsum[j] += __shfl_xor_sync(cmask, gsum[j], 8);
                  gsq[j] += __shfl_xor_sync(cmask, gsq[j], 8);
                  gsum[j] += __shfl_xor_sync(cmask, gsum[j], 16);
                  gsq[j] += __shfl_xor_sync(cmask, gsq[j], 16);
                }
                if (rsub == 0) {
                  float2* st = p.gn_stats + (long long)(m_warp >> 5) * p.ld_stats + n;
                  if (MODE >= 0 || n + 3 < p.N) {
                    *reinterpret_cast<float4*>(st) = make_float4(gsum[0], gsq[0], gsum[1], gsq[1]);
                    *reinterpret_cast<float4*>(st + 2) = make_float4(gsum[2], gsq[2], gsum[3], gsq[3]);
                  } else {
#pragma unroll
                    for (int j = 0; j < 4; ++j)
                      if (n + j < p.N) st[j] = make_float2(gsum[j], gsq[j]);
                  }
                }
              }
            }
            if constexpr (RES_TMA) {
              fence_proxy_async();      // this buffer's generic-proxy reads are ordered before the TMA write that reuses it
              if (++rd_buf == GEMM_RES_NBUF) { rd_buf = 0; rd_phase ^= 1; }
            }
            __syncwarp();
          }
        }
        release();
      }
    };

    if constexpr (!OVL) {
      // serial schedule (gemm_overlap): the eight consumer warps run the epilogue themselves
      // after each main loop; named barrier 1 keeps the dump behind the previous tile's last read, and the reads behind
      // the dump
      if constexpr (SPLITK) {
        for (int item = blockIdx.x; item < num_tiles; item += gridDim.x) consume(item, [] {});
      } else {
        epilogue(
            cw,
            [&](const int item) {
              consume(item, [] { named_bar_sync(1, 8 * 32); });
              named_bar_sync(1, 8 * 32);
            },
            [] {});
      }
    } else if (warp < 12) {
      // Overlapped schedule.  The CTA's j-th work item (j = 0, 1, ...; both sides walk the same item sequence) completes
      // phase j of acc_full (8 consumer-warp arrivals after the dump) and then phase j of acc_empty (EPI_WARPS arrivals
      // after the epilogue's last read).  A wait on parity P returns once the phase of parity P most recently begun has
      // completed; a fresh barrier counts as having just completed a phase of parity 1.  So:
      //   consumer, before dumping item j: wait(acc_empty, (j & 1) ^ 1) - j = 0 passes at once, j >= 1 waits for phase
      //     j - 1 (the epilogue of item j - 1).  Phase j - 1 cannot be mistaken for j - 3: acc_empty cannot run more than
      //     one phase ahead of this wait, since its phase j needs the dump of item j that follows it.
      //   epilogue warp, before reading item j: wait(acc_full, j & 1) - phase j, the dump of item j; phase j + 1 (the
      //     next dump) cannot complete before this warp arrives on acc_empty for item j.
      // The arrives release and the waits acquire (CTA scope), ordering the generic-proxy tile stores before the
      // epilogue's loads, and those loads before the next dump's stores; __syncwarp orders the other lanes' accesses
      // before lane 0's arrive.
      gemm_setmaxnreg<gemm_consumer_regs(MODE), gemm_launch_regs(MODE)>();
      uint32_t j = 0;
      for (int item = blockIdx.x; item < num_tiles; item += gridDim.x, ++j) {
        consume(item, [&] { mbar_wait(acc_empty, (j & 1) ^ 1); });
        __syncwarp();
        if (lane == 0) mbar_arrive(acc_full);
      }
    } else {
      gemm_setmaxnreg<gemm_epi_regs(MODE), gemm_launch_regs(MODE)>();
      uint32_t j = 0;
      epilogue(
          warp - 12, [&](int) { mbar_wait(acc_full, j & 1); },
          [&] {
            __syncwarp();
            if (lane == 0) mbar_arrive(acc_empty);
            ++j;
          });
    }
  }
}

// Second half of a split-K GEMM: sum the K slices (int32: exact in any order) and apply the fp32 epilogue of the plain
// kernel - zero-point correction (per border class for convs), scale, bias, per-image vector, residual - in the same
// operation order, plus the GroupNorm slab statistics when the consumer wants them.  Block = one 32-row slab x 32 columns:
// thread (row, column quad); a warp touches 4 rows x 128 contiguous bytes per access.  grid = (N / 32, M / 32).
__global__ void __launch_bounds__(256) splitk_finish_kernel(const GemmArgs p) {
  __shared__ float sy[32][33], sq[32][33];
  const int r = threadIdx.x >> 3, q = threadIdx.x & 7;
  const int m = blockIdx.y * 32 + r;
  const int n = blockIdx.x * 32 + q * 4;
  const bool ok = m < p.M && n < p.N;
  float4 y = make_float4(0.f, 0.f, 0.f, 0.f);
  if (ok) {
    const long long slice = (long long)p.M * p.N;
    const int32_t* w = p.ws + (long long)m * p.N + n;
    int4 a = *reinterpret_cast<const int4*>(w);
#pragma unroll 4
    for (int z = 1; z < p.splits; ++z) {
      const int4 v = *reinterpret_cast<const int4*>(w + z * slice);
      a.x += v.x; a.y += v.y; a.z += v.z; a.w += v.w;
    }
    int cls, img;
    gemm_row_meta(p, m, cls, img);
    if (p.corr) {
      const int4 c = __ldg(reinterpret_cast<const int4*>(p.corr + (p.taps == 9 ? (long long)cls * p.N : 0) + n));
      a.x -= c.x; a.y -= c.y; a.z -= c.z; a.w -= c.w;
    }
    const float4 sc = __ldg(reinterpret_cast<const float4*>(p.scale + n));
    float4 bi = make_float4(0.f, 0.f, 0.f, 0.f);
    if (p.bias) bi = __ldg(reinterpret_cast<const float4*>(p.bias + n));
    y = make_float4((float)a.x * sc.x + bi.x, (float)a.y * sc.y + bi.y, (float)a.z * sc.z + bi.z, (float)a.w * sc.w + bi.w);
    if (p.rowvec) {
      const float4 rv = __ldg(reinterpret_cast<const float4*>(p.rowvec + (long long)img * p.ld_rowvec + n));
      y.x += rv.x; y.y += rv.y; y.z += rv.z; y.w += rv.w;
    }
    if (p.residual) {
      const float4 rs = *reinterpret_cast<const float4*>(p.residual + (long long)m * p.ldr + n);
      y.x += rs.x; y.y += rs.y; y.z += rs.z; y.w += rs.w;
    }
    *reinterpret_cast<float4*>(p.out + (long long)m * p.ldo + n) = y;
  }
  if (p.gn_stats) {        // column sums of the slab's 32 rows (host: M % 32 == 0), fixed order
    sy[r][4 * q] = y.x; sy[r][4 * q + 1] = y.y; sy[r][4 * q + 2] = y.z; sy[r][4 * q + 3] = y.w;
    sq[r][4 * q] = y.x * y.x; sq[r][4 * q + 1] = y.y * y.y; sq[r][4 * q + 2] = y.z * y.z; sq[r][4 * q + 3] = y.w * y.w;
    __syncthreads();
    if (threadIdx.x < 32) {
      const int col = blockIdx.x * 32 + threadIdx.x;
      if (col < p.N) {
        float s0 = 0.f, s1 = 0.f;
#pragma unroll
        for (int i = 0; i < 32; ++i) { s0 += sy[i][threadIdx.x]; s1 += sq[i][threadIdx.x]; }
        p.gn_stats[(long long)blockIdx.y * p.ld_stats + col] = make_float2(s0, s1);
      }
    }
  }
}

}  // namespace qd
