// C ABI of libqdiff_b200.so (see include/qdiff_b200.h): per-op launchers + recorded-program engine.
#include <cuda.h>
#include <cuda_runtime.h>
#include <cudaTypedefs.h>

#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <new>
#include <utility>
#include <vector>

#include "../../include/qdiff_b200.h"
#include "attention.cuh"
#include "attention_wg.cuh"
#include "elem.cuh"
#include "gemm_i8.cuh"
#include "runtime.cuh"

namespace qdr {

thread_local char g_err[512] = "";
std::atomic<long long> g_launches{0};

int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(QD_ERR_CUDA, "%s: %s", what, cudaGetErrorString(e));
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return QD_OK;
}

int current_device() {
  int dev = -1;
  if (cudaGetDevice(&dev) != cudaSuccess) return -1;
  return dev;
}

}  // namespace qdr

namespace {

using namespace qdr;

std::atomic<int> g_num_sms[kMaxDevices];   // per device (zero-initialised): a process may drive several GPUs

// SM count of the CURRENT device (cached per device).
int num_sms() {
  const int dev = current_device();
  if (dev < 0 || dev >= kMaxDevices) {
    fail(QD_ERR_CUDA, "no CUDA device: qdiff_b200 has no CPU fallback");
    return 0;
  }
  int n = g_num_sms[dev].load(std::memory_order_relaxed);
  if (n == 0) {
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) {
      fail(QD_ERR_CUDA, "no CUDA device: qdiff_b200 has no CPU fallback");
      return 0;
    }
    g_num_sms[dev].store(n, std::memory_order_relaxed);
  }
  return n;
}

struct DeviceGuard {   // run a block on `device`, restoring the caller's current device afterwards
  int prev = -1;
  bool ok = true;
  explicit DeviceGuard(int device) {
    if (cudaGetDevice(&prev) != cudaSuccess) prev = -1;
    if (prev != device) ok = cudaSetDevice(device) == cudaSuccess;
  }
  ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
};

int grid_for(long long work_items, int threads, int per_sm = 8) {
  const int sms = num_sms();
  long long blocks = (work_items + threads - 1) / threads;
  long long cap = (long long)sms * per_sm;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return (int)blocks;
}

// ------------------------------------------------------------------ TMA descriptor encode
PFN_cuTensorMapEncodeTiled_v12000 get_encode() {
  static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(p);
  });
  return fn;
}

int encode_u8_map(CUtensorMap* m, const void* base, int rank, const cuuint64_t* dims, const cuuint64_t* strides_bytes,
                  const cuuint32_t* box, int swizzle_bytes = 128) {
  auto enc = get_encode();
  if (!enc) return fail(QD_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
  cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_UINT8, (cuuint32_t)rank, const_cast<void*>(base), dims, strides_bytes,
                   box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   swizzle_bytes == 0 ? CU_TENSOR_MAP_SWIZZLE_NONE :
                   swizzle_bytes == 32 ? CU_TENSOR_MAP_SWIZZLE_32B : swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(QD_ERR_CUDA, "cuTensorMapEncodeTiled failed (%d)", (int)r);
  return QD_OK;
}

// ------------------------------------------------------------------ GEMM plan
struct GemmPlan {
  CUtensorMap tmA, tmB, tmR;   // tmR: residual as bytes [M][N*4], 128 B x 32 row boxes (plain GEMMs with a residual)
  qd::GemmArgs args;
  int grid, mode;
};

// N-tile width (<= qd::GEMM_MAX_BN).  Heuristic cost of a 128 x BN tile on one SM, in cycles (the constants are a
// rough model, not a fit to measurements on this GPU; tools/sweep_bn.py sweeps BN per layer shape):
//   main loop  per 128-byte k-block: max(tensor time ~ 2.1*BN, L2->SM operand delivery ~ 3.0*(128 + BN)) -- with one CTA per SM
//              the big-K convs are bound by the operand bytes (128 + BN)*128 per k-block, so wide tiles (more reuse of the
//              A rows) win even when they leave the last wave less full;
//   epilogue   ~ BN columns (overlaps the producer's loads of the next tile's operands);
//   waves      = ceil(tiles / SMs).
// QDIFF_BN_MODEL=wave selects the round-1 rule (waves * (BN + 24)), kept for A/B comparisons.
int pick_bn(int N, int tiles_m, int sms, int hint, int step, long long K) {
  if (hint > 0) return hint;
  static const int wave_model = [] { const char* e = getenv("QDIFF_BN_MODEL"); return (e && !strcmp(e, "wave")) ? 1 : 0; }();
  int best = step;
  double best_cost = -1.0;
  const int n16 = (N + step - 1) / step * step;
  const double kb = (double)((K + 127) / 128);
  for (int bn = step; bn <= qd::GEMM_MAX_BN; bn += step) {
    if (bn > n16) break;
    const long long tiles = (long long)tiles_m * ((N + bn - 1) / bn);
    const long long waves = (tiles + sms - 1) / sms;
    double cost;
    if (wave_model) {
      cost = (double)waves * (bn + 24);
    } else {
      const double main_loop = kb * (2.1 * bn > 3.0 * (128 + bn) ? 2.1 * bn : 3.0 * (128 + bn));
      const double epilogue = 6.0 * bn + 300.0;
      cost = (double)waves * ((main_loop > epilogue ? main_loop : epilogue) + 200.0);
    }
    if (best_cost < 0 || cost < best_cost - 1e-9 || (cost < best_cost + 1e-9 && bn > best)) {
      best_cost = cost;
      best = bn;
    }
  }
  return best;
}

int gemm_mode(const qd::GemmArgs& a);

// Split-K workspace: ONE fixed-size buffer per device, allocated at the first plan that needs it and never moved (recorded
// programs and captured CUDA graphs hold the pointer).  Ops of a device run one after the other, so they can share it.
constexpr size_t kSplitWsBytes = 64u << 20;
int32_t* splitk_workspace() {
  static void* ws[kMaxDevices] = {};
  static std::mutex mu;
  const int dev = current_device();
  if (dev < 0 || dev >= kMaxDevices) return nullptr;
  std::lock_guard<std::mutex> lk(mu);
  if (!ws[dev] && cudaMalloc(&ws[dev], kSplitWsBytes) != cudaSuccess) { ws[dev] = nullptr; cudaGetLastError(); }
  return reinterpret_cast<int32_t*>(ws[dev]);
}

int plan_gemm(const qd_gemm_desc* d, GemmPlan* pl) {
  if (!d || !d->a || !d->w || !d->scale) return fail(QD_ERR_BAD_ARG, "gemm: null operand");
  if (d->taps != 1 && d->taps != 9) return fail(QD_ERR_UNSUPPORTED, "gemm: taps must be 1 or 9 (got %d)", d->taps);
  if (d->C <= 0 || (d->C % 32) != 0) return fail(QD_ERR_UNSUPPORTED, "gemm: C=%d must be a positive multiple of 32", d->C);
  if (d->a_bf16 && (d->corr || d->out_q || d->geglu || d->w_int4_packed || !d->out))
    return fail(QD_ERR_BAD_ARG, "gemm: a_bf16 (weight-only) layers take no corr / out_q / geglu / packed weights and write fp32");
  if (d->M <= 0 || d->N <= 0) return fail(QD_ERR_BAD_ARG, "gemm: bad M/N");
  if (!d->out && !d->out_q) return fail(QD_ERR_BAD_ARG, "gemm: no output");
  const int sms = num_sms();
  if (!sms) return QD_ERR_CUDA;

  qd::GemmArgs& a = pl->args;
  memset(&a, 0, sizeof(a));
  a.M = d->M; a.N = d->N; a.C = d->C; a.taps = d->taps;
  a.kdup = d->k_dup == 2 ? 2 : 1;
  if (d->k_dup != 0 && d->k_dup != 1 && d->k_dup != 2) return fail(QD_ERR_BAD_ARG, "gemm: k_dup must be 0, 1 or 2");
  if (a.kdup == 2 && d->w_int4_packed) return fail(QD_ERR_BAD_ARG, "gemm: k_dup 2 is for 8-bit weights (not packed INT4)");
  a.tiles_m = (d->M + qd::GEMM_BM - 1) / qd::GEMM_BM;
  a.geglu = d->geglu;
  if (d->geglu) {
    if ((d->N & 7) || !d->out_q || d->out || d->rowvec || d->residual || d->out_q_transposed || (d->ldq & 3) || d->taps != 1)
      return fail(QD_ERR_BAD_ARG, "gemm: geglu needs N %% 8 == 0, out_q only, plain GEMM");
  }
  a.BN = pick_bn(d->N, a.tiles_m, sms, d->bn_hint, d->geglu ? 32 : 16, (long long)d->C * d->taps * a.kdup);
  // the GEGLU epilogue finalises whole 32-column chunks (4 x 8 interleaved x / gate columns): a narrower last chunk would
  // read accumulator columns the tile never wrote and store codes into the next N tile's output columns
  if (d->geglu && (a.BN % 32))
    return fail(QD_ERR_BAD_ARG, "gemm: geglu needs an N tile that is a multiple of 32 (bn_hint %d)", d->bn_hint);
  const int bn_default = a.BN;
  // split-K candidates (see below) take the widest N tile: few tiles remain, and what is shared among the SMs is the K loop
  // (the split-K partial kernel takes up to qd::GEMM_MAX_BN_SPLITK columns; without split-K the tile reverts to bn_default)
  static const int splitk_enabled = [] { const char* e = getenv("QDIFF_SPLITK"); return (e && !strcmp(e, "0")) ? 0 : 1; }();
  const int num_kb_all = ((d->C + qd::GEMM_BK - 1) / qd::GEMM_BK) * d->taps * a.kdup;
  const bool splitk_candidate = splitk_enabled && !d->bn_hint && !d->a_bf16 && !d->w_int4_packed && d->out && !d->out_q && !d->geglu &&
                                !(d->N & 3) && !(d->ldo & 3) && (!d->residual || !(d->ldr & 3)) && (!d->rowvec || !(d->ld_rowvec & 3)) &&
                                num_kb_all >= 16;
  if (splitk_candidate) {
    const int bn_wide = d->N >= qd::GEMM_MAX_BN_SPLITK ? qd::GEMM_MAX_BN_SPLITK : (d->N + 15) / 16 * 16;
    if (2 * a.tiles_m * ((d->N + bn_wide - 1) / bn_wide) <= sms) a.BN = bn_wide;
  }
  if (a.BN % 16 || a.BN < 16 || a.BN > qd::GEMM_MAX_BN_SPLITK || (d->bn_hint && a.BN > qd::GEMM_MAX_BN))
    return fail(QD_ERR_BAD_ARG, "gemm: bad BN %d (16 .. %d)", a.BN, qd::GEMM_MAX_BN);
  a.tiles_n = (d->N + a.BN - 1) / a.BN;
  a.a_signed = d->a_signed; a.b_signed = 1;

  // pipeline depth / shared-memory size depend on the epilogue variant (8 or 16 staging tiles): launch_gemm_mode()

  // ---- A map (always rank 4)
  cuuint64_t dims[4], strides[3];
  cuuint32_t box[4];
  if (d->taps == 1) {
    if (d->lda % 16) return fail(QD_ERR_UNSUPPORTED, "gemm: lda=%lld must be a multiple of 16", d->lda);
    if (d->lda < d->C) return fail(QD_ERR_BAD_ARG, "gemm: lda < C");
    dims[0] = (cuuint64_t)d->C; dims[1] = (cuuint64_t)d->M; dims[2] = 1; dims[3] = 1;
    strides[0] = (cuuint64_t)d->lda; strides[1] = (cuuint64_t)d->lda * d->M; strides[2] = strides[1];
    box[0] = qd::GEMM_BK; box[1] = qd::GEMM_BM; box[2] = 1; box[3] = 1;
  } else {
    const int H = d->H, W = d->W, B = d->B;
    if (H <= 0 || W <= 0 || B <= 0 || (long long)B * H * W != d->M) return fail(QD_ERR_BAD_ARG, "gemm: conv geometry");
    const int hw = H * W;
    int bh, bn;
    int bw = W;
    if (W > 128) {                 // first-stage decoder maps (256, 512 wide): a tile is a 128-pixel segment of one row
      if (W % 128) return fail(QD_ERR_UNSUPPORTED, "gemm: conv W=%d must divide or be a multiple of 128", W);
      bw = 128; bh = 1; bn = 1;
    } else if (hw >= 128) {
      if (128 % W) return fail(QD_ERR_UNSUPPORTED, "gemm: conv W=%d must divide 128", W);
      bh = 128 / W; bn = 1;
      if (H % bh) return fail(QD_ERR_UNSUPPORTED, "gemm: conv H=%d not a multiple of %d", H, bh);
    } else {
      if (128 % hw) return fail(QD_ERR_UNSUPPORTED, "gemm: conv H*W=%d must divide 128", hw);
      bh = H; bn = 128 / hw;
    }
    a.H = H; a.W = W; a.bh = bh; a.bn = bn;
    // pixel pitch: lda when it exceeds C (a column range of a wider NHWC buffer: the leading bfloat16 planes of a split3
    // activation), else the dense C
    const cuuint64_t pitch = d->lda > d->C ? (cuuint64_t)d->lda : (cuuint64_t)d->C;
    if (pitch % 16) return fail(QD_ERR_UNSUPPORTED, "gemm: conv pixel pitch %llu must be a multiple of 16", (unsigned long long)pitch);
    dims[0] = (cuuint64_t)d->C; dims[1] = (cuuint64_t)W; dims[2] = (cuuint64_t)H; dims[3] = (cuuint64_t)B;
    strides[0] = pitch; strides[1] = pitch * W; strides[2] = pitch * W * H;
    box[0] = qd::GEMM_BK; box[1] = (cuuint32_t)bw; box[2] = (cuuint32_t)bh; box[3] = (cuuint32_t)bn;
  }
  int rc = encode_u8_map(&pl->tmA, d->a, 4, dims, strides, box);
  if (rc) return rc;
  if (d->w_int4_packed) {
    if (!d->w_zero) return fail(QD_ERR_BAD_ARG, "gemm: packed INT4 weights need w_zero");
    if (((uintptr_t)d->w) & 15) return fail(QD_ERR_BAD_ARG, "gemm: packed weights must be 16-byte aligned");
    a.w4 = 1;
    a.wzero = d->w_zero;
  }
  a.out = d->out; a.ldo = d->ldo;
  a.out_q = reinterpret_cast<int8_t*>(d->out_q); a.ldq = d->ldq;
  a.out_q_transposed = d->out_q_transposed;
  a.rows_per_batch = d->rows_per_batch;
  if ((d->rowvec || d->out_q_transposed) && d->rows_per_batch <= 0) return fail(QD_ERR_BAD_ARG, "gemm: rows_per_batch required");
  a.oq_d = d->out_q_head_dim; a.oq_pitch = d->out_q_head_pitch;
  a.oq_f16 = d->out_q_f16 ? 1 : 0;
  if (a.oq_f16 && (!d->out_q || d->out_q_transposed || d->geglu || (d->ldq & 3) || (((uintptr_t)d->out_q) & 7)))
    return fail(QD_ERR_BAD_ARG, "gemm: out_q_f16 needs a row-major out_q with ldq %% 4 == 0");
  if (a.oq_d > 0 && ((a.oq_d & 3) || (a.oq_pitch & 3) || a.oq_pitch < a.oq_d || d->out_q_transposed || !d->out_q))
    return fail(QD_ERR_BAD_ARG, "gemm: bad out_q head layout");
  if (d->out_q && d->oq.qmax - d->oq.qmin > 255)
    return fail(QD_ERR_UNSUPPORTED, "gemm: the epilogue emits 8-bit codes; quantizer range [%d, %d] is wider", d->oq.qmin, d->oq.qmax);
  a.q_delta = d->oq.delta; a.q_zp = d->oq.zero_point; a.q_lo = d->oq.qmin; a.q_hi = d->oq.qmax;
  a.scale = d->scale; a.bias = d->bias; a.corr = d->corr;
  a.scale_q = d->scale_q; a.bias_q = d->bias_q;
  a.gn_stats = reinterpret_cast<float2*>(d->gn_stats); a.ld_stats = d->ld_stats;
  a.bf16 = d->a_bf16;
  if (d->gn_stats && (!d->out || (d->ld_stats & 1) || (reinterpret_cast<uintptr_t>(d->gn_stats) & 15)))
    return fail(QD_ERR_BAD_ARG, "gemm: gn_stats needs an fp32 output, an even ld_stats and 16-byte alignment");
  if ((d->scale_q == nullptr) != (d->bias_q == nullptr)) return fail(QD_ERR_BAD_ARG, "gemm: scale_q and bias_q come together");
  a.rowvec = d->rowvec; a.ld_rowvec = d->ld_rowvec;
  a.residual = d->residual; a.ldr = d->ldr;
  const int tiles = a.tiles_m * a.tiles_n;
  pl->grid = tiles < sms ? tiles : sms;
  pl->mode = gemm_mode(a);
  // ---- split-K: short-M, long-K layers (the 4x4 / 8x8 levels: few output tiles, 90-220 k-blocks each).  A CTA's main loop
  // time per k-block depends little on the N tile, so the lever is to share a tile's K loop among idle SMs.  fp32-output
  // layers (GroupNorm slab statistics come from the finish pass).
  {
    const int num_kb = num_kb_all;
    const bool eligible = splitk_candidate && pl->mode >= 0 && 2 * tiles <= sms &&
                          (!a.gn_stats || (!(a.M & 31) && !(a.ld_stats & 1)));
    if (eligible) {
      int splits = sms / tiles;
      if (splits > 16) splits = 16;
      if (splits > num_kb / 4) splits = num_kb / 4;
      if (splits >= 2 && (size_t)splits * a.M * a.N * 4 <= kSplitWsBytes) {
        const int per = (num_kb + splits - 1) / splits;
        splits = (num_kb + per - 1) / per;
        int32_t* ws = splitk_workspace();
        if (ws && splits >= 2) {
          a.splits = splits; a.kb_per_split = per; a.ws = ws;
          pl->grid = tiles * splits < sms ? tiles * splits : sms;
        }
      }
    }
  }
  if (a.splits <= 1 && a.BN > qd::GEMM_MAX_BN) {      // no split-K after all: the N tile of the ordinary kernels
    a.BN = bn_default;
    a.tiles_n = (d->N + a.BN - 1) / a.BN;
    const int t = a.tiles_m * a.tiles_n;
    pl->grid = t < sms ? t : sms;
  }
  // ---- B map: [w_rows][taps*C] s8, or [w_rows][taps*C/2] packed 4-bit codes (unswizzled: the unpack warps re-lay it out)
  {
    const int w_rows = d->w_rows > 0 ? d->w_rows : d->N;
    if (d->w_int4_packed) {
      cuuint64_t bd[2] = {(cuuint64_t)d->taps * d->C / 2, (cuuint64_t)w_rows};
      cuuint64_t bs[1] = {(cuuint64_t)d->taps * d->C / 2};
      cuuint32_t bb[2] = {qd::GEMM_BK / 2, (cuuint32_t)a.BN};
      rc = encode_u8_map(&pl->tmB, d->w, 2, bd, bs, bb, 0);
    } else {
      cuuint64_t bd[2] = {(cuuint64_t)d->taps * d->C * a.kdup, (cuuint64_t)w_rows};
      cuuint64_t bs[1] = {(cuuint64_t)d->taps * d->C * a.kdup};
      cuuint32_t bb[2] = {qd::GEMM_BK, (cuuint32_t)a.BN};
      rc = encode_u8_map(&pl->tmB, d->w, 2, bd, bs, bb);
    }
    if (rc) return rc;
  }
  if (a.bf16 && pl->mode < 0)
    return fail(QD_ERR_UNSUPPORTED, "gemm: weight-only (a_bf16) layer needs a specialised epilogue (N %% 4 == 0, aligned leading dimensions)");
  memset(&pl->tmR, 0, sizeof(pl->tmR));
  if (qd::gemm_res_tma(pl->mode)) {
    cuuint64_t rd[2] = {(cuuint64_t)d->N * 4, (cuuint64_t)d->M};
    cuuint64_t rs[1] = {(cuuint64_t)d->ldr * 4};
    cuuint32_t rb[2] = {128, 32};
    rc = encode_u8_map(&pl->tmR, d->residual, 2, rd, rs, rb);
    if (rc) return rc;
  }
  return QD_OK;
}

template <int MODE, bool W4>
int launch_gemm_mode_w(const GemmPlan& pl, cudaStream_t s) {
  static std::atomic<unsigned long long> optin{0};
  if (int rc = ensure_smem_optin(qd::gemm_i8_kernel<MODE, W4>, 227 * 1024, optin, "gemm")) return rc;
  qd::GemmArgs a = pl.args;
  const int stage_bytes = qd::gemm_stage_footprint(a.BN, W4 ? 1 : 0);
  constexpr int res_bytes = qd::gemm_res_bytes(MODE);
  constexpr bool splitk = MODE >= 0 && (MODE & qd::EPI_SPLITK) != 0;
  if (a.BN > qd::gemm_max_bn(MODE)) return fail(QD_ERR_BAD_ARG, "gemm: BN=%d exceeds %d (mode %d)", a.BN, qd::gemm_max_bn(MODE), MODE);
  int stages = (232448 - 512 - qd::gemm_acc_tile_bytes(a.BN, splitk) - res_bytes - 1024 - 1024) / stage_bytes;
  if (stages > qd::GEMM_MAX_STAGES) stages = qd::GEMM_MAX_STAGES;
  if (stages < 2) stages = 2;
  a.stages = stages;
  const int smem = qd::gemm_smem_layout(a.BN, stages, W4 ? 1 : 0, res_bytes, splitk).total;
  if (smem > 232448) return fail(QD_ERR_UNSUPPORTED, "gemm: BN=%d needs %d bytes of shared memory for 2 stages (mode %d, w4 %d)", a.BN, smem, MODE, (int)W4);
  launch_k(qd::gemm_i8_kernel<MODE, W4>, pl.grid, qd::gemm_threads(MODE, W4), smem, s, pl.tmA, pl.tmB, pl.tmR, a);
  return check_launch("gemm_i8_kernel");
}

template <int MODE>
int launch_gemm_mode(const GemmPlan& pl, cudaStream_t s) {
  return pl.args.w4 ? launch_gemm_mode_w<MODE, true>(pl, s) : launch_gemm_mode_w<MODE, false>(pl, s);
}

// Specialised epilogues for the hot combinations; everything else runs the generic (-1) kernel.
int gemm_mode(const qd::GemmArgs& a) {
  const bool f = a.out != nullptr, q = a.out_q != nullptr;
  if (a.geglu) return qd::EPI_GEGLU | qd::EPI_OUT_Q | (a.corr ? qd::EPI_CORR : 0);
  if (q && !f && !a.geglu && !a.scale_q) return -1;     // specialised requantising epilogues take pre-divided constants
  if (a.out_q_transposed && q && !f && !a.rowvec && !a.residual && a.taps == 1 && a.oq_d == 0 &&
      a.rows_per_batch % 32 == 0 && (a.ldq & 15) == 0 && (reinterpret_cast<uintptr_t>(a.out_q) & 15) == 0)
    return qd::EPI_TRANS | qd::EPI_OUT_Q | (a.corr ? qd::EPI_CORR : 0);
  if (f == q || a.out_q_transposed || (a.N & 3)) return -1;
  if (a.rowvec && a.residual) return -1;
  if (q && a.rowvec) return -1;
  if (f && (a.ldo & 3)) return -1;
  if (q && (a.ldq & 3)) return -1;
  if (a.residual && (a.ldr & 3)) return -1;
  if (a.rowvec && (a.ld_rowvec & 3)) return -1;
  // short-K plain GEMMs with a residual (to_out / proj_out at the 64x64 and 32x32 levels, split-shortcut second halves):
  // the epilogue is the critical path and its residual loads are latency-bound -> TMA ring.  Longer K: the ring's shared
  // memory would cost pipeline stages (tools/sweep_bn.py: K = 1280 lost 10 % with 2 stages), registers-prefetch path.
  if (a.bf16) {      // weight-only: fp32 output with an optional per-image vector or residual; no ring (long byte-K)
    return qd::EPI_BF16 | qd::EPI_OUT_F32 | ((a.taps == 9) ? qd::EPI_CONV : 0) | (a.rowvec ? qd::EPI_ROWVEC : 0) |
           (a.residual ? qd::EPI_RESIDUAL : 0);
  }
  static const int ring_kb = [] { const char* e = getenv("QDIFF_RES_RING_KB"); return e ? atoi(e) : 5; }();
  const int num_kb = ((a.C + qd::GEMM_BK - 1) / qd::GEMM_BK) * a.taps * a.kdup;
  const bool ring = a.residual && a.taps == 1 && num_kb <= ring_kb && !(reinterpret_cast<uintptr_t>(a.residual) & 15) &&
                    !a.w4;    // packed INT4 stages already carry the staging area of the packed tile: no room for the ring
  return (a.corr ? qd::EPI_CORR : 0) | ((a.taps == 9) ? qd::EPI_CONV : 0) | (a.rowvec ? qd::EPI_ROWVEC : 0) |
         (a.residual ? qd::EPI_RESIDUAL : 0) | (f ? qd::EPI_OUT_F32 : qd::EPI_OUT_Q) | (ring ? qd::EPI_RESTMA : 0);
}

int launch_gemm(const GemmPlan& pl, cudaStream_t s) {
  using namespace qd;
  if (pl.args.splits > 1) {     // K slices -> workspace, then the epilogue pass
    if (int rc = launch_gemm_mode_w<EPI_SPLITK, false>(pl, s)) return rc;   // split-K never takes packed INT4 weights
    launch_k(qd::splitk_finish_kernel, dim3((pl.args.N + 31) / 32, (pl.args.M + 31) / 32), 256, 0, s, pl.args);
    return check_launch("splitk_finish_kernel");
  }
  switch (pl.mode) {
    case EPI_OUT_F32: return launch_gemm_mode<EPI_OUT_F32>(pl, s);
    case EPI_OUT_F32 | EPI_CORR: return launch_gemm_mode<EPI_OUT_F32 | EPI_CORR>(pl, s);
    case EPI_OUT_F32 | EPI_ROWVEC: return launch_gemm_mode<EPI_OUT_F32 | EPI_ROWVEC>(pl, s);
    case EPI_OUT_F32 | EPI_ROWVEC | EPI_CORR: return launch_gemm_mode<EPI_OUT_F32 | EPI_ROWVEC | EPI_CORR>(pl, s);
    case EPI_OUT_F32 | EPI_RESIDUAL: return launch_gemm_mode<EPI_OUT_F32 | EPI_RESIDUAL>(pl, s);
    case EPI_OUT_F32 | EPI_RESIDUAL | EPI_CORR: return launch_gemm_mode<EPI_OUT_F32 | EPI_RESIDUAL | EPI_CORR>(pl, s);
    case EPI_OUT_F32 | EPI_CORR | EPI_CONV: return launch_gemm_mode<EPI_OUT_F32 | EPI_CORR | EPI_CONV>(pl, s);
    case EPI_OUT_F32 | EPI_ROWVEC | EPI_CORR | EPI_CONV: return launch_gemm_mode<EPI_OUT_F32 | EPI_ROWVEC | EPI_CORR | EPI_CONV>(pl, s);
    case EPI_OUT_F32 | EPI_RESIDUAL | EPI_CORR | EPI_CONV: return launch_gemm_mode<EPI_OUT_F32 | EPI_RESIDUAL | EPI_CORR | EPI_CONV>(pl, s);
    case EPI_OUT_Q | EPI_CORR | EPI_CONV: return launch_gemm_mode<EPI_OUT_Q | EPI_CORR | EPI_CONV>(pl, s);
    // 3x3 convs on symmetric activation codes (zero point 0: no correction table): CIFAR-10, LSUN-bedroom
    case EPI_OUT_F32 | EPI_CONV: return launch_gemm_mode<EPI_OUT_F32 | EPI_CONV>(pl, s);
    case EPI_OUT_F32 | EPI_ROWVEC | EPI_CONV: return launch_gemm_mode<EPI_OUT_F32 | EPI_ROWVEC | EPI_CONV>(pl, s);
    case EPI_OUT_F32 | EPI_RESIDUAL | EPI_CONV: return launch_gemm_mode<EPI_OUT_F32 | EPI_RESIDUAL | EPI_CONV>(pl, s);
    case EPI_OUT_Q | EPI_CONV: return launch_gemm_mode<EPI_OUT_Q | EPI_CONV>(pl, s);
    case EPI_OUT_Q: return launch_gemm_mode<EPI_OUT_Q>(pl, s);
    case EPI_OUT_Q | EPI_CORR: return launch_gemm_mode<EPI_OUT_Q | EPI_CORR>(pl, s);
    case EPI_OUT_Q | EPI_RESIDUAL: return launch_gemm_mode<EPI_OUT_Q | EPI_RESIDUAL>(pl, s);
    case EPI_OUT_Q | EPI_RESIDUAL | EPI_CORR: return launch_gemm_mode<EPI_OUT_Q | EPI_RESIDUAL | EPI_CORR>(pl, s);
    case EPI_OUT_F32 | EPI_RESIDUAL | EPI_RESTMA: return launch_gemm_mode<EPI_OUT_F32 | EPI_RESIDUAL | EPI_RESTMA>(pl, s);
    case EPI_OUT_F32 | EPI_RESIDUAL | EPI_CORR | EPI_RESTMA: return launch_gemm_mode<EPI_OUT_F32 | EPI_RESIDUAL | EPI_CORR | EPI_RESTMA>(pl, s);
    case EPI_OUT_Q | EPI_RESIDUAL | EPI_RESTMA: return launch_gemm_mode<EPI_OUT_Q | EPI_RESIDUAL | EPI_RESTMA>(pl, s);
    case EPI_OUT_Q | EPI_RESIDUAL | EPI_CORR | EPI_RESTMA: return launch_gemm_mode<EPI_OUT_Q | EPI_RESIDUAL | EPI_CORR | EPI_RESTMA>(pl, s);
    // weight-only layers (bfloat16 x3 planes, fp32 accumulators)
    case EPI_BF16 | EPI_OUT_F32: return launch_gemm_mode_w<EPI_BF16 | EPI_OUT_F32, false>(pl, s);
    case EPI_BF16 | EPI_OUT_F32 | EPI_ROWVEC: return launch_gemm_mode_w<EPI_BF16 | EPI_OUT_F32 | EPI_ROWVEC, false>(pl, s);
    case EPI_BF16 | EPI_OUT_F32 | EPI_RESIDUAL: return launch_gemm_mode_w<EPI_BF16 | EPI_OUT_F32 | EPI_RESIDUAL, false>(pl, s);
    case EPI_BF16 | EPI_OUT_F32 | EPI_CONV: return launch_gemm_mode_w<EPI_BF16 | EPI_OUT_F32 | EPI_CONV, false>(pl, s);
    case EPI_BF16 | EPI_OUT_F32 | EPI_ROWVEC | EPI_CONV: return launch_gemm_mode_w<EPI_BF16 | EPI_OUT_F32 | EPI_ROWVEC | EPI_CONV, false>(pl, s);
    case EPI_BF16 | EPI_OUT_F32 | EPI_RESIDUAL | EPI_CONV: return launch_gemm_mode_w<EPI_BF16 | EPI_OUT_F32 | EPI_RESIDUAL | EPI_CONV, false>(pl, s);
    case EPI_TRANS | EPI_OUT_Q: return launch_gemm_mode<EPI_TRANS | EPI_OUT_Q>(pl, s);
    case EPI_TRANS | EPI_OUT_Q | EPI_CORR: return launch_gemm_mode<EPI_TRANS | EPI_OUT_Q | EPI_CORR>(pl, s);
    case EPI_GEGLU | EPI_OUT_Q: return launch_gemm_mode<EPI_GEGLU | EPI_OUT_Q>(pl, s);
    case EPI_GEGLU | EPI_OUT_Q | EPI_CORR: return launch_gemm_mode<EPI_GEGLU | EPI_OUT_Q | EPI_CORR>(pl, s);
    default: return launch_gemm_mode<-1>(pl, s);
  }
}

// ------------------------------------------------------------------ elementwise launchers
// Each launcher's descriptor checks live in a validate_* function that qd_engine_add_op runs too, so that a descriptor the
// kernels cannot take is refused when it is added to a program rather than surfacing mid-graph as a misaligned access.
// Vector paths need their base pointers and leading dimensions aligned to the access width; where a scalar kernel exists
// (quantize, split, im2col) a misaligned descriptor runs that one instead.
bool aligned(const void* p, int bytes) { return ((uintptr_t)p & (uintptr_t)(bytes - 1)) == 0; }

bool quantize_vec(const qd_quantize_desc& d) {
  return (d.C % 4 == 0) && (d.ld_src % 4 == 0) && (d.ld_dst % 4 == 0) && (d.split % 4 == 0) && aligned(d.src, 16) &&
         aligned(d.dst, 4);
}

int validate_quantize(const qd_quantize_desc& d) {
  if (!d.src || !d.dst || d.M <= 0 || d.C <= 0) return fail(QD_ERR_BAD_ARG, "quantize: bad args");
  if (d.q0.qmax - d.q0.qmin > 255 || d.q1.qmax - d.q1.qmin > 255)
    return fail(QD_ERR_UNSUPPORTED, "quantize: the engine emits 8-bit codes; quantizer range [%d, %d] is wider", d.q0.qmin, d.q0.qmax);
  if (!aligned(d.src, 4)) return fail(QD_ERR_UNSUPPORTED, "quantize: src must be 4-byte aligned");
  if (d.upsample2x && !quantize_vec(d))
    return fail(QD_ERR_UNSUPPORTED, "quantize: upsample needs C, ld_src, ld_dst, split %% 4 == 0, src 16-byte and dst 4-byte aligned");
  return QD_OK;
}

int launch_quantize(const qd_quantize_desc& d, cudaStream_t s) {
  if (int rc = validate_quantize(d)) return rc;
  if (quantize_vec(d)) {
    const long long rows = d.upsample2x ? (long long)d.B * 4 * d.H * d.W : d.M;
    launch_k(qd::quantize_kernel, grid_for(rows * (d.C / 4), 256), 256, 0, s, d);
  } else {
    launch_k(qd::quantize_scalar_kernel, grid_for((long long)d.M * d.C, 256), 256, 0, s, d);
  }
  return check_launch("quantize_kernel");
}

// slab / rows-per-block of the three-kernel GroupNorm: enough blocks to fill the GPU at every feature-map size
int gn_slab_rows(int B, int HW) {
  int sms = num_sms();
  if (sms <= 0) sms = 132;
  long long r = ((long long)B * HW) / (4LL * sms);
  int slab = 64;
  while (slab > 8 && slab > r) slab >>= 1;
  return slab;
}

long long gn_workspace_floats(int B, int HW, int C, int groups) {
  const int slab = gn_slab_rows(B, HW);
  const long long nslab = (HW + slab - 1) / slab;
  (void)C;
  return (long long)B * nslab * groups * 2 * 2 + (long long)B * groups * 2 + 16;   // doubles count as 2 floats
}

int use_stats_env() {
  static const int v = [] { const char* e = getenv("QDIFF_GN_STATS"); return (e && !strcmp(e, "0")) ? 0 : 1; }();
  return v;
}

enum GnPath { GN_FUSED, GN_FROM_STATS, GN_PARTIAL };

// Which of the three GroupNorm paths launch_groupnorm takes for a descriptor (the checks of validate_groupnorm passed).
GnPath gn_path(const qd_groupnorm_desc& d) {
  const int cpg = d.C / d.groups;
  // ---- single-kernel path: the (image, group) slab fits the registers of one block
  bool ok = (cpg % 2 == 0) && cpg <= 128 && (d.ld_x % 2 == 0) && (!d.out_f || d.ld_f % 2 == 0);
  for (int o = 0; o < d.n_out; ++o) ok = ok && (d.ld_q[o] % 2 == 0);
  const long long units = (long long)d.HW * (cpg / 2);
  static const int force = [] {   // QDIFF_GN=fused|split: A/B switch for profiling
    const char* e = getenv("QDIFF_GN");
    return !e ? 0 : (!strcmp(e, "fused") ? 1 : (!strcmp(e, "split") ? 2 : 0));
  }();
  const long long limit = force == 1 ? 512LL * qd::GN_NU : (force == 2 ? 0 : 256LL * qd::GN_NU);
  // The one-block-per-(image, group) kernel reads cpg * 4 bytes per pixel out of every C * 4 (sector-inefficient for
  // narrow groups) and launches B * groups blocks: it only pays in the launch-latency regime.  The three-kernel path
  // (statistics from the producing GEMMs' slab sums, then a coalesced apply pass) takes everything else: maps above ~2 M
  // elements or with more than 2048 blocks, and above ~0.5 M elements when the producing GEMMs left slab statistics.
  // (Thresholds from per-op timings on the previous GPU generation; not re-measured on the H100.)
  const long long elems = (long long)d.B * d.HW * d.C;
  const bool small_problem = elems <= ((d.stats_in && use_stats_env()) ? (512LL << 10) : (2LL << 20)) && (long long)d.B * d.groups <= 2048;
  if (ok && units <= limit && (force == 1 || small_problem)) return GN_FUSED;
  return (d.stats_in && use_stats_env()) ? GN_FROM_STATS : GN_PARTIAL;
}

int validate_groupnorm(const qd_groupnorm_desc& d) {
  if (!d.x || !d.gamma || !d.beta || d.B <= 0 || d.HW <= 0) return fail(QD_ERR_BAD_ARG, "groupnorm: null arg or empty map");
  if (d.groups <= 0 || d.groups > qd::GN_MAX_GROUPS || d.C <= 0 || d.C % 4 || d.C % d.groups || d.ld_x % 4)
    return fail(QD_ERR_UNSUPPORTED, "groupnorm: C=%d groups=%d", d.C, d.groups);
  if (d.n_out < 0 || d.n_out > 3) return fail(QD_ERR_BAD_ARG, "groupnorm: n_out");
  for (int o = 0; o < d.n_out; ++o)
    if (!d.out_q[o]) return fail(QD_ERR_BAD_ARG, "groupnorm: out_q[%d] is NULL", o);
  if (d.ss_scale && !d.ss_shift) return fail(QD_ERR_BAD_ARG, "groupnorm: scale-shift needs both operands");
  if (d.raw_q && ((d.raw_split & 3) || (d.ld_raw & 3) || d.raw_split < 0))
    return fail(QD_ERR_BAD_ARG, "groupnorm: raw output needs raw_split %% 4 == 0 and ld_raw %% 4 == 0");
  // the fused kernel moves channel pairs (float2 loads and stores, 16-bit code pairs); the apply kernel channel quads
  // (float4, 32-bit code quads)
  const GnPath path = gn_path(d);
  const int w = path == GN_FUSED ? 2 : 4;
  if (!aligned(d.x, 4 * w)) return fail(QD_ERR_UNSUPPORTED, "groupnorm: x must be %d-byte aligned", 4 * w);
  if (d.out_f && (!aligned(d.out_f, 4 * w) || d.ld_f % w))
    return fail(QD_ERR_UNSUPPORTED, "groupnorm: out_f needs %d-byte alignment and ld_f %% %d == 0", 4 * w, w);
  for (int o = 0; o < d.n_out; ++o)
    if (!aligned(d.out_q[o], w) || d.ld_q[o] % w)
      return fail(QD_ERR_UNSUPPORTED, "groupnorm: out_q[%d] needs %d-byte alignment and ld_q %% %d == 0", o, w, w);
  if (d.raw_q && !aligned(d.raw_q, w)) return fail(QD_ERR_UNSUPPORTED, "groupnorm: raw_q must be %d-byte aligned", w);
  if (path != GN_FUSED) {
    if (!d.ws) return fail(QD_ERR_BAD_ARG, "groupnorm: workspace required");
    if (!aligned(d.ws, 8)) return fail(QD_ERR_BAD_ARG, "groupnorm: workspace must be 8-byte aligned");
  }
  if (path == GN_FROM_STATS) {
    if (d.HW % 32) return fail(QD_ERR_BAD_ARG, "groupnorm: stats_in needs HW %% 32 == 0");
    if (!aligned(d.stats_in, 8)) return fail(QD_ERR_UNSUPPORTED, "groupnorm: stats_in must be 8-byte aligned");
  }
  return QD_OK;
}

int launch_groupnorm(const qd_groupnorm_desc& d, cudaStream_t s) {
  if (int rc = validate_groupnorm(d)) return rc;
  const int cpg = d.C / d.groups;
  const GnPath path = gn_path(d);
  if (path == GN_FUSED) {
    const long long units = (long long)d.HW * (cpg / 2);
    int threads = units <= 256LL * qd::GN_NU ? 256 : 512;
    if (units < 256) threads = (int)((units + 31) / 32 * 32);
    if (threads < cpg / 2) threads = (cpg / 2 + 31) / 32 * 32;
    launch_k(qd::gn_fused_small_kernel, dim3(d.groups, d.B), threads, 0, s, d);
    return check_launch("gn_fused_small_kernel");
  }
  const int slab = gn_slab_rows(d.B, d.HW);
  const int nslab = (d.HW + slab - 1) / slab;
  double* part = reinterpret_cast<double*>(d.ws);
  float* stats = d.ws + (long long)d.B * nslab * d.groups * 4;
  int threads = d.C / 4;
  threads = (threads + 31) / 32 * 32;
  if (threads > 256) threads = 256;
  if (threads < 2 * d.groups) threads = (2 * d.groups + 31) / 32 * 32;
  int rc;
  if (path == GN_FROM_STATS) {
    // the producing GEMMs left per-slab column sums: no pass over x for the statistics
    launch_k(qd::gn_finalize_from_stats_kernel, dim3(d.groups, d.B), 128, 0, s, reinterpret_cast<const float2*>(d.stats_in),
                                                                         d.ld_stats_in, d.HW, d.C, d.groups, d.eps, stats);
    rc = check_launch("gn_finalize_from_stats_kernel");
    if (rc) return rc;
  } else {
    launch_k(qd::gn_partial_kernel, dim3(nslab, d.B), threads, 2 * d.C * sizeof(float), s, d.x, d.ld_x, d.HW, d.C, d.groups, slab,
                                                                                     nslab, part);
    rc = check_launch("gn_partial_kernel");
    if (rc) return rc;
    launch_k(qd::gn_finalize_kernel, d.B, 256, 0, s, part, d.HW, d.C, d.groups, nslab, d.eps, stats);
    rc = check_launch("gn_finalize_kernel");
    if (rc) return rc;
  }
  // apply: block = TX channel quads x TY rows, 256 threads; rows per block sized so that the grid fills the GPU ~4x over
  const int cq = d.C / 4;
  const int slabs_x = (cq + 255) / 256;
  const int TX = (cq + slabs_x - 1) / slabs_x;
  int TY = 256 / TX;
  if (TY < 1) TY = 1;
  const int athreads = TX * TY;
  int rows = qd::GN_BATCH * TY;
  while ((long long)((d.HW + rows - 1) / rows) * slabs_x * d.B > 8LL * num_sms() && rows < 8 * qd::GN_BATCH * TY) rows += qd::GN_BATCH * TY;
  const dim3 grid(slabs_x, (d.HW + rows - 1) / rows, d.B);
  const bool raw = d.raw_q != nullptr;
#define QD_GN_APPLY(NOUT, RAW) launch_k(qd::gn_apply_kernel<NOUT, RAW>, grid, athreads, 0, s, d, stats, rows, TX)
  switch (d.n_out * 2 + (raw ? 1 : 0)) {
    case 0: QD_GN_APPLY(0, false); break;
    case 1: QD_GN_APPLY(0, true); break;
    case 2: QD_GN_APPLY(1, false); break;
    case 3: QD_GN_APPLY(1, true); break;
    case 4: QD_GN_APPLY(2, false); break;
    case 5: QD_GN_APPLY(2, true); break;
    case 6: QD_GN_APPLY(3, false); break;
    default: QD_GN_APPLY(3, true); break;
  }
#undef QD_GN_APPLY
  return check_launch("gn_apply_kernel");
}

template <int NVEC>
int launch_layernorm_t(const qd_layernorm_desc& d, cudaStream_t s) {
  const int wpb = 8;
  launch_k(qd::layernorm_quant_kernel<NVEC>, grid_for((long long)d.M * 32, wpb * 32, 8), wpb * 32, 0, s, d);
  return check_launch("layernorm_quant_kernel");
}

int validate_layernorm(const qd_layernorm_desc& d) {
  if (!d.x || !d.gamma || !d.beta || d.M <= 0) return fail(QD_ERR_BAD_ARG, "layernorm: null arg or M <= 0");
  if (d.C <= 0 || d.C % 4 || d.ld_x % 4) return fail(QD_ERR_UNSUPPORTED, "layernorm: C=%d", d.C);
  if (d.C > 2048) return fail(QD_ERR_UNSUPPORTED, "layernorm: C=%d exceeds 2048", d.C);
  if (d.n_out < 0 || d.n_out > 3 || (d.n_out == 0 && !d.out_f)) return fail(QD_ERR_BAD_ARG, "layernorm: n_out");
  if (d.out_f && (d.ld_f & 3)) return fail(QD_ERR_UNSUPPORTED, "layernorm: ld_f");
  // float4 loads of x, gamma, beta; float4 stores of out_f; 32-bit stores of four codes
  if (!aligned(d.x, 16) || !aligned(d.gamma, 16) || !aligned(d.beta, 16) || (d.out_f && !aligned(d.out_f, 16)))
    return fail(QD_ERR_UNSUPPORTED, "layernorm: x, gamma, beta and out_f must be 16-byte aligned");
  for (int o = 0; o < d.n_out; ++o)
    if (!d.out_q[o] || !aligned(d.out_q[o], 4) || (d.ld_q[o] & 3))
      return fail(QD_ERR_UNSUPPORTED, "layernorm: out_q[%d] needs 4-byte alignment and ld_q %% 4 == 0", o);
  return QD_OK;
}

int launch_layernorm(const qd_layernorm_desc& d, cudaStream_t s) {
  if (int rc = validate_layernorm(d)) return rc;
  const int nvec = (d.C / 4 + 31) / 32;
  switch (nvec) {
    case 1: return launch_layernorm_t<1>(d, s);
    case 2: return launch_layernorm_t<2>(d, s);
    case 3: return launch_layernorm_t<3>(d, s);
    case 4: return launch_layernorm_t<4>(d, s);
    case 5: return launch_layernorm_t<5>(d, s);
    case 6: case 7: case 8: return launch_layernorm_t<8>(d, s);
    case 9: case 10: return launch_layernorm_t<10>(d, s);
    case 11: case 12: case 13: case 14: case 15: case 16: return launch_layernorm_t<16>(d, s);
    default: return fail(QD_ERR_UNSUPPORTED, "layernorm: C=%d exceeds 2048", d.C);
  }
}

// the vector kernel loads float4 and stores four bfloat16 per plane as one 8-byte word
bool split_vec(const qd_split_desc& d) {
  return !(d.C & 3) && !(d.ld_src & 3) && aligned(d.src, 16) && aligned(d.dst, 8);
}

int validate_split3(const qd_split_desc& d) {
  if (!d.src || !d.dst || d.M <= 0 || d.C <= 0) return fail(QD_ERR_BAD_ARG, "split: bad args");
  if (d.act < 0 || d.act > 3) return fail(QD_ERR_BAD_ARG, "split: act %d", d.act);
  if ((d.Cp & 3) || d.Cp < d.C || d.ld_dst < 3LL * d.Cp || (d.ld_dst & 3))
    return fail(QD_ERR_UNSUPPORTED, "split: Cp=%d must be a multiple of 4, >= C, with ld_dst >= 3*Cp", d.Cp);
  if (!aligned(d.src, 4) || !aligned(d.dst, 2)) return fail(QD_ERR_UNSUPPORTED, "split: src / dst misaligned for their types");
  if (d.upsample2x && !split_vec(d))
    return fail(QD_ERR_UNSUPPORTED, "split: upsample needs C, ld_src %% 4 == 0, src 16-byte and dst 8-byte aligned");
  return QD_OK;
}

int launch_split3(const qd_split_desc& d, cudaStream_t s) {
  if (int rc = validate_split3(d)) return rc;
  if (!split_vec(d)) {
    launch_k(qd::split_bf16x3_scalar_kernel, grid_for((long long)d.M * d.C, 256), 256, 0, s, d);
    return check_launch("split_bf16x3_scalar_kernel");
  }
  const long long rows = d.upsample2x ? (long long)d.B * 4 * d.H * d.W : d.M;
  launch_k(qd::split_bf16x3_kernel, grid_for(rows * (d.C / 4), 256), 256, 0, s, d);
  return check_launch("split_bf16x3_kernel");
}

// long sequences (never causal: the text encoder's T = 77 takes the one-row kernel): AFP_R query rows per block share the
// K / V rows they read (K/V traffic / AFP_R).  Its phase 1 reads K as float4.
size_t afp_rows_smem(const qd_attention_fp_desc& d) {
  return (size_t)qd::AFP_R * (d.d + qd::afp_tk_pitch(d.Tk)) * sizeof(float);
}
bool afp_rows(const qd_attention_fp_desc& d) {
  const bool vec = !(d.d & 3) && !(d.ld_q & 3) && !(d.ld_k & 3) && !(d.q_off & 3) && !(d.k_off & 3) && !(d.head_stride_q & 3) &&
                   !(d.head_stride_k & 3) && aligned(d.q, 16) && aligned(d.k, 16);
  return !d.causal && d.Tq >= 256 && afp_rows_smem(d) <= 200 * 1024 && vec;
}

int validate_attention_fp(const qd_attention_fp_desc& d) {
  if (!d.q || !d.k || !d.v || !d.out || d.B <= 0 || d.heads <= 0 || d.d <= 0 || d.Tq <= 0 || d.Tk <= 0)
    return fail(QD_ERR_BAD_ARG, "attention_fp32: bad args");
  if (d.causal != 0 && d.causal != 1) return fail(QD_ERR_BAD_ARG, "attention_fp32: causal must be 0 or 1 (got %d)", d.causal);
  if (d.causal && d.Tq != d.Tk) return fail(QD_ERR_UNSUPPORTED, "attention_fp32: causal needs Tq == Tk (got %d, %d)", d.Tq, d.Tk);
  if (!aligned(d.q, 4) || !aligned(d.k, 4) || !aligned(d.v, 4) || !aligned(d.out, 4))
    return fail(QD_ERR_UNSUPPORTED, "attention_fp32: q, k, v and out must be 4-byte aligned");
  if (!afp_rows(d) && (size_t)(d.d + d.Tk) * sizeof(float) > 48 * 1024)
    return fail(QD_ERR_UNSUPPORTED, "attention_fp32: d + Tk = %d exceeds 12288 floats of shared memory", d.d + d.Tk);
  return QD_OK;
}

int launch_attention_fp(const qd_attention_fp_desc& d, cudaStream_t s) {
  if (int rc = validate_attention_fp(d)) return rc;
  if (afp_rows(d)) {
    static std::atomic<unsigned long long> optin{0};
    if (int rc = ensure_smem_optin(qd::attention_fp32_rows_kernel, 200 * 1024, optin, "attention_fp32_rows")) return rc;
    launch_k(qd::attention_fp32_rows_kernel, dim3((d.Tq + qd::AFP_R - 1) / qd::AFP_R, d.B * d.heads), 256, afp_rows_smem(d), s, d);
    return check_launch("attention_fp32_rows_kernel");
  }
  // the dynamic score row may take the whole default 48 KB: the kernel's static reduction slots come on top, which needs
  // the opt-in (without it d + Tk = 12288 failed to launch)
  static std::atomic<unsigned long long> optin1{0};
  if (int rc = ensure_smem_optin(qd::attention_fp32_kernel, 48 * 1024, optin1, "attention_fp32")) return rc;
  const size_t smem = (size_t)(d.d + d.Tk) * sizeof(float);
  launch_k(qd::attention_fp32_kernel, dim3(d.Tq, d.B * d.heads), 128, smem, s, d);
  return check_launch("attention_fp32_kernel");
}

int validate_embed(const qd_embed_desc& d) {
  if (!d.ids || !d.tok || !d.pos || !d.out || d.B <= 0 || d.T <= 0 || d.C <= 0 || d.vocab <= 0 || d.ld_out < d.C)
    return fail(QD_ERR_BAD_ARG, "embed_tokens: bad args (B=%d T=%d C=%d vocab=%d ld_out=%lld)", d.B, d.T, d.C, d.vocab, d.ld_out);
  if (!aligned(d.ids, 4) || !aligned(d.tok, 4) || !aligned(d.pos, 4) || !aligned(d.out, 4))
    return fail(QD_ERR_UNSUPPORTED, "embed_tokens: ids, tok, pos and out must be 4-byte aligned");
  return QD_OK;
}

int launch_embed(const qd_embed_desc& d, cudaStream_t s) {
  if (int rc = validate_embed(d)) return rc;
  launch_k(qd::embed_tokens_kernel, grid_for((long long)d.B * d.T * d.C, 256), 256, 0, s, d);
  return check_launch("embed_tokens_kernel");
}

// 16 channels of one tap per thread: uint4 loads and stores
bool im2col_vec(const qd_im2col_desc& d) {
  return (d.C % 16) == 0 && d.ld_dst == 9 * d.C && (d.ld_dst % 16) == 0 && aligned(d.src, 16) && aligned(d.dst, 16);
}

int validate_im2col(const qd_im2col_desc& d) {
  if (!d.src || !d.dst) return fail(QD_ERR_BAD_ARG, "im2col: null arg");
  if (d.B <= 0 || d.H <= 0 || d.W <= 0 || d.C <= 0 || d.Ho <= 0 || d.Wo <= 0 || d.stride <= 0)
    return fail(QD_ERR_BAD_ARG, "im2col: empty geometry");
  if (d.ld_dst < 9 * d.C) return fail(QD_ERR_BAD_ARG, "im2col: ld_dst too small");
  return QD_OK;
}

int launch_im2col(const qd_im2col_desc& d, cudaStream_t s) {
  if (int rc = validate_im2col(d)) return rc;
  if (im2col_vec(d)) {
    launch_k(qd::im2col_vec_kernel, grid_for((long long)d.B * d.Ho * d.Wo * 9 * (d.C / 16), 256), 256, 0, s, d);
    return check_launch("im2col_vec_kernel");
  }
  const long long total = (long long)d.B * d.Ho * d.Wo * d.ld_dst;
  launch_k(qd::im2col_kernel, grid_for(total, 256), 256, 0, s, d);
  return check_launch("im2col_kernel");
}

template <int DQ, int DV, bool QS, bool VS, bool S16, bool F16>
int launch_attention_inst(const qd_attention_desc& d, cudaStream_t s) {
  constexpr int MINB = (DV <= 48) ? 2 : 1;
  auto kern = qd::qattention_kernel<DQ, DV, QS, VS, S16, MINB, F16>;
  static std::atomic<unsigned long long> optin{0};
  if (int rc = ensure_smem_optin(kern, 200 * 1024, optin, "attention")) return rc;
  const bool zrk = !F16 && d.zq != 0;      // fp16 centred operands carry no zero-point cross term
  const qd::AttSmemLayout lay = qd::att_smem_layout(DQ, DV, d.Tk, zrk);
  if (lay.total > 200 * 1024) return fail(QD_ERR_UNSUPPORTED, "attention: Tk=%d needs %d B of shared memory", d.Tk, lay.total);
  if (zrk) {
    if (!d.ws) return fail(QD_ERR_BAD_ARG, "attention: workspace required when zq != 0");
    const int tk_pad = qd::att_ws_stride(d.Tk);
    launch_k(qd::att_krowsum_kernel<QS>, grid_for((long long)d.B * d.heads * tk_pad, 256), 256, 0, s, d, tk_pad, 0, 0);
    int rc = check_launch("att_krowsum_kernel");
    if (rc) return rc;
  }
  dim3 grid((d.Tq + qd::ATT_BM - 1) / qd::ATT_BM, d.B * d.heads);
  launch_k(kern, grid, qd::ATT_WARPS * 32, lay.total, s, d);
  return check_launch("qattention_kernel");
}

// DQ: bytes of the padded QK^T reduction (8-bit codes: d rounded up to 32; F16: 2 d rounded up to 32)
template <int DQ, int DV, bool F16 = false>
int launch_attention_t(const qd_attention_desc& d, cudaStream_t s) {
  const bool qs = d.q_signed != 0, vs = d.v_signed != 0, s16 = d.sm_bits > 8;
  if (qs && vs && s16) return launch_attention_inst<DQ, DV, true, true, true, F16>(d, s);
  if (qs && vs && !s16) return launch_attention_inst<DQ, DV, true, true, false, F16>(d, s);
  if (!qs && !vs && s16) return launch_attention_inst<DQ, DV, false, false, true, F16>(d, s);
  if (!qs && !vs && !s16) return launch_attention_inst<DQ, DV, false, false, false, F16>(d, s);
  return fail(QD_ERR_UNSUPPORTED, "attention: mixed signedness q=%d v=%d", d.q_signed, d.v_signed);
}

// small-Tk path (cross-attention): one key tile, K/V staged once per CTA, single-pass softmax
template <int DQ, int DV, bool QS, bool VS, bool S16>
int launch_attention_smallk_inst(const qd_attention_desc& d, cudaStream_t s) {
  constexpr int NKV = 3;
  auto kern = qd::qattention_smallk_kernel<DQ, DV, QS, VS, S16, NKV>;
  const int spw = d.Tq >= 2048 ? 4 : (d.Tq >= 512 ? 2 : 1);
  const int slabs = (d.Tq + 15) / 16;
  dim3 grid((slabs + spw * qd::ATS_WARPS - 1) / (spw * qd::ATS_WARPS), d.B * d.heads);
  launch_k(kern, grid, qd::ATS_WARPS * 32, qd::ats_smem_bytes<DQ, DV, NKV>(), s, d, spw);
  return check_launch("qattention_smallk_kernel");
}

template <int DQ, int DV>
int launch_attention_smallk(const qd_attention_desc& d, cudaStream_t s) {
  const bool qs = d.q_signed != 0, vs = d.v_signed != 0, s16 = d.sm_bits > 8;
  if (qs && vs && s16) return launch_attention_smallk_inst<DQ, DV, true, true, true>(d, s);
  if (qs && vs && !s16) return launch_attention_smallk_inst<DQ, DV, true, true, false>(d, s);
  if (!qs && !vs && s16) return launch_attention_smallk_inst<DQ, DV, false, false, true>(d, s);
  if (!qs && !vs && !s16) return launch_attention_smallk_inst<DQ, DV, false, false, false>(d, s);
  return fail(QD_ERR_UNSUPPORTED, "attention: mixed signedness q=%d v=%d", d.q_signed, d.v_signed);
}

// ---- wgmma attention (attention_wg.cuh): Q / K in the per-head padded layout (pitch P = 32 / 64 / 128 bytes, the K tile's
// TMA box and swizzle span), dense V^T; d in {16, 24, 32, 40, 48, 64, 80, 96} (fp16 Q / K: d <= 64)
bool attention_wg_eligible(const qd_attention_desc& d) {
  static const int forced_mma = [] { const char* e = getenv("QDIFF_ATTENTION"); return (e && !strcmp(e, "mma")) ? 1 : 0; }();
  if (forced_mma) return false;     // QDIFF_ATTENTION=mma: the mma.sync kernel (A/B comparisons)
  const int P = d.head_stride_q, rb = d.qk_f16 ? 2 * d.d : d.d;
  if (d.d != 16 && d.d != 24 && d.d != 32 && d.d != 40 && d.d != 48 && d.d != 64 && d.d != 80 && d.d != 96) return false;
  if (d.qk_f16 && d.d > 64) return false;
  if ((P != 32 && P != 64 && P != 128) || P < rb || d.head_stride_k != P) return false;
  if (d.q_off != 0 || d.k_off != 0 || (d.ld_k & 15) || (((uintptr_t)d.k) & 15) || (((uintptr_t)d.vt) & 15)) return false;
  if (d.v_off != 0 || d.head_stride_v != d.d || d.v_batch_stride != (long long)d.heads * d.d * d.ld_vt) return false;
  if (d.zq != 0 && !d.qk_f16 && !d.ws) return false;
  // 8-bit codes: the kernel converts zq * rowsum(k) to fp32 by a magic-number add, exact for zero points of the code range
  if (!d.qk_f16 && (d.zq > 255 || d.zq < (d.q_signed ? -255 : 0))) return false;
  return true;
}

template <int DQ, int DV, bool QS, bool VS, bool S16, bool F16>
int launch_attention_wg_inst(const qd_attention_desc& d, cudaStream_t s) {
  // d <= 40 fits 128 registers without spills: two CTAs per SM (DESIGN §6); larger d would spill there
  constexpr int MINB = DV <= 40 ? 2 : 1;
  auto kern = qd::qattention_wg_kernel<DQ, DV, QS, VS, S16, F16, MINB>;
  const int P = d.head_stride_q;
  const qd::AtwSmem lay = qd::atw_smem(P, qd::atw_nv(DV));
  static std::atomic<unsigned long long> optin{0};
  if (int rc = ensure_smem_optin(kern, 227 * 1024, optin, "attention_wg")) return rc;
  CUtensorMap tmK, tmV;
  {
    cuuint64_t dims[2] = {(cuuint64_t)d.ld_k, (cuuint64_t)d.B * d.Tk};
    cuuint64_t strides[1] = {(cuuint64_t)d.ld_k};
    cuuint32_t box[2] = {(cuuint32_t)P, (cuuint32_t)qd::ATT_BN};
    if (int rc = encode_u8_map(&tmK, d.k, 2, dims, strides, box, P)) return rc;
  }
  {
    cuuint64_t dims[2] = {(cuuint64_t)d.ld_vt, (cuuint64_t)d.B * d.heads * d.d};
    cuuint64_t strides[1] = {(cuuint64_t)d.ld_vt};
    cuuint32_t box[2] = {(cuuint32_t)qd::ATT_BN, (cuuint32_t)d.d};
    if (int rc = encode_u8_map(&tmV, d.vt, 2, dims, strides, box, 64)) return rc;
  }
  if (!F16 && d.zq != 0) {
    const int tk_pad = qd::att_ws_stride(d.Tk);
    launch_k(qd::att_krowsum_kernel<QS>, grid_for((long long)d.B * d.heads * tk_pad, 256), 256, 0, s, d, tk_pad, 0, 0);
    if (int rc = check_launch("att_krowsum_kernel")) return rc;
  }
  dim3 grid((d.Tq + qd::ATT_BM - 1) / qd::ATT_BM, d.B * d.heads);
  launch_k(kern, grid, qd::ATW_THREADS, lay.total, s, tmK, tmV, d, P);
  return check_launch("qattention_wg_kernel");
}

template <int DQ, int DV, bool F16>
int launch_attention_wg_t(const qd_attention_desc& d, cudaStream_t s) {
  const bool qs = d.q_signed != 0, vs = d.v_signed != 0, s16 = d.sm_bits > 8;
  if (qs && vs && s16) return launch_attention_wg_inst<DQ, DV, true, true, true, F16>(d, s);
  if (qs && vs && !s16) return launch_attention_wg_inst<DQ, DV, true, true, false, F16>(d, s);
  if (!qs && !vs && s16) return launch_attention_wg_inst<DQ, DV, false, false, true, F16>(d, s);
  if (!qs && !vs && !s16) return launch_attention_wg_inst<DQ, DV, false, false, false, F16>(d, s);
  return fail(QD_ERR_UNSUPPORTED, "attention: mixed signedness q=%d v=%d", d.q_signed, d.v_signed);
}

int launch_attention_wg(const qd_attention_desc& d, cudaStream_t s) {
  if (d.qk_f16) {
    switch (d.d) {
      case 16: return launch_attention_wg_t<32, 16, true>(d, s);
      case 24: return launch_attention_wg_t<64, 24, true>(d, s);
      case 32: return launch_attention_wg_t<64, 32, true>(d, s);
      case 40: return launch_attention_wg_t<96, 40, true>(d, s);
      case 48: return launch_attention_wg_t<96, 48, true>(d, s);
      default: return launch_attention_wg_t<128, 64, true>(d, s);
    }
  }
  switch (d.d) {
    case 16: return launch_attention_wg_t<32, 16, false>(d, s);
    case 24: return launch_attention_wg_t<32, 24, false>(d, s);
    case 32: return launch_attention_wg_t<32, 32, false>(d, s);
    case 40: return launch_attention_wg_t<64, 40, false>(d, s);
    case 48: return launch_attention_wg_t<64, 48, false>(d, s);
    case 64: return launch_attention_wg_t<64, 64, false>(d, s);
    case 80: return launch_attention_wg_t<96, 80, false>(d, s);
    default: return launch_attention_wg_t<96, 96, false>(d, s);
  }
}

int validate_attention(const qd_attention_desc& d) {
  if (!d.q || !d.k || !d.vt || (!d.out && !d.out_q)) return fail(QD_ERR_BAD_ARG, "attention: null arg");
  if (d.out_q && (d.ld_out_q & 1)) return fail(QD_ERR_UNSUPPORTED, "attention: ld_out_q");
  if (d.q_signed != d.k_signed) return fail(QD_ERR_UNSUPPORTED, "attention: q/k signedness differ");
  if (d.zw != 0) return fail(QD_ERR_UNSUPPORTED, "attention: softmax zero point must be 0 (got %d)", d.zw);
  if (d.sm_bits != 8 && d.sm_bits != 16) return fail(QD_ERR_UNSUPPORTED, "attention: sm_bits %d", d.sm_bits);
  // Keys beyond Tk get the score att_mask (attention.cuh).  On int32 scores at d > 64 that is INT_MIN, whose exponent lies
  // at least (2^31 - 255^2 d) * c below the row maximum's: ex2 flushes it to 0 once that exceeds 127 plus log2(1 / delta_w).
  if (!(d.sim_scale > 0.f)) return fail(QD_ERR_UNSUPPORTED, "attention: sim_scale must be positive (got %g)", d.sim_scale);
  if (!d.qk_f16 && d.d > 64 &&
      (2147483648.0 - 65025.0 * d.d) * d.sim_scale * 1.4426950408889634 < 128.0 + fmax(0.0, -log2((double)d.delta_w)))
    return fail(QD_ERR_UNSUPPORTED, "attention: sim_scale %g too small to mask the keys beyond Tk at d = %d", d.sim_scale, d.d);
  if (d.ld_vt % 16 || d.ld_vt < d.Tk) return fail(QD_ERR_BAD_ARG, "attention: ld_vt");
  if ((d.q_off | d.head_stride_q | (int)d.ld_q) & 3) return fail(QD_ERR_UNSUPPORTED, "attention: q needs 4-byte alignment");
  if ((d.k_off | d.head_stride_k | (int)d.ld_k | d.d) & 7) return fail(QD_ERR_UNSUPPORTED, "attention: k rows need 8-byte alignment");
  if (d.out && (d.ld_out % 2)) return fail(QD_ERR_UNSUPPORTED, "attention: ld_out");
  return QD_OK;
}

int launch_attention(const qd_attention_desc& d, cudaStream_t s) {
  if (int rc = validate_attention(d)) return rc;
  if (d.qk_f16) {      // fp16 centred-code Q / K (QK^T on f16 x f16 -> f32 MMAs, exact), d <= 64, any Tk
    if (attention_wg_eligible(d)) return launch_attention_wg(d, s);
    switch (d.d) {
      case 16: return launch_attention_t<32, 16, true>(d, s);
      case 24: return launch_attention_t<64, 24, true>(d, s);
      case 32: return launch_attention_t<64, 32, true>(d, s);
      case 40: return launch_attention_t<96, 40, true>(d, s);
      case 48: return launch_attention_t<96, 48, true>(d, s);
      case 64: return launch_attention_t<128, 64, true>(d, s);
      default: return fail(QD_ERR_UNSUPPORTED, "attention: qk_f16 needs d in {16, 24, 32, 40, 48, 64} (got %d)", d.d);
    }
  }
  if (d.Tk <= 96 && (d.d == 40 || d.d == 80)) {
    static const bool off = [] { const char* e = getenv("QDIFF_ATTENTION"); return e && !strcmp(e, "nosmallk"); }();
    if (!off) return d.d == 40 ? launch_attention_smallk<64, 40>(d, s) : launch_attention_smallk<96, 80>(d, s);
  }
  if (attention_wg_eligible(d)) return launch_attention_wg(d, s);
  switch (d.d) {
    case 16: return launch_attention_t<32, 16>(d, s);
    case 24: return launch_attention_t<32, 24>(d, s);
    case 32: return launch_attention_t<32, 32>(d, s);
    case 40: return launch_attention_t<64, 40>(d, s);
    case 48: return launch_attention_t<64, 48>(d, s);
    case 64: return launch_attention_t<64, 64>(d, s);
    case 80: return launch_attention_t<96, 80>(d, s);
    case 96: return launch_attention_t<96, 96>(d, s);
    case 160: return launch_attention_t<160, 160>(d, s);
    case 256: return launch_attention_t<256, 256>(d, s);
    default: return fail(QD_ERR_UNSUPPORTED, "attention: head dim %d not instantiated", d.d);
  }
}

int validate_misc(int kind, const qd_misc_desc& m) {
  if (!m.src || !m.dst) return fail(QD_ERR_BAD_ARG, "misc %d: null src / dst", kind);
  if (!aligned(m.src, 4) || !aligned(m.dst, 4)) return fail(QD_ERR_UNSUPPORTED, "misc %d: src / dst must be 4-byte aligned", kind);
  switch (kind) {
    case QD_OP_TIMESTEP_EMB:
      if (!m.aux) return fail(QD_ERR_BAD_ARG, "timestep_embedding: missing frequency table");
      return QD_OK;
    case QD_OP_COPY2D:      // float4 rows
      if (m.b % 4 || m.ld_src % 4 || m.ld_dst % 4 || !aligned(m.src, 16) || !aligned(m.dst, 16))
        return fail(QD_ERR_UNSUPPORTED, "copy2d: C, ld_src, ld_dst %% 4 == 0 and 16-byte aligned src / dst");
      return QD_OK;
    case QD_OP_NCHW_TO_NHWC:
    case QD_OP_NHWC_TO_NCHW:
      return QD_OK;
    case QD_OP_AVGPOOL2X:   // float4 channel quads
    case QD_OP_UPSAMPLE2X:
      if (m.d % 4 || !aligned(m.src, 16) || !aligned(m.dst, 16))
        return fail(QD_ERR_UNSUPPORTED, "%s: C %% 4 == 0 and 16-byte aligned src / dst", kind == QD_OP_AVGPOOL2X ? "avgpool" : "upsample");
      return QD_OK;
    case QD_OP_SOFTMAX_ROWS:
      if (m.a <= 0 || m.b <= 0 || m.ld_src < m.b || m.src != m.dst) return fail(QD_ERR_BAD_ARG, "softmax_rows: in place, rows=%d cols=%d", m.a, m.b);
      return QD_OK;
    case QD_OP_VQ_LOOKUP:
      if (!m.aux || m.a <= 0 || m.b <= 0 || m.b > qd::VQ_MAX_C || m.c <= 0 || m.ld_src < m.b || m.ld_dst < m.b)
        return fail(QD_ERR_BAD_ARG, "vq_lookup: bad args (rows=%d, C=%d <= %d, n_e=%d)", m.a, m.b, qd::VQ_MAX_C, m.c);
      if (!aligned(m.aux, 4)) return fail(QD_ERR_UNSUPPORTED, "vq_lookup: codebook must be 4-byte aligned");
      return QD_OK;
    default:
      return fail(QD_ERR_BAD_ARG, "misc: unknown kind %d", kind);
  }
}

int launch_misc(int kind, const qd_misc_desc& m, cudaStream_t s) {
  if (int rc = validate_misc(kind, m)) return rc;
  switch (kind) {
    case QD_OP_TIMESTEP_EMB:
      launch_k(qd::timestep_embedding_kernel, grid_for((long long)m.a * (m.b / 2), 128), 128, 0, s, m.src, m.aux, m.a, m.b, m.c, m.dst);
      return check_launch("timestep_embedding_kernel");
    case QD_OP_COPY2D:
      launch_k(qd::copy2d_kernel, grid_for((long long)m.a * (m.b / 4), 256), 256, 0, s, m.src, m.ld_src, m.dst, m.ld_dst, m.a, m.b);
      return check_launch("copy2d_kernel");
    case QD_OP_NCHW_TO_NHWC:
      launch_k(qd::nchw_to_nhwc_kernel, grid_for((long long)m.a * m.b * m.c, 256), 256, 0, s, m.src, m.dst, m.a, m.b, m.c);
      return check_launch("nchw_to_nhwc_kernel");
    case QD_OP_NHWC_TO_NCHW:
      launch_k(qd::nhwc_to_nchw_kernel, grid_for((long long)m.a * m.b * m.c, 256), 256, 0, s, m.src, m.dst, m.a, m.b, m.c);
      return check_launch("nhwc_to_nchw_kernel");
    case QD_OP_AVGPOOL2X:
      launch_k(qd::avgpool2x_kernel, grid_for((long long)m.a * (m.b / 2) * (m.c / 2) * (m.d / 4), 256), 256, 0, s, m.src, m.dst, m.a, m.b, m.c, m.d);
      return check_launch("avgpool2x_kernel");
    case QD_OP_UPSAMPLE2X:
      launch_k(qd::upsample2x_f32_kernel, grid_for((long long)m.a * m.b * m.c * m.d, 256), 256, 0, s, m.src, m.dst, m.a, m.b, m.c, m.d);
      return check_launch("upsample2x_f32_kernel");
    case QD_OP_SOFTMAX_ROWS:
      launch_k(qd::softmax_rows_kernel, dim3(m.a), 256, 0, s, m.dst, m.ld_src, m.b);
      return check_launch("softmax_rows_kernel");
    case QD_OP_VQ_LOOKUP:
      launch_k(qd::vq_lookup_kernel, grid_for((long long)m.a * 32, 256), 256, 0, s, m.src, m.ld_src, m.aux, m.dst, m.ld_dst, m.a, m.b, m.c);
      return check_launch("vq_lookup_kernel");
    default:
      return fail(QD_ERR_BAD_ARG, "misc: unknown kind %d", kind);
  }
}

struct Op {
  int kind;
  GemmPlan gemm;
  union {
    qd_quantize_desc quant;
    qd_groupnorm_desc gn;
    qd_layernorm_desc ln;
    qd_im2col_desc im2col;
    qd_attention_desc att;
    qd_misc_desc misc;
    qd_split_desc split;
    qd_attention_fp_desc attfp;
    qd_embed_desc embed;
  };
  Op() : kind(0) { memset(&gemm, 0, sizeof(gemm)); memset(&gn, 0, sizeof(gn)); }
};

int run_op(const Op& op, cudaStream_t s) {
  switch (op.kind) {
    case QD_OP_GEMM: return launch_gemm(op.gemm, s);
    case QD_OP_QUANTIZE: return launch_quantize(op.quant, s);
    case QD_OP_GROUPNORM: return launch_groupnorm(op.gn, s);
    case QD_OP_LAYERNORM: return launch_layernorm(op.ln, s);
    case QD_OP_IM2COL: return launch_im2col(op.im2col, s);
    case QD_OP_ATTENTION: return launch_attention(op.att, s);
    case QD_OP_SPLIT3: return launch_split3(op.split, s);
    case QD_OP_ATTENTION_FP: return launch_attention_fp(op.attfp, s);
    case QD_OP_EMBED: return launch_embed(op.embed, s);
    default: return launch_misc(op.kind, op.misc, s);
  }
}

}  // namespace

struct qd_engine {
  int device;
  bool finalized;
  std::vector<Op> ops;
};

extern "C" {

const char* qd_last_error(void) { return g_err; }
int qd_num_sms(void) { return num_sms(); }
long long qd_launch_count(void) { return g_launches.load(); }

int qd_qgemm_i8(const qd_gemm_desc* d, qd_stream_t stream) {
  GemmPlan pl;
  int rc = plan_gemm(d, &pl);
  if (rc) return rc;
  return launch_gemm(pl, (cudaStream_t)stream);
}
int qd_quantize(const qd_quantize_desc* d, qd_stream_t s) {
  if (!d) return fail(QD_ERR_BAD_ARG, "null desc");
  return launch_quantize(*d, (cudaStream_t)s);
}
long long qd_groupnorm_workspace_floats(int B, int HW, int C, int groups) {
  if (B <= 0 || HW <= 0 || C <= 0 || groups <= 0) return 0;
  return gn_workspace_floats(B, HW, C, groups);
}

int qd_groupnorm_quant(const qd_groupnorm_desc* d, qd_stream_t s) {
  if (!d) return fail(QD_ERR_BAD_ARG, "null desc");
  return launch_groupnorm(*d, (cudaStream_t)s);
}
int qd_layernorm_quant(const qd_layernorm_desc* d, qd_stream_t s) {
  if (!d) return fail(QD_ERR_BAD_ARG, "null desc");
  return launch_layernorm(*d, (cudaStream_t)s);
}
int qd_im2col_i8(const qd_im2col_desc* d, qd_stream_t s) {
  if (!d) return fail(QD_ERR_BAD_ARG, "null desc");
  return launch_im2col(*d, (cudaStream_t)s);
}
int qd_qattention(const qd_attention_desc* d, qd_stream_t s) {
  if (!d) return fail(QD_ERR_BAD_ARG, "null desc");
  return launch_attention(*d, (cudaStream_t)s);
}
int qd_lincomb3(float* out, float a, const float* x, float b, const float* y, float c, const float* z, long long n,
                qd_stream_t s) {
  if (!out || !x || n <= 0) return fail(QD_ERR_BAD_ARG, "lincomb3: bad args");
  launch_k(qd::lincomb3_kernel, grid_for(n, 256), 256, 0, (cudaStream_t)s, out, a, x, b, y, c, z, n);
  return check_launch("lincomb3_kernel");
}
int qd_split_bf16x3(const qd_split_desc* d, qd_stream_t s) {
  if (!d) return fail(QD_ERR_BAD_ARG, "null desc");
  return launch_split3(*d, (cudaStream_t)s);
}
int qd_attention_fp32(const qd_attention_fp_desc* d, qd_stream_t s) {
  if (!d) return fail(QD_ERR_BAD_ARG, "null desc");
  return launch_attention_fp(*d, (cudaStream_t)s);
}
int qd_embed_tokens(const qd_embed_desc* d, qd_stream_t s) {
  if (!d) return fail(QD_ERR_BAD_ARG, "null desc");
  return launch_embed(*d, (cudaStream_t)s);
}
int qd_timestep_embedding(const float* t, const float* freqs, int32_t B, int32_t dim, int32_t mode, float* out,
                          qd_stream_t s) {
  qd_misc_desc m{t, out, 0, 0, B, dim, mode, 0, freqs};
  return launch_misc(QD_OP_TIMESTEP_EMB, m, (cudaStream_t)s);
}
int qd_copy2d(const float* src, long long ld_src, float* dst, long long ld_dst, int32_t M, int32_t C, qd_stream_t s) {
  qd_misc_desc m{src, dst, ld_src, ld_dst, M, C, 0, 0, nullptr};
  return launch_misc(QD_OP_COPY2D, m, (cudaStream_t)s);
}
int qd_nchw_to_nhwc(const float* src, float* dst, int32_t B, int32_t C, int32_t HW, qd_stream_t s) {
  qd_misc_desc m{src, dst, 0, 0, B, C, HW, 0, nullptr};
  return launch_misc(QD_OP_NCHW_TO_NHWC, m, (cudaStream_t)s);
}
int qd_nhwc_to_nchw(const float* src, float* dst, int32_t B, int32_t C, int32_t HW, qd_stream_t s) {
  qd_misc_desc m{src, dst, 0, 0, B, C, HW, 0, nullptr};
  return launch_misc(QD_OP_NHWC_TO_NCHW, m, (cudaStream_t)s);
}
int qd_avgpool2x(const float* src, float* dst, int32_t B, int32_t H, int32_t W, int32_t C, qd_stream_t s) {
  qd_misc_desc m{src, dst, 0, 0, B, H, W, C, nullptr};
  return launch_misc(QD_OP_AVGPOOL2X, m, (cudaStream_t)s);
}
int qd_upsample2x_f32(const float* src, float* dst, int32_t B, int32_t H, int32_t W, int32_t C, qd_stream_t s) {
  qd_misc_desc m{src, dst, 0, 0, B, H, W, C, nullptr};
  return launch_misc(QD_OP_UPSAMPLE2X, m, (cudaStream_t)s);
}
int qd_softmax_rows(float* x, long long ld, int32_t rows, int32_t cols, qd_stream_t s) {
  qd_misc_desc m{x, x, ld, ld, rows, cols, 0, 0, nullptr};
  return launch_misc(QD_OP_SOFTMAX_ROWS, m, (cudaStream_t)s);
}
int qd_vq_lookup(const float* z, long long ld_z, const float* codebook, float* out, long long ld_out, int32_t rows, int32_t C,
                 int32_t n_e, qd_stream_t s) {
  qd_misc_desc m{z, out, ld_z, ld_out, rows, C, n_e, 0, codebook};
  return launch_misc(QD_OP_VQ_LOOKUP, m, (cudaStream_t)s);
}
int qd_sampler_step(const qd_sampler_desc* d, qd_stream_t s) {
  if (!d || !d->x || !d->eps || !d->x_prev || d->n <= 0) return fail(QD_ERR_BAD_ARG, "sampler: bad args");
  launch_k(qd::sampler_step_kernel, grid_for(d->n, 256), 256, 0, (cudaStream_t)s, *d);
  return check_launch("sampler_step_kernel");
}
int qd_ancestral_step(const qd_ancestral_desc* d, qd_stream_t s) {
  if (!d || !d->x || !d->eps || !d->x_prev || d->n <= 0) return fail(QD_ERR_BAD_ARG, "ancestral: bad args");
  launch_k(qd::ancestral_step_kernel, grid_for(d->n, 256), 256, 0, (cudaStream_t)s, *d);
  return check_launch("ancestral_step_kernel");
}

int qd_engine_create(int device, qd_engine** out) {
  if (!out) return fail(QD_ERR_BAD_ARG, "null out");
  {
    DeviceGuard g(device);    // the caller's current device (and with it torch's current stream) is left untouched
    if (!g.ok) return fail(QD_ERR_CUDA, "cudaSetDevice(%d) failed: no CPU fallback", device);
    if (!num_sms()) return QD_ERR_CUDA;
  }
  qd_engine* e = new (std::nothrow) qd_engine();
  if (!e) return fail(QD_ERR_BAD_ARG, "out of host memory");
  e->device = device;
  e->finalized = false;
  *out = e;
  return QD_OK;
}

int qd_engine_add_op(qd_engine* e, int kind, const void* desc) {
  if (!e || !desc) return fail(QD_ERR_BAD_ARG, "null arg");
  DeviceGuard g(e->device);   // tile choice (SM count) and descriptors are planned for the engine's device
  if (!g.ok) return fail(QD_ERR_CUDA, "cudaSetDevice(%d) failed", e->device);
  Op op;
  op.kind = kind;
  int rc = QD_OK;
  switch (kind) {
    case QD_OP_GEMM: rc = plan_gemm(reinterpret_cast<const qd_gemm_desc*>(desc), &op.gemm); break;
    // the launchers' own checks, so that a descriptor the kernels cannot take is refused here and not at replay
    case QD_OP_QUANTIZE: op.quant = *reinterpret_cast<const qd_quantize_desc*>(desc); rc = validate_quantize(op.quant); break;
    case QD_OP_GROUPNORM: op.gn = *reinterpret_cast<const qd_groupnorm_desc*>(desc); rc = validate_groupnorm(op.gn); break;
    case QD_OP_LAYERNORM: op.ln = *reinterpret_cast<const qd_layernorm_desc*>(desc); rc = validate_layernorm(op.ln); break;
    case QD_OP_IM2COL: op.im2col = *reinterpret_cast<const qd_im2col_desc*>(desc); rc = validate_im2col(op.im2col); break;
    case QD_OP_ATTENTION: op.att = *reinterpret_cast<const qd_attention_desc*>(desc); rc = validate_attention(op.att); break;
    case QD_OP_SPLIT3: op.split = *reinterpret_cast<const qd_split_desc*>(desc); rc = validate_split3(op.split); break;
    case QD_OP_ATTENTION_FP:
      op.attfp = *reinterpret_cast<const qd_attention_fp_desc*>(desc);
      rc = validate_attention_fp(op.attfp);
      break;
    case QD_OP_EMBED: op.embed = *reinterpret_cast<const qd_embed_desc*>(desc); rc = validate_embed(op.embed); break;
    case QD_OP_TIMESTEP_EMB: case QD_OP_COPY2D: case QD_OP_NCHW_TO_NHWC: case QD_OP_NHWC_TO_NCHW:
    case QD_OP_AVGPOOL2X: case QD_OP_UPSAMPLE2X: case QD_OP_VQ_LOOKUP: case QD_OP_SOFTMAX_ROWS:
      op.misc = *reinterpret_cast<const qd_misc_desc*>(desc);
      rc = validate_misc(kind, op.misc);
      break;
    default: return fail(QD_ERR_BAD_ARG, "unknown op kind %d", kind);
  }
  if (rc) return rc;
  e->ops.push_back(op);
  e->finalized = false;
  return QD_OK;
}

int qd_engine_num_ops(const qd_engine* e) { return e ? (int)e->ops.size() : 0; }

int qd_engine_finalize(qd_engine* e) {
  if (!e) return fail(QD_ERR_BAD_ARG, "null engine");
  e->finalized = true;
  return QD_OK;
}

int qd_engine_run_range(qd_engine* e, int first, int last, qd_stream_t stream) {
  if (!e) return fail(QD_ERR_BAD_ARG, "null engine");
  if (!e->finalized) return fail(QD_ERR_NOT_FINALIZED, "engine not finalized");
  if (first < 0 || last > (int)e->ops.size() || first > last) return fail(QD_ERR_BAD_ARG, "bad op range");
  if (current_device() != e->device)
    return fail(QD_ERR_BAD_ARG, "engine was built for device %d but the current device is %d", e->device, current_device());
  for (int i = first; i < last; ++i) {
    int rc = run_op(e->ops[i], (cudaStream_t)stream);
    if (rc) return rc;
  }
  return QD_OK;
}
int qd_engine_run(qd_engine* e, qd_stream_t stream) {
  if (!e) return fail(QD_ERR_BAD_ARG, "null engine");
  return qd_engine_run_range(e, 0, (int)e->ops.size(), stream);
}
void qd_engine_destroy(qd_engine* e) { delete e; }

}  // extern "C"
