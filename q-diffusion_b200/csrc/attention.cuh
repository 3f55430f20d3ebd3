// Quantised attention core (SURVEY 2.2 K9): integer QK^T, fp32 softmax, re-quantised P, integer PV.
//   S_int[i,j] = sum_d (q[i,d]-zq)(k[j,d]-zk)         exact int32 (mma.sync m16n8k32 u8/s8)
//   P = softmax_j(S_int * sim_scale)                    fp32, two passes because the reference
//                                                       quantises P AFTER normalisation with a fixed
//                                                       calibrated step (qdiff/quant_block.py:217)
//   Pq = min(rne(P / delta_w), p_qmax)                  8- or 16-bit codes (zero point 0)
//   O[i,:] = out_scale * (sum_j Pq[i,j] v[j,:] - zv * sum_j Pq[i,j])
// 16-bit codes are contracted exactly as two byte planes (hi, lo) against the 8-bit V codes, both
// accumulated in int32 over the whole key range (exact: 255*255*Tk < 2^31 for Tk < 33k).
//
// v2 (this file): the kernel is bound by the per-score scalar work (two exp2 + conversions per score:
// MUFU 16/clk/SM and issue slots), not by the tensor pipe, so the design minimises instructions per score:
//   * exp2 domain with the row maximum taken on the INTEGER scores and the normalisation folded into
//     the exponent:  code = rni(exp2(S*c + (rowconst - max*c + log2(1/(l*delta_w)))))  (1 FFMA + 1 MUFU)
//   * row sums of P codes come out of the PV MMA through an all-ones extra V^T row (no per-score add)
//   * int32 O accumulators live across the whole pass (no per-tile conversion)
//   * K / V^T tiles stream through a cp.async double buffer, one __syncthreads per tile
//   * 8 warps x 16 query rows per CTA; the key permutation lets the S accumulator fragment feed the PV
//     A-operand without shuffles: MMA k-slot (4t+e) <-> key 8*(e>>1)+2t+(e&1) inside each 32-key chunk.
// Tensor path: mma.sync IMMA (register-resident P).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <type_traits>
#include "../../include/qdiff_b200.h"
#include "quant_math.cuh"

namespace qd {

template <bool A_SIGNED, bool B_SIGNED>
__device__ __forceinline__ void mma_i8_16832(int (&c)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  if constexpr (A_SIGNED && B_SIGNED) {
    asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.s8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+r"(c[0]), "+r"(c[1]), "+r"(c[2]), "+r"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
  } else if constexpr (A_SIGNED && !B_SIGNED) {
    asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.s8.u8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+r"(c[0]), "+r"(c[1]), "+r"(c[2]), "+r"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
  } else if constexpr (!A_SIGNED && B_SIGNED) {
    asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.u8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+r"(c[0]), "+r"(c[1]), "+r"(c[2]), "+r"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
  } else {
    asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.u8.u8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+r"(c[0]), "+r"(c[1]), "+r"(c[2]), "+r"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
  }
}

__device__ __forceinline__ void cp_async8(void* smem_dst, const void* gsrc) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"((uint32_t)__cvta_generic_to_shared(smem_dst)), "l"(gsrc) : "memory");
}
// fp16 operands, fp32 accumulation (qd_attention_desc.qk_f16).  With the fragments loaded exactly like the 8-bit ones
// (8 bytes per lane and 32-byte chunk), the k-slots see the same consistent permutation of the head dim in A and B.
__device__ __forceinline__ void mma_f16_16816(float (&c)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((uint32_t)__cvta_generic_to_shared(smem_dst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// entries per (batch, head) of the zq*rowsum(k) workspace (padded for 128-key tiles)
__host__ __device__ __forceinline__ int att_ws_stride(int Tk) { return (Tk + 127) / 128 * 128; }

// Position of key t inside a V^T row: within each group of 16 keys, key 8a+2b+c sits at byte 4b+2a+c.
__host__ __device__ __forceinline__ int att_vt_perm(int t) {
  return (t & ~15) | (((t >> 1) & 3) << 2) | (((t >> 3) & 1) << 1) | (t & 1);
}

// zq * rowsum_d(k[b, j, head h]) for every key: the only zero-point cross term that survives the softmax.
// bias_minus = 0: ws = zq*rowsum (subtracted by the mma.sync kernel).  Otherwise ws = bias - zq*rowsum, to be ADDED to the
// raw score: with bias = 0x4B400000 the sum is at once the corrected score and its magic-number float form.
template <bool SIGNED>
__global__ void att_krowsum_kernel(const qd_attention_desc p, int tk_pad, int bias_minus = 0, int bias = 0) {
  const long long total = (long long)p.B * p.heads * tk_pad;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int j = (int)(i % tk_pad);
    const long long bh = i / tk_pad;
    const int h = (int)(bh % p.heads);
    const long long b = bh / p.heads;
    int s = 0;
    if (j < p.Tk) {
      const uint8_t* kr = reinterpret_cast<const uint8_t*>(p.k) + (b * p.Tk + j) * p.ld_k + p.k_off + h * p.head_stride_k;
      for (int w = 0; w < p.d / 4; ++w) {
        const uint32_t v = *reinterpret_cast<const uint32_t*>(kr + 4 * w);
        s += SIGNED ? __dp4a((int)v, 0x01010101, 0) : (int)__dp4a(v, 0x01010101u, 0u);
      }
    }
    reinterpret_cast<int*>(p.ws)[i] = bias_minus ? bias - p.zq * s : p.zq * s;
  }
}

constexpr int ATT_WARPS = 8;
constexpr int ATT_BM = 16 * ATT_WARPS;  // query rows per CTA
constexpr int ATT_BN = 64;              // keys per tile

template <bool SIGNED>
__device__ __forceinline__ int bytesum(uint32_t w) {
  if constexpr (SIGNED) return __dp4a((int)w, 0x01010101, 0);
  else return (int)__dp4a(w, 0x01010101u, 0u);
}

__host__ __device__ constexpr int att_kp(int DQ) { return ((DQ / 32) & 1) ? DQ : DQ + 32; }

struct AttSmemLayout {
  int kp, vp, k_bytes, v_bytes, zrk_off, total;
};
__host__ __device__ inline AttSmemLayout att_smem_layout(int DQ, int DV, int Tk, bool need_zrk) {
  AttSmemLayout l;
  l.kp = att_kp(DQ);
  l.vp = ATT_BN + 16;
  l.k_bytes = ATT_BN * l.kp;
  l.v_bytes = (DV + 8) * l.vp;
  l.zrk_off = 2 * l.k_bytes + 2 * l.v_bytes;
  l.total = l.zrk_off + 2 * ATT_BN * 4;   // double-buffered zq*rowsum(k) slices
  return l;
}

// int32 -> float without the XU pipe (valid for |s| < 2^22): 1.5*2^23 + s is exact in fp32.
template <bool MAGIC>
__device__ __forceinline__ float att_i2f(int s) {
  if constexpr (MAGIC) return __int_as_float(s + 0x4B400000) - 12582912.0f;
  else return (float)s;
}

// Score type of the two-pass kernels: int32 on 8-bit codes; on fp16 operands the fp32 accumulators, which already hold
// the exact integer scores (|S| < 2^22), so they skip the float -> int -> float round trip (F2I on the XU pipe).  Every
// value, maximum and exponent argument is the same in both forms.
template <bool F16>
using att_score_t = std::conditional_t<F16, float, int>;
template <bool MAGIC>
__device__ __forceinline__ float att_s2f(int s) { return att_i2f<MAGIC>(s); }
template <bool MAGIC>
__device__ __forceinline__ float att_s2f(float s) { return s; }
__device__ __forceinline__ int att_smax(int a, int b) { return max(a, b); }
__device__ __forceinline__ float att_smax(float a, float b) { return fmaxf(a, b); }
__device__ __forceinline__ int att_lowest(int) { return INT_MIN; }
__device__ __forceinline__ float att_lowest(float) { return -INFINITY; }
// Score of a masked key (beyond Tk in the last key tile).  It is below every reachable score and its exponent
// fmaf(att_s2f(mask), c, b) is -inf, so the key takes no part in the row maximum, the row sum or the P codes whatever the
// codes are: -inf as an fp32 score (fp16 operands); on int32 scores converted by att_i2f<true> the integer that the
// conversion turns into the bit pattern of -inf.  att_i2f<false> (d > 64) turns INT_MIN into -2^31 instead, at least
// 2^31 - 255^2 d below every score: its probability is exactly 0 for the sim_scale values launch_attention accepts.
template <bool MAGIC>
__device__ __forceinline__ int att_mask(int) { return MAGIC ? (int)(0xFF800000u - 0x4B400000u) : INT_MIN; }
template <bool MAGIC>
__device__ __forceinline__ float att_mask(float) { return -INFINITY; }

// DQ: reduction length of QK^T padded to a multiple of 32; DV: head dim d (multiple of 8).
// Shared-memory tiles are addressed from the array symbol (the
// pointer-array version compiled to generic LD + 64-bit IMAD address math), the
// int<->float conversions avoid the XU pipe (it was the binding unit: I2F + F2I + 2 MUFU per score at
// 16 lanes/clk/SM), and the d index inside a 32-byte k-chunk is permuted (slot 4t+e <-> d 8t+e, slot
// 16+4t+e <-> d 8t+4+e, identically for Q and K) so each B fragment is one 8-byte shared load.
// F16: Q / K hold fp16 centred codes (code - zero point; qd_attention_desc.qk_f16, d <= 64).  QK^T then runs as
// m16n8k16 f16 x f16 -> f32: every product and partial sum is an integer below 2^24, so the score is exact, and it is
// already free of zero-point cross terms (no zq*rowsum(k) pass).  DQ counts BYTES of the padded reduction in both forms.
template <int DQ, int DV, bool QK_SIGNED, bool V_SIGNED, bool SM16, int MINB, bool F16 = false>
__global__ void __launch_bounds__(ATT_WARPS * 32, MINB)
qattention_kernel(const qd_attention_desc p) {
  constexpr int KP = att_kp(DQ);    // K tile row pitch (bytes): odd multiple of 32 -> conflict-free 8-byte B-fragment loads
  constexpr int VP = ATT_BN + 16;   // V^T tile row pitch (bytes)
  constexpr int NKC = DQ / 32;      // k-chunks for QK^T
  constexpr int NDT = DV / 8 + 1;   // n8 tiles of the output + the all-ones row-sum tile
  constexpr int KB = ATT_BN * KP, VB = (DV + 8) * VP;
  constexpr int ZB = ATT_BN * 4;    // per-tile zq*rowsum(k) slice
  constexpr bool MAGIC = DV <= 64;  // |S| <= 255*255*d < 2^22
  constexpr int RB = F16 ? 2 * DV : DV;   // bytes of one head's Q / K row
  constexpr int WPR = RB / 8;       // 8-byte pieces per K row
  static_assert(!F16 || DV <= 64, "fp16 Q / K operands: d <= 64 keeps |S| below 2^22");
  extern __shared__ __align__(16) uint8_t att_smem[];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int bh = blockIdx.y;
  const int b = bh / p.heads, h = bh - b * p.heads;
  const int row0 = blockIdx.x * ATT_BM + warp * 16;
  const int* zrk_g = reinterpret_cast<const int*>(p.ws) + (long long)bh * (long long)att_ws_stride(p.Tk);

  const uint8_t* qbase = reinterpret_cast<const uint8_t*>(p.q) + (long long)b * p.Tq * p.ld_q + p.q_off +
                         h * p.head_stride_q;
  const uint8_t* kbase = reinterpret_cast<const uint8_t*>(p.k) + (long long)b * p.Tk * p.ld_k + p.k_off +
                         h * p.head_stride_k;
  const uint8_t* vbase = reinterpret_cast<const uint8_t*>(p.vt) + (long long)b * p.v_batch_stride +
                         (long long)(p.v_off + h * p.head_stride_v) * p.ld_vt;
  const int ntiles = (p.Tk + ATT_BN - 1) / ATT_BN;

  // ---- prologue: zero both K buffers (the d..DQ padding must stay 0) and V^T buffers, ones row for row sums
  for (int i = threadIdx.x; i < (2 * KB + 2 * VB) / 16; i += blockDim.x)
    reinterpret_cast<uint4*>(att_smem)[i] = make_uint4(0u, 0u, 0u, 0u);
  __syncthreads();
  for (int i = threadIdx.x; i < 2 * ATT_BN; i += blockDim.x)
    att_smem[2 * KB + (i / ATT_BN) * VB + DV * VP + (i % ATT_BN)] = 1;
  auto prefetch = [&](int tile, int pass, int buf) {
    const int j0 = tile * ATT_BN;
    const int rows = min(ATT_BN, p.Tk - j0);
    uint8_t* dK = att_smem + buf * KB;
    for (int idx = threadIdx.x; idx < rows * WPR; idx += ATT_WARPS * 32) {
      const int r = idx / WPR, w = idx - r * WPR;
      cp_async8(dK + r * KP + 8 * w, kbase + (long long)(j0 + r) * p.ld_k + 8 * w);
    }
    if (!F16 && p.zq != 0 && threadIdx.x < ATT_BN / 4)
      cp_async16(att_smem + 2 * KB + 2 * VB + buf * ZB + 16 * threadIdx.x, zrk_g + j0 + 4 * threadIdx.x);
    if (pass == 1) {
      uint8_t* dV = att_smem + 2 * KB + buf * VB;
      for (int idx = threadIdx.x; idx < DV * (ATT_BN / 16); idx += ATT_WARPS * 32) {
        const int r = idx / (ATT_BN / 16), w = idx - r * (ATT_BN / 16);
        if (j0 + 16 * w < p.Tk) cp_async16(dV + r * VP + 16 * w, vbase + (long long)r * p.ld_vt + j0 + 16 * w);
      }
    }
    cp_async_commit();
  };
  prefetch(0, 0, 0);

  // ---- Q fragments (rows g, g+8 of this warp's 16-row slab), zero-padded beyond d, d-permuted (see above).
  // Of the zero-point cross terms only -zq*rowsum(k_j) depends on the key; -zk*rowsum(q_i) + d*zq*zk is a
  // per-row constant and cancels in the softmax, so it is never formed.
  uint32_t qf[NKC][4];
  {
    const int r0 = min(row0 + g, p.Tq - 1), r1 = min(row0 + g + 8, p.Tq - 1);
    const uint8_t* q0 = qbase + (long long)r0 * p.ld_q;
    const uint8_t* q1 = qbase + (long long)r1 * p.ld_q;
#pragma unroll
    for (int kc = 0; kc < NKC; ++kc) {
      const int c0 = kc * 32 + 8 * t, c1 = c0 + 4;
      qf[kc][0] = c0 < RB ? *reinterpret_cast<const uint32_t*>(q0 + c0) : 0u;
      qf[kc][1] = c0 < RB ? *reinterpret_cast<const uint32_t*>(q1 + c0) : 0u;
      qf[kc][2] = c1 < RB ? *reinterpret_cast<const uint32_t*>(q0 + c1) : 0u;
      qf[kc][3] = c1 < RB ? *reinterpret_cast<const uint32_t*>(q1 + c1) : 0u;
    }
  }
  // s2 = S_int * c  with c = sim_scale * log2(e)
  const float c = p.sim_scale * 1.4426950408889634f;
  const bool has_zq = !F16 && p.zq != 0;
  const bool ragged = (p.Tk % ATT_BN) != 0;

  using SV = att_score_t<F16>;
  SV mi0 = att_lowest(SV{}), mi1 = att_lowest(SV{});   // running integer row maxima (of S_raw - zrk)
  float l0 = 0.f, l1 = 0.f;           // running sums of exp2((S - max) * c)
  float off0 = 0.f, off1 = 0.f;       // pass-2 exponent offsets
  int olo[NDT][4], ohi[SM16 ? NDT : 1][4];
#pragma unroll
  for (int i = 0; i < NDT; ++i) { olo[i][0] = olo[i][1] = olo[i][2] = olo[i][3] = 0; }
#pragma unroll
  for (int i = 0; i < (SM16 ? NDT : 1); ++i) { ohi[i][0] = ohi[i][1] = ohi[i][2] = ohi[i][3] = 0; }
  const float pmax = (float)p.p_qmax;
  const QuantK oqk = make_quantk(p.oq);

  int buf = 0;
  for (int pass = 0; pass < 2; ++pass) {
    if (pass == 1) {                       // freeze the softmax statistics
      l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
      l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
      l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
      l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
      // code = rne(exp2(S*c - max*c + log2(1/(l*delta_w))))
      off0 = -(float)mi0 * c + log2f(1.0f / (l0 * p.delta_w));
      off1 = -(float)mi1 * c + log2f(1.0f / (l1 * p.delta_w));
    }
    for (int tile = 0; tile < ntiles; ++tile, buf ^= 1) {
      const int j0 = tile * ATT_BN;
      cp_async_wait_all();
      __syncthreads();                     // this tile landed for everyone; everyone is done with the previous one
      if (tile + 1 < ntiles) prefetch(tile + 1, pass, buf ^ 1);
      else if (pass == 0) prefetch(0, 1, buf ^ 1);
      const uint8_t* sK = att_smem + buf * KB;
      const uint8_t* sV = att_smem + 2 * KB + buf * VB;
      const int* sZrk = reinterpret_cast<const int*>(att_smem + 2 * KB + 2 * VB + buf * ZB);

      // ---- S = Q K^T for this warp: 16 x 64 (int32, or exact integers in fp32 on fp16 operands)
      SV sacc[8][4];
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        sacc[nt][0] = sacc[nt][1] = sacc[nt][2] = sacc[nt][3] = 0;
#pragma unroll
        for (int kc = 0; kc < NKC; ++kc) {
          const uint2 kk = *reinterpret_cast<const uint2*>(sK + (8 * nt + g) * KP + kc * 32 + 8 * t);
          const uint32_t bf[2] = {kk.x, kk.y};
          if constexpr (F16) mma_f16_16816(sacc[nt], qf[kc], bf);
          else mma_i8_16832<QK_SIGNED, QK_SIGNED>(sacc[nt], qf[kc], bf);
        }
      }
      if (has_zq) {
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
          const int2 z = *reinterpret_cast<const int2*>(sZrk + 8 * nt + 2 * t);
          sacc[nt][0] -= z.x; sacc[nt][1] -= z.y; sacc[nt][2] -= z.x; sacc[nt][3] -= z.y;
        }
      }
      if (ragged && tile == ntiles - 1) {
        const SV mask = att_mask<MAGIC>(SV{});
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
          const int j = j0 + 8 * nt + 2 * t;
          if (j >= p.Tk) { sacc[nt][0] = mask; sacc[nt][2] = mask; }
          if (j + 1 >= p.Tk) { sacc[nt][1] = mask; sacc[nt][3] = mask; }
        }
      }
      if (pass == 0) {
        SV tm0 = sacc[0][0], tm1 = sacc[0][2];
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
          tm0 = att_smax(tm0, att_smax(sacc[nt][0], sacc[nt][1]));
          tm1 = att_smax(tm1, att_smax(sacc[nt][2], sacc[nt][3]));
        }
        tm0 = att_smax(tm0, __shfl_xor_sync(0xffffffffu, tm0, 1));
        tm0 = att_smax(tm0, __shfl_xor_sync(0xffffffffu, tm0, 2));
        tm1 = att_smax(tm1, __shfl_xor_sync(0xffffffffu, tm1, 1));
        tm1 = att_smax(tm1, __shfl_xor_sync(0xffffffffu, tm1, 2));
        if (tm0 > mi0) { l0 *= (mi0 == att_lowest(SV{})) ? 0.f : ex2_approx((float)(mi0 - tm0) * c); mi0 = tm0; }
        if (tm1 > mi1) { l1 *= (mi1 == att_lowest(SV{})) ? 0.f : ex2_approx((float)(mi1 - tm1) * c); mi1 = tm1; }
        const float b0 = -(float)mi0 * c, b1 = -(float)mi1 * c;
        float a0 = 0.f, a1 = 0.f;
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
          a0 += ex2_approx(fmaf(att_s2f<MAGIC>(sacc[nt][0]), c, b0)) + ex2_approx(fmaf(att_s2f<MAGIC>(sacc[nt][1]), c, b0));
          a1 += ex2_approx(fmaf(att_s2f<MAGIC>(sacc[nt][2]), c, b1)) + ex2_approx(fmaf(att_s2f<MAGIC>(sacc[nt][3]), c, b1));
        }
        l0 += a0;
        l1 += a1;
      } else {
        // ---- P codes, packed straight into PV A-fragments (byte planes), then O += P V.
        // rne(pr) for 0 <= pr < 2^22 sits in the low mantissa bits of pr + 1.5*2^23: no F2I (XU pipe) needed.
#pragma unroll
        for (int kc = 0; kc < 2; ++kc) {
          uint32_t plo[4], phi[4];
#pragma unroll
          for (int half = 0; half < 2; ++half) {      // a0/a1 (keys 0..15 of the chunk) then a2/a3 (16..31)
            const int ntA = 4 * kc + 2 * half, ntB = ntA + 1;
            uint32_t cd[8];
            const SV sv[8] = {sacc[ntA][0], sacc[ntA][1], sacc[ntB][0], sacc[ntB][1],
                              sacc[ntA][2], sacc[ntA][3], sacc[ntB][2], sacc[ntB][3]};
#pragma unroll
            for (int e = 0; e < 8; ++e) {
              const float pr = ex2_approx(fmaf(att_s2f<MAGIC>(sv[e]), c, e < 4 ? off0 : off1));
              cd[e] = __float_as_uint(fminf(pr, pmax) + 12582912.0f);
            }
            plo[2 * half] = __byte_perm(__byte_perm(cd[0], cd[1], 0x0040), __byte_perm(cd[2], cd[3], 0x0040), 0x5410);
            plo[2 * half + 1] = __byte_perm(__byte_perm(cd[4], cd[5], 0x0040), __byte_perm(cd[6], cd[7], 0x0040), 0x5410);
            if constexpr (SM16) {
              phi[2 * half] = __byte_perm(__byte_perm(cd[0], cd[1], 0x0051), __byte_perm(cd[2], cd[3], 0x0051), 0x5410);
              phi[2 * half + 1] = __byte_perm(__byte_perm(cd[4], cd[5], 0x0051), __byte_perm(cd[6], cd[7], 0x0051), 0x5410);
            }
          }
#pragma unroll
          for (int nd = 0; nd < NDT; ++nd) {
            // V^T rows are stored with the 16-key groups permuted (key 8a+2b+c at byte 4b+2a+c, see
            // att_vt_perm) so the k-slots of this thread are 4 contiguous bytes
            const uint8_t* vr = sV + (8 * nd + g) * VP + 32 * kc + 4 * t;
            const uint32_t bf[2] = {*reinterpret_cast<const uint32_t*>(vr), *reinterpret_cast<const uint32_t*>(vr + 16)};
            if (nd == NDT - 1) {   // all-ones row (unsigned) -> row sums of the codes
              mma_i8_16832<false, false>(olo[nd], plo, bf);
              if constexpr (SM16) mma_i8_16832<false, false>(ohi[nd], phi, bf);
            } else {
              mma_i8_16832<false, V_SIGNED>(olo[nd], plo, bf);
              if constexpr (SM16) mma_i8_16832<false, V_SIGNED>(ohi[nd], phi, bf);
            }
          }
        }
      }
    }
  }

  // ---- write O: (256*hi + lo - zv * rowsum) * out_scale.  Row sums sit in column 0 of the extra tile (t == 0).
  float rs0 = (float)olo[NDT - 1][0], rs1 = (float)olo[NDT - 1][2];
  if constexpr (SM16) { rs0 += 256.0f * (float)ohi[NDT - 1][0]; rs1 += 256.0f * (float)ohi[NDT - 1][2]; }
  rs0 = __shfl_sync(0xffffffffu, rs0, lane & ~3);
  rs1 = __shfl_sync(0xffffffffu, rs1, lane & ~3);
  const int r0 = row0 + g, r1 = row0 + g + 8;
  const float z0 = (float)p.zv * rs0, z1 = (float)p.zv * rs1;
#pragma unroll
  for (int nd = 0; nd < NDT - 1; ++nd) {
    const int col = h * DV + 8 * nd + 2 * t;
    float v0 = (float)olo[nd][0], v1 = (float)olo[nd][1], v2 = (float)olo[nd][2], v3 = (float)olo[nd][3];
    if constexpr (SM16) {
      v0 += 256.0f * (float)ohi[nd][0]; v1 += 256.0f * (float)ohi[nd][1];
      v2 += 256.0f * (float)ohi[nd][2]; v3 += 256.0f * (float)ohi[nd][3];
    }
    const float y0 = (v0 - z0) * p.out_scale, y1 = (v1 - z0) * p.out_scale;
    const float y2 = (v2 - z1) * p.out_scale, y3 = (v3 - z1) * p.out_scale;
    if (p.out) {
      if (r0 < p.Tq) *reinterpret_cast<float2*>(p.out + ((long long)b * p.Tq + r0) * p.ld_out + col) = make_float2(y0, y1);
      if (r1 < p.Tq) *reinterpret_cast<float2*>(p.out + ((long long)b * p.Tq + r1) * p.ld_out + col) = make_float2(y2, y3);
    }
    if (p.out_q) {   // consumer's activation quantizer (to_out.0 / proj_out input), qdiff/quant_layer.py:82-88
      uint8_t* oq = reinterpret_cast<uint8_t*>(p.out_q);
      if (r0 < p.Tq)
        *reinterpret_cast<uint16_t*>(oq + ((long long)b * p.Tq + r0) * p.ld_out_q + col) =
            (uint16_t)(quant_code(y0, oqk) | (quant_code(y1, oqk) << 8));
      if (r1 < p.Tq)
        *reinterpret_cast<uint16_t*>(oq + ((long long)b * p.Tq + r1) * p.ld_out_q + col) =
            (uint16_t)(quant_code(y2, oqk) | (quant_code(y3, oqk) << 8));
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Small-Tk variant (cross-attention: Tk = 77 context tokens).  The whole key range is one tile, so
//   * K, V^T and zq*rowsum(k) are staged in shared memory ONCE per CTA (the row sums are computed here: no
//     separate att_krowsum launch) and each warp then streams 16-query slabs past them;
//   * the softmax is a single pass over register-resident scores (max, sum, codes from the same accumulators).
// The two-pass kernel above pays its per-CTA prologue (tile ring, barriers) per 128 queries; with ~80 keys that
// prologue dominates the run time.
// Arithmetic is the same as qattention_kernel (same exp2-domain formulas, same fragment/key permutations).
constexpr int ATS_WARPS = 4;

template <int DQ, int DV, int NKV>
__host__ __device__ constexpr int ats_smem_bytes() {
  return NKV * 32 * att_kp(DQ) + (DV + 8) * (NKV * 32 + 16) + NKV * 32 * 4;
}

template <int DQ, int DV, bool QK_SIGNED, bool V_SIGNED, bool SM16, int NKV>
__global__ void __launch_bounds__(ATS_WARPS * 32)
qattention_smallk_kernel(const qd_attention_desc p, int slabs_per_warp) {
  constexpr int KP = att_kp(DQ);
  constexpr int TKP = NKV * 32;     // padded key count
  constexpr int NT8 = NKV * 4;      // n8 tiles of S
  constexpr int VP = TKP + 16;
  constexpr int NKC = DQ / 32;
  constexpr int NDT = DV / 8 + 1;
  constexpr int KB = TKP * KP, VB = (DV + 8) * VP;
  constexpr bool MAGIC = DV <= 64;
  constexpr int WPR = DV / 8;
  extern __shared__ __align__(16) uint8_t att_smem[];
  uint8_t* sK = att_smem;
  uint8_t* sV = att_smem + KB;
  int* sZrk = reinterpret_cast<int*>(att_smem + KB + VB);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int bh = blockIdx.y;
  const int b = bh / p.heads, h = bh - b * p.heads;
  const uint8_t* qbase = reinterpret_cast<const uint8_t*>(p.q) + (long long)b * p.Tq * p.ld_q + p.q_off +
                         h * p.head_stride_q;
  const uint8_t* kbase = reinterpret_cast<const uint8_t*>(p.k) + (long long)b * p.Tk * p.ld_k + p.k_off +
                         h * p.head_stride_k;
  const uint8_t* vbase = reinterpret_cast<const uint8_t*>(p.vt) + (long long)b * p.v_batch_stride +
                         (long long)(p.v_off + h * p.head_stride_v) * p.ld_vt;

  // ---- stage K (d..DQ padding and rows >= Tk stay 0), V^T (+ all-ones row) and zq*rowsum(k)
  for (int i = threadIdx.x; i < (KB + VB) / 16; i += blockDim.x)
    reinterpret_cast<uint4*>(att_smem)[i] = make_uint4(0u, 0u, 0u, 0u);
  __syncthreads();
  for (int idx = threadIdx.x; idx < p.Tk * WPR; idx += blockDim.x) {
    const int r = idx / WPR, w = idx - r * WPR;
    *reinterpret_cast<uint2*>(sK + r * KP + 8 * w) = *reinterpret_cast<const uint2*>(kbase + (long long)r * p.ld_k + 8 * w);
  }
  for (int idx = threadIdx.x; idx < DV * (TKP / 16); idx += blockDim.x) {
    const int r = idx / (TKP / 16), w = idx - r * (TKP / 16);
    if (16 * w < p.Tk)
      *reinterpret_cast<uint4*>(sV + r * VP + 16 * w) = *reinterpret_cast<const uint4*>(vbase + (long long)r * p.ld_vt + 16 * w);
  }
  for (int i = threadIdx.x; i < TKP; i += blockDim.x) sV[DV * VP + i] = 1;
  __syncthreads();
  for (int j = threadIdx.x; j < TKP; j += blockDim.x) {
    int sum = 0;
    if (p.zq != 0 && j < p.Tk) {
#pragma unroll
      for (int w = 0; w < DV / 4; ++w) sum += bytesum<QK_SIGNED>(*reinterpret_cast<const uint32_t*>(sK + j * KP + 4 * w));
    }
    sZrk[j] = p.zq * sum;
  }
  __syncthreads();

  const float c = p.sim_scale * 1.4426950408889634f;
  const float pmax = (float)p.p_qmax;
  const QuantK oqk = make_quantk(p.oq);

  for (int sl = 0; sl < slabs_per_warp; ++sl) {
    const int row0 = ((blockIdx.x * slabs_per_warp + sl) * ATS_WARPS + warp) * 16;
    if (row0 >= p.Tq) break;
    uint32_t qf[NKC][4];
    {
      const int r0 = min(row0 + g, p.Tq - 1), r1 = min(row0 + g + 8, p.Tq - 1);
      const uint8_t* q0 = qbase + (long long)r0 * p.ld_q;
      const uint8_t* q1 = qbase + (long long)r1 * p.ld_q;
#pragma unroll
      for (int kc = 0; kc < NKC; ++kc) {
        const int c0 = kc * 32 + 8 * t, c1 = c0 + 4;
        qf[kc][0] = c0 < DV ? *reinterpret_cast<const uint32_t*>(q0 + c0) : 0u;
        qf[kc][1] = c0 < DV ? *reinterpret_cast<const uint32_t*>(q1 + c0) : 0u;
        qf[kc][2] = c1 < DV ? *reinterpret_cast<const uint32_t*>(q0 + c1) : 0u;
        qf[kc][3] = c1 < DV ? *reinterpret_cast<const uint32_t*>(q1 + c1) : 0u;
      }
    }
    // ---- S = Q K^T (16 x TKP), minus zq*rowsum(k), masked beyond Tk
    int sacc[NT8][4];
#pragma unroll
    for (int nt = 0; nt < NT8; ++nt) {
      sacc[nt][0] = sacc[nt][1] = sacc[nt][2] = sacc[nt][3] = 0;
#pragma unroll
      for (int kc = 0; kc < NKC; ++kc) {
        const uint2 kk = *reinterpret_cast<const uint2*>(sK + (8 * nt + g) * KP + kc * 32 + 8 * t);
        const uint32_t bf[2] = {kk.x, kk.y};
        mma_i8_16832<QK_SIGNED, QK_SIGNED>(sacc[nt], qf[kc], bf);
      }
      const int2 z = *reinterpret_cast<const int2*>(sZrk + 8 * nt + 2 * t);
      sacc[nt][0] -= z.x; sacc[nt][1] -= z.y; sacc[nt][2] -= z.x; sacc[nt][3] -= z.y;
      const int j = 8 * nt + 2 * t;
      if (j >= p.Tk) { sacc[nt][0] = att_mask<MAGIC>(0); sacc[nt][2] = att_mask<MAGIC>(0); }
      if (j + 1 >= p.Tk) { sacc[nt][1] = att_mask<MAGIC>(0); sacc[nt][3] = att_mask<MAGIC>(0); }
    }
    // ---- row statistics (rows g and g+8; a row lives in the 4 lanes of a quad)
    int mi0 = sacc[0][0], mi1 = sacc[0][2];
#pragma unroll
    for (int nt = 0; nt < NT8; ++nt) {
      mi0 = max(mi0, max(sacc[nt][0], sacc[nt][1]));
      mi1 = max(mi1, max(sacc[nt][2], sacc[nt][3]));
    }
    mi0 = max(mi0, __shfl_xor_sync(0xffffffffu, mi0, 1));
    mi0 = max(mi0, __shfl_xor_sync(0xffffffffu, mi0, 2));
    mi1 = max(mi1, __shfl_xor_sync(0xffffffffu, mi1, 1));
    mi1 = max(mi1, __shfl_xor_sync(0xffffffffu, mi1, 2));
    const float b0 = -(float)mi0 * c, b1 = -(float)mi1 * c;
    float l0 = 0.f, l1 = 0.f;
#pragma unroll
    for (int nt = 0; nt < NT8; ++nt) {
      l0 += ex2_approx(fmaf(att_i2f<MAGIC>(sacc[nt][0]), c, b0)) + ex2_approx(fmaf(att_i2f<MAGIC>(sacc[nt][1]), c, b0));
      l1 += ex2_approx(fmaf(att_i2f<MAGIC>(sacc[nt][2]), c, b1)) + ex2_approx(fmaf(att_i2f<MAGIC>(sacc[nt][3]), c, b1));
    }
    l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
    l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
    const float off0 = b0 + log2f(1.0f / (l0 * p.delta_w));
    const float off1 = b1 + log2f(1.0f / (l1 * p.delta_w));

    // ---- P codes -> PV (same packing as qattention_kernel)
    int olo[NDT][4], ohi[SM16 ? NDT : 1][4];
#pragma unroll
    for (int i = 0; i < NDT; ++i) { olo[i][0] = olo[i][1] = olo[i][2] = olo[i][3] = 0; }
#pragma unroll
    for (int i = 0; i < (SM16 ? NDT : 1); ++i) { ohi[i][0] = ohi[i][1] = ohi[i][2] = ohi[i][3] = 0; }
#pragma unroll
    for (int kc = 0; kc < NKV; ++kc) {
      uint32_t plo[4], phi[4];
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        const int ntA = 4 * kc + 2 * half, ntB = ntA + 1;
        uint32_t cd[8];
        const int sv[8] = {sacc[ntA][0], sacc[ntA][1], sacc[ntB][0], sacc[ntB][1],
                           sacc[ntA][2], sacc[ntA][3], sacc[ntB][2], sacc[ntB][3]};
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const float pr = ex2_approx(fmaf(att_i2f<MAGIC>(sv[e]), c, e < 4 ? off0 : off1));
          cd[e] = __float_as_uint(fminf(pr, pmax) + 12582912.0f);
        }
        plo[2 * half] = __byte_perm(__byte_perm(cd[0], cd[1], 0x0040), __byte_perm(cd[2], cd[3], 0x0040), 0x5410);
        plo[2 * half + 1] = __byte_perm(__byte_perm(cd[4], cd[5], 0x0040), __byte_perm(cd[6], cd[7], 0x0040), 0x5410);
        if constexpr (SM16) {
          phi[2 * half] = __byte_perm(__byte_perm(cd[0], cd[1], 0x0051), __byte_perm(cd[2], cd[3], 0x0051), 0x5410);
          phi[2 * half + 1] = __byte_perm(__byte_perm(cd[4], cd[5], 0x0051), __byte_perm(cd[6], cd[7], 0x0051), 0x5410);
        }
      }
#pragma unroll
      for (int nd = 0; nd < NDT; ++nd) {
        const uint8_t* vr = sV + (8 * nd + g) * VP + 32 * kc + 4 * t;
        const uint32_t bf[2] = {*reinterpret_cast<const uint32_t*>(vr), *reinterpret_cast<const uint32_t*>(vr + 16)};
        if (nd == NDT - 1) {
          mma_i8_16832<false, false>(olo[nd], plo, bf);
          if constexpr (SM16) mma_i8_16832<false, false>(ohi[nd], phi, bf);
        } else {
          mma_i8_16832<false, V_SIGNED>(olo[nd], plo, bf);
          if constexpr (SM16) mma_i8_16832<false, V_SIGNED>(ohi[nd], phi, bf);
        }
      }
    }
    // ---- O = (256*hi + lo - zv*rowsum) * out_scale
    float rs0 = (float)olo[NDT - 1][0], rs1 = (float)olo[NDT - 1][2];
    if constexpr (SM16) { rs0 += 256.0f * (float)ohi[NDT - 1][0]; rs1 += 256.0f * (float)ohi[NDT - 1][2]; }
    rs0 = __shfl_sync(0xffffffffu, rs0, lane & ~3);
    rs1 = __shfl_sync(0xffffffffu, rs1, lane & ~3);
    const int r0 = row0 + g, r1 = row0 + g + 8;
    const float z0 = (float)p.zv * rs0, z1 = (float)p.zv * rs1;
#pragma unroll
    for (int nd = 0; nd < NDT - 1; ++nd) {
      const int col = h * DV + 8 * nd + 2 * t;
      float v0 = (float)olo[nd][0], v1 = (float)olo[nd][1], v2 = (float)olo[nd][2], v3 = (float)olo[nd][3];
      if constexpr (SM16) {
        v0 += 256.0f * (float)ohi[nd][0]; v1 += 256.0f * (float)ohi[nd][1];
        v2 += 256.0f * (float)ohi[nd][2]; v3 += 256.0f * (float)ohi[nd][3];
      }
      const float y0 = (v0 - z0) * p.out_scale, y1 = (v1 - z0) * p.out_scale;
      const float y2 = (v2 - z1) * p.out_scale, y3 = (v3 - z1) * p.out_scale;
      if (p.out) {
        if (r0 < p.Tq) *reinterpret_cast<float2*>(p.out + ((long long)b * p.Tq + r0) * p.ld_out + col) = make_float2(y0, y1);
        if (r1 < p.Tq) *reinterpret_cast<float2*>(p.out + ((long long)b * p.Tq + r1) * p.ld_out + col) = make_float2(y2, y3);
      }
      if (p.out_q) {
        uint8_t* oq = reinterpret_cast<uint8_t*>(p.out_q);
        if (r0 < p.Tq)
          *reinterpret_cast<uint16_t*>(oq + ((long long)b * p.Tq + r0) * p.ld_out_q + col) =
              (uint16_t)(quant_code(y0, oqk) | (quant_code(y1, oqk) << 8));
        if (r1 < p.Tq)
          *reinterpret_cast<uint16_t*>(oq + ((long long)b * p.Tq + r1) * p.ld_out_q + col) =
              (uint16_t)(quant_code(y2, oqk) | (quant_code(y3, oqk) << 8));
      }
    }
  }
}

}  // namespace qd
