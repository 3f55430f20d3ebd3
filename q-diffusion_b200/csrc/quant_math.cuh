// Activation-quantizer arithmetic shared by every kernel that emits codes
// (UniformAffineQuantizer.forward, qdiff/quant_layer.py:82-87:  code = clamp(rne(y / delta) + zp, lo, hi)).
//
// The straightforward form rintf(__fdiv_rn(y, d)) + zp -> clamp -> (int) costs 4 XU-pipe operations per
// element (FCHK, MUFU.RCP, FRND, F2I; the XU pipe runs at 16 lanes/clk/SM), which made the "memory-bound"
// norm/quantise kernels XU-bound well below HBM bandwidth.  This
// version uses no XU operation per element:
//   * y/d as q0 = y*r, q = fma(fma(-q0, d, y), r, q0) with r = RN(1/d): one Newton step on the FMA pipe,
//     correctly rounded except for vanishingly rare halfway cases;
//   * rne() and float->int through the 1.5*2^23 magic constant (valid for |q| < 2^22, enforced by a clamp);
//   * zero point and clamp in integer arithmetic.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../include/qdiff_b200.h"

namespace qd {

struct QuantK {
  float delta, rdelta;
  int bias;        // 0x4B400000 - zero_point
  float flo, fhi;  // clamp range of q = y/delta BEFORE rounding: [qmin - zp, qmax - zp] (integers, so
                   // clamp-then-round == round-then-clamp, and |q| stays inside the magic-constant range)
};

__device__ __forceinline__ QuantK make_quantk(float delta, int zero_point, int lo, int hi) {
  QuantK k;
  k.delta = delta;
  k.rdelta = __frcp_rn(delta);
  k.bias = 0x4B400000 - zero_point;
  k.flo = (float)(lo - zero_point);
  k.fhi = (float)(hi - zero_point);
  return k;
}
__device__ __forceinline__ QuantK make_quantk(const qd_qparams& q) {
  return make_quantk(q.delta, q.zero_point, q.qmin, q.qmax);
}

// y / delta with one Newton step.  When q0 = y * r overflows (y = +-inf, or |y| / delta beyond FLT_MAX) the step computes
// fma(-inf, delta, y) = NaN, which the clamp below would turn into the LOW rail; q0 itself is then the right infinity.
// Finite quotients never take the select, so their codes are unchanged.  NaN inputs stay NaN and clamp to the low rail.
__device__ __forceinline__ float quant_quotient(float y, const QuantK& k) {
  const float q0 = y * k.rdelta;
  const float q = fmaf(fmaf(-q0, k.delta, y), k.rdelta, q0);
  return q == q ? q : q0;
}

// Exact form (8 instructions): used where the input fp32 value is itself exact w.r.t. the reference
// (standalone quantizer, GEMM epilogues).
__device__ __forceinline__ uint32_t quant_code(float y, const QuantK& k) {
  const float q = fminf(fmaxf(quant_quotient(y, k), k.flo), k.fhi);
  return (uint32_t)(__float_as_int(q + 12582912.0f) - k.bias) & 0xFFu;   // rne(q) + zero_point
}

// rne(y / delta) clamped to [qmin - zp, qmax - zp]: the code minus its zero point, as a float (fp16 attention operands)
__device__ __forceinline__ float quant_centered(float y, const QuantK& k) {
  const float q = fminf(fmaxf(quant_quotient(y, k), k.flo), k.fhi);
  return (q + 12582912.0f) - 12582912.0f;
}

// Fast form (5 instructions, reciprocal multiply without the Newton step): y*r differs from y/delta by <= 1 ulp,
// which can move a code only when the quotient sits within 1 ulp of a rounding boundary (~1e-5 of elements).
// Used behind SiLU / GELU / normalisation, whose inputs already differ from the reference by ulps.
__device__ __forceinline__ uint32_t quant_code_fast(float y, const QuantK& k) {
  const float q = fminf(fmaxf(y * k.rdelta, k.flo), k.fhi);
  return (uint32_t)(__float_as_int(q + 12582912.0f) - k.bias) & 0xFFu;
}

// Pre-scaled form (3 instructions + a quarter of the 3-PRMT pack): the caller's value is already t = y / delta + zero_point
// (qd_gemm_desc.scale_q / bias_q); clamp to the code range, round through the magic constant.  Returns the float's bit
// pattern: its LOW BYTE is the code (two's complement for signed codes), because 0x4B400000 ends in 0x00.
__device__ __forceinline__ QuantK make_quantk_pre(float delta, int lo, int hi) {
  QuantK k;
  k.delta = delta;
  k.rdelta = __frcp_rn(delta);     // multiplies a residual into code units
  k.bias = 0x4B400000;
  k.flo = (float)lo;
  k.fhi = (float)hi;
  return k;
}
__device__ __forceinline__ uint32_t quant_bits_pre(float t, const QuantK& k) {
  return __float_as_uint(fminf(fmaxf(t, k.flo), k.fhi) + 12582912.0f);
}
__device__ __forceinline__ uint32_t pack4_low_bytes(uint32_t r0, uint32_t r1, uint32_t r2, uint32_t r3) {
  return __byte_perm(__byte_perm(r0, r1, 0x0040), __byte_perm(r2, r3, 0x0040), 0x5410);
}

// x * sigmoid(x) with 2 XU operations (ex2, rcp); ~2 ulp, inside the reference's own fp32 noise band.
__device__ __forceinline__ float silu_fast(float x) {
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(-1.4426950408889634f * x));
  return __fdividef(x, 1.0f + e);
}

// exact-erf GELU (F.gelu default, ldm/modules/attention.py:44)
__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)); }

// The same function in ~15 instructions (libm erff is ~40, which made the GEGLU GEMM epilogue issue-bound).  erfc(z) = t*P(t)*exp(-z^2), t = 1/(1 + p z) (Abramowitz-Stegun 7.1.26) with
// the 1/2 and the 1/sqrt(2) folded into the constants, evaluated on the complementary side so that negative
// gates lose no precision:  gelu(g) = g - h (g >= 0), -h (g < 0), h = |g| * erfc(|g|/sqrt2) / 2.
// Max |error| 3.3e-7 over [-8, 8] in fp32 (torch's own fp32 F.gelu: 1.2e-6), measured in tools/check_gelu.py.
__device__ __forceinline__ float gelu_fast(float g) {
  const float ag = fabsf(g);
  float t, e;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(ag, 0.3275911f * 0.70710678118654752440f, 1.0f)));
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"((g * (-0.5f * 1.4426950408889634f)) * g));
  float poly = fmaf(0.5f * 1.061405429f, t, 0.5f * -1.453152027f);
  poly = fmaf(poly, t, 0.5f * 1.421413741f);
  poly = fmaf(poly, t, 0.5f * -0.284496736f);
  poly = fmaf(poly, t, 0.5f * 0.254829592f);
  const float h = ag * ((poly * t) * e);
  return g >= 0.f ? g - h : -h;
}

}  // namespace qd
