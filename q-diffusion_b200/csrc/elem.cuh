// Memory-bound fused kernels on the UNet path: activation quantizers with their elementwise
// producers (SiLU / GEGLU / nearest-2x upsample / split-shortcut), GroupNorm(+SiLU)+quant,
// LayerNorm+multi-consumer quant, im2col for the strided convs, layout changes, sampler update.
// All are HBM-bound: 128-bit loads, channel-contiguous (NHWC) coalescing, grids sized in
// multiples of the SM count with grid-stride loops.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../include/qdiff_b200.h"
#include "quant_math.cuh"

namespace qd {

__device__ __forceinline__ uint32_t pack4(uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  return a | (b << 8) | (c << 16) | (d << 24);
}
__device__ __forceinline__ float silu_f(float x) { return silu_fast(x); }
__device__ __forceinline__ float gelu_erf_f(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)); }
// quick_gelu of transformers' activations.py (x * sigmoid(1.702 x)), the CLIP text encoder's MLP activation; expf, not
// __expf: the weight-only planes carry the value to 2^-24
__device__ __forceinline__ float quick_gelu_f(float x) { return x * (1.0f / (1.0f + expf(-1.702f * x))); }
// SiLU of the weight-only planes (temb / emb_layers): expf (2 ulp), not __expf, whose error grows as 2 + 1.17 |x| ulp
__device__ __forceinline__ float silu_accurate_f(float x) { return x / (1.0f + expf(-x)); }

// ------------------------------------------------------------------------------------ quantize
// One thread = 4 consecutive channels of one row.
__global__ void quantize_kernel(const qd_quantize_desc p) {
  const int cq = p.C >> 2;
  const long long rows_out = p.upsample2x ? (long long)p.B * (2 * p.H) * (2 * p.W) : (long long)p.M;
  const long long total = rows_out * cq;
  const QuantK k0 = make_quantk(p.q0), k1 = make_quantk(p.q1);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long ro = i / cq;
    const int c = (int)(i - ro * cq) << 2;
    long long rs = ro;
    if (p.upsample2x) {
      const int W2 = 2 * p.W, H2 = 2 * p.H;
      const int w2 = (int)(ro % W2);
      const long long t = ro / W2;
      const int h2 = (int)(t % H2);
      const long long b = t / H2;
      rs = (b * p.H + (h2 >> 1)) * p.W + (w2 >> 1);
    }
    const float* s = p.src + rs * p.ld_src + c;
    float4 v = *reinterpret_cast<const float4*>(s);
    if (p.act == 1) {
      v.x = silu_f(v.x); v.y = silu_f(v.y); v.z = silu_f(v.z); v.w = silu_f(v.w);
    } else if (p.act == 2) {
      const float4 g = *reinterpret_cast<const float4*>(s + p.C);
      v.x *= gelu_erf_f(g.x); v.y *= gelu_erf_f(g.y); v.z *= gelu_erf_f(g.z); v.w *= gelu_erf_f(g.w);
    }
    uint32_t out;
    if (p.split > 0 && c >= p.split) {
      out = pack4(quant_code(v.x, k1), quant_code(v.y, k1), quant_code(v.z, k1), quant_code(v.w, k1));
    } else {
      out = pack4(quant_code(v.x, k0), quant_code(v.y, k0), quant_code(v.z, k0), quant_code(v.w, k0));
    }
    *reinterpret_cast<uint32_t*>(reinterpret_cast<uint8_t*>(p.dst) + ro * p.ld_dst + c) = out;
  }
}

// scalar tail variant for C % 4 != 0 (conv_in with 3 input channels, etc.)
__global__ void quantize_scalar_kernel(const qd_quantize_desc p) {
  const long long total = (long long)p.M * p.C;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / p.C;
    const int c = (int)(i - r * p.C);
    float v = p.src[r * p.ld_src + c];
    if (p.act == 1) v = silu_f(v);
    else if (p.act == 2) v *= gelu_erf_f(p.src[r * p.ld_src + p.C + c]);
    const QuantK k = make_quantk((p.split > 0 && c >= p.split) ? p.q1 : p.q0);
    reinterpret_cast<uint8_t*>(p.dst)[r * p.ld_dst + c] = (uint8_t)quant_code(v, k);
  }
}

// ------------------------------------------------------------------------------------ weight-only operands
// fp32 activation -> three bfloat16 planes (hi, mid, lo): x = hi + mid + lo up to 2^-24 |x|, so that a bfloat16 tensor-core
// contraction against integer weight codes (exact in bfloat16) with fp32 accumulation reproduces the fp32 conv of the
// reference's weight-only path (quant_layer.py:263-279, use_act_quant False).  One thread = 4 channels of one row.
__device__ __forceinline__ uint32_t bf16_bits(float x) { return __float_as_uint(x) >> 16; }   // x already on the bf16 grid
__device__ __forceinline__ float bf16_rn(float x) {       // round-to-nearest-even to the bfloat16 grid, kept as float
  const uint32_t u = __float_as_uint(x);
  const uint32_t r = u + 0x7FFFu + ((u >> 16) & 1u);
  return __uint_as_float(r & 0xFFFF0000u);
}
__global__ void split_bf16x3_kernel(const qd_split_desc p) {
  const int cq = p.C >> 2;
  const long long rows_out = p.upsample2x ? (long long)p.B * (2 * p.H) * (2 * p.W) : (long long)p.M;
  const long long total = rows_out * cq;
  uint16_t* dst = reinterpret_cast<uint16_t*>(p.dst);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long ro = i / cq;
    const int c = (int)(i - ro * cq) << 2;
    long long rs = ro;
    if (p.upsample2x) {
      const int W2 = 2 * p.W, H2 = 2 * p.H;
      const int w2 = (int)(ro % W2);
      const long long t = ro / W2;
      const int h2 = (int)(t % H2);
      const long long b = t / H2;
      rs = (b * p.H + (h2 >> 1)) * p.W + (w2 >> 1);
    }
    const float4 v4 = *reinterpret_cast<const float4*>(p.src + rs * p.ld_src + c);
    float v[4] = {v4.x, v4.y, v4.z, v4.w};
    if (p.act == 2) {       // GEGLU (ldm/modules/attention.py:42-44) with the exact-erf GELU
      const float4 g4 = *reinterpret_cast<const float4*>(p.src + rs * p.ld_src + p.C + c);
      v[0] *= gelu_erf_f(g4.x); v[1] *= gelu_erf_f(g4.y); v[2] *= gelu_erf_f(g4.z); v[3] *= gelu_erf_f(g4.w);
    }
    uint32_t pl[3][4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float x = v[j];
      if (p.act == 1) x = silu_accurate_f(x);
      else if (p.act == 3) x = quick_gelu_f(x);
      const float h = bf16_rn(x);
      const float r1 = x - h;
      const float m = bf16_rn(r1);
      const float l = bf16_rn(r1 - m);
      pl[0][j] = bf16_bits(h); pl[1][j] = bf16_bits(m); pl[2][j] = bf16_bits(l);
    }
    uint16_t* o = dst + ro * p.ld_dst + c;
#pragma unroll
    for (int q = 0; q < 3; ++q)
      *reinterpret_cast<uint2*>(o + (long long)q * p.Cp) = make_uint2(pl[q][0] | (pl[q][1] << 16), pl[q][2] | (pl[q][3] << 16));
  }
}

// element-wise variant for C % 4 != 0 (conv_in with 3 input channels)
__global__ void split_bf16x3_scalar_kernel(const qd_split_desc p) {
  const long long total = (long long)p.M * p.C;
  uint16_t* dst = reinterpret_cast<uint16_t*>(p.dst);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / p.C;
    const int c = (int)(i - r * p.C);
    float x = p.src[r * p.ld_src + c];
    if (p.act == 1) x = silu_accurate_f(x);
    else if (p.act == 2) x *= gelu_erf_f(p.src[r * p.ld_src + p.C + c]);
    else if (p.act == 3) x = quick_gelu_f(x);
    const float h = bf16_rn(x);
    const float r1 = x - h;
    const float m = bf16_rn(r1);
    const float l = bf16_rn(r1 - m);
    uint16_t* o = dst + r * p.ld_dst + c;
    o[0] = (uint16_t)bf16_bits(h);
    o[p.Cp] = (uint16_t)bf16_bits(m);
    o[2 * p.Cp] = (uint16_t)bf16_bits(l);
  }
}

// fp32 attention of the weight-only path: one block per (query row, batch*head).  Scores of the row live in shared
// memory (Tk <= 8192), exact expf, fp32 accumulation in a fixed order.  Small problems only (CIFAR 16x16, LDM latents):
// correctness path of BASELINE configs[0], not a throughput kernel.
__global__ void __launch_bounds__(128) attention_fp32_kernel(const qd_attention_fp_desc p) {
  extern __shared__ float afp_sh[];
  float* qs = afp_sh;                 // [d]
  float* sc = afp_sh + p.d;           // [Tk]
  __shared__ float red[4];
  const int bh = blockIdx.y, b = bh / p.heads, h = bh - b * p.heads;
  const int r = blockIdx.x;
  // causal: keys r+1.. are never read, so they take no probability whatever they hold (the launcher checks Tq == Tk)
  const int nk = p.causal ? min(r + 1, p.Tk) : p.Tk;
  const float* q = p.q + ((long long)b * p.Tq + r) * p.ld_q + p.q_off + h * p.head_stride_q;
  for (int i = threadIdx.x; i < p.d; i += blockDim.x) qs[i] = q[i];
  __syncthreads();
  float mx = -INFINITY;
  for (int j = threadIdx.x; j < nk; j += blockDim.x) {
    const float* k = p.k + ((long long)b * p.Tk + j) * p.ld_k + p.k_off + h * p.head_stride_k;
    float acc = 0.f;
    for (int i = 0; i < p.d; ++i) acc = fmaf(qs[i], k[i], acc);
    acc *= p.scale;
    sc[j] = acc;
    mx = fmaxf(mx, acc);
  }
  for (int off = 16; off > 0; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  mx = fmaxf(fmaxf(red[0], red[1]), fmaxf(red[2], red[3]));
  __syncthreads();
  float sum = 0.f;
  for (int j = threadIdx.x; j < nk; j += blockDim.x) {
    const float e = expf(sc[j] - mx);
    sc[j] = e;
    sum += e;
  }
  for (int off = 16; off > 0; off >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, off);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sum;
  __syncthreads();
  const float inv = 1.0f / (red[0] + red[1] + red[2] + red[3]);
  float* o = p.out + ((long long)b * p.Tq + r) * p.ld_out + h * p.d;
  for (int c = threadIdx.x; c < p.d; c += blockDim.x) {
    const float* v = p.v + (long long)b * p.Tk * p.ld_v + p.v_off + h * p.head_stride_v + c;
    float acc = 0.f;
    for (int j = 0; j < nk; ++j) acc = fmaf(sc[j] * inv, v[(long long)j * p.ld_v], acc);
    o[c] = acc;
  }
}

// ------------------------------------------------------------------------------------ text encoder input embedding
// out[b*T + t] = tok[ids[b, t]] + pos[t] (CLIPTextEmbeddings.forward): one thread per channel, rows over the grid
__global__ void embed_tokens_kernel(const qd_embed_desc p) {
  const long long total = (long long)p.B * p.T * p.C;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long row = i / p.C;
    const int c = (int)(i - row * p.C);
    const int t = (int)(row % p.T);
    const int id = p.ids[row];
    p.out[row * p.ld_out + c] = (id >= 0 && id < p.vocab) ? p.tok[(long long)id * p.C + c] + p.pos[(long long)t * p.C + c]
                                                          : __int_as_float(0x7fc00000);
  }
}

// The same attention for long sequences (first-stage decoder mid block: T = 4096, d = 512; LDM / SD weight-only levels):
// AFP_R query rows per block share every K and V row that is read, so K/V cross L2 T / AFP_R times instead of T times
// (T = 4096, d = 512: 8 GB instead of 64 GB per image).  Phase 1: a warp per key, lanes over d, AFP_R dot products per K row;
// phase 2: a warp per query row (max, exp, sum in shared memory); phase 3: a thread per output column, AFP_R accumulators.
constexpr int AFP_R = 8;
__host__ __device__ inline int afp_tk_pitch(int Tk) { return (Tk + 3) & ~3; }     // score row pitch (16-byte aligned rows)
__global__ void __launch_bounds__(256) attention_fp32_rows_kernel(const qd_attention_fp_desc p) {
  extern __shared__ float afp_sh[];
  const int tkp = afp_tk_pitch(p.Tk);
  float* qs = afp_sh;                        // [AFP_R][d]
  float* sc = afp_sh + AFP_R * p.d;          // [AFP_R][tkp]
  __shared__ float inv_s[AFP_R];
  const int bh = blockIdx.y, b = bh / p.heads, h = bh - b * p.heads;
  const int r0 = blockIdx.x * AFP_R;
  const int nr = min(AFP_R, p.Tq - r0);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < AFP_R * p.d; i += blockDim.x) {
    const int r = i / p.d, c = i - r * p.d;
    qs[i] = r < nr ? p.q[((long long)b * p.Tq + r0 + r) * p.ld_q + p.q_off + h * p.head_stride_q + c] : 0.f;
  }
  __syncthreads();
  // phase 1: a lane owns 4 consecutive channels per step: one 16-byte K load and AFP_R 16-byte shared loads of q feed
  // 4 * AFP_R FMAs (the scalar form issued one shared load per FMA and was LSU-bound).  d % 4 == 0 (checked by the launcher).
  for (int j = warp; j < p.Tk; j += 8) {
    const float* k = p.k + ((long long)b * p.Tk + j) * p.ld_k + p.k_off + h * p.head_stride_k;
    float acc[AFP_R];
#pragma unroll
    for (int r = 0; r < AFP_R; ++r) acc[r] = 0.f;
    for (int i = 4 * lane; i < p.d; i += 128) {
      const float4 kv = *reinterpret_cast<const float4*>(k + i);
#pragma unroll
      for (int r = 0; r < AFP_R; ++r) {
        const float4 qv = *reinterpret_cast<const float4*>(qs + r * p.d + i);
        acc[r] = fmaf(qv.x, kv.x, acc[r]); acc[r] = fmaf(qv.y, kv.y, acc[r]);
        acc[r] = fmaf(qv.z, kv.z, acc[r]); acc[r] = fmaf(qv.w, kv.w, acc[r]);
      }
    }
    float mine = 0.f;
#pragma unroll
    for (int r = 0; r < AFP_R; ++r) {
      float a = acc[r];
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) a += __shfl_xor_sync(0xffffffffu, a, off);
      if (lane == r) mine = a;
    }
    if (lane < AFP_R) sc[lane * tkp + j] = mine * p.scale;
  }
  __syncthreads();
  if (warp < AFP_R) {
    float* row = sc + warp * tkp;
    float mx = -INFINITY;
    for (int j = lane; j < p.Tk; j += 32) mx = fmaxf(mx, row[j]);
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
    float sum = 0.f;
    for (int j = lane; j < tkp; j += 32) {
      const float e = j < p.Tk ? expf(row[j] - mx) : 0.f;     // the pitch padding takes part in phase 3 as zeros
      row[j] = e;
      sum += e;
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, off);
    if (lane == 0) inv_s[warp] = 1.0f / sum;
  }
  __syncthreads();
  // phase 3: a thread owns an output column; 4 keys per step: AFP_R 16-byte shared loads of the probabilities (broadcast)
  // and 4 V loads feed 4 * AFP_R FMAs
  for (int c = threadIdx.x; c < p.d; c += blockDim.x) {
    const float* v = p.v + (long long)b * p.Tk * p.ld_v + p.v_off + h * p.head_stride_v + c;
    float acc[AFP_R];
#pragma unroll
    for (int r = 0; r < AFP_R; ++r) acc[r] = 0.f;
    const int t4 = p.Tk & ~3;
#pragma unroll 2
    for (int j = 0; j < t4; j += 4) {
      const float v0 = v[(long long)j * p.ld_v], v1 = v[(long long)(j + 1) * p.ld_v];
      const float v2 = v[(long long)(j + 2) * p.ld_v], v3 = v[(long long)(j + 3) * p.ld_v];
#pragma unroll
      for (int r = 0; r < AFP_R; ++r) {
        const float4 pr = *reinterpret_cast<const float4*>(sc + r * tkp + j);
        acc[r] = fmaf(pr.x, v0, acc[r]); acc[r] = fmaf(pr.y, v1, acc[r]);
        acc[r] = fmaf(pr.z, v2, acc[r]); acc[r] = fmaf(pr.w, v3, acc[r]);
      }
    }
    for (int j = t4; j < p.Tk; ++j) {
      const float vv = v[(long long)j * p.ld_v];
#pragma unroll
      for (int r = 0; r < AFP_R; ++r) acc[r] = fmaf(sc[r * tkp + j], vv, acc[r]);
    }
#pragma unroll
    for (int r = 0; r < AFP_R; ++r)
      if (r < nr) p.out[((long long)b * p.Tq + r0 + r) * p.ld_out + h * p.d + c] = acc[r] * inv_s[r];
  }
}

// ------------------------------------------------------------------------------------ groupnorm
// Three-kernel path (large feature maps).  Pass 1: a block reduces `slab` pixels x all channels to per-GROUP
// partial sums (fp32 per thread over the slab, then double, in a fixed order: results are run-to-run
// identical).  The slab length is chosen by the launcher so that the grid fills the GPU at every level of the
// UNet (fixed 64-pixel slabs would leave the 8x8 / 16x16 levels with only 16-64 blocks).
// ws layout: double part[B][nslab][groups][2], then float stats[B][groups][2].
constexpr int GN_MAX_GROUPS = 64;
__global__ void __launch_bounds__(256) gn_partial_kernel(const float* __restrict__ x, long long ld_x, int HW, int C,
                                                         int groups, int slab, int nslab, double* __restrict__ part) {
  extern __shared__ float gn_sh[];   // [2][C] per-channel sums of this slab
  const int b = blockIdx.y, sl = blockIdx.x;
  const int p0 = sl * slab;
  const int p1 = min(HW, p0 + slab);
  const int cq = C >> 2;
  for (int q = threadIdx.x; q < cq; q += blockDim.x) {
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f), ss = make_float4(0.f, 0.f, 0.f, 0.f);
    const float* base = x + ((long long)b * HW + p0) * ld_x + (q << 2);
#pragma unroll 8
    for (int p = p0; p < p1; ++p) {
      const float4 v = *reinterpret_cast<const float4*>(base);
      base += ld_x;
      s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
      ss.x += v.x * v.x; ss.y += v.y * v.y; ss.z += v.z * v.z; ss.w += v.w * v.w;
    }
    *reinterpret_cast<float4*>(gn_sh + (q << 2)) = s;
    *reinterpret_cast<float4*>(gn_sh + C + (q << 2)) = ss;
  }
  __syncthreads();
  if (threadIdx.x < 2 * groups) {
    const int g = threadIdx.x >> 1, which = threadIdx.x & 1;
    const int cpg = C / groups;
    const float* src = gn_sh + which * C + g * cpg;
    double acc = 0.0;
    for (int i = 0; i < cpg; ++i) acc += (double)src[i];
    part[(((long long)b * nslab + sl) * groups + g) * 2 + which] = acc;
  }
}
// Pass 2: per image: reduce the slabs (fixed order) -> mean, rstd per group.  One block per image.
__global__ void __launch_bounds__(256) gn_finalize_kernel(const double* __restrict__ part, int HW, int C, int groups,
                                                          int nslab, float eps, float* __restrict__ stats) {
  __shared__ double sh[4][2 * GN_MAX_GROUPS];
  const int b = blockIdx.x;
  const int n2 = 2 * groups;
  const int item = threadIdx.x % (2 * GN_MAX_GROUPS), lane4 = threadIdx.x / (2 * GN_MAX_GROUPS);   // 256 = 2 x 128
  const int nl = blockDim.x / (2 * GN_MAX_GROUPS);
  double acc = 0.0;
  if (item < n2)
    for (int sl = lane4; sl < nslab; sl += nl) acc += part[((long long)b * nslab + sl) * n2 + item];
  sh[lane4][item] = acc;
  __syncthreads();
  if (threadIdx.x < groups) {
    const int g = threadIdx.x;
    double s = 0.0, ss = 0.0;
    for (int l = 0; l < nl; ++l) { s += sh[l][2 * g]; ss += sh[l][2 * g + 1]; }
    const double cnt = (double)HW * (C / groups);
    const double mean = s / cnt;
    double var = ss / cnt - mean * mean;
    if (var < 0.0) var = 0.0;
    stats[((long long)b * groups + g) * 2] = (float)mean;
    stats[((long long)b * groups + g) * 2 + 1] = (float)(1.0 / sqrt(var + (double)eps));
  }
}
// Statistics from the producing GEMMs' epilogues (qd_gemm_desc.gn_stats): per 32-row slab and channel (sum, sum of squares).
// One block per (group, image): 128 threads stride over the group's (slab, channel) items, accumulate in double, reduce
// in a fixed order (warp shuffles, then the 4 warps through shared memory).  Replaces gn_partial + gn_finalize, i.e. one
// full read of the fp32 tensor.  (One block per IMAGE instead leaves most SMs idle.)
__global__ void __launch_bounds__(128) gn_finalize_from_stats_kernel(const float2* __restrict__ slabs, long long ld_stats,
                                                                    int HW, int C, int groups, float eps,
                                                                    float* __restrict__ stats) {
  __shared__ double sh[2][4];
  const int g = blockIdx.x, b = blockIdx.y;
  const int cpg = C / groups;
  const int nsl = HW >> 5;
  const float2* base = slabs + (long long)b * nsl * ld_stats + g * cpg;
  double s = 0.0, ss = 0.0;
  const int items = nsl * cpg;
  for (int i = threadIdx.x; i < items; i += blockDim.x) {
    const int sl = i / cpg, ch = i - sl * cpg;
    const float2 v = base[(long long)sl * ld_stats + ch];
    s += (double)v.x;
    ss += (double)v.y;
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, off);
    ss += __shfl_xor_sync(0xffffffffu, ss, off);
  }
  if ((threadIdx.x & 31) == 0) { sh[0][threadIdx.x >> 5] = s; sh[1][threadIdx.x >> 5] = ss; }
  __syncthreads();
  if (threadIdx.x == 0) {
    s = (sh[0][0] + sh[0][1]) + (sh[0][2] + sh[0][3]);
    ss = (sh[1][0] + sh[1][1]) + (sh[1][2] + sh[1][3]);
    const double cnt = (double)HW * cpg;
    const double mean = s / cnt;
    double var = ss / cnt - mean * mean;
    if (var < 0.0) var = 0.0;
    stats[((long long)b * groups + g) * 2] = (float)mean;
    stats[((long long)b * groups + g) * 2 + 1] = (float)(1.0 / sqrt(var + (double)eps));
  }
}

// Pass 3: normalise + affine (+scale-shift) (+SiLU) + quantise for each consumer.
// Block = TX channel quads x TY rows (TX * TY <= 256); grid (channel slabs, row chunks, B).  A thread owns ONE channel
// quad: it folds mean / rstd / gamma / beta (/ scale-shift) into y = a*x + b once (8 registers) and then streams its rows,
// GN_BATCH independent 16-byte loads in flight before the first store.  The first version (one block of C/4 threads per
// 32 rows, up to 4 quads per thread) needed 118 registers and ran 96-thread blocks at 21 % occupancy: every warp sat
// on its first FFMA waiting for DRAM.  The consumer count and the raw
// output are template parameters so that the common single-consumer case carries one quantizer's constants only.
// Occupancy: the single-consumer kernel runs 4-row load batches under a 64-register cap (4 blocks = 32 warps per SM) so
// that more warps wait on DRAM at once; the multi-consumer / raw-output variants keep 8 rows.
constexpr int GN_BATCH = 8;                                   // host: rows per block are multiples of GN_BATCH * TY
__host__ __device__ constexpr int gn_apply_batch(int NOUT, bool RAW) { return (NOUT <= 1 && !RAW) ? 4 : 8; }
__host__ __device__ constexpr int gn_apply_minblocks(int NOUT, bool RAW) { return (NOUT <= 1 && !RAW) ? 4 : 1; }
template <int NOUT, bool RAW>
__global__ void __launch_bounds__(256, gn_apply_minblocks(NOUT, RAW)) gn_apply_kernel(const qd_groupnorm_desc p, const float* __restrict__ stats,
                                                       int rows_per_block, int TX) {
  constexpr int NB = gn_apply_batch(NOUT, RAW);      // rows per thread and load batch
  const int b = blockIdx.z;
  const int tx = threadIdx.x % TX, ty = threadIdx.x / TX;
  const int TY = blockDim.x / TX;
  const int q = blockIdx.x * TX + tx;                 // channel quad
  const int cq = p.C >> 2;
  if (q >= cq || ty >= TY) return;
  const int c = q << 2;
  const int cpg = p.C / p.groups;
  float ca[4], cb[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int ch = c + j;
    const int g = ch / cpg;
    const float mean = stats[((long long)b * p.groups + g) * 2];
    const float rstd = stats[((long long)b * p.groups + g) * 2 + 1];
    float a = rstd * p.gamma[ch];
    float bb = p.beta[ch] - mean * a;
    if (p.ss_scale) {
      const float s1 = 1.0f + p.ss_scale[(long long)b * p.ld_ss + ch];
      a *= s1;
      bb = bb * s1 + p.ss_shift[(long long)b * p.ld_ss + ch];
    }
    ca[j] = a;
    cb[j] = bb;
  }
  QuantK qk[NOUT > 0 ? NOUT : 1];
#pragma unroll
  for (int o = 0; o < NOUT; ++o) qk[o] = make_quantk(p.q[o]);
  QuantK kr = make_quantk(p.q_raw[0]);
  if (RAW && c >= p.raw_split) kr = make_quantk(p.q_raw[1]);
  const int r0 = blockIdx.y * rows_per_block;
  const int r1 = min(p.HW, r0 + rows_per_block);
  const long long step = (long long)TY * p.ld_x;
  for (int rb = r0 + ty; rb < r1; rb += NB * TY) {
    const float* xp = p.x + ((long long)b * p.HW + rb) * p.ld_x + c;
    float4 vv[NB];
#pragma unroll
    for (int i = 0; i < NB; ++i)
      if (rb + i * TY < r1) vv[i] = *reinterpret_cast<const float4*>(xp + i * step);
#pragma unroll
    for (int i = 0; i < NB; ++i) {
      const int r = rb + i * TY;
      if (r >= r1) break;
      const float4 v = vv[i];
      const long long row = (long long)b * p.HW + r;
      if (RAW)
        *reinterpret_cast<uint32_t*>(reinterpret_cast<uint8_t*>(p.raw_q) + row * p.ld_raw + c) =
            pack4(quant_code(v.x, kr), quant_code(v.y, kr), quant_code(v.z, kr), quant_code(v.w, kr));
      float y[4] = {fmaf(v.x, ca[0], cb[0]), fmaf(v.y, ca[1], cb[1]), fmaf(v.z, ca[2], cb[2]), fmaf(v.w, ca[3], cb[3])};
      if (p.silu) {
#pragma unroll
        for (int j = 0; j < 4; ++j) y[j] = silu_f(y[j]);
      }
      if (p.out_f) *reinterpret_cast<float4*>(p.out_f + row * p.ld_f + c) = make_float4(y[0], y[1], y[2], y[3]);
#pragma unroll
      for (int o = 0; o < NOUT; ++o)
        *reinterpret_cast<uint32_t*>(reinterpret_cast<uint8_t*>(p.out_q[o]) + row * p.ld_q[o] + c) =
            pack4(quant_code_fast(y[0], qk[o]), quant_code_fast(y[1], qk[o]), quant_code_fast(y[2], qk[o]),
                  quant_code_fast(y[3], qk[o]));
    }
  }
}

// Single-kernel path (small feature maps: HW * C/groups <= 512 threads x 2*GN_NU values).  One block per
// (image, group): the group's HW x cpg values are read ONCE into registers, mean and variance are computed in
// two passes over those registers (block reductions in double, fixed order), then normalised / activated /
// quantised straight from registers.  No workspace, one launch instead of three, x read once.
constexpr int GN_NU = 20;   // float2 units per thread
__device__ __forceinline__ double gn_block_sum(double v, double* sh) {
  for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  __syncthreads();                 // sh may still be read from the previous reduction
  if (l == 0) sh[w] = v;
  __syncthreads();
  double t = 0.0;
  const int nw = blockDim.x >> 5;
  for (int i = 0; i < nw; ++i) t += sh[i];   // same order in every thread
  return t;
}
__global__ void __launch_bounds__(512) gn_fused_small_kernel(const qd_groupnorm_desc p) {
  __shared__ double red[16];
  __shared__ float2 coef[2][64];   // per channel pair of the group: (a0, a1), (b0, b1); cpg <= 128
  const int b = blockIdx.y, g = blockIdx.x;
  const int cpg = p.C / p.groups;
  const int U = cpg >> 1;                 // float2 units per row
  const int total = p.HW * U;
  const int T = blockDim.x;
  const float* xg = p.x + (long long)b * p.HW * p.ld_x + g * cpg;
  float2 v[GN_NU];
  // unit u = threadIdx.x + k*T -> (row, cu); advanced incrementally (no division in the loop)
  const int dr = T / U, dc = T - dr * U;
  int row = threadIdx.x / U, cu = threadIdx.x - row * U;
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < GN_NU; ++k) {
    v[k] = make_float2(0.f, 0.f);
    if (threadIdx.x + k * T < total) v[k] = *reinterpret_cast<const float2*>(xg + (long long)row * p.ld_x + 2 * cu);
    s += v[k].x + v[k].y;
    row += dr; cu += dc;
    if (cu >= U) { cu -= U; ++row; }
  }
  const double cnt = (double)p.HW * cpg;
  const float mean = (float)(gn_block_sum((double)s, red) / cnt);
  float s2 = 0.f;
#pragma unroll
  for (int k = 0; k < GN_NU; ++k) {
    if (threadIdx.x + k * T < total) {
      const float dx = v[k].x - mean, dy = v[k].y - mean;
      s2 += dx * dx + dy * dy;
    }
  }
  const float rstd = (float)(1.0 / sqrt(gn_block_sum((double)s2, red) / cnt + (double)p.eps));
  if (threadIdx.x < U) {
    float a[2], bb[2];
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int ch = g * cpg + 2 * threadIdx.x + j;
      a[j] = rstd * p.gamma[ch];
      bb[j] = p.beta[ch] - mean * a[j];
      if (p.ss_scale) {
        const float s1 = 1.0f + p.ss_scale[(long long)b * p.ld_ss + ch];
        a[j] *= s1;
        bb[j] = bb[j] * s1 + p.ss_shift[(long long)b * p.ld_ss + ch];
      }
    }
    coef[0][threadIdx.x] = make_float2(a[0], a[1]);
    coef[1][threadIdx.x] = make_float2(bb[0], bb[1]);
  }
  __syncthreads();
  const QuantK qk[3] = {make_quantk(p.q[0]), make_quantk(p.q[1]), make_quantk(p.q[2])};
  const QuantK qraw[2] = {make_quantk(p.q_raw[0]), make_quantk(p.q_raw[1])};
  row = threadIdx.x / U; cu = threadIdx.x - row * U;
#pragma unroll
  for (int k = 0; k < GN_NU; ++k) {
    if (threadIdx.x + k * T < total) {
      const float2 a = coef[0][cu], bb = coef[1][cu];
      float y0 = fmaf(v[k].x, a.x, bb.x), y1 = fmaf(v[k].y, a.y, bb.y);
      if (p.silu) { y0 = silu_f(y0); y1 = silu_f(y1); }
      const long long r = (long long)b * p.HW + row;
      const int c = g * cpg + 2 * cu;
      if (p.out_f) *reinterpret_cast<float2*>(p.out_f + r * p.ld_f + c) = make_float2(y0, y1);
      if (p.raw_q) {
        const QuantK& kr = qraw[c < p.raw_split ? 0 : 1];
        *reinterpret_cast<uint16_t*>(reinterpret_cast<uint8_t*>(p.raw_q) + r * p.ld_raw + c) =
            (uint16_t)(quant_code(v[k].x, kr) | (quant_code(v[k].y, kr) << 8));
      }
#pragma unroll
      for (int o = 0; o < 3; ++o) {
        if (o < p.n_out)
          *reinterpret_cast<uint16_t*>(reinterpret_cast<uint8_t*>(p.out_q[o]) + r * p.ld_q[o] + c) =
              (uint16_t)(quant_code_fast(y0, qk[o]) | (quant_code_fast(y1, qk[o]) << 8));
      }
    }
    row += dr; cu += dc;
    if (cu >= U) { cu -= U; ++row; }
  }
}

// ------------------------------------------------------------------------------------ layernorm
// One warp per row; the row lives in registers (NVEC float4 per lane, compile-time so it is NOT demoted to local
// memory: the first version indexed a float4[32] array with a run-time trip count and spilled it),
// two-pass mean / variance in fp32, then 1-3 consumer quantizers.
template <int NVEC>
__global__ void __launch_bounds__(256) layernorm_quant_kernel(const qd_layernorm_desc p) {
  const int warps_per_block = blockDim.x >> 5;
  const int lane = threadIdx.x & 31;
  const int cq = p.C >> 2;
  const QuantK qk[3] = {make_quantk(p.q[0]), make_quantk(p.q[1]), make_quantk(p.q[2])};
  float4 g[NVEC], be[NVEC];
#pragma unroll
  for (int k = 0; k < NVEC; ++k) {
    const int q = lane + 32 * k;
    g[k] = q < cq ? *reinterpret_cast<const float4*>(p.gamma + (q << 2)) : make_float4(0.f, 0.f, 0.f, 0.f);
    be[k] = q < cq ? *reinterpret_cast<const float4*>(p.beta + (q << 2)) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  const float inv_c = 1.0f / (float)p.C;
  // the next row of this warp is fetched while the current one is reduced / quantised (register double buffer)
  auto load_row = [&](long long r, float4 (&dst)[NVEC]) {
    const float* xr = p.x + r * p.ld_x;
#pragma unroll
    for (int k = 0; k < NVEC; ++k) {
      const int q = lane + 32 * k;
      dst[k] = q < cq ? *reinterpret_cast<const float4*>(xr + (q << 2)) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  };
  const long long stride = (long long)gridDim.x * warps_per_block;
  long long row = (long long)blockIdx.x * warps_per_block + (threadIdx.x >> 5);
  constexpr bool DB = NVEC <= 5;          // wider rows: the second buffer would cost occupancy (or spill)
  float4 v[NVEC], vn[DB ? NVEC : 1];
  if (DB && row < p.M) load_row(row, v);
  for (; row < p.M; row += stride) {
    if constexpr (DB) {
      if (row + stride < p.M) load_row(row + stride, vn);
    } else {
      load_row(row, v);
    }
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < NVEC; ++k) s += (v[k].x + v[k].y) + (v[k].z + v[k].w);
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
    const float mean = s * inv_c;
    float ss = 0.f;
#pragma unroll
    for (int k = 0; k < NVEC; ++k) {
      if (lane + 32 * k < cq) {
        const float a = v[k].x - mean, b = v[k].y - mean, c = v[k].z - mean, d = v[k].w - mean;
        ss += (a * a + b * b) + (c * c + d * d);
      }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, off);
    const float rstd = rsqrtf(ss * inv_c + p.eps);
#pragma unroll
    for (int k = 0; k < NVEC; ++k) {
      const int q = lane + 32 * k;
      if (q < cq) {
        const int c = q << 2;
        const float y0 = (v[k].x - mean) * rstd * g[k].x + be[k].x;
        const float y1 = (v[k].y - mean) * rstd * g[k].y + be[k].y;
        const float y2 = (v[k].z - mean) * rstd * g[k].z + be[k].z;
        const float y3 = (v[k].w - mean) * rstd * g[k].w + be[k].w;
        if (p.out_f) *reinterpret_cast<float4*>(p.out_f + row * p.ld_f + c) = make_float4(y0, y1, y2, y3);
#pragma unroll
        for (int o = 0; o < 3; ++o) {
          if (o < p.n_out) {
            const uint32_t code = pack4(quant_code_fast(y0, qk[o]), quant_code_fast(y1, qk[o]), quant_code_fast(y2, qk[o]),
                                        quant_code_fast(y3, qk[o]));
            *reinterpret_cast<uint32_t*>(reinterpret_cast<uint8_t*>(p.out_q[o]) + row * p.ld_q[o] + c) = code;
          }
        }
      }
    }
    if constexpr (DB) {
#pragma unroll
      for (int k = 0; k < NVEC; ++k) v[k] = vn[k];
    }
  }
}

// ------------------------------------------------------------------------------------ im2col
__global__ void im2col_kernel(const qd_im2col_desc p) {
  // one thread = one byte-quad where possible; generic byte path keeps it simple (small tensors).
  const long long rows = (long long)p.B * p.Ho * p.Wo;
  const int K = 9 * p.C;
  const long long total = rows * p.ld_dst;
  const uint8_t* src = reinterpret_cast<const uint8_t*>(p.src);
  uint8_t* dst = reinterpret_cast<uint8_t*>(p.dst);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / p.ld_dst;
    const int k = (int)(i - r * p.ld_dst);
    uint8_t val = 0;
    if (k < K) {
      const int tap = k / p.C, c = k - tap * p.C;
      const int ky = tap / 3, kx = tap - ky * 3;
      const int wo = (int)(r % p.Wo);
      const long long t = r / p.Wo;
      const int ho = (int)(t % p.Ho);
      const long long b = t / p.Ho;
      const int h = ho * p.stride - p.pad_top + ky;
      const int w = wo * p.stride - p.pad_left + kx;
      if (h >= 0 && h < p.H && w >= 0 && w < p.W)
        val = src[((b * p.H + h) * p.W + w) * p.C + c];
      else
        val = (uint8_t)p.pad_code;
    }
    dst[i] = val;
  }
}

// 16-byte variant (C % 16 == 0: the stride-2 Downsample convs): one thread = 16 channels of one tap of one output pixel
__global__ void im2col_vec_kernel(const qd_im2col_desc p) {
  const int c16 = p.C >> 4;
  const long long total = (long long)p.B * p.Ho * p.Wo * 9 * c16;
  const uint8_t* src = reinterpret_cast<const uint8_t*>(p.src);
  uint8_t* dst = reinterpret_cast<uint8_t*>(p.dst);
  const uint32_t pc = (uint32_t)(p.pad_code & 0xFF) * 0x01010101u;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int cc = (int)(i % c16);
    long long t = i / c16;
    const int tap = (int)(t % 9);
    const long long r = t / 9;
    const int ky = tap / 3, kx = tap - ky * 3;
    const int wo = (int)(r % p.Wo);
    const long long t2 = r / p.Wo;
    const int ho = (int)(t2 % p.Ho);
    const long long b = t2 / p.Ho;
    const int h = ho * p.stride - p.pad_top + ky;
    const int w = wo * p.stride - p.pad_left + kx;
    uint4 v = make_uint4(pc, pc, pc, pc);
    if (h >= 0 && h < p.H && w >= 0 && w < p.W)
      v = *reinterpret_cast<const uint4*>(src + ((b * p.H + h) * p.W + w) * (long long)p.C + (cc << 4));
    *reinterpret_cast<uint4*>(dst + r * p.ld_dst + tap * p.C + (cc << 4)) = v;
  }
}

// ------------------------------------------------------------------------------------ misc fp32
__global__ void timestep_embedding_kernel(const float* __restrict__ t, const float* __restrict__ freqs, int B, int dim,
                                          int mode, float* __restrict__ out) {
  const int half = dim / 2;
  const int total = B * half;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int b = i / half, k = i - b * half;
    // mode 0 (ldm util.py:162-166): emb = [cos, sin]; mode 1 (ddim diffusion.py:16-21): emb = [sin, cos].
    // freqs[] comes from the host (identical fp32 expression as the reference) so a = t*freq is bit-identical.
    const float a = t[b] * freqs[k];
    const float sv = sinf(a), cv = cosf(a);
    float* o = out + (long long)b * dim;
    if (mode == 0) { o[k] = cv; o[half + k] = sv; }
    else           { o[k] = sv; o[half + k] = cv; }
    if ((dim & 1) && k == 0) o[dim - 1] = 0.f;
  }
}

__global__ void copy2d_kernel(const float* __restrict__ src, long long ld_src, float* __restrict__ dst,
                              long long ld_dst, int M, int C) {
  const int cq = C >> 2;
  const long long total = (long long)M * cq;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / cq;
    const int c = (int)(i - r * cq) << 2;
    *reinterpret_cast<float4*>(dst + r * ld_dst + c) = *reinterpret_cast<const float4*>(src + r * ld_src + c);
  }
}

__global__ void nchw_to_nhwc_kernel(const float* __restrict__ src, float* __restrict__ dst, int B, int C, int HW) {
  const long long total = (long long)B * C * HW;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    // i indexes dst (b, p, c)
    const int c = (int)(i % C);
    const long long t = i / C;
    const int p = (int)(t % HW);
    const long long b = t / HW;
    dst[i] = src[(b * C + c) * HW + p];
  }
}
__global__ void nhwc_to_nchw_kernel(const float* __restrict__ src, float* __restrict__ dst, int B, int C, int HW) {
  const long long total = (long long)B * C * HW;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    // i indexes dst (b, c, p)
    const int p = (int)(i % HW);
    const long long t = i / HW;
    const int c = (int)(t % C);
    const long long b = t / C;
    dst[i] = src[(b * HW + p) * C + c];
  }
}

__global__ void avgpool2x_kernel(const float* __restrict__ src, float* __restrict__ dst, int B, int H, int W, int C) {
  const int Ho = H / 2, Wo = W / 2, cq = C >> 2;
  const long long total = (long long)B * Ho * Wo * cq;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % cq) << 2;
    long long t = i / cq;
    const int wo = (int)(t % Wo); t /= Wo;
    const int ho = (int)(t % Ho);
    const long long b = t / Ho;
    const float* s = src + ((b * H + 2 * ho) * W + 2 * wo) * (long long)C + c;
    const float4 a = *reinterpret_cast<const float4*>(s);
    const float4 bq = *reinterpret_cast<const float4*>(s + C);
    const float4 cc = *reinterpret_cast<const float4*>(s + (long long)W * C);
    const float4 d = *reinterpret_cast<const float4*>(s + (long long)W * C + C);
    float4 o;
    o.x = (a.x + bq.x + cc.x + d.x) * 0.25f;
    o.y = (a.y + bq.y + cc.y + d.y) * 0.25f;
    o.z = (a.z + bq.z + cc.z + d.z) * 0.25f;
    o.w = (a.w + bq.w + cc.w + d.w) * 0.25f;
    *reinterpret_cast<float4*>(dst + ((b * Ho + ho) * Wo + wo) * (long long)C + c) = o;
  }
}
__global__ void upsample2x_f32_kernel(const float* __restrict__ src, float* __restrict__ dst, int B, int H, int W,
                                      int C) {
  const int H2 = 2 * H, W2 = 2 * W, cq = C >> 2;
  const long long total = (long long)B * H2 * W2 * cq;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % cq) << 2;
    long long t = i / cq;
    const int w2 = (int)(t % W2); t /= W2;
    const int h2 = (int)(t % H2);
    const long long b = t / H2;
    *reinterpret_cast<float4*>(dst + ((b * H2 + h2) * W2 + w2) * (long long)C + c) =
        *reinterpret_cast<const float4*>(src + ((b * H + (h2 >> 1)) * W + (w2 >> 1)) * (long long)C + c);
  }
}

// In-place softmax over the rows of an fp32 matrix (first-stage AttnBlock on the tensor cores: scores from the plane GEMM,
// probabilities into the next plane split; model.py:190-192).  One block per row, exact expf, fixed reduction order.
__global__ void __launch_bounds__(256) softmax_rows_kernel(float* __restrict__ x, long long ld, int cols) {
  __shared__ float red[8];
  float* row = x + (long long)blockIdx.x * ld;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float mx = -INFINITY;
  for (int j = threadIdx.x; j < cols; j += blockDim.x) mx = fmaxf(mx, row[j]);
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
  if (lane == 0) red[warp] = mx;
  __syncthreads();
  mx = red[0];
#pragma unroll
  for (int i = 1; i < 8; ++i) mx = fmaxf(mx, red[i]);
  __syncthreads();
  float sum = 0.f;
  for (int j = threadIdx.x; j < cols; j += blockDim.x) {
    const float e = expf(row[j] - mx);
    row[j] = e;
    sum += e;
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, off);
  if (lane == 0) red[warp] = sum;
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) tot += red[i];
  const float inv = 1.0f / tot;
  for (int j = threadIdx.x; j < cols; j += blockDim.x) row[j] *= inv;
}

// ------------------------------------------------------------------------------------ VQ first stage
// Nearest codebook entry per latent pixel (VectorQuantizer2.forward of taming-transformers, the `quantize` step of
// VQModelInterface.decode, ldm/models/autoencoder.py:274-283): d_j = sum(z^2) + sum(e_j^2) - 2 z.e_j in fp32 with the
// reference's association, argmin with the lowest index on ties, output z + (e - z) (the straight-through form: it
// rounds).  One warp per pixel, lanes stride over the codebook.
constexpr int VQ_MAX_C = 16;
constexpr int VQ_NONE = 0x7fffffff;       // a lane that saw no codebook entry (n_e < 32)
// torch.argmin's order: a NaN distance is smaller than every number (the first NaN wins), then the lowest index on ties.
// Every real entry beats VQ_NONE, so the index stays in range even when every distance is +inf or NaN.
__device__ __forceinline__ bool vq_better(float d, int i, float best, int bi) {
  if (i == VQ_NONE) return false;
  if (bi == VQ_NONE) return true;
  const bool dn = d != d, bn = best != best;
  if (dn || bn) return dn && (!bn || i < bi);
  return d < best || (d == best && i < bi);
}
__global__ void __launch_bounds__(256) vq_lookup_kernel(const float* __restrict__ z, long long ld_z, const float* __restrict__ cb,
                                                        float* __restrict__ out, long long ld_out, int rows, int C, int n_e) {
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long r = warp; r < rows; r += nwarps) {
    float zv[VQ_MAX_C];
    float zz = 0.f;
#pragma unroll
    for (int c = 0; c < VQ_MAX_C; ++c) {
      zv[c] = c < C ? z[r * ld_z + c] : 0.f;
      if (c < C) zz = __fadd_rn(zz, __fmul_rn(zv[c], zv[c]));
    }
    float best = INFINITY;
    int bi = VQ_NONE;
    for (int j = lane; j < n_e; j += 32) {
      const float* e = cb + (long long)j * C;
      float ee = 0.f, dot = 0.f;
#pragma unroll
      for (int c = 0; c < VQ_MAX_C; ++c) {
        if (c < C) {
          const float ev = __ldg(e + c);
          ee = __fadd_rn(ee, __fmul_rn(ev, ev));
          dot = fmaf(zv[c], ev, dot);
        }
      }
      const float dj = __fsub_rn(__fadd_rn(zz, ee), __fmul_rn(2.0f, dot));
      if (vq_better(dj, j, best, bi)) { best = dj; bi = j; }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      const float ob = __shfl_xor_sync(0xffffffffu, best, off);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, off);
      if (vq_better(ob, oi, best, bi)) { best = ob; bi = oi; }
    }
    if (lane < C) {
      const float zc = z[r * ld_z + lane];
      out[r * ld_out + lane] = __fadd_rn(zc, __fsub_rn(__ldg(cb + (long long)bi * C + lane), zc));
    }
  }
}

// ------------------------------------------------------------------------------------ sampler
__global__ void lincomb3_kernel(float* __restrict__ out, float a, const float* __restrict__ x, float b,
                                const float* __restrict__ y, float c, const float* __restrict__ z, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float v = a * x[i];
    if (y) v = fmaf(b, y[i], v);
    if (z) v = fmaf(c, z[i], v);
    out[i] = v;
  }
}

__global__ void sampler_step_kernel(const qd_sampler_desc p) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < p.n;
       i += (long long)gridDim.x * blockDim.x) {
    float e;
    if (p.cfg_scale != 0.f) {
      const float eu = p.eps[i], ec = p.eps[p.n + i];
      e = eu + p.cfg_scale * (ec - eu);
    } else {
      e = p.eps[i];
    }
    if (p.eps_out) p.eps_out[i] = e;
    float ep = p.c_e0 * e;
    if (p.old1) ep += p.c_e1 * p.old1[i];
    if (p.old2) ep += p.c_e2 * p.old2[i];
    if (p.old3) ep += p.c_e3 * p.old3[i];
    const float x = p.x[i];
    const float x0 = (x - p.sqrt_one_minus_at * ep) / p.sqrt_at;
    float xp = p.sqrt_a_prev * x0 + p.dir_coef * ep;
    if (p.noise) xp += p.sigma * p.noise[i];
    if (p.pred_x0) p.pred_x0[i] = x0;
    p.x_prev[i] = xp;
  }
}

// Ancestral (posterior-mean) update: x0 = c_x x - c_e eps, optionally clamped to [-1, 1] (NaN passes through like
// torch.clamp), x_prev = m_x0 x0 + m_x x + sigma noise.
__global__ void ancestral_step_kernel(const qd_ancestral_desc p) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < p.n;
       i += (long long)gridDim.x * blockDim.x) {
    const float x = p.x[i];
    float x0 = p.c_x * x - p.c_e * p.eps[i];
    if (p.clamp) x0 = x0 < -1.f ? -1.f : (x0 > 1.f ? 1.f : x0);
    float xp = p.m_x0 * x0 + p.m_x * x;
    if (p.noise) xp += p.sigma * p.noise[i];
    if (p.pred_x0) p.pred_x0[i] = x0;
    p.x_prev[i] = xp;
  }
}

}  // namespace qd
