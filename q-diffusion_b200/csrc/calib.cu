// Calibration entry points of libqdiff_b200.so (see include/qdiff_b200.h): the channel-wise 'mse' weight scale search.
// Its own translation unit: calibration runs once per checkpoint, never inside a recorded engine program.
#include <cuda_runtime.h>

#include <cstdint>
#include <vector>

#include "../../include/qdiff_b200.h"
#include "runtime.cuh"

namespace qd {

constexpr int WS_THREADS = 256;
constexpr int WS_WARPS = WS_THREADS / 32;
constexpr int WS_CANDIDATES = 80;
constexpr int WS_SMEM_MAX = 200 * 1024;   // rows up to 51200 elements are staged in shared memory, longer ones read from L2

struct WsCandidate {
  float delta, zp;
};

// Candidate i of UniformAffineQuantizer.quantize(x, x_max * s_i, x_min * s_i), qdiff/quant_layer.py:166-190: the ratio is
// a Python double rounded to fp32 when torch multiplies the fp32 extremes by it; every step after that is one fp32 IEEE
// operation (the explicit _rn intrinsics keep nvcc from contracting the double or fp32 steps into FMAs).
__device__ __forceinline__ WsCandidate ws_candidate(float x_max, float x_min, int i, float levels) {
  const float s = (float)__dsub_rn(1.0, __dmul_rn((double)i, 0.01));
  const float new_max = __fmul_rn(x_max, s), new_min = __fmul_rn(x_min, s);
  WsCandidate c;
  c.delta = __fdiv_rn(__fsub_rn(new_max, new_min), levels);
  c.zp = rintf(__fdiv_rn(-new_min, c.delta));
  return c;
}

// One CTA per row.  The row is read once into shared memory (or, past WS_SMEM_MAX, straight from global memory); each
// candidate is then one pass over it.  Every thread sums its own elements k = tid, tid + 256, ... in float64, the warp
// folds its lanes by a fixed shuffle tree and the 8 warp sums are added in warp order: the score does not depend on
// scheduling.  The quantise step is the reference's own fp32 sequence, not quant_math.cuh's code path: the zero point can
// lie outside [0, 2^n - 1] (single-signed rows) and rne(x / delta) + zp is an fp32 addition in the reference.
__global__ void __launch_bounds__(WS_THREADS) weight_scale_search_kernel(qd_wsearch_desc d) {
  extern __shared__ float ws_row[];
  __shared__ double part[WS_WARPS][WS_CANDIDATES];
  __shared__ float red_max[WS_WARPS], red_min[WS_WARPS];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const long long r = blockIdx.x;
  const int K = d.k1 - d.k0;
  const float* src = d.w + r * d.ld + d.k0;
  const bool staged = (long long)K * 4 <= WS_SMEM_MAX;
  const float* x = staged ? ws_row : src;

  float mx = -INFINITY, mn = INFINITY;
  bool bad = false;
  for (int k = tid; k < K; k += WS_THREADS) {
    const float v = src[k];
    if (staged) ws_row[k] = v;
    bad |= !isfinite(v);
    mx = fmaxf(mx, v);
    mn = fminf(mn, v);
  }
  for (int o = 16; o > 0; o >>= 1) {
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
  }
  if (lane == 0) red_max[warp] = mx, red_min[warp] = mn;
  bad = __syncthreads_or(bad);
  mx = red_max[0];
  mn = red_min[0];
  for (int w = 1; w < WS_WARPS; ++w) mx = fmaxf(mx, red_max[w]), mn = fminf(mn, red_min[w]);
  if (bad || !(mx > mn)) {     // non-finite or constant row: no candidate has a usable step
    if (tid == 0) d.index[r] = -1;
    return;
  }

  const float levels = (float)((1 << d.n_bits) - 1);
  for (int i = 0; i < WS_CANDIDATES; ++i) {
    const WsCandidate c = ws_candidate(mx, mn, i, levels);
    double acc = 0.0;
    if (c.delta > 0.f && isfinite(c.delta)) {
      for (int k = tid; k < K; k += WS_THREADS) {
        const float v = x[k];
        const float t = fminf(fmaxf(__fadd_rn(rintf(__fdiv_rn(v, c.delta)), c.zp), 0.f), levels);
        const float xq = __fmul_rn(__fsub_rn(t, c.zp), c.delta);
        const float e = fabsf(__fsub_rn(v, xq));
        if (e > 0.f) acc += pow((double)e, 2.4);
      }
    } else {
      acc = INFINITY;        // the reference's score is NaN here and never wins the strict comparison
    }
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) part[warp][i] = acc;
  }
  __syncthreads();
  if (tid == 0) {
    int best_i = -1;
    double best = INFINITY;
    for (int i = 0; i < WS_CANDIDATES; ++i) {
      double s = part[0][i];
      for (int w = 1; w < WS_WARPS; ++w) s += part[w][i];
      if (s < best) best = s, best_i = i;
    }
    d.index[r] = best_i;
    if (best_i >= 0) {
      const WsCandidate c = ws_candidate(mx, mn, best_i, levels);
      d.delta[r] = c.delta;
      d.zero_point[r] = c.zp;
      if (d.score) d.score[r] = best;
    }
  }
}

}  // namespace qd

namespace {

using namespace qdr;

int launch_weight_scale_search(const qd_wsearch_desc& d, cudaStream_t s) {
  if (!d.w || !d.delta || !d.zero_point || !d.index) return fail(QD_ERR_BAD_ARG, "weight_scale_search: null pointer");
  if (d.N <= 0 || d.k0 < 0 || d.k1 <= d.k0 || d.k1 > d.ld)
    return fail(QD_ERR_BAD_ARG, "weight_scale_search: N=%d, columns [%d, %d) of rows with pitch %lld", d.N, d.k0, d.k1, d.ld);
  if (d.n_bits < 2 || d.n_bits > 8) return fail(QD_ERR_UNSUPPORTED, "weight_scale_search: n_bits=%d not in [2, 8]", d.n_bits);
  const long long K = d.k1 - d.k0;
  const int smem = K * 4 <= qd::WS_SMEM_MAX ? (int)(K * 4) : 0;
  static std::atomic<unsigned long long> optin{0};
  if (int rc = ensure_smem_optin(qd::weight_scale_search_kernel, qd::WS_SMEM_MAX, optin, "weight_scale_search")) return rc;
  launch_k(qd::weight_scale_search_kernel, dim3(d.N), qd::WS_THREADS, smem, s, d);
  if (int rc = check_launch("weight_scale_search_kernel")) return rc;
  std::vector<int32_t> idx(d.N);
  cudaError_t e = cudaMemcpyAsync(idx.data(), d.index, sizeof(int32_t) * d.N, cudaMemcpyDeviceToHost, s);
  if (e == cudaSuccess) e = cudaStreamSynchronize(s);
  if (e != cudaSuccess) return fail(QD_ERR_CUDA, "weight_scale_search: %s", cudaGetErrorString(e));
  for (int r = 0; r < d.N; ++r)
    if (idx[r] < 0)
      return fail(QD_ERR_UNSUPPORTED, "weight_scale_search: row %d (columns [%d, %d)) is constant or not finite: no "
                  "candidate has a usable step", r, d.k0, d.k1);
  return QD_OK;
}

}  // namespace

extern "C" {

int qd_weight_scale_search(const qd_wsearch_desc* d, qd_stream_t s) {
  if (!d) return fail(QD_ERR_BAD_ARG, "null desc");
  return launch_weight_scale_search(*d, (cudaStream_t)s);
}

}  // extern "C"
