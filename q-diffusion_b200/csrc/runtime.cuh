// Host-side plumbing shared by every translation unit of libqdiff_b200.so: the thread's last-error text behind
// qd_last_error, the launch counter behind qd_launch_count, the one launch helper and the shared-memory opt-in.
// Defined once in engine.cu; calib.cu uses the same objects so an error raised there reads back through qd_last_error.
#pragma once
#include <cuda_runtime.h>

#include <atomic>
#include <utility>

#include "../../include/qdiff_b200.h"

namespace qdr {

extern thread_local char g_err[512];
extern std::atomic<long long> g_launches;
constexpr int kMaxDevices = 64;

int fail(int code, const char* fmt, ...);
int check_launch(const char* what);
int current_device();

// Every kernel launch of the library goes through here.
// Programmatic dependent launch (cudaLaunchAttributeProgrammaticStreamSerialization on every launch + griddepcontrol.wait /
// launch_dependents in every kernel) showed no gain inside the CUDA graphs on the previous GPU generation (not re-measured
// on the H100), so the launches stay plain.
template <typename... KArgs, typename... Args>
void launch_k(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = s;
  cudaLaunchKernelEx(&cfg, kern, KArgs(std::forward<Args>(args))...);
}

// cudaFuncAttributeMaxDynamicSharedMemorySize is a PER-DEVICE attribute of a kernel: opt in once per (kernel, device).
// `done` is the kernel instantiation's own bitmask of devices already configured.
template <typename K>
int ensure_smem_optin(K kern, int bytes, std::atomic<unsigned long long>& done, const char* what) {
  const int dev = current_device();
  if (dev < 0 || dev >= kMaxDevices) return fail(QD_ERR_CUDA, "%s: no current CUDA device", what);
  const unsigned long long bit = 1ull << dev;
  if (done.load(std::memory_order_acquire) & bit) return QD_OK;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e != cudaSuccess) return fail(QD_ERR_CUDA, "%s: cudaFuncSetAttribute: %s", what, cudaGetErrorString(e));
  done.fetch_or(bit, std::memory_order_release);
  return QD_OK;
}

}  // namespace qdr
