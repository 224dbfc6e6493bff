// Shared helpers for the sm_90a kernels of libtriforce_b200.so.
#pragma once

#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/triforce_b200.h"

namespace tf {

void set_error(const char* fmt, ...);

#define TF_CHECK_ARG(cond, ...)            \
  do {                                     \
    if (!(cond)) {                         \
      ::tf::set_error(__VA_ARGS__);        \
      return TF_ERR_INVALID;               \
    }                                      \
  } while (0)

#define TF_CHECK_SUPPORTED(cond, ...)      \
  do {                                     \
    if (!(cond)) {                         \
      ::tf::set_error(__VA_ARGS__);        \
      return TF_ERR_UNSUPPORTED;           \
    }                                      \
  } while (0)

#define TF_CHECK_CUDA(expr)                                                                      \
  do {                                                                                           \
    cudaError_t _e = (expr);                                                                     \
    if (_e != cudaSuccess) {                                                                     \
      ::tf::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
      return TF_ERR_CUDA;                                                                        \
    }                                                                                            \
  } while (0)

#define TF_CHECK_LAUNCH() TF_CHECK_CUDA(cudaGetLastError())

// Opt a kernel into more than 48 KB of dynamic shared memory.  The attribute is per (function, DEVICE): remembered per device
// (one static table per call site), so a process that drives several GPUs configures each of them.
#define TF_ENSURE_DYNAMIC_SMEM(kern, bytes)                                                                       \
  do {                                                                                                            \
    static bool _tf_done[64] = {false};                                                                           \
    int _tf_dev = 0;                                                                                              \
    TF_CHECK_CUDA(cudaGetDevice(&_tf_dev));                                                                       \
    if (_tf_dev < 0 || _tf_dev >= 64 || !_tf_done[_tf_dev]) {                                                     \
      TF_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(bytes)));       \
      if (_tf_dev >= 0 && _tf_dev < 64) _tf_done[_tf_dev] = true;                                                 \
    }                                                                                                             \
  } while (0)

int sm_count();
// tf_set_pdl() mask: which decode-path kernels are launched with programmatic stream serialization
enum PdlBit { kPdlNorm = 1, kPdlSilu = 2, kPdlRope = 4, kPdlDraftAttn = 8, kPdlVerifyAttn = 16, kPdlSkinny = 32, kPdlSkinnyPrefetch = 64, kPdlStream = 128, kPdlAllReduce = 256 };
bool pdl_enabled(int bit);

// Launch with (optionally) the programmatic-dependent-launch attribute: the kernel may start while its predecessor on the
// stream is still running and must execute pdl_wait() before it touches anything the predecessor writes.
template <typename... KArgs, typename... Args>
inline cudaError_t launch_kernel(int pdl_bit, void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled(pdl_bit) ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

__host__ __device__ inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// ---- device helpers -------------------------------------------------------------------------------------------------
// Programmatic dependent launch (sm_90+): both are no-ops when the grid was launched without the attribute.
//   pdl_launch_dependents(): the next kernel on the stream may start launching (its pre-wait part only reads constants);
//   pdl_wait(): blocks until the previous kernel on the stream has completed and its writes are visible.
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ uint4 ld_nc_v4(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// mbarrier / TMA (cp.async.bulk.tensor) wrappers — sm_90+ PTX, SASS: SYNCS / UTMALDG
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
// 4-D tiled TMA load: coordinates (c0 = d element, c1 = key row, c2 = head, c3 = layer)
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1,
                                            int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void prefetch_tensormap(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}

}  // namespace tf
