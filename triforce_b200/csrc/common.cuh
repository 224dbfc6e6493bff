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

// ---- E4M3 full-KV store ---------------------------------------------------------------------------------------------
// A row x of d fp16 values (K after RoPE, or V) of one (layer, KV head, slot) is stored as one int8 exponent e and d codes
//   e    = the smallest integer with max|x| <= 448 * 2^e (0 for an all-zero row; in [-32, 8] for finite fp16 input),
//   code = e4m3_rn(x / 2^e)   (round to nearest even; x / 2^e is exact and |x / 2^e| <= 448, so nothing saturates).
// The row the store stands for is D = fp16_rn(code * 2^e).  Every kernel that reads the store computes what its fp16
// counterpart computes on D; tests/kv_e4m3_oracle.py restates the rule.  These functions are the only place it is coded.
__device__ __forceinline__ int kv_e4m3_exponent(float amax) {
  if (!(amax > 0.f)) return 0;
  const uint32_t b = __float_as_uint(amax);  // amax = 1.m * 2^E; 448 = 1.75 * 2^8
  const int E = (int)(b >> 23) - 127;
  return (b & 0x7fffffu) <= 0x600000u ? E - 8 : E - 7;
}
__device__ __forceinline__ float kv_e4m3_pow2(int e) { return __uint_as_float((uint32_t)(e + 127) << 23); }
// codes of (lo, hi) at exponent e: lo in the low byte
__device__ __forceinline__ uint16_t kv_e4m3_quantize2(float lo, float hi, int e) {
  const float s = kv_e4m3_pow2(-e);
  uint16_t r;
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(hi * s), "f"(lo * s));
  return r;
}
// two codes (lo in the low byte) -> their exact fp16 values
__device__ __forceinline__ __half2 kv_e4m3_codes2(uint16_t c) {
  uint32_t r;
  asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(r) : "h"(c));
  return *reinterpret_cast<__half2*>(&r);
}
// D = fp16_rn(fp16_rn(c * a) * b) with (a, b) = (1, 2^e), or (2^-8, 2^(e+8)) below e = -24 where 2^e has no fp16: the
// first product is exact (codes are multiples of 2^-9), so D is rounded once
__device__ __forceinline__ void kv_e4m3_factors(int e, __half& a, __half& b) {
  a = __float2half_rn(e < -24 ? 0.00390625f : 1.f);
  b = __float2half_rn(kv_e4m3_pow2(e < -24 ? e + 8 : e));
}
__device__ __forceinline__ __half2 kv_e4m3_apply(__half2 c, __half2 a, __half2 b) { return __hmul2_rn(__hmul2_rn(c, a), b); }
// two codes of one row (exponent e) -> D
__device__ __forceinline__ __half2 kv_e4m3_dequant2(uint16_t c, int e) {
  __half a, b;
  kv_e4m3_factors(e, a, b);
  return kv_e4m3_apply(kv_e4m3_codes2(c), __half2half2(a), __half2half2(b));
}
// 8 codes of one row -> 8 fp16 values of D
__device__ __forceinline__ uint4 kv_e4m3_dequant8(uint2 c, int e) {
  uint4 r;
  __half2* o = reinterpret_cast<__half2*>(&r);
  o[0] = kv_e4m3_dequant2((uint16_t)(c.x & 0xffffu), e);
  o[1] = kv_e4m3_dequant2((uint16_t)(c.x >> 16), e);
  o[2] = kv_e4m3_dequant2((uint16_t)(c.y & 0xffffu), e);
  o[3] = kv_e4m3_dequant2((uint16_t)(c.y >> 16), e);
  return r;
}

}  // namespace tf
