// Library-level entry points: version, error string, SM count, TMA descriptor encoding.
#include <stdarg.h>
#include <string.h>

#include "common.cuh"

namespace tf {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

static int g_pdl = 0;
bool pdl_enabled(int bit) { return (g_pdl & bit) != 0; }

int sm_count() {
  static int cached = 0;
  if (cached > 0) return cached;
  int dev = 0, n = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return -1;
  if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return -1;
  cached = n;
  return n;
}

}  // namespace tf

extern "C" {

int tf_version(void) { return 100; /* 0.1.0 */ }

const char* tf_last_error(void) { return tf::g_err; }

int tf_set_pdl(int on) {
  tf::g_pdl = on;
  return TF_OK;
}

int tf_sm_count(void) {
  int n = tf::sm_count();
  if (n <= 0) {
    tf::set_error("no CUDA device");
    return TF_ERR_CUDA;
  }
  return n;
}

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// eb = element bytes: 2 = fp16 (boxes of 64 elements = 128 B, SWIZZLE_128B), 1 = E4M3 codes (a box is one whole row of d
// bytes: SWIZZLE_128B at d = 128, SWIZZLE_64B at d = 64)
static int kv_tensormap_encode(const char* what, void* out, const void* base, int eb, int d, long long cap, int heads, int layers,
                               long long head_stride, long long layer_stride, int box_keys) {
  TF_CHECK_ARG(out && base, "%s: NULL pointer", what);
  TF_CHECK_ARG(d == 64 || d == 128, "%s: head_dim must be 64 or 128 (got %d)", what, d);
  TF_CHECK_ARG(cap > 0 && heads > 0 && layers > 0, "%s: bad extents", what);
  TF_CHECK_ARG(box_keys > 0 && box_keys <= 256, "%s: box_keys out of range", what);
  TF_CHECK_ARG(((uintptr_t)base & 15) == 0, "%s: base must be 16-byte aligned", what);
  TF_CHECK_ARG((head_stride * eb) % 16 == 0 && (layer_stride * eb) % 16 == 0, "%s: strides must be multiples of 16 bytes", what);

  static PFN_encodeTiled encode = nullptr;
  if (!encode) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
    if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || !fn) {
      tf::set_error("cuTensorMapEncodeTiled not available from the driver (%s)", cudaGetErrorString(e));
      return TF_ERR_CUDA;
    }
    encode = (PFN_encodeTiled)fn;
  }
  // dims fastest-first: (d, slot, head, layer).  Box: 128 B (one SWIZZLE_128B span) or one 64 B e4m3 row x box_keys rows.
  cuuint64_t gdim[4] = {(cuuint64_t)d, (cuuint64_t)cap, (cuuint64_t)heads, (cuuint64_t)layers};
  cuuint64_t gstride[3] = {(cuuint64_t)d * eb, (cuuint64_t)head_stride * eb,
                           (cuuint64_t)(layers > 1 ? layer_stride : head_stride * heads) * eb};
  cuuint32_t box[4] = {eb == 2 ? 64u : (cuuint32_t)d, (cuuint32_t)box_keys, 1, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUtensorMap map;
  CUresult r = encode(&map, eb == 2 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_UINT8, 4, const_cast<void*>(base), gdim,
                      gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                      eb == 1 && d == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                      CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    tf::set_error("cuTensorMapEncodeTiled failed with CUresult %d", (int)r);
    return TF_ERR_CUDA;
  }
  memcpy(out, &map, sizeof(map));
  static_assert(sizeof(CUtensorMap) == 128, "CUtensorMap is 128 bytes");
  return TF_OK;
}

int tf_kv_tensormap_encode(void* out, const void* base, int d, long long cap, int heads, int layers,
                           long long head_stride, long long layer_stride, int box_keys) {
  return kv_tensormap_encode("tf_kv_tensormap_encode", out, base, 2, d, cap, heads, layers, head_stride, layer_stride, box_keys);
}

int tf_kv_tensormap_encode_e4m3(void* out, const void* base, int d, long long cap, int heads, int layers,
                                long long head_stride, long long layer_stride, int box_keys) {
  return kv_tensormap_encode("tf_kv_tensormap_encode_e4m3", out, base, 1, d, cap, heads, layers, head_stride, layer_stride, box_keys);
}

}  // extern "C"
