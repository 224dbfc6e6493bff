// (i) Retrieval-cache build: chunk mean + q·k̄ score + per-head top-k + KV gather.
// Replaces models/cache.py:154-175 of the reference (ATen mean, cuBLAS bmm, ATen topk, 2x gather, 2x copy).
// Arithmetic contract (bit-compared against oracle/triforce_oracle.py):
//   k̄[c]   = fp16( fp32 sum over the chunk's rows in row order * fp32(1/chunk) )
//   score  = fp16( fp64 dot: slices of 8 consecutive d elements summed in order, slice partials butterfly-combined )
//   order  = descending score, ascending chunk index on ties, -0 == +0, NaN greatest; chunk 0 forced first.
// Grouped-query attention (tf_retrieval_build_gqa, rule "group_sum"): scores, top-k and gather run per (layer, KV head) and
// the score's query is q̄ = fp64 sum of the grp query heads of the group (exact for grp <= 64 fp16 values); grp = 1 is MHA.
// E4M3 store (tf_retrieval_build_e4m3, the format of common.cuh): scores and gather read the codes and exponents, and every
// K or V value they use is D, so results are those of the fp16 build on D; the gather writes D into the fp16 retrieval cache.
// All three kernels are HBM/latency bound integer+fp work; no tensor cores (task statement ①).
#include "common.cuh"

namespace tf {

// --------------------------------------------------------------------------------------------------------------------
// kernel 1: scores.  One lane group (d/8 lanes) owns one chunk: every lane keeps an 8-wide slice of the running mean.
// A warp therefore streams 32/(d/8) chunks at once; loads are 16-byte, fully coalesced (a row = d*2 contiguous bytes).
// --------------------------------------------------------------------------------------------------------------------
// 8 consecutive fp16 values of row `row` of a head, from the fp16 store or (Ke != NULL) as D of the E4M3 store
template <bool E4M3>
__device__ __forceinline__ uint4 load8(const void* base, size_t off, const int8_t* __restrict__ Ke, size_t row) {
  if constexpr (E4M3) return kv_e4m3_dequant8(__ldg(reinterpret_cast<const uint2*>(reinterpret_cast<const uint8_t*>(base) + off)), Ke[row]);
  else return ld_nc_v4(reinterpret_cast<const __half*>(base) + off);
}

template <int D, int CHUNK /* 0 = runtime */, bool E4M3>
__global__ void __launch_bounds__(256) chunk_score_kernel(const void* __restrict__ K, long long layer_stride,
                                                          long long head_stride, const __half* __restrict__ q,
                                                          int H, int qg, int chunks, int chunk_rt, __half* __restrict__ scores,
                                                          const int8_t* __restrict__ Ke) {
  constexpr int LPR = D / 8;        // lanes per row
  constexpr int CPW = 32 / LPR;     // chunks per warp pass
  const int chunk = CHUNK ? CHUNK : chunk_rt;
  const int h = blockIdx.y, layer = blockIdx.z;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int grp = lane / LPR, li = lane % LPR;
  const size_t head0 = (size_t)layer * layer_stride + (size_t)h * head_stride;  // elements (fp16) or bytes (codes)
  const __half* qh = q + ((size_t)layer * H + h) * qg * D + li * 8;  // the qg query heads of KV head h
  double q64[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) q64[i] = 0.0;
  for (int g = 0; g < qg; ++g) {
    uint4 raw = *reinterpret_cast<const uint4*>(qh + (size_t)g * D);
    const __half* qq = reinterpret_cast<const __half*>(&raw);
#pragma unroll
    for (int i = 0; i < 8; ++i) q64[i] += (double)__half2float(qq[i]);
  }
  const float inv = 1.0f / (float)chunk;
  const int warps_per_grid = gridDim.x * (blockDim.x >> 5);
  const int passes = (chunks + CPW - 1) / CPW;
  for (int p = blockIdx.x * (blockDim.x >> 5) + warp; p < passes; p += warps_per_grid) {
    const int c = p * CPW + grp;
    const bool valid = c < chunks;
    float acc[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = 0.f;
    if (valid) {
      const size_t base = head0 + (size_t)c * chunk * D + li * 8;
      const size_t row0 = head0 / D + (size_t)c * chunk;
      if (CHUNK == 8) {
        uint4 raw[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) raw[j] = load8<E4M3>(K, base + (size_t)j * D, Ke, row0 + j);  // 8 independent loads in flight
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const __half2* h2 = reinterpret_cast<const __half2*>(&raw[j]);
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            float2 f = __half22float2(h2[i]);
            acc[2 * i] = __fadd_rn(acc[2 * i], f.x);
            acc[2 * i + 1] = __fadd_rn(acc[2 * i + 1], f.y);
          }
        }
      } else {
        for (int j = 0; j < chunk; ++j) {
          uint4 raw = load8<E4M3>(K, base + (size_t)j * D, Ke, row0 + j);
          const __half2* h2 = reinterpret_cast<const __half2*>(&raw);
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            float2 f = __half22float2(h2[i]);
            acc[2 * i] = __fadd_rn(acc[2 * i], f.x);
            acc[2 * i + 1] = __fadd_rn(acc[2 * i + 1], f.y);
          }
        }
      }
    }
    double part = 0.0;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float mean16 = __half2float(__float2half_rn(__fmul_rn(acc[i], inv)));
      part = __dadd_rn(part, __dmul_rn((double)mean16, q64[i]));  // not fused: a group sum q̄ may carry more than 42 bits
    }
#pragma unroll
    for (int m = LPR / 2; m >= 1; m >>= 1) part += __shfl_xor_sync(0xffffffffu, part, m);
    if (valid && li == 0) scores[((size_t)layer * H + h) * chunks + c] = __double2half(part);
  }
}

// --------------------------------------------------------------------------------------------------------------------
// kernel 2: per-(layer, head) top-k in shared memory.  key = sortable16(score) << 16 | (0xFFFF - idx): unique keys, so a
// 4-pass MSB radix select finds the k-th largest exactly, a compaction collects the k winners and a bitonic sort orders
// them.  Candidates are chunks 1..chunks-1 (chunk 0 is always slot 0, cache.py:159-162).
// --------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t sortable16(uint16_t b) {
  if (b == 0x8000u) b = 0;  // -0 == +0
  return (b & 0x8000u) ? (uint32_t)(~b & 0xFFFFu) : (uint32_t)(b | 0x8000u);
}

__global__ void __launch_bounds__(1024) topk_kernel(const __half* __restrict__ scores, int chunks, int k /* = select_sets-1 */,
                                                    int kpad /* pow2 >= k */, int32_t* __restrict__ idx_out /* [.., k+1] */) {
  extern __shared__ uint32_t sm[];
  uint32_t* keys = sm;                  // [chunks-1]
  uint32_t* sel = sm + (chunks - 1);    // [kpad]
  __shared__ uint32_t hist[256];
  __shared__ uint32_t s_prefix, s_krem, s_count;
  const int n = chunks - 1;
  const int tid = threadIdx.x;
  const size_t row = (size_t)blockIdx.x;  // layer*H + h
  const uint16_t* sc = reinterpret_cast<const uint16_t*>(scores) + row * chunks + 1;
  for (int i = tid; i < n; i += blockDim.x) keys[i] = (sortable16(sc[i]) << 16) | (uint32_t)(0xFFFF - i);
  if (tid == 0) { s_prefix = 0; s_krem = (uint32_t)k; s_count = 0; }
  __syncthreads();
  if (k > 0) {
    for (int shift = 24; shift >= 0; shift -= 8) {
      for (int i = tid; i < 256; i += blockDim.x) hist[i] = 0;
      __syncthreads();
      const uint32_t prefix = s_prefix;
      const uint32_t himask = (shift == 24) ? 0u : (0xFFFFFFFFu << (shift + 8));
      for (int base = 0; base < n; base += blockDim.x) {  // trip count is block-uniform (full-mask ballots below)
        const int i = base + tid;
        const uint32_t key = i < n ? keys[i] : 0u;
        const bool in = i < n && (key & himask) == prefix;
        const uint32_t bin = (key >> shift) & 0xFFu;
        // warp-aggregated histogram: scores cluster in few bins, so aggregate equal bins before the shared atomic
        const unsigned active = __ballot_sync(0xffffffffu, in);
        if (in) {
          const unsigned peers = __match_any_sync(active, bin);
          if ((int)(__ffs(peers) - 1) == (tid & 31)) atomicAdd(&hist[bin], (uint32_t)__popc(peers));
        }
      }
      __syncthreads();
      if (tid == 0) {
        uint32_t krem = s_krem, cum = 0;
        int b = 255;
        for (; b >= 0; --b) {
          if (cum + hist[b] >= krem) break;
          cum += hist[b];
        }
        s_krem = krem - cum;
        s_prefix = prefix | ((uint32_t)b << shift);
      }
      __syncthreads();
    }
    const uint32_t kth = s_prefix;  // exact k-th largest key
    for (int i = tid; i < kpad; i += blockDim.x) sel[i] = 0;  // padding sorts last (real keys have bit 15.. set or idx>0)
    __syncthreads();
    for (int i = tid; i < n; i += blockDim.x) {
      const uint32_t key = keys[i];
      if (key >= kth) sel[atomicAdd(&s_count, 1u)] = key;
    }
    __syncthreads();
    // bitonic sort, descending, kpad elements
    for (int size = 2; size <= kpad; size <<= 1) {
      for (int stride = size >> 1; stride > 0; stride >>= 1) {
        for (int i = tid; i < (kpad >> 1); i += blockDim.x) {
          const int lo = ((i / stride) * (stride << 1)) + (i % stride);
          const int hi = lo + stride;
          const bool desc = ((lo & size) == 0);
          const uint32_t a = sel[lo], b = sel[hi];
          if ((a < b) == desc) { sel[lo] = b; sel[hi] = a; }
        }
        __syncthreads();
      }
    }
  }
  int32_t* out = idx_out + row * (size_t)(k + 1);
  if (tid == 0) out[0] = 0;
  for (int i = tid; i < k; i += blockDim.x) out[1 + i] = (int32_t)(0xFFFF - (sel[i] & 0xFFFFu)) + 1;
}

// --------------------------------------------------------------------------------------------------------------------
// kernel 3: gather.  In the head-major layout one chunk of one head is `chunk*d*2` contiguous bytes in both source and
// destination, so the gather is a batch of small contiguous copies (16 B per thread).
// --------------------------------------------------------------------------------------------------------------------
template <bool E4M3>
__global__ void __launch_bounds__(256) gather_kernel(const void* __restrict__ K, const void* __restrict__ V,
                                                     long long kv_layer_stride, long long kv_head_stride,
                                                     __half* __restrict__ rK, __half* __restrict__ rV,
                                                     long long r_layer_stride, long long r_head_stride,
                                                     const int32_t* __restrict__ idx, int H, int select_sets,
                                                     int chunk_elems /* chunk*d */, int d, const int8_t* __restrict__ Ke,
                                                     const int8_t* __restrict__ Ve) {
  const int h = blockIdx.y, layer = blockIdx.z;
  const int vec_per_chunk = chunk_elems / 8;
  const size_t row = (size_t)layer * H + h;
  const int32_t* id = idx + row * select_sets;
  const size_t src_base = (size_t)layer * kv_layer_stride + (size_t)h * kv_head_stride;
  const size_t dst_base = (size_t)layer * r_layer_stride + (size_t)h * r_head_stride;
  const int total = select_sets * vec_per_chunk;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int slot = i / vec_per_chunk, v = i % vec_per_chunk;
    const size_t src = src_base + (size_t)id[slot] * chunk_elems + (size_t)v * 8;
    const size_t dst = dst_base + (size_t)slot * chunk_elems + (size_t)v * 8;
    const size_t src_row = src / d;  // exponent index of the source row
    const uint4 a = load8<E4M3>(K, src, Ke, src_row);
    const uint4 b = load8<E4M3>(V, src, Ve, src_row);
    *reinterpret_cast<uint4*>(rK + dst) = a;
    *reinterpret_cast<uint4*>(rV + dst) = b;
  }
}

static int next_pow2(int x) {
  int p = 1;
  while (p < x) p <<= 1;
  return p;
}

}  // namespace tf

extern "C" {

// H = KV heads of the store; the query has H * grp heads (grp = 1: MHA)
// Ke / Ve non-NULL: K / V are E4M3 code stores with these exponents (strides in bytes; exponent strides = code strides / d)
static int retrieval_build_impl(const void* K, const void* V, long long kv_layer_stride, long long kv_head_stride, const void* q,
                                int n_layers, int H, int grp, int d, int prefill, int chunk, int budget, void* retrK, void* retrV,
                                long long r_layer_stride, long long r_head_stride, int32_t* out_idx, void* out_scores,
                                void* workspace, size_t workspace_bytes, tf_stream_t stream_, const int8_t* Ke = nullptr,
                                const int8_t* Ve = nullptr);

size_t tf_retrieval_build_workspace_bytes(int n_layers, int H, int d, int prefill, int chunk, int budget) {
  if (n_layers <= 0 || H <= 0 || chunk <= 0) return 0;
  const size_t chunks = (size_t)(prefill / chunk), sel = (size_t)(budget / chunk);
  return tf::align_up((size_t)n_layers * H * chunks * sizeof(__half), 256) +
         tf::align_up((size_t)n_layers * H * sel * sizeof(int32_t), 256);
}

int tf_retrieval_build(const void* K, const void* V, long long kv_layer_stride, long long kv_head_stride, const void* q,
                       int n_layers, int H, int d, int prefill, int chunk, int budget, void* retrK, void* retrV,
                       long long r_layer_stride, long long r_head_stride, int32_t* out_idx, void* out_scores,
                       void* workspace, size_t workspace_bytes, tf_stream_t stream) {
  return retrieval_build_impl(K, V, kv_layer_stride, kv_head_stride, q, n_layers, H, 1, d, prefill, chunk, budget, retrK, retrV,
                              r_layer_stride, r_head_stride, out_idx, out_scores, workspace, workspace_bytes, stream);
}

int tf_retrieval_build_e4m3(const void* K, const void* V, const int8_t* Kexp, const int8_t* Vexp, long long kv_layer_stride,
                            long long kv_head_stride, const void* q, int n_layers, int Hq, int Hkv, int d, int prefill, int chunk,
                            int budget, void* retrK, void* retrV, long long r_layer_stride, long long r_head_stride, int32_t* out_idx,
                            void* out_scores, void* workspace, size_t workspace_bytes, tf_stream_t stream) {
  if (Hkv <= 0 || Hq <= 0 || Hq % Hkv != 0 || Hq / Hkv > 64) {
    tf::set_error("tf_retrieval_build_e4m3: Hq (%d) must be a multiple of Hkv (%d), at most 64 per KV head", Hq, Hkv);
    return TF_ERR_INVALID;
  }
  if (!Kexp || !Vexp) {
    tf::set_error("tf_retrieval_build_e4m3: NULL exponent pointer");
    return TF_ERR_INVALID;
  }
  if (d <= 0 || kv_layer_stride % d != 0 || kv_head_stride % d != 0) {
    tf::set_error("tf_retrieval_build_e4m3: code strides must be multiples of d");
    return TF_ERR_INVALID;
  }
  return retrieval_build_impl(K, V, kv_layer_stride, kv_head_stride, q, n_layers, Hkv, Hq / Hkv, d, prefill, chunk, budget, retrK,
                              retrV, r_layer_stride, r_head_stride, out_idx, out_scores, workspace, workspace_bytes, stream, Kexp, Vexp);
}

int tf_retrieval_build_gqa(const void* K, const void* V, long long kv_layer_stride, long long kv_head_stride, const void* q,
                           int n_layers, int Hq, int Hkv, int d, int prefill, int chunk, int budget, void* retrK, void* retrV,
                           long long r_layer_stride, long long r_head_stride, int32_t* out_idx, void* out_scores,
                           void* workspace, size_t workspace_bytes, tf_stream_t stream) {
  if (Hkv <= 0 || Hq <= 0 || Hq % Hkv != 0 || Hq / Hkv > 64) {
    tf::set_error("tf_retrieval_build_gqa: Hq (%d) must be a multiple of Hkv (%d), at most 64 per KV head", Hq, Hkv);
    return TF_ERR_INVALID;
  }
  return retrieval_build_impl(K, V, kv_layer_stride, kv_head_stride, q, n_layers, Hkv, Hq / Hkv, d, prefill, chunk, budget, retrK,
                              retrV, r_layer_stride, r_head_stride, out_idx, out_scores, workspace, workspace_bytes, stream);
}

static int retrieval_build_impl(const void* K, const void* V, long long kv_layer_stride, long long kv_head_stride, const void* q,
                                int n_layers, int H, int grp, int d, int prefill, int chunk, int budget, void* retrK, void* retrV,
                                long long r_layer_stride, long long r_head_stride, int32_t* out_idx, void* out_scores,
                                void* workspace, size_t workspace_bytes, tf_stream_t stream_, const int8_t* Ke, const int8_t* Ve) {
  using namespace tf;
  const bool e4m3 = Ke != nullptr;
  cudaStream_t stream = (cudaStream_t)stream_;
  TF_CHECK_ARG(K && V && q && retrK && retrV, "tf_retrieval_build: NULL pointer");
  TF_CHECK_ARG(n_layers > 0 && H > 0 && chunk > 0, "tf_retrieval_build: bad extents");
  TF_CHECK_ARG(prefill % chunk == 0, "prefill should be multiple of chunk_size, got %d %% %d", prefill, chunk);
  TF_CHECK_ARG(budget % chunk == 0, "max_budget should be multiple of chunk_size, got %d %% %d", budget, chunk);
  TF_CHECK_SUPPORTED(d == 64 || d == 128 || d == 256, "tf_retrieval_build: head_dim %d not in {64,128,256}", d);
  TF_CHECK_SUPPORTED(!e4m3 || d != 256, "tf_retrieval_build_e4m3: head_dim %d not in {64,128}", d);
  const int chunks = prefill / chunk, sel = budget / chunk;
  TF_CHECK_ARG(sel >= 1 && sel - 1 <= chunks - 1, "selected index k out of range (k=%d, candidates=%d)", sel - 1, chunks - 1);
  TF_CHECK_ARG(((uintptr_t)K & 15) == 0 && ((uintptr_t)V & 15) == 0 && ((uintptr_t)retrK & 15) == 0 &&
                   ((uintptr_t)retrV & 15) == 0 && ((uintptr_t)q & 15) == 0,
               "tf_retrieval_build: pointers must be 16-byte aligned");
  TF_CHECK_ARG(kv_head_stride % 8 == 0 && kv_layer_stride % 8 == 0 && r_head_stride % 8 == 0 && r_layer_stride % 8 == 0,
               "tf_retrieval_build: strides must be multiples of 8 elements");
  TF_CHECK_SUPPORTED(chunks - 1 <= 65536, "tf_retrieval_build: more than 65537 chunks per head (%d)", chunks);
  const int kpad = next_pow2(sel - 1 > 1 ? sel - 1 : 2);
  const size_t topk_smem = ((size_t)(chunks - 1) + kpad) * sizeof(uint32_t);
  TF_CHECK_SUPPORTED(topk_smem <= 220 * 1024, "tf_retrieval_build: %zu B of shared memory needed for top-k (chunks=%d, k=%d)",
                     topk_smem, chunks, sel - 1);

  const size_t need = tf_retrieval_build_workspace_bytes(n_layers, H, d, prefill, chunk, budget);
  char* ws = (char*)workspace;
  __half* scores = (__half*)out_scores;
  int32_t* idx = out_idx;
  if (!scores || !idx) {
    TF_CHECK_ARG(workspace && workspace_bytes >= need, "tf_retrieval_build: workspace too small (%zu < %zu)", workspace_bytes, need);
    if (!scores) scores = (__half*)ws;
    if (!idx) idx = (int32_t*)(ws + align_up((size_t)n_layers * H * chunks * sizeof(__half), 256));
  }

  const int sms = sm_count() > 0 ? sm_count() : 132;
  {
    const int per_pass = 32 / (d / 8);
    const int passes = (chunks + per_pass - 1) / per_pass;
    int gx = (passes + 7) / 8;  // 8 warps per CTA
    const int cap = (sms * 8 + H * n_layers - 1) / (H * n_layers);
    if (gx > cap) gx = cap < 1 ? 1 : cap;
    dim3 grid(gx, H, n_layers);
#define LAUNCH_SCORE(D_, C_, E_)                                                                                    \
  chunk_score_kernel<D_, C_, E_><<<grid, 256, 0, stream>>>(K, kv_layer_stride, kv_head_stride, (const __half*)q, H, grp, \
                                                           chunks, chunk, scores, Ke)
    if (e4m3) {
      if (d == 128) { if (chunk == 8) LAUNCH_SCORE(128, 8, true); else LAUNCH_SCORE(128, 0, true); }
      else { if (chunk == 8) LAUNCH_SCORE(64, 8, true); else LAUNCH_SCORE(64, 0, true); }
    } else if (d == 128) { if (chunk == 8) LAUNCH_SCORE(128, 8, false); else LAUNCH_SCORE(128, 0, false); }
    else if (d == 64) { if (chunk == 8) LAUNCH_SCORE(64, 8, false); else LAUNCH_SCORE(64, 0, false); }
    else { if (chunk == 8) LAUNCH_SCORE(256, 8, false); else LAUNCH_SCORE(256, 0, false); }
#undef LAUNCH_SCORE
    TF_CHECK_LAUNCH();
  }
  {
    TF_ENSURE_DYNAMIC_SMEM(topk_kernel, 220 * 1024);
    topk_kernel<<<n_layers * H, 1024, topk_smem, stream>>>(scores, chunks, sel - 1, kpad, idx);
    TF_CHECK_LAUNCH();
  }
  {
    const int total_vec = sel * (chunk * d / 8);
    int gx = (total_vec + 255) / 256;
    if (gx > 64) gx = 64;
    dim3 grid(gx, H, n_layers);
    if (e4m3)
      gather_kernel<true><<<grid, 256, 0, stream>>>(K, V, kv_layer_stride, kv_head_stride, (__half*)retrK, (__half*)retrV,
                                                    r_layer_stride, r_head_stride, idx, H, sel, chunk * d, d, Ke, Ve);
    else
      gather_kernel<false><<<grid, 256, 0, stream>>>(K, V, kv_layer_stride, kv_head_stride, (__half*)retrK, (__half*)retrV,
                                                     r_layer_stride, r_head_stride, idx, H, sel, chunk * d, d, nullptr, nullptr);
    TF_CHECK_LAUNCH();
  }
  return TF_OK;
}

}  // extern "C"
