// Per-layer glue around the attention kernels: fused RoPE + KV append, the draft's sliding-window attention with
// RoPE-on-read, cache maintenance (budget-tail overwrite, StreamingLLM window slide) and the fp16 elementwise ops of the
// decoder layer (residual add + RMSNorm, SiLU*up).  All HBM/latency-bound byte work — no tensor cores.
// Rounding points restate the reference's fp16 tensors (see include/triforce_b200.h for file:line of each site).
#include "common.cuh"

namespace tf {

// ---- RoPE on a half2 pair (a = elements (2j,2j+1) of the first half, b = same of the second half) -------------------
__device__ __forceinline__ void rope_pair(__half2 a, __half2 b, __half2 cos_lo, __half2 cos_hi, __half2 sin_lo,
                                          __half2 sin_hi, __half2& out_lo, __half2& out_hi) {
  // x_embed = (x * cos) + (rotate_half(x) * sin), rotate_half(x) = cat(-x2, x1); every op rounds to fp16
  out_lo = __hadd2_rn(__hmul2_rn(a, cos_lo), __hmul2_rn(__hneg2(b), sin_lo));
  out_hi = __hadd2_rn(__hmul2_rn(b, cos_hi), __hmul2_rn(a, sin_hi));
}

// the amax of a row held by the D/4 threads of a rope_append CTA (one warp at d = 128, half a warp at d = 64)
template <int D>
__device__ __forceinline__ float row_amax(__half2 lo, __half2 hi) {
  const __half2 a = __hmax2(__habs2(lo), __habs2(hi));
  float m = fmaxf(__low2float(a), __high2float(a));
#pragma unroll
  for (int o = D / 8; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(D == 128 ? 0xffffffffu : 0xffffu, m, o));
  return m;
}

// E4M3 row store (common.cuh): thread j holds elements (2j, 2j+1) and (D/2 + 2j, D/2 + 2j + 1) of the row
template <int D>
__device__ __forceinline__ void store_row_e4m3(__half2 lo, __half2 hi, uint8_t* codes_row, int8_t* exp, int j) {
  const int e = kv_e4m3_exponent(row_amax<D>(lo, hi));
  const float2 l = __half22float2(lo), u = __half22float2(hi);
  reinterpret_cast<uint16_t*>(codes_row)[j] = kv_e4m3_quantize2(l.x, l.y, e);
  reinterpret_cast<uint16_t*>(codes_row)[j + D / 4] = kv_e4m3_quantize2(u.x, u.y, e);
  if (j == 0) *exp = (int8_t)e;
}

// E4M3: Kc / Vc are the code stores [Hkv][cap][D] (head stride cap * D), Ke / Ve the exponents [Hkv][cap]
template <int D, bool E4M3>
__global__ void __launch_bounds__(D / 4) rope_append_kernel(const __half* __restrict__ q, const __half* __restrict__ k,
                                                            const __half* __restrict__ v, long long row_stride,
                                                            const __half* __restrict__ cos, const __half* __restrict__ sin,
                                                            int max_pos, const int32_t* __restrict__ pos_ids, int pos0,
                                                            const int32_t* __restrict__ pos0_dev, int slot0,
                                                            const int32_t* __restrict__ slot0_dev, int H, int Hkv, int rotate_q,
                                                            int rotate_k, __half* __restrict__ q_out,
                                                            void* __restrict__ Kc, void* __restrict__ Vc,
                                                            long long head_stride, long long cap, int8_t* __restrict__ Ke,
                                                            int8_t* __restrict__ Ve) {
  pdl_launch_dependents();
  pdl_wait();
  // one CTA per (row, query head); the first Hkv of them also append K/V head h (grouped-query attention: Hkv < H)
  const int r = blockIdx.x, h = blockIdx.y, j = threadIdx.x;  // j-th half2 of the first half
  int pos = pos_ids ? pos_ids[r] : pos0 + (pos0_dev ? *pos0_dev : 0) + r;
  pos = min(max(pos, 0), max_pos - 1);
  const long long slot = (long long)slot0 + (slot0_dev ? *slot0_dev : 0) + r;
  const size_t in = (size_t)r * row_stride + (size_t)h * D;
  const __half2* c2 = reinterpret_cast<const __half2*>(cos + (size_t)pos * D);
  const __half2* s2 = reinterpret_cast<const __half2*>(sin + (size_t)pos * D);
  const __half2 cl = c2[j], ch = c2[j + D / 4], sl = s2[j], sh = s2[j + D / 4];
  {
    const __half2* x = reinterpret_cast<const __half2*>(q + in);
    __half2 lo = x[j], hi = x[j + D / 4];
    if (rotate_q) rope_pair(lo, hi, cl, ch, sl, sh, lo, hi);
    __half2* o = reinterpret_cast<__half2*>(q_out + ((size_t)r * H + h) * D);
    o[j] = lo;
    o[j + D / 4] = hi;
  }
  if (h < Hkv && slot >= 0 && slot < cap) {
    const size_t dst = (size_t)h * head_stride + (size_t)slot * D;
    const __half2* x = reinterpret_cast<const __half2*>(k + in);
    __half2 lo = x[j], hi = x[j + D / 4];
    if (rotate_k) rope_pair(lo, hi, cl, ch, sl, sh, lo, hi);
    const __half2* xv = reinterpret_cast<const __half2*>(v + in);
    if constexpr (E4M3) {
      const size_t ex = (size_t)h * cap + (size_t)slot;
      store_row_e4m3<D>(lo, hi, reinterpret_cast<uint8_t*>(Kc) + dst, Ke + ex, j);
      store_row_e4m3<D>(xv[j], xv[j + D / 4], reinterpret_cast<uint8_t*>(Vc) + dst, Ve + ex, j);
    } else {
      __half2* o = reinterpret_cast<__half2*>(reinterpret_cast<__half*>(Kc) + dst);
      o[j] = lo;
      o[j + D / 4] = hi;
      __half2* ov = reinterpret_cast<__half2*>(reinterpret_cast<__half*>(Vc) + dst);
      ov[j] = xv[j];
      ov[j + D / 4] = xv[j + D / 4];
    }
  }
}

// fp16 rows [slot0, slot0 + n) of one layer -> E4M3 codes and exponents, one warp per (row, KV head)
template <int D>
__global__ void __launch_bounds__(128) kv_quantize_kernel(const __half* __restrict__ src, long long src_head_stride, int slot0, int n,
                                                          uint8_t* __restrict__ codes, int8_t* __restrict__ exps, long long cap) {
  const int r = blockIdx.x * 4 + (threadIdx.x >> 5), h = blockIdx.y, lane = threadIdx.x & 31;
  if (r >= n) return;
  const size_t slot = (size_t)slot0 + r;
  kv_e4m3_quantize_row_warp<D>(src + (size_t)h * src_head_stride + slot * D, codes + ((size_t)h * cap + slot) * D,
                               exps + (size_t)h * cap + slot, lane);
}

// ---- (ii) draft attention --------------------------------------------------------------------------------------------
// One CTA per (head, block of 16 query rows).  Keys are rotated at their slot index while staged into shared memory
// (the reference re-applies RoPE to the whole cache each step, modeling_llama_68m.py:161-162), then each warp computes
// one query row at a time: lanes split the keys for q·K, then split the d columns for P·V.
constexpr int kDraftRowsPerCta = 16;
constexpr int kDraftThreads = 256;

template <int D>
__global__ void __launch_bounds__(kDraftThreads) draft_attn_kernel(const __half* __restrict__ q, const __half* __restrict__ K,
                                                                   const __half* __restrict__ V, long long head_stride,
                                                                   const __half* __restrict__ cos, const __half* __restrict__ sin,
                                                                   int kv_len, int R, int H, float scale_log2,
                                                                   __half* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  constexpr int LD = D + 8;  // padded row (halfs): 16-byte row reads by consecutive lanes are bank-conflict free
  extern __shared__ __align__(16) uint8_t dsm[];
  __half* Ks = reinterpret_cast<__half*>(dsm);          // [kv_len][LD]
  __half* Vs = Ks + (size_t)kv_len * LD;                // [kv_len][LD]
  float* Ps = reinterpret_cast<float*>(Vs + (size_t)kv_len * LD);  // [8 warps][kv_len]
  const int h = blockIdx.x, rb = blockIdx.y * kDraftRowsPerCta;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const __half* Kh = K + (size_t)h * head_stride;
  const __half* Vh = V + (size_t)h * head_stride;
  const int rows_here = min(kDraftRowsPerCta, R - rb);
  const int max_key = min(kv_len, kv_len - R + rb + rows_here);  // keys beyond the last row's limit are never read

  // stage K (rotated) and V: one thread per half2 pair (j, j + D/4)
  for (int idx = threadIdx.x; idx < max_key * (D / 4); idx += kDraftThreads) {
    const int row = idx / (D / 4), j = idx % (D / 4);
    const __half2* x = reinterpret_cast<const __half2*>(Kh + (size_t)row * D);
    const __half2* c2 = reinterpret_cast<const __half2*>(cos + (size_t)row * D);
    const __half2* s2 = reinterpret_cast<const __half2*>(sin + (size_t)row * D);
    __half2 lo, hi;
    rope_pair(x[j], x[j + D / 4], c2[j], c2[j + D / 4], s2[j], s2[j + D / 4], lo, hi);
    __half2* kd = reinterpret_cast<__half2*>(Ks + (size_t)row * LD);
    kd[j] = lo;
    kd[j + D / 4] = hi;
    const __half2* xv = reinterpret_cast<const __half2*>(Vh + (size_t)row * D);
    __half2* vd = reinterpret_cast<__half2*>(Vs + (size_t)row * LD);
    vd[j] = xv[j];
    vd[j + D / 4] = xv[j + D / 4];
  }
  __syncthreads();

  float* P = Ps + (size_t)warp * kv_len;
  for (int rr = warp; rr < rows_here; rr += kDraftThreads / 32) {
    const int r = rb + rr;
    const int limit = kv_len - R + r;  // last visible key
    const __half* qr = q + ((size_t)r * H + h) * D;
    // q row in registers (fp32)
    float qf[D];
#pragma unroll
    for (int i = 0; i < D / 8; ++i) {
      const uint4 raw = *reinterpret_cast<const uint4*>(qr + i * 8);
      const __half2* h2 = reinterpret_cast<const __half2*>(&raw);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 f = __half22float2(h2[e]);
        qf[i * 8 + 2 * e] = f.x;
        qf[i * 8 + 2 * e + 1] = f.y;
      }
    }
    float mx = -INFINITY;
    for (int j = lane; j <= limit; j += 32) {
      const __half* kr = Ks + (size_t)j * LD;
      float acc = 0.f;
#pragma unroll
      for (int i = 0; i < D / 8; ++i) {
        const uint4 raw = *reinterpret_cast<const uint4*>(kr + i * 8);
        const __half2* h2 = reinterpret_cast<const __half2*>(&raw);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float2 f = __half22float2(h2[e]);
          acc = fmaf(qf[i * 8 + 2 * e], f.x, acc);
          acc = fmaf(qf[i * 8 + 2 * e + 1], f.y, acc);
        }
      }
      P[j] = acc;
      mx = fmaxf(mx, acc);
    }
    mx = warp_max(mx);
    float sum = 0.f;
    for (int j = lane; j <= limit; j += 32) {
      const float p = exp2f((P[j] - mx) * scale_log2);
      P[j] = p;
      sum += p;
    }
    sum = warp_sum(sum);
    __syncwarp();
    // O = P V: each lane owns D/32 consecutive columns
    constexpr int CPL = D / 32;
    float o[CPL];
#pragma unroll
    for (int c = 0; c < CPL; ++c) o[c] = 0.f;
    for (int j = 0; j <= limit; ++j) {
      const float p = P[j];
      const __half* vr = Vs + (size_t)j * LD + lane * CPL;
#pragma unroll
      for (int c = 0; c < CPL; c += 2) {
        const float2 f = __half22float2(*reinterpret_cast<const __half2*>(vr + c));
        o[c] = fmaf(p, f.x, o[c]);
        o[c + 1] = fmaf(p, f.y, o[c + 1]);
      }
    }
    const float inv = 1.f / sum;
    __half* orow = out + ((size_t)r * H + h) * D + lane * CPL;
#pragma unroll
    for (int c = 0; c < CPL; c += 2) *reinterpret_cast<__half2*>(orow + c) = __floats2half2_rn(o[c] * inv, o[c + 1] * inv);
    __syncwarp();
  }
}

// ---- cache maintenance ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) tail_update_kernel(const __half* __restrict__ K, const __half* __restrict__ V,
                                                          long long kls, long long khs, __half* __restrict__ rK,
                                                          __half* __restrict__ rV, long long rls, long long rhs, int D,
                                                          int prefill, int budget, int seq_len_host,
                                                          const int32_t* __restrict__ seq_len_dev) {
  const int h = blockIdx.y, layer = blockIdx.z;
  // rows [seq_len - n_new, seq_len) go to [budget - n_new, budget): never more than the budget, whatever length the device
  // holds (the hosts refuse a step that would pass it; this keeps a wrong length from writing outside the budget)
  const int seq_len = seq_len_host + (seq_len_dev ? *seq_len_dev : 0);
  const int n_new = min(seq_len - prefill, budget);
  if (n_new <= 0) return;
  const int src_row = seq_len - n_new;
  const int vec_per_row = D / 8;
  const int total = n_new * vec_per_row;
  const size_t src0 = (size_t)layer * kls + (size_t)h * khs + (size_t)src_row * D;
  const size_t dst0 = (size_t)layer * rls + (size_t)h * rhs + (size_t)(budget - n_new) * D;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const size_t off = (size_t)i * 8;
    *reinterpret_cast<uint4*>(rK + dst0 + off) = *reinterpret_cast<const uint4*>(K + src0 + off);
    *reinterpret_cast<uint4*>(rV + dst0 + off) = *reinterpret_cast<const uint4*>(V + src0 + off);
  }
}

// tail_update_kernel over an E4M3 store: codes and their exponents in, D out (exponent strides = code strides / D)
__global__ void __launch_bounds__(256) tail_update_e4m3_kernel(const uint8_t* __restrict__ K, const uint8_t* __restrict__ V,
                                                               const int8_t* __restrict__ Ke, const int8_t* __restrict__ Ve,
                                                               long long kls, long long khs, __half* __restrict__ rK,
                                                               __half* __restrict__ rV, long long rls, long long rhs, int D,
                                                               int prefill, int budget, int seq_len_host,
                                                               const int32_t* __restrict__ seq_len_dev) {
  const int h = blockIdx.y, layer = blockIdx.z;
  // the rows of tail_update_kernel: the last min(seq_len - prefill, budget), never outside the budget
  const int seq_len = seq_len_host + (seq_len_dev ? *seq_len_dev : 0);
  const int n_new = min(seq_len - prefill, budget);
  if (n_new <= 0) return;
  const int src_row = seq_len - n_new;
  const int vec_per_row = D / 8;
  const int total = n_new * vec_per_row;
  const size_t head = (size_t)layer * kls + (size_t)h * khs;
  const size_t dst0 = (size_t)layer * rls + (size_t)h * rhs + (size_t)(budget - n_new) * D;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const size_t slot = (size_t)src_row + i / vec_per_row;
    const size_t src = head + slot * D + (size_t)(i % vec_per_row) * 8;
    const size_t ex = head / D + slot;
    *reinterpret_cast<uint4*>(rK + dst0 + (size_t)i * 8) = kv_e4m3_dequant8(*reinterpret_cast<const uint2*>(K + src), Ke[ex]);
    *reinterpret_cast<uint4*>(rV + dst0 + (size_t)i * 8) = kv_e4m3_dequant8(*reinterpret_cast<const uint2*>(V + src), Ve[ex]);
  }
}

// tail_update_kernel into an E4M3 retrieval cache (tf_tail_update_to_e4m3): one warp per row, quantized from an fp16 store or
// copied from an E4M3 one (rows index exponents; strides are multiples of D)
template <int D, bool SRC_E4M3>
__global__ void __launch_bounds__(256) tail_update_to_e4m3_kernel(const void* __restrict__ K, const void* __restrict__ V,
                                                                  const int8_t* __restrict__ Ke, const int8_t* __restrict__ Ve,
                                                                  long long kls, long long khs, uint8_t* __restrict__ rK,
                                                                  uint8_t* __restrict__ rV, int8_t* __restrict__ rKe,
                                                                  int8_t* __restrict__ rVe, long long rls, long long rhs, int prefill,
                                                                  int budget, int seq_len_host, const int32_t* __restrict__ seq_len_dev) {
  const int h = blockIdx.y, layer = blockIdx.z, lane = threadIdx.x & 31;
  // the rows of tail_update_kernel: the last min(seq_len - prefill, budget), never outside the budget
  const int seq_len = seq_len_host + (seq_len_dev ? *seq_len_dev : 0);
  const int n_new = min(seq_len - prefill, budget);
  if (n_new <= 0) return;
  const int src_row = seq_len - n_new;
  const size_t src0 = ((size_t)layer * kls + (size_t)h * khs) / D + src_row;
  const size_t dst0 = ((size_t)layer * rls + (size_t)h * rhs) / D + (budget - n_new);
  for (int r = blockIdx.x * 8 + (threadIdx.x >> 5); r < n_new; r += gridDim.x * 8) {
    kv_e4m3_row_into<D, SRC_E4M3>(K, Ke, src0 + r, rK, rKe, dst0 + r, lane);
    kv_e4m3_row_into<D, SRC_E4M3>(V, Ve, src0 + r, rV, rVe, dst0 + r, lane);
  }
}

// StreamingLLM window slide (cache.py:263-265 evict_for_spec): rows [src, src + n_rows) → [dst_start, …) of every (layer, head),
// K and V, with src = src_start + *shift_dev, or src_start when shift_dev is NULL (the device loop reads its shift from device
// memory)
__global__ void __launch_bounds__(256) window_slide_kernel(__half* __restrict__ K, __half* __restrict__ V, long long ls,
                                                           long long hs, int D, int src_start, const int32_t* __restrict__ shift_dev,
                                                           int dst_start, int n_rows) {
  extern __shared__ __align__(16) uint8_t wsm[];
  uint4* buf = reinterpret_cast<uint4*>(wsm);
  const int h = blockIdx.x, layer = blockIdx.y;
  const int src_row = src_start + (shift_dev ? *shift_dev : 0);
  const int nvec = n_rows * D / 8;
  __half* bases[2] = {K + (size_t)layer * ls + (size_t)h * hs, V + (size_t)layer * ls + (size_t)h * hs};
#pragma unroll
  for (int w = 0; w < 2; ++w) {
    const uint4* src = reinterpret_cast<const uint4*>(bases[w] + (size_t)src_row * D);
    uint4* dst = reinterpret_cast<uint4*>(bases[w] + (size_t)dst_start * D);
    for (int i = threadIdx.x; i < nvec; i += blockDim.x) buf[i] = src[i];  // clone semantics: read everything first
    __syncthreads();
    for (int i = threadIdx.x; i < nvec; i += blockDim.x) dst[i] = buf[i];
    __syncthreads();
  }
}

// gather_kv_incremental (cache.py:333-343): rows src_idx[i] -> dst_start + i of every (layer, head), K and V, clone
// semantics (all sources are read before anything is written)
__global__ void __launch_bounds__(128) kv_compact_kernel(__half* __restrict__ K, __half* __restrict__ V, long long ls, long long hs,
                                                         int D, const int32_t* __restrict__ src_idx, int n, int dst_start) {
  extern __shared__ __align__(16) uint8_t csm[];
  uint4* buf = reinterpret_cast<uint4*>(csm);
  const int h = blockIdx.x, layer = blockIdx.y;
  const int vec_per_row = D / 8;
  const int nvec = n * vec_per_row;
  __half* bases[2] = {K + (size_t)layer * ls + (size_t)h * hs, V + (size_t)layer * ls + (size_t)h * hs};
#pragma unroll
  for (int w = 0; w < 2; ++w) {
    for (int i = threadIdx.x; i < nvec; i += blockDim.x) {
      const int r = i / vec_per_row, v = i % vec_per_row;
      buf[i] = *reinterpret_cast<const uint4*>(bases[w] + (size_t)src_idx[r] * D + v * 8);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < nvec; i += blockDim.x) {
      const int r = i / vec_per_row, v = i % vec_per_row;
      *reinterpret_cast<uint4*>(bases[w] + (size_t)(dst_start + r) * D + v * 8) = buf[i];
    }
    __syncthreads();
  }
}

// The same over an E4M3 store ([L][H][cap] rows of d code bytes and one exponent): one CTA per (head, layer) stages the n source
// rows of K codes, V codes and both exponents in shared memory before it writes any destination row (clone semantics).
__global__ void __launch_bounds__(128) kv_compact_e4m3_kernel(uint8_t* __restrict__ Kc, uint8_t* __restrict__ Vc, int8_t* __restrict__ Ke,
                                                              int8_t* __restrict__ Ve, long long cap, int H, int D,
                                                              const int32_t* __restrict__ src_idx, int n, int dst_start) {
  extern __shared__ __align__(16) uint8_t csm[];
  uint4* buf = reinterpret_cast<uint4*>(csm);  // [2][n][D / 16]
  int8_t* ebuf = reinterpret_cast<int8_t*>(buf + 2 * (size_t)n * (D / 16));  // [2][n]
  const int h = blockIdx.x, layer = blockIdx.y;
  const size_t row0 = ((size_t)layer * H + h) * (size_t)cap;
  const int vec_per_row = D / 16;
  const int nvec = n * vec_per_row;
  uint8_t* codes[2] = {Kc + row0 * D, Vc + row0 * D};
  int8_t* exps[2] = {Ke + row0, Ve + row0};
  for (int i = threadIdx.x; i < 2 * nvec; i += blockDim.x) {
    const int w = i / nvec, r = (i % nvec) / vec_per_row, v = i % vec_per_row;
    buf[i] = *reinterpret_cast<const uint4*>(codes[w] + (size_t)src_idx[r] * D + v * 16);
  }
  for (int i = threadIdx.x; i < 2 * n; i += blockDim.x) ebuf[i] = exps[i / n][src_idx[i % n]];
  __syncthreads();
  for (int i = threadIdx.x; i < 2 * nvec; i += blockDim.x) {
    const int w = i / nvec, r = (i % nvec) / vec_per_row, v = i % vec_per_row;
    *reinterpret_cast<uint4*>(codes[w] + (size_t)(dst_start + r) * D + v * 16) = buf[i];
  }
  for (int i = threadIdx.x; i < 2 * n; i += blockDim.x) exps[i / n][dst_start + i % n] = ebuf[i];
}

// ---- elementwise glue ------------------------------------------------------------------------------------------------
// One CTA per row, one 16-byte vector (8 halfs) per thread per pass: for hidden = 4096 that is 512 threads with the whole
// row in registers — a single load, one block reduction, a single store (launch-latency bound: ~3 us).
template <int VPT /* vectors per thread */>
__global__ void __launch_bounds__(1024) add_rmsnorm_kernel(__half* __restrict__ h, const __half* __restrict__ delta,
                                                           const __half* __restrict__ w, float eps, __half* __restrict__ out,
                                                           int hidden) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float red[32];
  const size_t base = (size_t)blockIdx.x * hidden;
  const int nvec = hidden / 8;
  uint4 xv[VPT];
  float ss = 0.f;
#pragma unroll
  for (int v = 0; v < VPT; ++v) {
    const int i = threadIdx.x + v * blockDim.x;
    if (i < nvec) {
      uint4 x = *reinterpret_cast<const uint4*>(h + base + (size_t)i * 8);
      if (delta) {
        const uint4 dl = *reinterpret_cast<const uint4*>(delta + base + (size_t)i * 8);
        __half2* x2 = reinterpret_cast<__half2*>(&x);
        const __half2* d2 = reinterpret_cast<const __half2*>(&dl);
#pragma unroll
        for (int e = 0; e < 4; ++e) x2[e] = __hadd2_rn(x2[e], d2[e]);
        *reinterpret_cast<uint4*>(h + base + (size_t)i * 8) = x;
      }
      xv[v] = x;
      const __half2* x2 = reinterpret_cast<const __half2*>(&x);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 f = __half22float2(x2[e]);
        ss += f.x * f.x + f.y * f.y;
      }
    }
  }
  ss = warp_sum(ss);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
  __syncthreads();
  float tot = (threadIdx.x & 31) < ((blockDim.x + 31) >> 5) ? red[threadIdx.x & 31] : 0.f;
  tot = warp_sum(tot);
  const float inv = rsqrtf(tot / (float)hidden + eps);
#pragma unroll
  for (int v = 0; v < VPT; ++v) {
    const int i = threadIdx.x + v * blockDim.x;
    if (i < nvec) {
      const uint4 wv = *reinterpret_cast<const uint4*>(w + (size_t)i * 8);
      const __half2* x2 = reinterpret_cast<const __half2*>(&xv[v]);
      const __half2* w2 = reinterpret_cast<const __half2*>(&wv);
      uint4 o;
      __half2* o2 = reinterpret_cast<__half2*>(&o);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 f = __half22float2(x2[e]);
        o2[e] = __hmul2_rn(w2[e], __floats2half2_rn(f.x * inv, f.y * inv));
      }
      *reinterpret_cast<uint4*>(out + base + (size_t)i * 8) = o;
    }
  }
}

__global__ void __launch_bounds__(256) silu_mul_kernel(const __half* __restrict__ gu, __half* __restrict__ out, int inter) {
  pdl_launch_dependents();
  pdl_wait();
  const size_t r = blockIdx.y;
  const __half2* g2 = reinterpret_cast<const __half2*>(gu + r * 2 * (size_t)inter);
  const __half2* u2 = g2 + inter / 2;
  __half2* o2 = reinterpret_cast<__half2*>(out + r * (size_t)inter);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < inter / 2; i += gridDim.x * blockDim.x) {
    const float2 g = __half22float2(g2[i]);
    const __half2 s = __floats2half2_rn(g.x / (1.f + expf(-g.x)), g.y / (1.f + expf(-g.y)));
    o2[i] = __hmul2_rn(s, u2[i]);
  }
}

}  // namespace tf

extern "C" {

// H query heads, Hkv K/V heads (Hkv == H: MHA)
// Kexp / Vexp non-NULL: Kcache / Vcache are E4M3 code stores of one layer ([Hkv][cap][d], head stride cap * d) with these
// exponents [Hkv][cap]
static int rope_append_impl(const void* q, const void* k, const void* v, long long qkv_row_stride, const void* cos, const void* sin,
                            int max_pos, const int32_t* pos_ids_dev, int pos0, const int32_t* pos0_dev, int slot0,
                            const int32_t* slot0_dev, int R, int H, int Hkv, int d, int rotate_q, int rotate_k, void* q_out,
                            void* Kcache, void* Vcache, long long kv_head_stride, long long cap, tf_stream_t stream_,
                            int8_t* Kexp = nullptr, int8_t* Vexp = nullptr) {
  using namespace tf;
  TF_CHECK_ARG(q && k && v && cos && sin && q_out && Kcache && Vcache, "tf_rope_append: NULL pointer");
  TF_CHECK_ARG(R >= 1 && H >= 1 && max_pos >= 1 && cap >= 1, "tf_rope_append: bad extents");
  TF_CHECK_ARG(Hkv >= 1 && H % Hkv == 0, "tf_rope_append_gqa: Hq (%d) must be a positive multiple of Hkv (%d)", H, Hkv);
  TF_CHECK_SUPPORTED(d == 64 || d == 128, "tf_rope_append: head_dim %d not in {64,128}", d);
  TF_CHECK_ARG(qkv_row_stride % 2 == 0 && kv_head_stride % 2 == 0, "tf_rope_append: strides must be even");
  if (!slot0_dev) TF_CHECK_ARG(slot0 >= 0 && (long long)slot0 + R <= cap, "tf_rope_append: slots [%d,%d) exceed capacity %lld", slot0, slot0 + R, cap);
  dim3 grid(R, H);
  cudaStream_t stream = (cudaStream_t)stream_;
#define TF_LAUNCH_ROPE(D_, E4M3_)                                                                                                   \
  TF_CHECK_CUDA(launch_kernel(kPdlRope, rope_append_kernel<D_, E4M3_>, grid, D_ / 4, 0, stream, (const __half*)q, (const __half*)k,  \
                              (const __half*)v, qkv_row_stride, (const __half*)cos, (const __half*)sin, max_pos, pos_ids_dev, pos0, \
                              pos0_dev, slot0, slot0_dev, H, Hkv, rotate_q, rotate_k, (__half*)q_out, Kcache, Vcache,              \
                              kv_head_stride, cap, Kexp, Vexp))
  if (Kexp) {
    if (d == 128) TF_LAUNCH_ROPE(128, true);
    else TF_LAUNCH_ROPE(64, true);
  } else {
    if (d == 128) TF_LAUNCH_ROPE(128, false);
    else TF_LAUNCH_ROPE(64, false);
  }
#undef TF_LAUNCH_ROPE
  TF_CHECK_LAUNCH();
  return TF_OK;
}

int tf_rope_append(const void* q, const void* k, const void* v, long long qkv_row_stride, const void* cos, const void* sin,
                   int max_pos, const int32_t* pos_ids_dev, int pos0, const int32_t* pos0_dev, int slot0,
                   const int32_t* slot0_dev, int R, int H, int d, int rotate_q, int rotate_k, void* q_out, void* Kcache,
                   void* Vcache, long long kv_head_stride, long long cap, tf_stream_t stream) {
  return rope_append_impl(q, k, v, qkv_row_stride, cos, sin, max_pos, pos_ids_dev, pos0, pos0_dev, slot0, slot0_dev, R, H, H, d,
                          rotate_q, rotate_k, q_out, Kcache, Vcache, kv_head_stride, cap, stream);
}

int tf_rope_append_gqa(const void* q, const void* k, const void* v, long long qkv_row_stride, const void* cos, const void* sin,
                       int max_pos, const int32_t* pos_ids_dev, int pos0, const int32_t* pos0_dev, int slot0,
                       const int32_t* slot0_dev, int R, int Hq, int Hkv, int d, int rotate_q, int rotate_k, void* q_out,
                       void* Kcache, void* Vcache, long long kv_head_stride, long long cap, tf_stream_t stream) {
  return rope_append_impl(q, k, v, qkv_row_stride, cos, sin, max_pos, pos_ids_dev, pos0, pos0_dev, slot0, slot0_dev, R, Hq, Hkv, d,
                          rotate_q, rotate_k, q_out, Kcache, Vcache, kv_head_stride, cap, stream);
}

int tf_rope_append_e4m3(const void* q, const void* k, const void* v, long long qkv_row_stride, const void* cos, const void* sin,
                        int max_pos, const int32_t* pos_ids_dev, int pos0, const int32_t* pos0_dev, int slot0,
                        const int32_t* slot0_dev, int R, int Hq, int Hkv, int d, void* q_out, void* Kcodes, void* Vcodes,
                        int8_t* Kexp, int8_t* Vexp, long long cap, tf_stream_t stream) {
  TF_CHECK_ARG(Kexp && Vexp, "tf_rope_append_e4m3: NULL exponent pointer");
  return rope_append_impl(q, k, v, qkv_row_stride, cos, sin, max_pos, pos_ids_dev, pos0, pos0_dev, slot0, slot0_dev, R, Hq, Hkv, d,
                          1, 1, q_out, Kcodes, Vcodes, cap * d, cap, stream, Kexp, Vexp);
}

int tf_kv_quantize_e4m3(const void* src, long long src_head_stride, int slot0, int n, int Hkv, int d, void* codes, int8_t* exps,
                        long long cap, tf_stream_t stream_) {
  using namespace tf;
  TF_CHECK_ARG(src && codes && exps, "tf_kv_quantize_e4m3: NULL pointer");
  TF_CHECK_SUPPORTED(d == 64 || d == 128, "tf_kv_quantize_e4m3: head_dim %d not in {64,128}", d);
  TF_CHECK_ARG(Hkv >= 1 && n >= 0 && slot0 >= 0 && (long long)slot0 + n <= cap, "tf_kv_quantize_e4m3: rows [%d,%d) outside [0,%lld)",
               slot0, slot0 + n, cap);
  TF_CHECK_ARG(src_head_stride >= cap * d && src_head_stride % 8 == 0 && ((uintptr_t)src & 15) == 0 && ((uintptr_t)codes & 15) == 0,
               "tf_kv_quantize_e4m3: src must be 16-byte aligned with a head stride of at least cap*d elements (a multiple of 8)");
  if (n == 0) return TF_OK;
  dim3 grid((n + 3) / 4, Hkv);
  cudaStream_t stream = (cudaStream_t)stream_;
  if (d == 128) kv_quantize_kernel<128><<<grid, 128, 0, stream>>>((const __half*)src, src_head_stride, slot0, n, (uint8_t*)codes, exps, cap);
  else kv_quantize_kernel<64><<<grid, 128, 0, stream>>>((const __half*)src, src_head_stride, slot0, n, (uint8_t*)codes, exps, cap);
  TF_CHECK_LAUNCH();
  return TF_OK;
}

int tf_draft_attn(const void* q, const void* K, const void* V, long long kv_head_stride, const void* cos, const void* sin,
                  int kv_len, int R, int H, int d, float scale, void* out, tf_stream_t stream_) {
  using namespace tf;
  TF_CHECK_ARG(q && K && V && cos && sin && out, "tf_draft_attn: NULL pointer");
  TF_CHECK_ARG(R >= 1 && H >= 1 && kv_len >= R, "tf_draft_attn: need kv_len >= R >= 1 (kv_len=%d, R=%d)", kv_len, R);
  TF_CHECK_SUPPORTED(d == 64 || d == 128, "tf_draft_attn: head_dim %d not in {64,128}", d);
  const size_t smem = (size_t)kv_len * (d + 8) * 2 * 2 + (size_t)(kDraftThreads / 32) * kv_len * 4;
  TF_CHECK_SUPPORTED(smem <= 200 * 1024, "tf_draft_attn: window of %d keys needs %zu B of shared memory", kv_len, smem);
  const float scale_log2 = scale * 1.4426950408889634f;
  dim3 grid(H, (R + kDraftRowsPerCta - 1) / kDraftRowsPerCta);
  cudaStream_t stream = (cudaStream_t)stream_;
  if (d == 64) {
    TF_ENSURE_DYNAMIC_SMEM(draft_attn_kernel<64>, 200 * 1024);
    TF_CHECK_CUDA(launch_kernel(kPdlDraftAttn, draft_attn_kernel<64>, grid, kDraftThreads, smem, stream, (const __half*)q, (const __half*)K, (const __half*)V, kv_head_stride,
                                                                 (const __half*)cos, (const __half*)sin, kv_len, R, H, scale_log2, (__half*)out));
  } else {
    TF_ENSURE_DYNAMIC_SMEM(draft_attn_kernel<128>, 200 * 1024);
    TF_CHECK_CUDA(launch_kernel(kPdlDraftAttn, draft_attn_kernel<128>, grid, kDraftThreads, smem, stream, (const __half*)q, (const __half*)K, (const __half*)V, kv_head_stride,
                                                                  (const __half*)cos, (const __half*)sin, kv_len, R, H, scale_log2, (__half*)out));
  }
  TF_CHECK_LAUNCH();
  return TF_OK;
}

int tf_tail_update(const void* K, const void* V, long long kv_layer_stride, long long kv_head_stride, void* retrK,
                   void* retrV, long long r_layer_stride, long long r_head_stride, int n_layers, int H, int d, int prefill,
                   int budget, int seq_len_host, const int32_t* seq_len_dev, int max_new, tf_stream_t stream_) {
  using namespace tf;
  TF_CHECK_ARG(K && V && retrK && retrV, "tf_tail_update: NULL pointer");
  TF_CHECK_ARG(n_layers >= 1 && H >= 1 && d % 8 == 0, "tf_tail_update: bad extents");
  TF_CHECK_ARG(max_new >= 0 && max_new <= budget, "tf_tail_update: max_new %d exceeds budget %d", max_new, budget);
  if (!seq_len_dev) {
    TF_CHECK_ARG(seq_len_host - prefill <= budget, "tf_tail_update: %d new tokens exceed budget %d", seq_len_host - prefill, budget);
    if (seq_len_host <= prefill) return TF_OK;
    max_new = seq_len_host - prefill;
  }
  if (max_new == 0) return TF_OK;
  int gx = (max_new * (d / 8) + 255) / 256;
  if (gx > 16) gx = 16;
  dim3 grid(gx, H, n_layers);
  tail_update_kernel<<<grid, 256, 0, (cudaStream_t)stream_>>>((const __half*)K, (const __half*)V, kv_layer_stride, kv_head_stride,
                                                              (__half*)retrK, (__half*)retrV, r_layer_stride, r_head_stride, d,
                                                              prefill, budget, seq_len_host, seq_len_dev);
  TF_CHECK_LAUNCH();
  return TF_OK;
}

int tf_tail_update_e4m3(const void* K, const void* V, const int8_t* Kexp, const int8_t* Vexp, long long kv_layer_stride,
                        long long kv_head_stride, void* retrK, void* retrV, long long r_layer_stride, long long r_head_stride,
                        int n_layers, int H, int d, int prefill, int budget, int seq_len_host, const int32_t* seq_len_dev,
                        int max_new, tf_stream_t stream_) {
  using namespace tf;
  TF_CHECK_ARG(K && V && Kexp && Vexp && retrK && retrV, "tf_tail_update_e4m3: NULL pointer");
  TF_CHECK_ARG(n_layers >= 1 && H >= 1 && d % 8 == 0, "tf_tail_update_e4m3: bad extents");
  TF_CHECK_ARG(kv_layer_stride % d == 0 && kv_head_stride % d == 0 && ((((uintptr_t)K | (uintptr_t)V)) & 7) == 0,
               "tf_tail_update_e4m3: code strides must be multiples of d and codes 8-byte aligned");
  TF_CHECK_ARG(max_new >= 0 && max_new <= budget, "tf_tail_update_e4m3: max_new %d exceeds budget %d", max_new, budget);
  if (!seq_len_dev) {
    TF_CHECK_ARG(seq_len_host - prefill <= budget, "tf_tail_update_e4m3: %d new tokens exceed budget %d", seq_len_host - prefill, budget);
    if (seq_len_host <= prefill) return TF_OK;
    max_new = seq_len_host - prefill;
  }
  if (max_new == 0) return TF_OK;
  int gx = (max_new * (d / 8) + 255) / 256;
  if (gx > 16) gx = 16;
  dim3 grid(gx, H, n_layers);
  tail_update_e4m3_kernel<<<grid, 256, 0, (cudaStream_t)stream_>>>((const uint8_t*)K, (const uint8_t*)V, Kexp, Vexp, kv_layer_stride,
                                                                   kv_head_stride, (__half*)retrK, (__half*)retrV, r_layer_stride,
                                                                   r_head_stride, d, prefill, budget, seq_len_host, seq_len_dev);
  TF_CHECK_LAUNCH();
  return TF_OK;
}

int tf_tail_update_to_e4m3(const void* K, const void* V, const int8_t* Kexp, const int8_t* Vexp, long long kv_layer_stride,
                           long long kv_head_stride, void* retrK, void* retrV, int8_t* retrKexp, int8_t* retrVexp,
                           long long r_layer_stride, long long r_head_stride, int n_layers, int H, int d, int prefill, int budget,
                           int seq_len_host, const int32_t* seq_len_dev, int max_new, tf_stream_t stream_) {
  using namespace tf;
  TF_CHECK_ARG(K && V && retrK && retrV && retrKexp && retrVexp, "tf_tail_update_to_e4m3: NULL pointer");
  TF_CHECK_ARG(!Kexp == !Vexp, "tf_tail_update_to_e4m3: the source's exponents are both NULL (fp16 store) or both set");
  TF_CHECK_ARG(n_layers >= 1 && H >= 1, "tf_tail_update_to_e4m3: bad extents");
  TF_CHECK_SUPPORTED(d == 64 || d == 128, "tf_tail_update_to_e4m3: head_dim %d not in {64,128}", d);
  TF_CHECK_ARG(kv_layer_stride % d == 0 && kv_head_stride % d == 0 && r_layer_stride % d == 0 && r_head_stride % d == 0,
               "tf_tail_update_to_e4m3: strides must be multiples of d");
  TF_CHECK_ARG(((((uintptr_t)K | (uintptr_t)V | (uintptr_t)retrK | (uintptr_t)retrV)) & 7) == 0,
               "tf_tail_update_to_e4m3: stores must be 8-byte aligned");
  TF_CHECK_ARG(max_new >= 0 && max_new <= budget, "tf_tail_update_to_e4m3: max_new %d exceeds budget %d", max_new, budget);
  if (!seq_len_dev) {
    TF_CHECK_ARG(seq_len_host - prefill <= budget, "tf_tail_update_to_e4m3: %d new tokens exceed budget %d", seq_len_host - prefill,
                 budget);
    if (seq_len_host <= prefill) return TF_OK;
    max_new = seq_len_host - prefill;
  }
  if (max_new == 0) return TF_OK;
  int gx = (max_new + 7) / 8;  // 8 warps per CTA, one row each
  if (gx > 16) gx = 16;
  dim3 grid(gx, H, n_layers);
  cudaStream_t stream = (cudaStream_t)stream_;
#define LAUNCH_TAIL8(D_, E_)                                                                                                      \
  tail_update_to_e4m3_kernel<D_, E_><<<grid, 256, 0, stream>>>(K, V, Kexp, Vexp, kv_layer_stride, kv_head_stride, (uint8_t*)retrK, \
                                                               (uint8_t*)retrV, retrKexp, retrVexp, r_layer_stride, r_head_stride,  \
                                                               prefill, budget, seq_len_host, seq_len_dev)
  if (d == 128) { if (Kexp) LAUNCH_TAIL8(128, true); else LAUNCH_TAIL8(128, false); }
  else { if (Kexp) LAUNCH_TAIL8(64, true); else LAUNCH_TAIL8(64, false); }
#undef LAUNCH_TAIL8
  TF_CHECK_LAUNCH();
  return TF_OK;
}

int tf_window_slide(void* K, void* V, long long layer_stride, long long head_stride, int n_layers, int H, int d,
                    int src_start, int dst_start, int n_rows, tf_stream_t stream_) {
  using namespace tf;
  TF_CHECK_ARG(K && V && n_layers >= 1 && H >= 1 && d % 8 == 0, "tf_window_slide: bad arguments");
  TF_CHECK_ARG(src_start >= 0 && dst_start >= 0 && n_rows >= 0, "tf_window_slide: negative range");
  if (n_rows == 0 || src_start == dst_start) return TF_OK;
  const size_t smem = (size_t)n_rows * d * 2;
  TF_CHECK_SUPPORTED(smem <= 200 * 1024, "tf_window_slide: window of %d rows needs %zu B of shared memory", n_rows, smem);
  TF_ENSURE_DYNAMIC_SMEM(window_slide_kernel, 200 * 1024);
  dim3 grid(H, n_layers);
  window_slide_kernel<<<grid, 256, smem, (cudaStream_t)stream_>>>((__half*)K, (__half*)V, layer_stride, head_stride, d, src_start,
                                                                  nullptr, dst_start, n_rows);
  TF_CHECK_LAUNCH();
  return TF_OK;
}

int tf_window_slide_dev(void* K, void* V, long long layer_stride, long long head_stride, int L, int H, int d, int src_base,
                        const int32_t* shift_dev, int dst_start, int n_rows, tf_stream_t stream) {
  using namespace tf;
  TF_CHECK_ARG(K && V && shift_dev && L >= 1 && H >= 1 && n_rows >= 1 && d % 8 == 0, "tf_window_slide_dev: bad arguments");
  const size_t smem = (size_t)n_rows * d * 2;
  TF_CHECK_SUPPORTED(smem <= 200 * 1024, "tf_window_slide_dev: window of %d rows does not fit in shared memory", n_rows);
  TF_ENSURE_DYNAMIC_SMEM(window_slide_kernel, 200 * 1024);
  window_slide_kernel<<<dim3(H, L), 256, smem, (cudaStream_t)stream>>>((__half*)K, (__half*)V, layer_stride, head_stride, d, src_base,
                                                                      shift_dev, dst_start, n_rows);
  TF_CHECK_LAUNCH();
  return TF_OK;
}

int tf_kv_compact(void* K, void* V, long long layer_stride, long long head_stride, int n_layers, int H, int d,
                  const int32_t* src_idx_dev, int n, int dst_start, tf_stream_t stream_) {
  using namespace tf;
  TF_CHECK_ARG(K && V && src_idx_dev && n_layers >= 1 && H >= 1 && d % 8 == 0, "tf_kv_compact: bad arguments");
  TF_CHECK_ARG(n >= 0 && dst_start >= 0, "tf_kv_compact: negative range");
  if (n == 0) return TF_OK;
  const size_t smem = (size_t)n * d * 2;
  TF_CHECK_SUPPORTED(smem <= 48 * 1024, "tf_kv_compact: %d rows need %zu B of shared memory", n, smem);
  dim3 grid(H, n_layers);
  kv_compact_kernel<<<grid, 128, smem, (cudaStream_t)stream_>>>((__half*)K, (__half*)V, layer_stride, head_stride, d, src_idx_dev, n,
                                                               dst_start);
  TF_CHECK_LAUNCH();
  return TF_OK;
}

int tf_kv_compact_e4m3(void* k_codes, void* v_codes, int8_t* k_exp, int8_t* v_exp, long long cap, int n_layers, int H, int d,
                       const int32_t* src_idx_dev, int n, int dst_start, tf_stream_t stream_) {
  using namespace tf;
  TF_CHECK_ARG(k_codes && v_codes && src_idx_dev, "tf_kv_compact_e4m3: NULL pointer");
  TF_CHECK_ARG(k_exp && v_exp, "tf_kv_compact_e4m3: NULL exponent pointer");
  TF_CHECK_ARG(n_layers >= 1 && H >= 1 && (d == 64 || d == 128) && cap >= 1, "tf_kv_compact_e4m3: bad arguments");
  TF_CHECK_ARG((((uintptr_t)k_codes | (uintptr_t)v_codes) & 15) == 0, "tf_kv_compact_e4m3: codes must be 16-byte aligned");
  TF_CHECK_ARG(n >= 0 && dst_start >= 0 && dst_start + (long long)n <= cap, "tf_kv_compact_e4m3: destination rows outside [0, cap)");
  if (n == 0) return TF_OK;
  const size_t smem = (size_t)2 * n * d + 2 * n;
  TF_CHECK_SUPPORTED(smem <= 48 * 1024, "tf_kv_compact_e4m3: %d rows need %zu B of shared memory", n, smem);
  kv_compact_e4m3_kernel<<<dim3(H, n_layers), 128, smem, (cudaStream_t)stream_>>>((uint8_t*)k_codes, (uint8_t*)v_codes, k_exp, v_exp, cap,
                                                                                  H, d, src_idx_dev, n, dst_start);
  TF_CHECK_LAUNCH();
  return TF_OK;
}

int tf_add_rmsnorm(void* h, const void* delta, const void* weight, float eps, void* out, int rows, int hidden,
                   tf_stream_t stream_) {
  using namespace tf;
  TF_CHECK_ARG(h && weight && out && rows >= 1 && hidden >= 8 && hidden % 8 == 0, "tf_add_rmsnorm: hidden must be a positive multiple of 8");
  TF_CHECK_SUPPORTED(hidden <= 32768, "tf_add_rmsnorm: hidden %d > 32768", hidden);
  TF_CHECK_ARG((((uintptr_t)h | (uintptr_t)weight | (uintptr_t)out | (uintptr_t)delta) & 15) == 0, "tf_add_rmsnorm: pointers must be 16-byte aligned");
  const int nvec = hidden / 8;
  int vpt = (nvec + 1023) / 1024;
  int threads = ((nvec + vpt - 1) / vpt + 31) / 32 * 32;
  cudaStream_t stream = (cudaStream_t)stream_;
  if (vpt == 1) TF_CHECK_CUDA(launch_kernel(kPdlNorm, add_rmsnorm_kernel<1>, rows, threads, 0, stream, (__half*)h, (const __half*)delta, (const __half*)weight, eps, (__half*)out, hidden));
  else if (vpt == 2) TF_CHECK_CUDA(launch_kernel(kPdlNorm, add_rmsnorm_kernel<2>, rows, threads, 0, stream, (__half*)h, (const __half*)delta, (const __half*)weight, eps, (__half*)out, hidden));
  else TF_CHECK_CUDA(launch_kernel(kPdlNorm, add_rmsnorm_kernel<4>, rows, threads, 0, stream, (__half*)h, (const __half*)delta, (const __half*)weight, eps, (__half*)out, hidden));
  TF_CHECK_LAUNCH();
  return TF_OK;
}

int tf_silu_mul(const void* gate_up, void* out, int rows, int inter, tf_stream_t stream_) {
  using namespace tf;
  TF_CHECK_ARG(gate_up && out && rows >= 1 && inter >= 2 && inter % 2 == 0, "tf_silu_mul: bad arguments");
  int gx = (inter / 2 + 255) / 256;
  dim3 grid(gx, rows);
  TF_CHECK_CUDA(launch_kernel(kPdlSilu, silu_mul_kernel, grid, 256, 0, (cudaStream_t)stream_, (const __half*)gate_up, (__half*)out, inter));
  TF_CHECK_LAUNCH();
  return TF_OK;
}

}  // extern "C"
