// Sampling kernels: temperature + top-p + softmax (utils/sampling.py:5-60), multinomial-as-argmax (:63-65),
// residual max_fn (:68-75) and the fused speculative accept/reject walks of utils/decoding.py:97-134,192-220.
// One CTA per logits row; everything a row needs lives in shared memory (32768 floats = 128 KB).
#include <float.h>

#include "common.cuh"

namespace tf {

constexpr int kThreads = 1024;

// ---- block-wide primitives (1024 threads) ---------------------------------------------------------------------------
__device__ __forceinline__ float block_reduce_max(float v, float* red) {
  v = warp_max(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = (threadIdx.x & 31) < (blockDim.x >> 5) ? red[threadIdx.x & 31] : -INFINITY;
  r = warp_max(r);
  return r;
}
__device__ __forceinline__ float block_reduce_sum(float v, float* red) {
  v = warp_sum(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = (threadIdx.x & 31) < (blockDim.x >> 5) ? red[threadIdx.x & 31] : 0.f;
  r = warp_sum(r);
  return r;
}
__device__ __forceinline__ int block_reduce_sum_int(int v, int* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  int r = (threadIdx.x & 31) < (blockDim.x >> 5) ? red[threadIdx.x & 31] : 0;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) r += __shfl_xor_sync(0xffffffffu, r, o);
  return r;
}
__device__ __forceinline__ uint32_t block_reduce_max_u32(uint32_t v, uint32_t* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = max(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  uint32_t r = (threadIdx.x & 31) < (blockDim.x >> 5) ? red[threadIdx.x & 31] : 0u;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) r = max(r, __shfl_xor_sync(0xffffffffu, r, o));
  return r;
}
// exclusive prefix sum of one value per thread, in thread order
template <typename T>
__device__ __forceinline__ T block_exclusive_scan(T v, T* red /* [32] */) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  T inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    T t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += t;
  }
  __syncthreads();
  if (lane == 31) red[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    T w = lane < (int)(blockDim.x >> 5) ? red[lane] : T(0);
    T winc = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      T t = __shfl_up_sync(0xffffffffu, winc, o);
      if (lane >= o) winc += t;
    }
    red[lane] = winc - w;  // exclusive warp offsets
  }
  __syncthreads();
  return red[warp] + inc - v;
}

struct ArgBest {
  float v;
  int i;
};
__device__ __forceinline__ bool arg_better(float v, int i, float bv, int bi) {
  // torch.argmax: NaN counts as the maximum; first index on ties
  const bool vn = v != v, bn = bv != bv;
  if (vn != bn) return vn;
  if (vn && bn) return i < bi;
  return v > bv || (v == bv && i < bi);
}
__device__ __forceinline__ ArgBest block_argmax(ArgBest b, float* redv, int* redi) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, b.v, o);
    const int oi = __shfl_xor_sync(0xffffffffu, b.i, o);
    if (arg_better(ov, oi, b.v, b.i)) { b.v = ov; b.i = oi; }
  }
  __syncthreads();
  if ((threadIdx.x & 31) == 0) { redv[threadIdx.x >> 5] = b.v; redi[threadIdx.x >> 5] = b.i; }
  __syncthreads();
  ArgBest r{redv[threadIdx.x & 31], redi[threadIdx.x & 31]};
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, r.v, o);
    const int oi = __shfl_xor_sync(0xffffffffu, r.i, o);
    if (arg_better(ov, oi, r.v, r.i)) { r.v = ov; r.i = oi; }
  }
  return r;
}

// IEEE division out of line: the correctly rounded quotient the reference's `/` gives (ATen), without replicating the
// special-case path of div.rn at every unrolled call site, which would bloat the 25 K-instruction norm_logits body and stall
// it on instruction fetch.
__device__ __noinline__ float div_rn(float a, float b) { return __fdiv_rn(a, b); }

// argmax_i num(i) / expo[i] over [0,V); every thread returns the winner.  Eight independent iterations in flight per thread.
template <typename F>
__device__ __forceinline__ int block_sample(F num, const float* __restrict__ expo, int V, float* redv, int* redi) {
  ArgBest b{-INFINITY, 0x7fffffff};
  const int step = blockDim.x;
  int i = threadIdx.x;
  for (; i + 7 * step < V; i += 8 * step) {
    float n[8], e[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) { n[u] = num(i + u * step); e[u] = expo[i + u * step]; }
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const float v = __fdiv_rn(n[u], e[u]);
      if (arg_better(v, i + u * step, b.v, b.i)) { b.v = v; b.i = i + u * step; }
    }
  }
  for (; i < V; i += step) {
    const float v = __fdiv_rn(num(i), expo[i]);
    if (arg_better(v, i, b.v, b.i)) { b.v = v; b.i = i; }
  }
  return block_argmax(b, redv, redi).i;
}

// --------------------------------------------------------------------------------------------------------------------
// norm_logits (temperature, top-p, softmax) — sort-free and deterministic.
//
// The reference sorts the row, takes the cumulative softmax mass and keeps sorted position j iff the mass BEFORE it is
// <= top_p (sampling.py:20-26).  Equivalent without a sort: find the threshold value v* = the smallest logit whose
// strictly-greater mass is <= top_p; keep everything above v*, and of the tokens equal to v* the first `quota` in ascending
// index order (what a stable descending sort yields).  v* is found by bisection on the order-preserving 32-bit key of the
// logit (2 key bits per pass, 16 passes); masses are 31-bit fixed point (p * 2^31: the masses of a row sum to ~2^31, so a
// thread's 32 items can never overflow 32 bits; warp/block totals are 64-bit), so the
// result does not depend on summation order and the tie quota is exact integer arithmetic.
// Each of the 512 threads owns elements {tid + 512 j}, j < 64: keys live in registers, fixed-point masses in shared memory
// (128 KB).
// --------------------------------------------------------------------------------------------------------------------
constexpr int kNlThreads = 512;                                // 128 registers per thread: the 64 keys stay in registers
constexpr int kItems = TF_SAMPLING_MAX_VOCAB / kNlThreads;     // 64
constexpr int kNlWarps = kNlThreads / 32;                      // 16

__device__ __forceinline__ uint32_t float_key(float x) {
  if (x == 0.f) x = 0.f;  // -0 == +0
  const uint32_t b = __float_as_uint(x);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float key_float(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}
__device__ __forceinline__ unsigned long long warp_sum_u64(unsigned long long v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__global__ void __launch_bounds__(kNlThreads) norm_logits_kernel(const float* __restrict__ logits, long long row_stride,
                                                               int V, float temperature, float top_p,
                                                               float* __restrict__ probs) {
  extern __shared__ uint32_t mass_s[];  // [kItems * kNlThreads]
  __shared__ float redf[32];
  __shared__ int redi[32];
  __shared__ unsigned long long red64[2][3][32];  // (16 warps write, lanes >= 16 read zeros)
  __shared__ int tie_tab[kItems * kNlWarps];  // [round j][warp] = 1024 entries, index order
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* lg = logits + (size_t)blockIdx.x * row_stride;
  float* out = probs + (size_t)blockIdx.x * V;

  uint32_t key[kItems];
  float mx = -INFINITY;
#pragma unroll
  for (int j = 0; j < kItems; ++j) {
    const int i = tid + j * kNlThreads;
    if (i < V) {
      const float x = div_rn(lg[i], temperature);
      key[j] = float_key(x);
      mx = fmaxf(mx, x);
    } else {
      key[j] = 0u;  // below every real key; mass 0
    }
  }
  mx = block_reduce_max(mx, redf);
  float z = 0.f;
#pragma unroll
  for (int j = 0; j < kItems; ++j)
    if (tid + j * kNlThreads < V) z += expf(key_float(key[j]) - mx);
  const float Z1 = block_reduce_sum(z, redf);

  uint32_t kstar = 0u;       // threshold key: keys above are kept, keys below dropped
  int quota = 0x7fffffff;    // how many of the tokens equal to the threshold are kept (ascending index)
  const bool filter = top_p > 0.f && top_p < 1.f;
  if (filter) {
    const float scale = 2147483648.f / Z1;  // 2^31
#pragma unroll
    for (int j = 0; j < kItems; ++j) {
      const int i = tid + j * kNlThreads;
      mass_s[i] = (i < V) ? __float2uint_rn(expf(key_float(key[j]) - mx) * scale) : 0u;  // <= 2^31
    }
    const unsigned long long tp = (unsigned long long)((double)top_p * 2147483648.0);
    // largest key kf with mass(key > kf) > tp  (predicate false); the threshold is kf + 1
    uint32_t kf = 0u;
    bool any_false;
    {
      uint32_t s0_32 = 0;
#pragma unroll
      for (int j = 0; j < kItems; ++j) s0_32 += (key[j] > 0u) ? mass_s[tid + j * kNlThreads] : 0u;
      unsigned long long s0 = warp_sum_u64(s0_32);
      if (lane == 0) red64[0][0][warp] = s0;
      __syncthreads();
      unsigned long long t0 = warp_sum_u64(lane < kNlWarps ? red64[0][0][lane] : 0ull);
      any_false = t0 > tp;  // if even "everything above key 0" fits under top_p, every token is kept
      __syncthreads();
    }
    if (any_false) {
      int buf = 0;
#pragma unroll 1
      for (int bit = 30; bit >= 0; bit -= 2) {
        const uint32_t cb = kf | (1u << bit), ca = kf | (2u << bit), cc = kf | (3u << bit);  // cb < ca < cc
        uint32_t sa32 = 0, sb32 = 0, sc32 = 0;  // cannot overflow: all masses of the row sum to ~2^31
#pragma unroll
        for (int j = 0; j < kItems; ++j) {
          const uint32_t m = mass_s[tid + j * kNlThreads];
          const uint32_t k = key[j];
          sa32 += (k > ca) ? m : 0u;
          sb32 += (k > cb) ? m : 0u;
          sc32 += (k > cc) ? m : 0u;
        }
        const unsigned long long sa = warp_sum_u64(sa32), sb = warp_sum_u64(sb32), sc = warp_sum_u64(sc32);
        if (lane == 0) { red64[buf][0][warp] = sa; red64[buf][1][warp] = sb; red64[buf][2][warp] = sc; }
        __syncthreads();
        const unsigned long long ta = warp_sum_u64(lane < kNlWarps ? red64[buf][0][lane] : 0ull);
        const unsigned long long tb = warp_sum_u64(lane < kNlWarps ? red64[buf][1][lane] : 0ull);
        const unsigned long long tc = warp_sum_u64(lane < kNlWarps ? red64[buf][2][lane] : 0ull);
        if (tc > tp) kf = cc;
        else if (ta > tp) kf = ca;
        else if (tb > tp) kf = cb;
        buf ^= 1;  // double-buffered: the next pass writes the other buffer, one barrier per pass suffices
      }
      kstar = kf + 1u;  // an existing key: mass(key > k) is constant between consecutive existing keys
      // mass above the threshold, and count / unit mass of the tokens sitting exactly on it
      uint32_t sg32 = 0;
      int cnt = 0;
      uint32_t unit = 0u;
#pragma unroll
      for (int j = 0; j < kItems; ++j) {
        const uint32_t m = mass_s[tid + j * kNlThreads];
        if (key[j] > kstar) sg32 += m;
        else if (key[j] == kstar) { ++cnt; unit = m; }
      }
      const unsigned long long sg = warp_sum_u64(sg32);
      __syncthreads();
      if (lane == 0) red64[0][0][warp] = sg;
      const int cnt_eq = block_reduce_sum_int(cnt, redi);  // (contains the barriers that publish red64)
      const uint32_t unit_m = block_reduce_max_u32(unit, reinterpret_cast<uint32_t*>(redi));
      const unsigned long long m_gt = warp_sum_u64(lane < kNlWarps ? red64[0][0][lane] : 0ull);
      unsigned long long q = cnt_eq;
      if (unit_m > 0u && m_gt <= tp) q = (tp - m_gt) / unit_m + 1ull;
      quota = (int)(q < (unsigned long long)cnt_eq ? q : (unsigned long long)cnt_eq);
      if (quota < cnt_eq) {
        // rank of each tied token in ascending index order: index = tid + 512 j = (warp, lane) within round j
#pragma unroll
        for (int j = 0; j < kItems; ++j) {
          const unsigned bal = __ballot_sync(0xffffffffu, key[j] == kstar);
          if (lane == 0) tie_tab[j * kNlWarps + warp] = __popc(bal);
        }
        __syncthreads();
        // exclusive scan of the 1024 table entries (index order) with 512 threads: two consecutive entries per thread
        const int m0 = tie_tab[2 * tid], m1 = tie_tab[2 * tid + 1];
        const int pre = block_exclusive_scan<int>(m0 + m1, redi);
        __syncthreads();
        tie_tab[2 * tid] = pre;
        tie_tab[2 * tid + 1] = pre + m0;
        __syncthreads();
      }
      // drop what falls outside the quota by clearing its key below the threshold marker (key 0 == "dropped")
      if (quota < cnt_eq) {
#pragma unroll
        for (int j = 0; j < kItems; ++j) {
          const bool eq = key[j] == kstar;
          const unsigned bal = __ballot_sync(0xffffffffu, eq);
          if (eq) {
            const int rank = tie_tab[j * kNlWarps + warp] + __popc(bal & ((1u << lane) - 1u));
            if (rank >= quota) key[j] = 0u;
          }
        }
      }
    }
  }

  float z2 = 0.f;
#pragma unroll
  for (int j = 0; j < kItems; ++j) {
    const int i = tid + j * kNlThreads;
    const bool keep = (i < V) && (!filter || kstar == 0u || key[j] >= kstar);
    if (!keep) key[j] = 0u;
    else z2 += expf(key_float(key[j]) - mx);
  }
  const float Z2 = block_reduce_sum(z2, redf);
#pragma unroll
  for (int j = 0; j < kItems; ++j) {
    const int i = tid + j * kNlThreads;
    if (i < V) out[i] = key[j] ? div_rn(expf(key_float(key[j]) - mx), Z2) : 0.f;
  }
}

__global__ void __launch_bounds__(kThreads) sample_argmax_kernel(const float* __restrict__ probs, long long ps,
                                                                 const float* __restrict__ expo, long long es, int V,
                                                                 int64_t* __restrict__ out) {
  __shared__ float redv[32];
  __shared__ int redi[32];
  const float* p = probs + (size_t)blockIdx.x * ps;
  const float* e = expo + (size_t)blockIdx.x * es;
  const int t = block_sample([&](int i) { return p[i]; }, e, V, redv, redi);
  if (threadIdx.x == 0) out[blockIdx.x] = (int64_t)t;
}

__global__ void __launch_bounds__(kThreads) residual_probs_kernel(const float* __restrict__ p, const float* __restrict__ q,
                                                                  int V, float* __restrict__ out) {
  __shared__ float redf[32];
  float s = 0.f;
  for (int i = threadIdx.x; i < V; i += kThreads) {
    const float x = p[i] - q[i];
    s += x > 0.f ? x : 0.f;
  }
  const float S = block_reduce_sum(s, redf);
  for (int i = threadIdx.x; i < V; i += kThreads) {
    const float x = p[i] - q[i];
    out[i] = __fdiv_rn(x > 0.f ? x : 0.f, S);
  }
}

// --------------------------------------------------------------------------------------------------------------------
// fused speculative decisions
// --------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ bool accept_test(float r, float p, float q, bool strict_less) {
  const float ratio = __fdiv_rn(p, q);
  if (ratio != ratio) return false;  // torch.min propagates NaN → comparison is False
  const float m = fminf(1.f, ratio);
  return strict_less ? (r < m) : (r <= m);
}

__global__ void __launch_bounds__(kThreads) middle_accept_kernel(const float* __restrict__ sp, const float* __restrict__ vp,
                                                                 int64_t* __restrict__ verify_tokens,
                                                                 const float* __restrict__ uniform,
                                                                 const float* __restrict__ expo, int gamma, int V,
                                                                 int32_t* __restrict__ st, int64_t* __restrict__ out_ids,
                                                                 float* __restrict__ spec_probs) {
  __shared__ float redv[32];
  __shared__ int redi[32];
  const int n = st[0];
  const int k = st[1];
  const int64_t t = verify_tokens[n + 1];
  const float* vpn = vp + (size_t)n * V;
  const bool accept = accept_test(uniform[0], vpn[t], sp[t], true);
  const int row = accept ? n + 1 : n;
  const float* vrow = vp + (size_t)row * V;
  const int t2 = block_sample([&](int i) { return vrow[i]; }, expo, V, redv, redi);  // contains __syncthreads
  // proposal rows attributed to the emitted ids (decoding.py:194,202 / :213)
  float* d0 = spec_probs + (size_t)k * V;
  if ((V & 3) == 0) {  // rows are 16-byte aligned (V * 4 B per row on top of 256-byte-aligned allocations)
    const float4* s0 = reinterpret_cast<const float4*>(vpn);
    float4* t0 = reinterpret_cast<float4*>(d0);
    for (int i = threadIdx.x; i < V / 4; i += kThreads) t0[i] = s0[i];
    if (accept) {
      const float4* s1 = reinterpret_cast<const float4*>(vrow);
      float4* t1 = reinterpret_cast<float4*>(spec_probs + (size_t)(k + 1) * V);
      for (int i = threadIdx.x; i < V / 4; i += kThreads) t1[i] = s1[i];
    }
  } else {
    for (int i = threadIdx.x; i < V; i += kThreads) d0[i] = vpn[i];
    if (accept) {
      float* d1 = spec_probs + (size_t)(k + 1) * V;
      for (int i = threadIdx.x; i < V; i += kThreads) d1[i] = vrow[i];
    }
  }
  if (threadIdx.x == 0) {
    int nn, kk;
    if (accept) {
      out_ids[k] = t;
      out_ids[k + 1] = (int64_t)t2;
      nn = n + 2; kk = k + 2;
    } else {
      out_ids[k] = (int64_t)t2;
      nn = n + 1; kk = k + 1;
    }
    if (nn <= gamma) verify_tokens[nn] = (int64_t)t2;
    st[0] = nn; st[1] = kk; st[2] = accept ? 1 : 0; st[3] += accept ? 1 : 0; st[4] += 1;
  }
}

__global__ void verify_accept_kernel(const float* __restrict__ p_rows, const float* __restrict__ q_rows,
                                     const int64_t* __restrict__ gen, int g2, const float* __restrict__ uniforms, int V,
                                     int strict_less, int64_t eos, int64_t first_token, int32_t* __restrict__ res,
                                     int64_t* __restrict__ pass_tokens) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  int count = 0, rejected = 0, examined = 0, hit_eos = 0;
  pass_tokens[0] = first_token;
  for (int i = 1; i < g2 + 2; ++i) pass_tokens[i] = 100;  // decoding.py:94
  for (int i = 0; i < g2; ++i) {
    const int64_t t = gen[i];
    ++examined;
    if (accept_test(uniforms[i], p_rows[(size_t)i * V + t], q_rows[(size_t)i * V + t], strict_less != 0)) {
      ++count;
      pass_tokens[count] = t;
      if (t == eos) { hit_eos = 1; break; }
    } else {
      rejected = 1;
      break;
    }
  }
  res[0] = count; res[1] = rejected; res[2] = examined; res[3] = hit_eos;
}

__global__ void __launch_bounds__(kThreads) verify_resample_kernel(const float* __restrict__ p_rows,
                                                                   const float* __restrict__ q_rows,
                                                                   const int64_t* __restrict__ gen, int g2,
                                                                   const float* __restrict__ expo, int V,
                                                                   int32_t* __restrict__ res, int64_t* __restrict__ out_token,
                                                                   int64_t* __restrict__ pass_tokens) {
  __shared__ float redv[32];
  __shared__ int redi[32];
  const int count = res[0];
  const int rejected = res[1];
  __syncthreads();
  if (rejected) {
    const float* p = p_rows + (size_t)count * V;
    const float* q = q_rows + (size_t)count * V;
    float s = 0.f;
    for (int i = threadIdx.x; i < V; i += kThreads) {
      const float x = p[i] - q[i];
      s += x > 0.f ? x : 0.f;
    }
    const float S = block_reduce_sum(s, redv);
    const int t = block_sample([&](int i) { const float x = p[i] - q[i]; return __fdiv_rn(x > 0.f ? x : 0.f, S); },
                               expo, V, redv, redi);
    if (threadIdx.x == 0) { out_token[0] = t; pass_tokens[count + 1] = t; }
  } else if (count == g2) {
    const float* p = p_rows + (size_t)g2 * V;
    const int t = block_sample([&](int i) { return p[i]; }, expo, V, redv, redi);
    if (threadIdx.x == 0) { out_token[0] = t; pass_tokens[count + 1] = t; res[0] = count + 1; }
  } else {
    if (threadIdx.x == 0) out_token[0] = gen[count - 1];  // stopped on an accepted EOS: nothing is drawn
  }
}

// --------------------------------------------------------------------------------------------------------------------
// Sequoia accept walk — utils/SpecTree_TP.py: accept_step (:147-165) driven by verify (:181-197), one CTA.
//   cur = 0 (the root = last committed token).  At node `cur`: p = target_probs[cur]; for each child (in order): token =
//   verify_tokens[child]; q = softmax(draft_logits[cur] / T); r = next uniform; accept child iff p[token] > r * q[token];
//   otherwise p = relu(p - q) / sum and draft_logits[cur][token] = -FLT_MAX (so the next q excludes it).  An accepted child
//   becomes `cur` (tokens 0 / 2 end the generation: "terminal"); when every child is rejected, or a leaf is reached, the
//   current p is the distribution the next token is drawn from.
// out (int32[32]): [0] accepted count, [1] code (-1 all children rejected, -2 leaf), [2] uniforms consumed, [3] terminal,
//                  [4] residual has NaN / zero mass, [8..] accepted node ids.
// --------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) tree_accept_walk_kernel(const float* __restrict__ target_probs, float* __restrict__ draft_logits,
                                                                    const int64_t* __restrict__ verify_tokens,
                                                                    const int32_t* __restrict__ succ_off, const int32_t* __restrict__ succ,
                                                                    const float* __restrict__ uniforms, float inv_T, int V,
                                                                    int max_accept, int32_t* __restrict__ out,
                                                                    float* __restrict__ residual, float* __restrict__ pbuf) {
  __shared__ float redf[32];
  __shared__ int s_accept;
  const int tid = threadIdx.x;
  int cur = 0, n_acc = 0, used = 0, code = 0, terminal = 0;
  bool nan_res = false;
  while (true) {
    const int c0 = succ_off[cur], c1 = succ_off[cur + 1];
    const float* p = target_probs + (size_t)cur * V;  // accept_step starts from the node's own target row
    if (c0 == c1) {  // leaf
      for (int i = tid; i < V; i += kThreads) residual[i] = p[i];
      code = -2;
      break;
    }
    float* dl = draft_logits + (size_t)cur * V;
    bool accepted = false;
    int child = -1;
    for (int c = c0; c < c1; ++c) {
      child = succ[c];
      const int64_t token = verify_tokens[child];
      // q = softmax(dl / T)
      float mx = -INFINITY;
      for (int i = tid; i < V; i += kThreads) mx = fmaxf(mx, dl[i] * inv_T);
      mx = block_reduce_max(mx, redf);
      float z = 0.f;
      for (int i = tid; i < V; i += kThreads) z += expf(dl[i] * inv_T - mx);
      const float Z = block_reduce_sum(z, redf);
      const float q_tok = __fdiv_rn(expf(dl[token] * inv_T - mx), Z);
      const float r = uniforms[used];
      ++used;
      if (tid == 0) s_accept = p[token] > r * q_tok;
      __syncthreads();
      accepted = s_accept != 0;
      __syncthreads();
      if (accepted) break;
      // p = relu(p - q) / sum ; draft_logits[token] = finfo(float32).min
      float sm = 0.f;
      for (int i = tid; i < V; i += kThreads) {
        const float qi = __fdiv_rn(expf(dl[i] * inv_T - mx), Z);
        const float x = p[i] - qi;
        const float v = x > 0.f ? x : 0.f;
        pbuf[i] = v;
        sm += v;
      }
      const float S = block_reduce_sum(sm, redf);
      for (int i = tid; i < V; i += kThreads) pbuf[i] = __fdiv_rn(pbuf[i], S);
      if (tid == 0) dl[token] = -FLT_MAX;
      __threadfence_block();
      __syncthreads();
      p = pbuf;
    }
    if (accepted) {
      if (tid == 0 && n_acc < max_accept) out[8 + n_acc] = child;
      ++n_acc;
      cur = child;
      const int64_t tok = verify_tokens[child];
      if (tok == 0 || tok == 2) { terminal = 1; break; }
      continue;
    }
    for (int i = tid; i < V; i += kThreads) residual[i] = p[i];
    code = -1;
    break;
  }
  __syncthreads();
  if (!terminal) {  // NaN / empty residual → the reference declares the run terminal (SpecTree_TP.py:199-200)
    float bad = 0.f;
    for (int i = tid; i < V; i += kThreads) { const float v = residual[i]; bad += (v != v) ? 1.f : 0.f; }
    nan_res = block_reduce_sum(bad, redf) > 0.f;
  }
  if (tid == 0) { out[0] = n_acc; out[1] = code; out[2] = used; out[3] = terminal; out[4] = nan_res ? 1 : 0; }
}

static int next_pow2(int x) {
  int p = 1;
  while (p < x) p <<= 1;
  return p;
}

}  // namespace tf

extern "C" {

size_t tf_norm_logits_workspace_bytes(int rows, int V) { (void)rows; (void)V; return 0; }

int tf_norm_logits(const float* logits, long long row_stride, int rows, int V, float temperature, float top_p,
                   float* probs, void* workspace, size_t workspace_bytes, tf_stream_t stream_) {
  using namespace tf;
  (void)workspace; (void)workspace_bytes;
  TF_CHECK_ARG(logits && probs && rows >= 0 && V > 0, "tf_norm_logits: bad arguments");
  TF_CHECK_SUPPORTED(V <= TF_SAMPLING_MAX_VOCAB, "tf_norm_logits: vocab %d > %d", V, TF_SAMPLING_MAX_VOCAB);
  TF_CHECK_ARG(temperature > 0.f, "tf_norm_logits: temperature must be > 0");
  if (rows == 0) return TF_OK;
  const size_t smem = (size_t)TF_SAMPLING_MAX_VOCAB * sizeof(uint32_t);
  TF_ENSURE_DYNAMIC_SMEM(norm_logits_kernel, smem);
  norm_logits_kernel<<<rows, kNlThreads, smem, (cudaStream_t)stream_>>>(logits, row_stride, V, temperature, top_p, probs);
  TF_CHECK_LAUNCH();
  return TF_OK;
}

int tf_sample_argmax(const float* probs, long long probs_row_stride, const float* expo, long long expo_row_stride,
                     int rows, int V, int64_t* out_tokens, tf_stream_t stream_) {
  using namespace tf;
  TF_CHECK_ARG(probs && expo && out_tokens && rows > 0 && V > 0, "tf_sample_argmax: bad arguments");
  sample_argmax_kernel<<<rows, kThreads, 0, (cudaStream_t)stream_>>>(probs, probs_row_stride, expo, expo_row_stride, V,
                                                                     out_tokens);
  TF_CHECK_LAUNCH();
  return TF_OK;
}

int tf_residual_probs(const float* p, const float* q, int V, float* out, tf_stream_t stream_) {
  using namespace tf;
  TF_CHECK_ARG(p && q && out && V > 0, "tf_residual_probs: bad arguments");
  residual_probs_kernel<<<1, kThreads, 0, (cudaStream_t)stream_>>>(p, q, V, out);
  TF_CHECK_LAUNCH();
  return TF_OK;
}

int tf_middle_accept(const float* draft_probs, const float* verify_probs, int64_t* verify_tokens, const float* uniform,
                     const float* expo, int gamma, int V, int32_t* st, int64_t* out_ids, float* spec_probs,
                     tf_stream_t stream_) {
  using namespace tf;
  TF_CHECK_ARG(draft_probs && verify_probs && verify_tokens && uniform && expo && st && out_ids && spec_probs,
               "tf_middle_accept: NULL pointer");
  TF_CHECK_ARG(gamma >= 1 && V > 0, "tf_middle_accept: bad gamma/V");
  middle_accept_kernel<<<1, kThreads, 0, (cudaStream_t)stream_>>>(draft_probs, verify_probs, verify_tokens, uniform, expo,
                                                                  gamma, V, st, out_ids, spec_probs);
  TF_CHECK_LAUNCH();
  return TF_OK;
}

int tf_tree_accept_walk(const float* target_probs, float* draft_logits, const int64_t* verify_tokens, const int32_t* succ_off,
                        const int32_t* succ, const float* uniforms, float temperature, int V, int max_accept, int32_t* out,
                        float* residual, float* scratch_V, tf_stream_t stream_) {
  using namespace tf;
  TF_CHECK_ARG(target_probs && draft_logits && verify_tokens && succ_off && succ && uniforms && out && residual && scratch_V,
               "tf_tree_accept_walk: NULL pointer");
  TF_CHECK_ARG(V > 0 && temperature > 0.f && max_accept >= 1 && max_accept <= 24, "tf_tree_accept_walk: bad V / temperature / max_accept");
  tree_accept_walk_kernel<<<1, kThreads, 0, (cudaStream_t)stream_>>>(target_probs, draft_logits, verify_tokens, succ_off, succ, uniforms,
                                                                     1.0f / temperature, V, max_accept, out, residual, scratch_V);
  TF_CHECK_LAUNCH();
  return TF_OK;
}

int tf_verify_accept(const float* p_rows, const float* q_rows, const int64_t* gen, int g2, const float* uniforms, int V,
                     int strict_less, int64_t eos_token, int64_t first_token, int32_t* res, int64_t* pass_tokens,
                     tf_stream_t stream_) {
  using namespace tf;
  TF_CHECK_ARG(p_rows && q_rows && gen && uniforms && res && pass_tokens && g2 >= 1 && V > 0, "tf_verify_accept: bad arguments");
  verify_accept_kernel<<<1, 32, 0, (cudaStream_t)stream_>>>(p_rows, q_rows, gen, g2, uniforms, V, strict_less, eos_token,
                                                            first_token, res, pass_tokens);
  TF_CHECK_LAUNCH();
  return TF_OK;
}

int tf_verify_resample(const float* p_rows, const float* q_rows, const int64_t* gen, int g2, const float* expo, int V,
                       int32_t* res, int64_t* out_token, int64_t* pass_tokens, tf_stream_t stream_) {
  using namespace tf;
  TF_CHECK_ARG(p_rows && q_rows && gen && expo && res && out_token && pass_tokens && g2 >= 1 && V > 0,
               "tf_verify_resample: bad arguments");
  verify_resample_kernel<<<1, kThreads, 0, (cudaStream_t)stream_>>>(p_rows, q_rows, gen, g2, expo, V, res, out_token,
                                                                    pass_tokens);
  TF_CHECK_LAUNCH();
  return TF_OK;
}

}  // extern "C"
