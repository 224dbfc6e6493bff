// The speculative decisions of the TriForce decode loop, written once for its two forms:
//   * the step-wise loop (sampling.cu: tf_sample_argmax, tf_middle_accept, tf_verify_accept, tf_verify_resample) reads its
//     uniforms and exponentials from buffers;
//   * the device loop (loop_graph.cu: tf_loop_draft_sample, tf_loop_middle_accept, tf_loop_verify) computes them inline from a
//     counter-based Philox stream.
// The kernels of both differ only in where a uniform or an exponential comes from; the argmax order, the sampler, the accept
// test and the bookkeeping of each decision are the functions below, so the two loops emit the same tokens from the same noise.
// Unless a comment says otherwise, a function here is called by every thread of one CTA of kThreads threads.
#pragma once

#include "common.cuh"

namespace tf {

constexpr int kThreads = 1024;

__device__ __forceinline__ float block_reduce_sum(float v, float* red) {
  v = warp_sum(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = (threadIdx.x & 31) < (blockDim.x >> 5) ? red[threadIdx.x & 31] : 0.f;
  r = warp_sum(r);
  return r;
}

// ---- torch.argmax order -------------------------------------------------------------------------------------------------
// A strict total order on (value, index), so the winner of a block does not depend on how elements are split across threads
// or in which order partial winners are combined.
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
// the winner of the per-thread bests of 32 full warps; every thread returns it
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

// accept iff r < min(1, p / q) (r <= min(1, p / q) when !strict_less); utils/decoding.py:98-99,192-193
__device__ __forceinline__ bool accept_test(float r, float p, float q, bool strict_less) {
  const float ratio = __fdiv_rn(p, q);
  if (ratio != ratio) return false;  // torch.min propagates NaN → comparison is False
  const float m = fminf(1.f, ratio);
  return strict_less ? (r < m) : (r <= m);
}

// ---- Philox4x32-10 stream ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
  constexpr uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(M0, c.x), lo0 = M0 * c.x;
    const uint32_t hi1 = __umulhi(M1, c.z), lo1 = M1 * c.z;
    c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
    k.x += W0;
    k.y += W1;
  }
  return c;
}
// Philox word -> uniform in (0, 1): (top 24 bits + 1/2) * 2^-24.  Above 2^23 the float sum is a tie that rounds to even, so the
// word 0xFFFFFF.. would give exactly 1.0, whose -log is -0.0 (p / -0 is NaN for p = 0, and NaN wins the sampling argmax).  That
// one value becomes 1 - 2^-24, which the rounded sum never produces: every other word keeps its bits.
__device__ __forceinline__ float philox_to_uniform(uint32_t x) {
  const float u = ((float)(x >> 8) + 0.5f) * (1.0f / 16777216.0f);
  return u < 1.0f ? u : __uint_as_float(0x3f7fffffu);
}
__device__ __forceinline__ float philox_uniform(unsigned long long seed, unsigned long long draw, uint32_t elem) {
  const uint4 r = philox4x32_10(make_uint4(elem >> 2, (uint32_t)draw, (uint32_t)(draw >> 32), 0u), make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
  return philox_to_uniform((elem & 3u) == 0 ? r.x : ((elem & 3u) == 1 ? r.y : ((elem & 3u) == 2 ? r.z : r.w)));
}
__device__ __forceinline__ float philox_exponential(unsigned long long seed, unsigned long long draw, uint32_t elem) {
  return -logf(philox_uniform(seed, draw, elem));
}

// ---- multinomial as argmax_i num(i) / e_i over [0, V), e_i ~ Exp(1) (utils/sampling.py:63-65) ---------------------------
// A noise source's scan(num, V) returns this thread's best of num(i) / e_i; block_sample reduces the bests.  Both scans visit
// every element once with the same division, so with the same e_i they give the same token.
//
// e_i = expo[i], read from a buffer.  Eight independent iterations in flight per thread.
struct ExpoFromBuffer {
  const float* __restrict__ expo;
  template <typename F>
  __device__ __forceinline__ ArgBest scan(F num, int V) const {
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
    return b;
  }
};
// e_i = philox_exponential(seed, draw, i), computed in place: one Philox call serves the four elements 4g .. 4g+3.
struct ExpoFromPhilox {
  unsigned long long seed, draw;
  template <typename F>
  __device__ __forceinline__ ArgBest scan(F num, int V) const {
    ArgBest b{-INFINITY, 0x7fffffff};
    const uint2 key = make_uint2((uint32_t)seed, (uint32_t)(seed >> 32));
    for (int g4 = threadIdx.x; g4 * 4 < V; g4 += blockDim.x) {
      const uint4 r = philox4x32_10(make_uint4((uint32_t)g4, (uint32_t)draw, (uint32_t)(draw >> 32), 0u), key);
      const uint32_t x[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int i = g4 * 4 + e;
        if (i < V) {
          const float v = __fdiv_rn(num(i), -logf(philox_to_uniform(x[e])));
          if (arg_better(v, i, b.v, b.i)) { b.v = v; b.i = i; }
        }
      }
    }
    return b;
  }
};
// every thread returns the sampled index
template <typename F, typename Expo>
__device__ __forceinline__ int block_sample(F num, const Expo& expo, int V, float* redv, int* redi) {
  return block_argmax(expo.scan(num, V), redv, redi).i;
}

// ---- the decisions --------------------------------------------------------------------------------------------------------
// One Middle_Spec decision (decoding.py:190-220).  n = st[0], k = st[1]; the draft token t = verify_tokens[n + 1] came from
// the draft row `sp`.  Accept t iff u < min(1, vp[n][t] / sp[t]); then sample t2 from vp row n + 1 (the bonus, on accept) or
// row n (the replacement, on reject), copy the proposal rows behind the emitted ids to spec_probs (decoding.py:194,202 / :213),
// emit [t, t2] or [t2] to out_ids, write t2 to verify_tokens[nn] (nn = the new n) and update
// st = {n, k, last accept flag, accepted draft tokens, inner iterations}.
template <typename Expo>
__device__ __forceinline__ void middle_spec_decision(const float* __restrict__ sp, const float* __restrict__ vp,
                                                     int64_t* __restrict__ verify_tokens, float u, const Expo& expo, int gamma,
                                                     int V, int32_t* __restrict__ st, int64_t* __restrict__ out_ids,
                                                     float* __restrict__ spec_probs, float* redv, int* redi) {
  const int n = st[0];
  const int k = st[1];
  const int64_t t = verify_tokens[n + 1];
  const float* vpn = vp + (size_t)n * V;
  const bool accept = accept_test(u, vpn[t], sp[t], true);
  const int row = accept ? n + 1 : n;
  const float* vrow = vp + (size_t)row * V;
  const int t2 = block_sample([&](int i) { return vrow[i]; }, expo, V, redv, redi);  // contains __syncthreads
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

// The outer accept walk (decoding.py:97-134), run by ONE thread: accept gen[i] iff uniform(i) < min(1, p_i[gen[i]] /
// q_i[gen[i]]) for i = 0, 1, ... until the first rejection, an accepted EOS or the end of gen[0, g2).
// pass_tokens[0, pass_len) = [first_token, the accepted ids, placeholders 100] (decoding.py:94).
struct AcceptWalk {
  int count;     // accepted ids: gen[0, count)
  int rejected;  // gen[count] was rejected
  int examined;  // ids tested
  int hit_eos;   // the walk stopped on an accepted EOS
};
template <typename U>
__device__ __forceinline__ AcceptWalk accept_walk(const float* __restrict__ p_rows, const float* __restrict__ q_rows,
                                                  const int64_t* __restrict__ gen, int g2, U uniform, int V, bool strict_less,
                                                  int64_t eos, int64_t first_token, int64_t* __restrict__ pass_tokens, int pass_len) {
  AcceptWalk w{0, 0, 0, 0};
  pass_tokens[0] = first_token;
  for (int i = 1; i < pass_len; ++i) pass_tokens[i] = 100;  // decoding.py:94
  for (int i = 0; i < g2; ++i) {
    const int64_t t = gen[i];
    ++w.examined;
    if (accept_test(uniform(i), p_rows[(size_t)i * V + t], q_rows[(size_t)i * V + t], strict_less)) {
      ++w.count;
      pass_tokens[w.count] = t;
      if (t == eos) { w.hit_eos = 1; break; }
    } else {
      w.rejected = 1;
      break;
    }
  }
  return w;
}

// The token that closes an outer step, after a walk that accepted gen[0, count) of gen[0, g2):
//   rejected            → sampled from the residual norm(max(p - q, 0)) of row `count` (sampling.py:68-75), decoding.py:114;
//   all g2 accepted     → the bonus token, sampled from the target's row g2 (decoding.py:127-134);
//   stopped on an EOS   → nothing is drawn: the accepted EOS gen[count - 1] is the next token.
// A drawn token is appended to pass_tokens[count + 1].  Every thread returns the next token.
template <typename Expo>
__device__ __forceinline__ int64_t resample_after_walk(const float* __restrict__ p_rows, const float* __restrict__ q_rows,
                                                       const int64_t* __restrict__ gen, int g2, int count, bool rejected,
                                                       const Expo& expo, int V, int64_t* __restrict__ pass_tokens,
                                                       float* redv, int* redi) {
  int t;
  if (rejected) {
    const float* p = p_rows + (size_t)count * V;
    const float* q = q_rows + (size_t)count * V;
    float s = 0.f;
    for (int i = threadIdx.x; i < V; i += kThreads) {
      const float x = p[i] - q[i];
      s += x > 0.f ? x : 0.f;
    }
    const float S = block_reduce_sum(s, redv);
    t = block_sample([&](int i) { const float x = p[i] - q[i]; return __fdiv_rn(x > 0.f ? x : 0.f, S); }, expo, V, redv, redi);
  } else if (count == g2) {
    const float* p = p_rows + (size_t)g2 * V;
    t = block_sample([&](int i) { return p[i]; }, expo, V, redv, redi);
  } else {
    return gen[count - 1];
  }
  if (threadIdx.x == 0) pass_tokens[count + 1] = t;
  return t;
}

}  // namespace tf
