// The whole draft → retrieve → verify iteration as ONE graph launch with a device-side loop — the replacement for the
// reference's utils/graph_infer.py (GraphInferenceEngine :129-194: one CUDA graph per draft offset + one verify graph, driven
// by utils/decoding.py:163-223 with a host synchronisation after every sampled token, :186,193,203) that north_star asks for.
//
//   parent graph = [ begin ] → WHILE(n < gamma) { draft forward (gamma rows) → draft sample → retrieval verify forward →
//                  accept / resample / bookkeeping → set condition } → [ full-KV verify of gamma+2 rows → accept walk + residual
//                  resample → KV / retrieval-tail / draft-window maintenance → results to pinned host memory ]
//
// The three bracketed parts are captured from the engine's own forwards (torch stream capture, kept as cudaGraph_t); this file
// holds what makes them a loop: the CUDA conditional WHILE node (cudaGraphConditionalHandle, set from a kernel with
// cudaGraphSetConditional), the device-side state machine of Middle_Spec (`n`, accepted ids, proposal rows — decoding.py:180-220)
// and of the outer accept walk (:97-134) in kernels that read their control variables from device memory, and a counter-based
// Philox4x32-10 noise source so that no random number has to come from the host.  Per outer iteration the host launches ONE
// graph and reads ONE small result record.
//
// Random numbers: draw `c` of stream (seed) = Philox4x32-10(counter = (element / 4, c_lo, c_hi, 0), key = seed); element i takes
// lane i % 4.  Uniforms u strictly inside (0, 1) (philox_to_uniform); exponentials -log(u) > 0.  The consumption order is the
// reference's (decoding.py:185,192,201/212,98,114/130): per inner iteration exponential (draft sample), uniform, exponential
// (accept / resample); per outer iteration one block of uniforms, then one exponential when a token is drawn.  `tf_philox_fill` replays the same draws for the step-wise
// (host-driven) loop, which is how the two loops are checked against each other event for event.
#include <float.h>
#include <string.h>

#include "common.cuh"

namespace tf {

constexpr int kLoopThreads = 1024;

struct PhiloxState {
  unsigned long long seed;
  unsigned long long ctr;  // next draw index
};

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

struct LoopBest {
  float v;
  int i;
};
__device__ __forceinline__ bool loop_better(float v, int i, float bv, int bi) {  // torch.argmax: NaN is the maximum, first index on ties
  const bool vn = v != v, bn = bv != bv;
  if (vn != bn) return vn;
  if (vn && bn) return i < bi;
  return v > bv || (v == bv && i < bi);
}
// argmax_i num(i) / Exp_i over [0, V) with Exp_i = exponential `draw` of the stream; every thread returns the winner.
// One Philox call serves the four elements 4g .. 4g+3 (the same element -> lane mapping as philox_uniform).
template <typename F>
__device__ __forceinline__ int loop_sample(F num, unsigned long long seed, unsigned long long draw, int V, float* redv, int* redi) {
  LoopBest b{-INFINITY, 0x7fffffff};
  const uint2 key = make_uint2((uint32_t)seed, (uint32_t)(seed >> 32));
  for (int g4 = threadIdx.x; g4 * 4 < V; g4 += blockDim.x) {
    const uint4 r = philox4x32_10(make_uint4((uint32_t)g4, (uint32_t)draw, (uint32_t)(draw >> 32), 0u), key);
    const uint32_t x[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int i = g4 * 4 + e;
      if (i < V) {
        const float v = __fdiv_rn(num(i), -logf(philox_to_uniform(x[e])));
        if (loop_better(v, i, b.v, b.i)) { b.v = v; b.i = i; }
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, b.v, o);
    const int oi = __shfl_xor_sync(0xffffffffu, b.i, o);
    if (loop_better(ov, oi, b.v, b.i)) { b.v = ov; b.i = oi; }
  }
  __syncthreads();
  if ((threadIdx.x & 31) == 0) { redv[threadIdx.x >> 5] = b.v; redi[threadIdx.x >> 5] = b.i; }
  __syncthreads();
  LoopBest r{(threadIdx.x & 31) < (blockDim.x >> 5) ? redv[threadIdx.x & 31] : -INFINITY, (threadIdx.x & 31) < (blockDim.x >> 5) ? redi[threadIdx.x & 31] : 0x7fffffff};
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, r.v, o);
    const int oi = __shfl_xor_sync(0xffffffffu, r.i, o);
    if (loop_better(ov, oi, r.v, r.i)) { r.v = ov; r.i = oi; }
  }
  __syncthreads();
  return r.i;
}
__device__ __forceinline__ bool loop_accept(float r, float p, float q, bool strict_less) {  // utils/decoding.py:98-99,192-193
  const float ratio = __fdiv_rn(p, q);
  if (ratio != ratio) return false;
  const float m = fminf(1.f, ratio);
  return strict_less ? (r < m) : (r <= m);
}

// ---- replay of the stream for the step-wise loop (and tests) ----------------------------------------------------------------
__global__ void __launch_bounds__(kLoopThreads) philox_fill_kernel(PhiloxState* st, int kind, float* __restrict__ out, int n) {
  const unsigned long long seed = st->seed, draw = st->ctr;
  for (int i = threadIdx.x; i < n; i += blockDim.x) out[i] = kind ? philox_exponential(seed, draw, (uint32_t)i) : philox_uniform(seed, draw, (uint32_t)i);
  __syncthreads();
  if (threadIdx.x == 0) st->ctr = draw + 1;
}

// ---- loop state: st[0] = n, st[1] = k (ids emitted), st[2] = last accept flag, st[3] = accepted draft tokens, st[4] = inner iterations
__global__ void loop_begin_kernel(int32_t* __restrict__ st, int64_t* __restrict__ verify_tokens, const int64_t* __restrict__ first_token,
                                  int gamma, const int32_t* __restrict__ seq_len_dev, int64_t* __restrict__ position_ids) {
  const int t = threadIdx.x;
  if (t < 8) st[t] = 0;
  if (t <= gamma) {
    verify_tokens[t] = t == 0 ? first_token[0] : 100;  // decoding.py:177: placeholders are token 100
    position_ids[t] = (int64_t)(*seq_len_dev) + t;     // decoding.py:180
  }
}

// draft token of inner iteration n: multinomial(draft_probs[n]) → verify_tokens[n + 1]   (decoding.py:183-186)
__global__ void __launch_bounds__(kLoopThreads) loop_draft_sample_kernel(const float* __restrict__ draft_probs, int V, const int32_t* __restrict__ st,
                                                                         PhiloxState* rng, int64_t* __restrict__ verify_tokens) {
  __shared__ float redv[32];
  __shared__ int redi[32];
  const int n = st[0];
  const float* row = draft_probs + (size_t)n * V;
  const unsigned long long seed = rng->seed, draw = rng->ctr;
  const int tkn = loop_sample([&](int i) { return row[i]; }, seed, draw, V, redv, redi);
  if (threadIdx.x == 0) {
    verify_tokens[n + 1] = (int64_t)tkn;
    rng->ctr = draw + 1;
  }
}

// one inner decision (decoding.py:190-220): accept test of the draft token against the retrieval-cache distribution, the
// sample that follows (bonus from row n+1 on accept, replacement from row n on reject), ids / proposal rows / slot bookkeeping
__global__ void __launch_bounds__(kLoopThreads) loop_middle_accept_kernel(const float* __restrict__ draft_probs, const float* __restrict__ vp,
                                                                          int64_t* __restrict__ verify_tokens, PhiloxState* rng, int gamma, int V,
                                                                          int32_t* __restrict__ st, int64_t* __restrict__ out_ids,
                                                                          float* __restrict__ spec_probs) {
  __shared__ float redv[32];
  __shared__ int redi[32];
  const int n = st[0], k = st[1];
  const unsigned long long seed = rng->seed, draw = rng->ctr;
  const float* sp = draft_probs + (size_t)n * V;
  const int64_t t = verify_tokens[n + 1];
  const float* vpn = vp + (size_t)n * V;
  const float u = philox_uniform(seed, draw, 0u);
  const bool accept = loop_accept(u, vpn[t], sp[t], true);
  const float* vrow = vp + (size_t)(accept ? n + 1 : n) * V;
  const int t2 = loop_sample([&](int i) { return vrow[i]; }, seed, draw + 1, V, redv, redi);
  float* d0 = spec_probs + (size_t)k * V;
  for (int i = threadIdx.x; i < V; i += blockDim.x) d0[i] = vpn[i];
  if (accept) {
    float* d1 = spec_probs + (size_t)(k + 1) * V;
    for (int i = threadIdx.x; i < V; i += blockDim.x) d1[i] = vrow[i];
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
    rng->ctr = draw + 2;
  }
}

// body of the WHILE node ends here: run another inner iteration iff n < gamma (decoding.py:182)
__global__ void loop_set_condition_kernel(cudaGraphConditionalHandle handle, const int32_t* __restrict__ st, int gamma) {
  if (threadIdx.x == 0) cudaGraphSetConditional(handle, st[0] < gamma ? 1u : 0u);
}

// input of the full-KV verify: [first token, the k ids of Middle_Spec, placeholders] — always gamma + 2 rows (decoding.py:84-85
// feeds 1 + k rows; rows beyond are causally invisible to the valid ones and their K/V slots are rolled back)
__global__ void loop_prepare_full_kernel(const int32_t* __restrict__ st, const int64_t* __restrict__ out_ids, const int64_t* __restrict__ first_token,
                                         int64_t* __restrict__ full_ids, int rows) {
  const int t = threadIdx.x, k = st[1];
  if (t < rows) full_ids[t] = t == 0 ? first_token[0] : (t <= k ? out_ids[t - 1] : 100);
}

// outer accept walk + residual / bonus sample + all the integer bookkeeping of decoding.py:97-139 in one CTA.
//   res (int32[16]): [0] tokens produced by this step, [1] count (accepted ids), [2] rejected, [3] gamma2 (= k), [4] examined,
//   [5] hit_eos, [6] inner iterations, [7] inner accepts, [8] window shift of the draft cache, [9] new seq_len
//   tokens (int64[gamma + 3]): the tokens this step appended to the output, in order
__global__ void __launch_bounds__(kLoopThreads) loop_verify_kernel(const float* __restrict__ p_rows, const float* __restrict__ q_rows,
                                                                   const int64_t* __restrict__ out_ids, const int32_t* __restrict__ st,
                                                                   PhiloxState* rng, int V, int strict_less, int64_t eos,
                                                                   int64_t* __restrict__ first_token, int32_t* __restrict__ res,
                                                                   int64_t* __restrict__ tokens, int64_t* __restrict__ pass_tokens, int pass_len,
                                                                   int32_t* __restrict__ seq_len_dev) {
  __shared__ float redv[32];
  __shared__ int redi[32];
  __shared__ int s_count, s_rejected, s_examined, s_eos;
  const int g2 = st[1];
  const unsigned long long seed = rng->seed, draw = rng->ctr;
  if (threadIdx.x == 0) {
    int count = 0, rejected = 0, examined = 0, hit_eos = 0;
    pass_tokens[0] = first_token[0];
    for (int i = 1; i < pass_len; ++i) pass_tokens[i] = 100;  // decoding.py:94
    for (int i = 0; i < g2; ++i) {
      const int64_t t = out_ids[i];
      ++examined;
      if (loop_accept(philox_uniform(seed, draw, (uint32_t)i), p_rows[(size_t)i * V + t], q_rows[(size_t)i * V + t], strict_less != 0)) {
        ++count;
        pass_tokens[count] = t;
        tokens[count - 1] = t;
        if (t == eos) { hit_eos = 1; break; }
      } else {
        rejected = 1;
        break;
      }
    }
    s_count = count; s_rejected = rejected; s_examined = examined; s_eos = hit_eos;
  }
  __syncthreads();
  const int count = s_count, rejected = s_rejected;
  const bool draws = rejected || count == g2;
  int tok = 0;
  if (rejected) {  // residual norm(max(p - q, 0)) (sampling.py:68-75), decoding.py:114
    const float* p = p_rows + (size_t)count * V;
    const float* q = q_rows + (size_t)count * V;
    float s = 0.f;
    for (int i = threadIdx.x; i < V; i += blockDim.x) {
      const float x = p[i] - q[i];
      s += x > 0.f ? x : 0.f;
    }
    s = warp_sum(s);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) redv[threadIdx.x >> 5] = s;
    __syncthreads();
    float S = (threadIdx.x & 31) < (blockDim.x >> 5) ? redv[threadIdx.x & 31] : 0.f;
    S = warp_sum(S);
    __syncthreads();
    tok = loop_sample([&](int i) { const float x = p[i] - q[i]; return __fdiv_rn(x > 0.f ? x : 0.f, S); }, seed, draw + 1, V, redv, redi);
  } else if (count == g2) {  // everything accepted: bonus token from the target's last row (decoding.py:127-134)
    const float* p = p_rows + (size_t)g2 * V;
    tok = loop_sample([&](int i) { return p[i]; }, seed, draw + 1, V, redv, redi);
  }
  if (threadIdx.x == 0) {
    int produced = count;
    int64_t next = draws ? (int64_t)tok : out_ids[count - 1];  // stopped on an accepted EOS: nothing is drawn
    if (draws) {
      pass_tokens[count + 1] = next;
      tokens[produced] = next;
      ++produced;
    }
    int shift = count;
    if (!rejected && count == g2) ++shift;  // decoding.py:131-139: the bonus token also moves the draft window
    const int new_len = *seq_len_dev + count + 1;  // the first token + the accepted ids stay in the full KV (decoding.py:124)
    *seq_len_dev = new_len;
    first_token[0] = next;
    res[0] = produced; res[1] = count; res[2] = rejected; res[3] = g2; res[4] = s_examined; res[5] = s_eos;
    res[6] = st[4]; res[7] = st[3]; res[8] = shift; res[9] = new_len;
    rng->ctr = draw + 1 + (draws ? 1 : 0);
  }
}

// StreamingLLM window slide with the shift read from device memory (cache.py:263-265 evict_for_spec): rows
// [src_base + *shift, … + n_rows) → [dst_start, …), clone semantics, all layers and heads
__global__ void __launch_bounds__(256) window_slide_dev_kernel(__half* __restrict__ K, __half* __restrict__ V, long long ls, long long hs, int D,
                                                               int src_base, const int32_t* __restrict__ shift, int dst_start, int n_rows) {
  extern __shared__ __align__(16) uint8_t lwsm[];
  uint4* buf = reinterpret_cast<uint4*>(lwsm);
  const int h = blockIdx.x, layer = blockIdx.y;
  const int src_start = src_base + *shift;
  const int nvec = n_rows * D / 8;
  __half* bases[2] = {K + (size_t)layer * ls + (size_t)h * hs, V + (size_t)layer * ls + (size_t)h * hs};
#pragma unroll
  for (int w = 0; w < 2; ++w) {
    const uint4* src = reinterpret_cast<const uint4*>(bases[w] + (size_t)src_start * D);
    uint4* dst = reinterpret_cast<uint4*>(bases[w] + (size_t)dst_start * D);
    for (int i = threadIdx.x; i < nvec; i += blockDim.x) buf[i] = src[i];
    __syncthreads();
    for (int i = threadIdx.x; i < nvec; i += blockDim.x) dst[i] = buf[i];
    __syncthreads();
  }
}

}  // namespace tf

extern "C" {

int tf_philox_fill(void* state, int kind, float* out, int n, tf_stream_t stream) {
  using namespace tf;
  TF_CHECK_ARG(state && out && n >= 1 && (kind == 0 || kind == 1), "tf_philox_fill: bad arguments");
  philox_fill_kernel<<<1, kLoopThreads, 0, (cudaStream_t)stream>>>((PhiloxState*)state, kind, out, n);
  TF_CHECK_LAUNCH();
  return TF_OK;
}

int tf_loop_begin(int32_t* state, int64_t* verify_tokens, const int64_t* first_token, int gamma, const int32_t* seq_len_dev,
                  int64_t* position_ids, tf_stream_t stream) {
  using namespace tf;
  TF_CHECK_ARG(state && verify_tokens && first_token && seq_len_dev && position_ids && gamma >= 1 && gamma < 64, "tf_loop_begin: bad arguments");
  loop_begin_kernel<<<1, 64, 0, (cudaStream_t)stream>>>(state, verify_tokens, first_token, gamma, seq_len_dev, position_ids);
  TF_CHECK_LAUNCH();
  return TF_OK;
}

int tf_loop_draft_sample(const float* draft_probs, int V, const int32_t* state, void* rng, int64_t* verify_tokens, tf_stream_t stream) {
  using namespace tf;
  TF_CHECK_ARG(draft_probs && state && rng && verify_tokens && V >= 1, "tf_loop_draft_sample: bad arguments");
  loop_draft_sample_kernel<<<1, kLoopThreads, 0, (cudaStream_t)stream>>>(draft_probs, V, state, (PhiloxState*)rng, verify_tokens);
  TF_CHECK_LAUNCH();
  return TF_OK;
}

int tf_loop_middle_accept(const float* draft_probs, const float* verify_probs, int64_t* verify_tokens, void* rng, int gamma, int V,
                          int32_t* state, int64_t* out_ids, float* spec_probs, tf_stream_t stream) {
  using namespace tf;
  TF_CHECK_ARG(draft_probs && verify_probs && verify_tokens && rng && state && out_ids && spec_probs, "tf_loop_middle_accept: NULL pointer");
  loop_middle_accept_kernel<<<1, kLoopThreads, 0, (cudaStream_t)stream>>>(draft_probs, verify_probs, verify_tokens, (PhiloxState*)rng, gamma, V, state,
                                                                           out_ids, spec_probs);
  TF_CHECK_LAUNCH();
  return TF_OK;
}

int tf_loop_prepare_full(const int32_t* state, const int64_t* out_ids, const int64_t* first_token, int64_t* full_ids, int rows,
                         tf_stream_t stream) {
  using namespace tf;
  TF_CHECK_ARG(state && out_ids && first_token && full_ids && rows >= 2 && rows <= 64, "tf_loop_prepare_full: bad arguments");
  loop_prepare_full_kernel<<<1, 64, 0, (cudaStream_t)stream>>>(state, out_ids, first_token, full_ids, rows);
  TF_CHECK_LAUNCH();
  return TF_OK;
}

int tf_loop_verify(const float* p_rows, const float* q_rows, const int64_t* out_ids, const int32_t* state, void* rng, int V, int strict_less,
                   int64_t eos, int64_t* first_token, int32_t* res, int64_t* tokens, int64_t* pass_tokens, int pass_len,
                   int32_t* seq_len_dev, tf_stream_t stream) {
  using namespace tf;
  TF_CHECK_ARG(p_rows && q_rows && out_ids && state && rng && first_token && res && tokens && pass_tokens && seq_len_dev && pass_len >= 3,
               "tf_loop_verify: bad arguments");
  loop_verify_kernel<<<1, kLoopThreads, 0, (cudaStream_t)stream>>>(p_rows, q_rows, out_ids, state, (PhiloxState*)rng, V, strict_less, eos, first_token, res,
                                                                    tokens, pass_tokens, pass_len, seq_len_dev);
  TF_CHECK_LAUNCH();
  return TF_OK;
}

int tf_window_slide_dev(void* K, void* V, long long layer_stride, long long head_stride, int L, int H, int d, int src_base,
                        const int32_t* shift_dev, int dst_start, int n_rows, tf_stream_t stream) {
  using namespace tf;
  TF_CHECK_ARG(K && V && shift_dev && L >= 1 && H >= 1 && n_rows >= 1 && d % 8 == 0, "tf_window_slide_dev: bad arguments");
  const size_t smem = (size_t)n_rows * d * 2;
  TF_CHECK_SUPPORTED(smem <= 200 * 1024, "tf_window_slide_dev: window of %d rows does not fit in shared memory", n_rows);
  int dev = 0;
  TF_CHECK_CUDA(cudaGetDevice(&dev));
  static size_t configured[64] = {0};
  if (dev < 64 && smem > configured[dev]) {
    TF_CHECK_CUDA(cudaFuncSetAttribute(window_slide_dev_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    configured[dev] = smem;
  }
  window_slide_dev_kernel<<<dim3(H, L), 256, smem, (cudaStream_t)stream>>>((__half*)K, (__half*)V, layer_stride, head_stride, d, src_base, shift_dev,
                                                                        dst_start, n_rows);
  TF_CHECK_LAUNCH();
  return TF_OK;
}

// parent graph = pre → WHILE(handle) { body → set condition } → post.  `pre`, `body`, `post`: cudaGraph_t captured by the caller
// (they are cloned into child-graph nodes; the caller keeps their memory alive).  Returns a cudaGraphExec_t in *exec_out.
int tf_loop_graph_build(void* pre, void* body, void* post, const int32_t* state, int gamma, void** exec_out) {
  using namespace tf;
  TF_CHECK_ARG(pre && body && post && state && exec_out, "tf_loop_graph_build: NULL pointer");
  cudaGraph_t G = nullptr;
  TF_CHECK_CUDA(cudaGraphCreate(&G, 0));
  cudaGraphNode_t n_pre, n_while, n_post;
  TF_CHECK_CUDA(cudaGraphAddChildGraphNode(&n_pre, G, nullptr, 0, (cudaGraph_t)pre));
  cudaGraphConditionalHandle handle;
  TF_CHECK_CUDA(cudaGraphConditionalHandleCreate(&handle, G, 1, cudaGraphCondAssignDefault));  // every launch starts with "run"
  cudaGraphNodeParams wp = {cudaGraphNodeTypeConditional};
  wp.type = cudaGraphNodeTypeConditional;
  wp.conditional.handle = handle;
  wp.conditional.type = cudaGraphCondTypeWhile;
  wp.conditional.size = 1;
  TF_CHECK_CUDA(cudaGraphAddNode(&n_while, G, &n_pre, 1, &wp));
  cudaGraph_t loop_body = wp.conditional.phGraph_out[0];
  cudaGraphNode_t b_body, b_cond;
  TF_CHECK_CUDA(cudaGraphAddChildGraphNode(&b_body, loop_body, nullptr, 0, (cudaGraph_t)body));
  cudaKernelNodeParams kp;
  memset(&kp, 0, sizeof(kp));
  const int32_t* st = state;
  int g = gamma;
  void* kargs[3] = {(void*)&handle, (void*)&st, (void*)&g};
  kp.func = (void*)loop_set_condition_kernel;
  kp.gridDim = dim3(1);
  kp.blockDim = dim3(32);
  kp.sharedMemBytes = 0;
  kp.kernelParams = kargs;
  TF_CHECK_CUDA(cudaGraphAddKernelNode(&b_cond, loop_body, &b_body, 1, &kp));
  TF_CHECK_CUDA(cudaGraphAddChildGraphNode(&n_post, G, &n_while, 1, (cudaGraph_t)post));
  cudaGraphExec_t exec = nullptr;
  TF_CHECK_CUDA(cudaGraphInstantiate(&exec, G, 0));
  TF_CHECK_CUDA(cudaGraphDestroy(G));
  *exec_out = (void*)exec;
  return TF_OK;
}

int tf_loop_graph_launch(void* exec, tf_stream_t stream) {
  TF_CHECK_ARG(exec, "tf_loop_graph_launch: NULL graph");
  TF_CHECK_CUDA(cudaGraphLaunch((cudaGraphExec_t)exec, (cudaStream_t)stream));
  return TF_OK;
}

int tf_loop_graph_destroy(void* exec) {
  if (exec) TF_CHECK_CUDA(cudaGraphExecDestroy((cudaGraphExec_t)exec));
  return TF_OK;
}

}  // extern "C"
