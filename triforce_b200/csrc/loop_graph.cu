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
// cudaGraphSetConditional), the device-side state of Middle_Spec (`n`, accepted ids, proposal rows — decoding.py:180-220) and
// of the outer accept walk (:97-134) in kernels that read their control variables from device memory, and the counters of a
// Philox4x32-10 noise stream so that no random number has to come from the host.  The decisions themselves (sampler, accept
// test, Middle_Spec step, accept walk, residual / bonus resample) are spec_decisions.cuh's, the same code the step-wise loop
// runs over buffered noise.  Per outer iteration the host launches ONE graph and reads ONE small result record.
//
// Random numbers: draw `c` of stream (seed) = Philox4x32-10(counter = (element / 4, c_lo, c_hi, 0), key = seed); element i takes
// lane i % 4.  Uniforms u strictly inside (0, 1) (philox_to_uniform); exponentials -log(u) > 0.  The consumption order is the
// reference's (decoding.py:185,192,201/212,98,114/130): per inner iteration exponential (draft sample), uniform, exponential
// (accept / resample); per outer iteration one block of uniforms, then one exponential when a token is drawn.  `tf_philox_fill`
// replays the same draws for the step-wise (host-driven) loop, which is how the two loops are checked against each other event
// for event.
#include <string.h>

#include "spec_decisions.cuh"

namespace tf {

struct PhiloxState {
  unsigned long long seed;
  unsigned long long ctr;  // next draw index
};

// ---- replay of the stream for the step-wise loop (and tests) ----------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) philox_fill_kernel(PhiloxState* st, int kind, float* __restrict__ out, int n) {
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
__global__ void __launch_bounds__(kThreads) loop_draft_sample_kernel(const float* __restrict__ draft_probs, int V, const int32_t* __restrict__ st,
                                                                     PhiloxState* rng, int64_t* __restrict__ verify_tokens) {
  __shared__ float redv[32];
  __shared__ int redi[32];
  const int n = st[0];
  const float* row = draft_probs + (size_t)n * V;
  const unsigned long long seed = rng->seed, draw = rng->ctr;
  const int tkn = block_sample([&](int i) { return row[i]; }, ExpoFromPhilox{seed, draw}, V, redv, redi);
  if (threadIdx.x == 0) {
    verify_tokens[n + 1] = (int64_t)tkn;
    rng->ctr = draw + 1;
  }
}

// one inner decision (decoding.py:190-220) on uniform 0 of draw `ctr` and exponentials of draw `ctr + 1`
__global__ void __launch_bounds__(kThreads) loop_middle_accept_kernel(const float* __restrict__ draft_probs, const float* __restrict__ vp,
                                                                      int64_t* __restrict__ verify_tokens, PhiloxState* rng, int gamma, int V,
                                                                      int32_t* __restrict__ st, int64_t* __restrict__ out_ids,
                                                                      float* __restrict__ spec_probs) {
  __shared__ float redv[32];
  __shared__ int redi[32];
  const unsigned long long seed = rng->seed, draw = rng->ctr;
  middle_spec_decision(draft_probs + (size_t)st[0] * V, vp, verify_tokens, philox_uniform(seed, draw, 0u), ExpoFromPhilox{seed, draw + 1},
                       gamma, V, st, out_ids, spec_probs, redv, redi);
  if (threadIdx.x == 0) rng->ctr = draw + 2;
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

// outer accept walk + residual / bonus sample + all the integer bookkeeping of decoding.py:97-139 in one CTA; the walk takes
// uniforms of draw `ctr`, the sample exponentials of draw `ctr + 1`.
//   res (int32[16]): [0] tokens produced by this step, [1] count (accepted ids), [2] rejected, [3] gamma2 (= k), [4] examined,
//   [5] hit_eos, [6] inner iterations, [7] inner accepts, [8] window shift of the draft cache, [9] new seq_len
//   tokens (int64[gamma + 3]): the tokens this step appended to the output, in order
__global__ void __launch_bounds__(kThreads) loop_verify_kernel(const float* __restrict__ p_rows, const float* __restrict__ q_rows,
                                                               const int64_t* __restrict__ out_ids, const int32_t* __restrict__ st,
                                                               PhiloxState* rng, int V, int strict_less, int64_t eos,
                                                               int64_t* __restrict__ first_token, int32_t* __restrict__ res,
                                                               int64_t* __restrict__ tokens, int64_t* __restrict__ pass_tokens, int pass_len,
                                                               int32_t* __restrict__ seq_len_dev) {
  __shared__ float redv[32];
  __shared__ int redi[32];
  __shared__ AcceptWalk s_walk;
  const int g2 = st[1];
  const unsigned long long seed = rng->seed, draw = rng->ctr;
  if (threadIdx.x == 0) {
    s_walk = accept_walk(p_rows, q_rows, out_ids, g2, [&](int i) { return philox_uniform(seed, draw, (uint32_t)i); }, V, strict_less != 0,
                         eos, first_token[0], pass_tokens, pass_len);
    for (int i = 0; i < s_walk.count; ++i) tokens[i] = out_ids[i];  // the accepted ids
  }
  __syncthreads();
  const AcceptWalk w = s_walk;
  const bool draws = w.rejected || w.count == g2;
  const int64_t next = resample_after_walk(p_rows, q_rows, out_ids, g2, w.count, w.rejected != 0, ExpoFromPhilox{seed, draw + 1}, V,
                                           pass_tokens, redv, redi);
  if (threadIdx.x == 0) {
    int produced = w.count;
    if (draws) tokens[produced++] = next;
    int shift = w.count;
    if (!w.rejected && w.count == g2) ++shift;  // decoding.py:131-139: the bonus token also moves the draft window
    const int new_len = *seq_len_dev + w.count + 1;  // the first token + the accepted ids stay in the full KV (decoding.py:124)
    *seq_len_dev = new_len;
    first_token[0] = next;
    res[0] = produced; res[1] = w.count; res[2] = w.rejected; res[3] = g2; res[4] = w.examined; res[5] = w.hit_eos;
    res[6] = st[4]; res[7] = st[3]; res[8] = shift; res[9] = new_len;
    rng->ctr = draw + 1 + (draws ? 1 : 0);
  }
}

}  // namespace tf

extern "C" {

int tf_philox_fill(void* state, int kind, float* out, int n, tf_stream_t stream) {
  using namespace tf;
  TF_CHECK_ARG(state && out && n >= 1 && (kind == 0 || kind == 1), "tf_philox_fill: bad arguments");
  philox_fill_kernel<<<1, kThreads, 0, (cudaStream_t)stream>>>((PhiloxState*)state, kind, out, n);
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
  loop_draft_sample_kernel<<<1, kThreads, 0, (cudaStream_t)stream>>>(draft_probs, V, state, (PhiloxState*)rng, verify_tokens);
  TF_CHECK_LAUNCH();
  return TF_OK;
}

int tf_loop_middle_accept(const float* draft_probs, const float* verify_probs, int64_t* verify_tokens, void* rng, int gamma, int V,
                          int32_t* state, int64_t* out_ids, float* spec_probs, tf_stream_t stream) {
  using namespace tf;
  TF_CHECK_ARG(draft_probs && verify_probs && verify_tokens && rng && state && out_ids && spec_probs, "tf_loop_middle_accept: NULL pointer");
  loop_middle_accept_kernel<<<1, kThreads, 0, (cudaStream_t)stream>>>(draft_probs, verify_probs, verify_tokens, (PhiloxState*)rng, gamma, V, state,
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
  loop_verify_kernel<<<1, kThreads, 0, (cudaStream_t)stream>>>(p_rows, q_rows, out_ids, state, (PhiloxState*)rng, V, strict_less, eos, first_token, res,
                                                                    tokens, pass_tokens, pass_len, seq_len_dev);
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
