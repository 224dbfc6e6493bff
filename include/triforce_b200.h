/*
 * triforce_b200 — C ABI of the GPU-native TriForce hot path (libtriforce_b200.so, sm_90a / H100 only).
 *
 * The reference (Infini-AI-Lab/TriForce) has no FFI/plugin layer: its hot path crosses into native code only through
 * third-party Python bindings (flash_attn.flash_attn_with_kvcache, ATen ops, NCCL via torch.distributed — SURVEY.md
 * §2b).  Each entry point below replaces one of those library call sites; the reference file:line it replaces is cited
 * on every declaration.  `INTEGRATION.md` shows the ctypes stub a maintainer of the reference would add.
 *
 * Conventions
 *   - plain pointers and sizes only; every device pointer is caller-owned; nothing here allocates or synchronises;
 *   - every function enqueues on `stream` (a cudaStream_t) and is CUDA-graph capturable;
 *   - returns 0 on success, a negative TF_ERR_* otherwise; `tf_last_error()` gives the message (thread-local);
 *   - "fp16" = IEEE binary16; KV caches are HEAD-MAJOR: [layer][head][slot][d], `*_head_stride` / `*_layer_stride`
 *     are in ELEMENTS, rows of one head are contiguous (d elements apart);
 *   - `*_dev` int pointers may be NULL; when given, the device value is ADDED to the host value at kernel run time
 *     (lets a captured graph follow `kv_cache.seq_len` without re-capture).
 */
#ifndef TRIFORCE_B200_H_
#define TRIFORCE_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* tf_stream_t; /* cudaStream_t */

enum {
  TF_OK = 0,
  TF_ERR_INVALID = -1,     /* bad argument (shape, alignment, NULL) */
  TF_ERR_UNSUPPORTED = -2, /* shape outside what the sm_90a kernels were built for */
  TF_ERR_WORKSPACE = -3,   /* workspace too small */
  TF_ERR_CUDA = -4         /* a CUDA runtime/driver call failed */
};

/* ---- misc ---------------------------------------------------------------------------------------------------- */
int tf_version(void);
const char* tf_last_error(void);
/* number of SMs of the current device (grid sizing); <0 on error */
int tf_sm_count(void);
/* Programmatic dependent launch for the decode-path kernels (tf_add_rmsnorm, tf_silu_mul, tf_rope_append, tf_draft_attn,
 * tf_verify_attn[_tree], tf_skinny_gemm): when on, they are launched with the programmatic-stream-serialization attribute,
 * start while their predecessor on the stream drains (barrier setup, descriptor and weight prefetch) and execute
 * griddepcontrol.wait before touching its outputs.  Process-wide bit mask, default 0 (off); graph-capturable:
 * 1 add_rmsnorm, 2 silu_mul, 4 rope_append, 8 draft_attn, 16 verify_attn, 32 skinny_gemm, 64 skinny_gemm pulls its weight rows
 * towards L2 before it waits, 128 stream_linear (weight ring filled before it waits), 256 allreduce_oneshot (lets the next projection prefetch during the exchange). */
int tf_set_pdl(int mask);

/* 128-byte TMA descriptor (CUtensorMap) over a head-major fp16 KV tensor [layers][heads][cap][d]; written to
 * `out_tensormap_128B` in HOST memory and passed by value to the attention kernels.  `box_keys` = keys per TMA box. */
int tf_kv_tensormap_encode(void* out_tensormap_128B, const void* base, int d, long long cap, int heads, int layers,
                           long long head_stride, long long layer_stride, int box_keys);

/* ---- E4M3 full-KV store (opt-in; fp16 stays the default) -----------------------------------------------------------
 * A store of L layers, Hkv KV heads and `cap` slots is, for K and for V:
 *   codes     uint8 [L][Hkv][cap][d] (torch.float8_e4m3fn bits), head-major like the fp16 store, strides in bytes;
 *   exponents int8  [L][Hkv][cap], one per row (the code strides divided by d).
 * Row x (d fp16 values: K after RoPE, or V): e = the smallest integer with max|x| <= 448 * 2^e (0 for an all-zero row; in
 * [-32, 8] for finite fp16 x); code = e4m3_rn(x / 2^e), round to nearest even (exact division, nothing saturates).  The row
 * the store holds is D = fp16_rn(code * 2^e).  Every entry below that reads the store computes what its fp16 counterpart
 * computes on D; the retrieval cache it fills stays fp16.  Entries take Hq, Hkv (Hq == Hkv is MHA).
 * tf_kv_tensormap_encode_e4m3: tf_kv_tensormap_encode over a code store (box = one row of d bytes x box_keys rows,
 *   SWIZZLE_128B at d = 128, SWIZZLE_64B at d = 64); strides in bytes.
 * tf_kv_quantize_e4m3: fp16 rows [slot0, slot0 + n) of one layer (`src` [Hkv][..][d], head stride in elements, >= cap*d)
 *   -> the same slots of one layer's codes [Hkv][cap][d] and exponents [Hkv][cap].
 * tf_rope_append_e4m3: tf_rope_append_gqa (rotate_q = rotate_k = 1; same position, slot and *_dev arguments, same PDL bit 4)
 *   with the appended K and V rows stored into one layer's codes [Hkv][cap][d] and exponents [Hkv][cap]; q_out is bit-identical.
 * tf_verify_attn_e4m3: tf_verify_attn_gqa over an E4M3 store (tensor maps from tf_kv_tensormap_encode_e4m3 with box_keys =
 *   TF_VERIFY_BOX_KEYS; exponents [L][Hkv][cap], 16-byte aligned; cap % TF_VERIFY_BOX_KEYS == 0).  Same stream-K split,
 *   in-kernel merge, device-side length, R·G packing and workspace (tf_verify_attn_gqa_workspace_bytes).  No calibrated split,
 *   no L2 prefetch, no tree mode.  V is dequantized exactly to D before the PV product; K enters as (q·code)·2^e in fp32, which is
 *   q·D exactly unless D rounds: for e < -15 codes below fp16's subnormal step, and a row holding ±65504 (code 256 at e = 8,
 *   D = ±inf, where this kernel keeps finite scores).  Otherwise results equal the fp16 kernel's on D up to the order of fp32
 *   sums.
 * tf_retrieval_build_e4m3: tf_retrieval_build_gqa (Hq == Hkv: tf_retrieval_build) over an E4M3 store; indices, scores and the
 *   gathered fp16 rows are bit-identical to that build run on D.
 * tf_tail_update_e4m3: tf_tail_update from an E4M3 store into the fp16 retrieval cache (writes D).
 */
int tf_kv_tensormap_encode_e4m3(void* out_tensormap_128B, const void* base, int d, long long cap, int heads, int layers,
                                long long head_stride, long long layer_stride, int box_keys);
int tf_kv_quantize_e4m3(const void* src, long long src_head_stride, int slot0, int n, int Hkv, int d, void* codes, int8_t* exps,
                        long long cap, tf_stream_t stream);
int tf_rope_append_e4m3(const void* q, const void* k, const void* v, long long qkv_row_stride, const void* cos, const void* sin,
                        int max_pos, const int32_t* pos_ids_dev, int pos0, const int32_t* pos0_dev, int slot0,
                        const int32_t* slot0_dev, int R, int Hq, int Hkv, int d, void* q_out, void* Kcodes, void* Vcodes,
                        int8_t* Kexp, int8_t* Vexp, long long cap, tf_stream_t stream);
int tf_verify_attn_e4m3(const void* q, const void* k_tensormap, const void* v_tensormap, const int8_t* k_exp, const int8_t* v_exp,
                        long long cap, int layer, int kv_len_host, const int32_t* kv_len_dev, int kv_len_max, int R, int Hq, int Hkv,
                        int d, float scale, void* out, void* workspace, size_t workspace_bytes, tf_stream_t stream);
int tf_retrieval_build_e4m3(const void* K, const void* V, const int8_t* Kexp, const int8_t* Vexp, long long kv_layer_stride,
                            long long kv_head_stride, const void* q, int n_layers, int Hq, int Hkv, int d, int prefill, int chunk,
                            int budget, void* retrK, void* retrV, long long r_layer_stride, long long r_head_stride, int32_t* out_idx,
                            void* out_scores, void* workspace, size_t workspace_bytes, tf_stream_t stream);
int tf_tail_update_e4m3(const void* K, const void* V, const int8_t* Kexp, const int8_t* Vexp, long long kv_layer_stride,
                        long long kv_head_stride, void* retrK, void* retrV, long long r_layer_stride, long long r_head_stride,
                        int n_layers, int H, int d, int prefill, int budget, int seq_len_host, const int32_t* seq_len_dev,
                        int max_new, tf_stream_t stream);

/* ---- (i) retrieval-cache build ---------------------------------------------------------------------------------
 * replaces models/cache.py:154-175 (RetrievalCache.init_graph_cache: ATen mean + cuBLAS bmm + ATen topk + 2 gathers;
 * TP twins :418-453, :517-556).  For each of `n_layers` layers and each head: k̄ = fp16(mean of each `chunk` rows of
 * K[:prefill]); score = fp16(q·k̄) (fp64 accumulate, see oracle/triforce_oracle.py for the fixed order);
 * idx = [0] + top-(budget/chunk - 1) of chunks 1.. (descending score, ascending index on ties) ; the chunk rows of K
 * and V are gathered into retrieval slots [0, budget) in that order.
 *   K, V        fp16 head-major full cache (layer 0 of the call), strides in elements
 *   q           fp16 [n_layers][H][d] (post-RoPE query of the last prompt token), contiguous
 *   retrK/retrV fp16 head-major retrieval cache (layer 0 of the call)
 *   out_idx     int32 [n_layers][H][budget/chunk] or NULL; out_scores fp16 [n_layers][H][prefill/chunk] or NULL
 */
size_t tf_retrieval_build_workspace_bytes(int n_layers, int H, int d, int prefill, int chunk, int budget);
int tf_retrieval_build(const void* K, const void* V, long long kv_layer_stride, long long kv_head_stride,
                       const void* q, int n_layers, int H, int d, int prefill, int chunk, int budget,
                       void* retrK, void* retrV, long long r_layer_stride, long long r_head_stride,
                       int32_t* out_idx, void* out_scores, void* workspace, size_t workspace_bytes, tf_stream_t stream);
/* tf_retrieval_build_gqa: the build of a grouped-query-attention target (Hq query heads over Hkv KV heads, query head h reads
 *   KV head h / (Hq/Hkv)) under the "group_sum" rule.  The reference defines no GQA rule (cache.py:157 broadcasts q over KV
 *   heads); this one scores each (layer, KV head) with q̄ = the sum of its group's query heads, taken in fp64 (exact for up to
 *   64 heads per group):  score = fp16(q̄·k̄) with the dot as above, then top-k and gather per (layer, KV head) exactly as above.
 *   Hkv == Hq gives tf_retrieval_build's bits.  q fp16 [n_layers][Hq][d]; out_idx [n_layers][Hkv][budget/chunk];
 *   out_scores [n_layers][Hkv][prefill/chunk]; the workspace is tf_retrieval_build_workspace_bytes(n_layers, Hkv, ...). */
int tf_retrieval_build_gqa(const void* K, const void* V, long long kv_layer_stride, long long kv_head_stride,
                           const void* q, int n_layers, int Hq, int Hkv, int d, int prefill, int chunk, int budget,
                           void* retrK, void* retrV, long long r_layer_stride, long long r_head_stride,
                           int32_t* out_idx, void* out_scores, void* workspace, size_t workspace_bytes, tf_stream_t stream);

/* ---- fused RoPE + KV append --------------------------------------------------------------------------------------
 * replaces models/modeling_llama.py:217-230 (apply_rotary_pos_emb + FlashSimpleCache.update cache.py:52-53 /
 * RetrievalCache.update cache.py:186-187) and models/modeling_llama_68m.py:145-152 (+ StreamingLLMEvictionCache
 * .update/.spec_update cache.py:227-228,242-243).  fp16 arithmetic with the reference's rounding points:
 * out = fp16(fp16(x*cos) + fp16(rotate_half(x)*sin)).
 *   q,k,v      fp16 [R][H*d] with row stride `qkv_row_stride` elements (slices of one fused QKV GEMM output)
 *   cos,sin    fp16 [max_pos][d]
 *   pos        position of row i = pos0 + (pos0_dev ? *pos0_dev : 0) + i, or pos_ids_dev[i] when pos_ids_dev != NULL
 *   slot       cache slot of row i = slot0 + (slot0_dev ? *slot0_dev : 0) + i
 *   rotate_q / rotate_k: the draft stores UN-rotated keys (modeling_llama_68m.py:152 then :161-162) → rotate_k = 0
 *   q_out      fp16 [R][H][d] contiguous
 */
int tf_rope_append(const void* q, const void* k, const void* v, long long qkv_row_stride, const void* cos,
                   const void* sin, int max_pos, const int32_t* pos_ids_dev, int pos0, const int32_t* pos0_dev,
                   int slot0, const int32_t* slot0_dev, int R, int H, int d, int rotate_q, int rotate_k, void* q_out,
                   void* Kcache, void* Vcache, long long kv_head_stride, long long cap, tf_stream_t stream);
/* tf_rope_append_gqa: the same for Hq query heads and Hkv K/V heads (Hq % Hkv == 0): q [R][Hq*d] → q_out [R][Hq][d], k / v
 *   [R][Hkv*d] (row stride qkv_row_stride, e.g. slices of one [Hq·d | Hkv·d | Hkv·d] GEMM row) appended to Hkv cache heads.
 *   Hkv == Hq gives tf_rope_append's bits. */
int tf_rope_append_gqa(const void* q, const void* k, const void* v, long long qkv_row_stride, const void* cos,
                       const void* sin, int max_pos, const int32_t* pos_ids_dev, int pos0, const int32_t* pos0_dev,
                       int slot0, const int32_t* slot0_dev, int R, int Hq, int Hkv, int d, int rotate_q, int rotate_k,
                       void* q_out, void* Kcache, void* Vcache, long long kv_head_stride, long long cap, tf_stream_t stream);

/* ---- (iii) verify attention over the retrieval budget or the full KV ------------------------------------------
 * replaces flash_attn_with_kvcache at models/modeling_llama.py:240 (and tensor_op.py:166-168,316): causal,
 * bottom-right aligned attention of R <= TF_VERIFY_MAX_ROWS new rows over kv_len keys (the R new rows already
 * appended), fp16 in/out, fp32 softmax/accumulate, scale passed by the caller (the reference's is fp16-rounded).
 * Split-KV ("stream-K" over (head, key-tile) work units, one CTA per SM slot) with TMA-staged K/V tiles, followed by
 * an in-kernel merge by the last CTA of each head.  kv_len = kv_len_host + (kv_len_dev ? *kv_len_dev : 0); `kv_len_max` bounds it (workspace/grid).
 *   q    fp16 [R][H][d] contiguous ; out fp16 [R][H][d] contiguous
 *   k_tensormap / v_tensormap: HOST pointers to descriptors from tf_kv_tensormap_encode (box_keys = TF_VERIFY_BOX_KEYS)
 *   variant: 0 = auto, 1 = mma.sync kernel
 *   clean_keys: keys [0, clean_keys) of this layer are NOT written by the kernels enqueued just before this one (e.g. the
 *              retrieval budget below the gamma+1 fresh slots); with tf_set_pdl the kernel then fills its TMA ring from that
 *              region before `griddepcontrol.wait`.  0 = make no such promise.  Ignored with a device-side length.
 *   workspace: tf_verify_attn_workspace_bytes() bytes, ZERO-FILLED before its first use (it holds per-head arrival
 *              counters that the kernel leaves at zero, and the optional split tables of tf_verify_attn_calibrate);
 *              one workspace per stream — launches sharing it must be ordered.
 */
#define TF_VERIFY_MAX_ROWS 32
#define TF_VERIFY_BOX_KEYS 64
size_t tf_verify_attn_workspace_bytes(int R, int H, int d);
int tf_verify_attn(const void* q, const void* k_tensormap, const void* v_tensormap, int layer, int kv_len_host,
                   const int32_t* kv_len_dev, int kv_len_max, int R, int H, int d, float scale, void* out,
                   void* workspace, size_t workspace_bytes, int variant, int clean_keys, tf_stream_t stream);

/* tf_verify_attn_prefetch: tf_verify_attn that also pulls `next_weight_bytes` of `next_weights` — the matrix the NEXT kernel on the
 *   stream will stream (o_proj: models/modeling_llama.py:243) — into L2 with `cp.async.bulk.prefetch.L2`, a few 4 KB requests per
 *   K/V tile so that they queue behind the kernel's own loads.  Only acts behind a short store (kv_len_max < 16384: the retrieval
 *   budget), where attention is latency-bound and HBM has idle time; NULL / 0 = plain tf_verify_attn.  Results are unaffected. */
int tf_verify_attn_prefetch(const void* q, const void* k_tensormap, const void* v_tensormap, int layer, int kv_len_host,
                            const int32_t* kv_len_dev, int kv_len_max, int R, int H, int d, float scale, void* out, void* workspace,
                            size_t workspace_bytes, int variant, int clean_keys, const void* next_weights, size_t next_weight_bytes,
                            tf_stream_t stream);

/* tf_verify_attn_gqa: tf_verify_attn for grouped-query attention — Hq query heads over a store of Hkv KV heads, Hq % Hkv == 0,
 *   query head h reads KV head h / G (G = Hq / Hkv, Hugging Face `repeat_kv` order).  q / out fp16 [R][Hq][d].  The stream-K
 *   units are (KV head, key tile); one CTA computes the R·G rows of a whole group against each tile it loads, so every K/V byte
 *   is read once per launch (kv_len·Hkv·d·2·2 bytes).  Packed row i = token row i / G of query head kvh·G + i % G; the causal
 *   limit and the tree-mask row are those of the token row.  R·G <= TF_VERIFY_MAX_ROWS (larger requests are cut into blocks
 *   of token rows by the caller, each with the kv_len that keeps it bottom-right aligned).  Workspace:
 *   tf_verify_attn_gqa_workspace_bytes (partials and arrival counters per KV head), zero-filled before first use.  G = 1 runs
 *   the code and gives the bits of tf_verify_attn.  There is no calibrated split or L2 prefetch for these launches.
 * tf_verify_attn_tree_gqa: the same for tf_verify_attn_tree; tree_mask is [R][tree_cols/32] over TOKEN rows. */
size_t tf_verify_attn_gqa_workspace_bytes(int R, int Hq, int Hkv, int d);
int tf_verify_attn_gqa(const void* q, const void* k_tensormap, const void* v_tensormap, int layer, int kv_len_host,
                       const int32_t* kv_len_dev, int kv_len_max, int R, int Hq, int Hkv, int d, float scale, void* out,
                       void* workspace, size_t workspace_bytes, int variant, int clean_keys, tf_stream_t stream);
int tf_verify_attn_tree_gqa(const void* q, const void* k_tensormap, const void* v_tensormap, int layer, int kv_len_host,
                            const int32_t* kv_len_dev, int kv_len_max, int R, int Hq, int Hkv, int d, float scale,
                            const uint32_t* tree_mask, int tree_cols, void* out, void* workspace, size_t workspace_bytes,
                            tf_stream_t stream);

/* tf_tree_attn_tc: the tree (Sequoia) verify attention on the Hopper tensor cores — `variant 2` of the verify attention, for
 *   R = 128·k query rows (the 512 tree nodes of BASELINE cfg5) against the full KV of one layer; replaces the SDPA call with an
 *   additive [512, S+512] mask at models/tensor_op.py:230-272 / utils/SpecTree_TP.py:168-175.  One CTA = (128-row block, head, KV
 *   split): TMA (SWIZZLE_128B) → S = Q·K^T and O += P·V as wgmma m64n128k16 (two 64-row warpgroups, fp16 → fp32 accumulators in
 *   registers, P fed from registers, V consumed MN-major), online softmax in registers, tree bitmask as in tf_verify_attn_tree;
 *   the splits are merged by a second small kernel.  Every KV byte is read once per 128-row block (4x for 512 rows) instead of
 *   once per 32-row block (16x).  d must be 128; tree_cols = 0 → plain attention over kv_len keys.  causal = 1 (tree_cols = 0):
 *   the bottom-right causal attention of R new rows — the PREFILL attention of a prompt chunk (utils/graph_infer.py:28-37 →
 *   modeling_llama.py:240); tiles above a 128-row block's diagonal are skipped.
 *   `debug_scores`: NULL, or fp32 [128][128] that receives the raw Q·K^T tile of (block 0, head 0, split 0) — test hook.
 */
size_t tf_tree_attn_tc_workspace_bytes(int R, int H, int kv_len_max);
int tf_tree_attn_tc(const void* q, const void* k_tensormap, const void* v_tensormap, int layer, int kv_len, int R, int H, int d,
                    float scale, const uint32_t* tree_mask, int tree_cols, int causal, void* out, void* workspace,
                    size_t workspace_bytes, float* debug_scores, tf_stream_t stream);
/* tf_tree_attn_tc_gqa: tf_tree_attn_tc for Hq query heads over Hkv KV heads (query head h reads KV head h / (Hq/Hkv)).  The grid,
 *   the workspace (tf_tree_attn_tc_workspace_bytes(R, Hq, kv_len_max)), q, out and the merge stay per query head; the CTAs of
 *   one group read the same K/V tiles, through L2 (the kernel is tensor-bound). */
int tf_tree_attn_tc_gqa(const void* q, const void* k_tensormap, const void* v_tensormap, int layer, int kv_len, int R, int Hq,
                        int Hkv, int d, float scale, const uint32_t* tree_mask, int tree_cols, int causal, void* out,
                        void* workspace, size_t workspace_bytes, tf_stream_t stream);

/* Init-time load balancing of tf_verify_attn (no reference counterpart; the reference has no such knob).  The kernel cuts
 * its (head, key-tile) axis into one contiguous range per CTA.  Where the SMs of a GPU do not all pull the same HBM bandwidth,
 * an equal cut leaves the kernel waiting for the slowest GPCs; this call measures the per-CTA streaming time of the
 * kernel on the caller's own KV store (R rows over kv_len keys of `layer`; contents are irrelevant) for `rounds`
 * iterations and stores a split table in the workspace, which later launches with the same grid follow.  Results stay
 * deterministic for a given table.  SYNCHRONISES the stream (never call it inside a graph capture).  rounds = 0 removes
 * the table.  report (host, nullable): {max/min per-CTA time before, after, median ns before, after}.
 */
int tf_verify_attn_calibrate(const void* q, const void* k_tensormap, const void* v_tensormap, int layer, int kv_len, int R,
                             int H, int d, float scale, void* out, void* workspace, size_t workspace_bytes, int rounds,
                             double* report, tf_stream_t stream);

/* Tree (Sequoia) variant of the verify attention — replaces F.scaled_dot_product_attention with an explicit additive
 * mask at models/tensor_op.py:217,265 (tree growth over the retrieval cache) and the masked 512-row verify of
 * utils/SpecTree_TP.py:168-175: the first kv_len - tree_cols keys are visible to every row, the LAST tree_cols columns
 * follow `tree_mask` (uint32 [R][tree_cols/32], bit c of row i set = node i may attend tree column c, i.e. the
 * reference's `tree_mask == 0` entries).  R <= 32 rows per call (callers loop over row blocks of the 512-node tree).
 */
int tf_verify_attn_tree(const void* q, const void* k_tensormap, const void* v_tensormap, int layer, int kv_len_host,
                        const int32_t* kv_len_dev, int kv_len_max, int R, int H, int d, float scale, const uint32_t* tree_mask,
                        int tree_cols, void* out, void* workspace, size_t workspace_bytes, tf_stream_t stream);

/* ---- (ii) draft sliding-window attention with RoPE-on-read ---------------------------------------------------------
 * replaces models/modeling_llama_68m.py:159-186 (full-cache key re-rotation + repeat_kv + flash_attn_with_kvcache):
 * keys are stored un-rotated and rotated at their SLOT index while being staged; causal bottom-right over kv_len keys.
 *   q fp16 [R][H][d] (already rotated), K/V head-major [H][cap][d] of one layer, out fp16 [R][H][d]
 */
int tf_draft_attn(const void* q, const void* K, const void* V, long long kv_head_stride, const void* cos,
                  const void* sin, int kv_len, int R, int H, int d, float scale, void* out, tf_stream_t stream);

/* ---- cache maintenance ---------------------------------------------------------------------------------------------
 * tf_tail_update: RetrievalCache.update_graph_cache, cache.py:180-182 — copy rows [prefill, seq_len) of the full cache
 *   over retrieval slots [budget-(seq_len-prefill), budget) for all layers/heads, K and V.  seq_len = host + *dev.
 * tf_window_slide: StreamingLLMEvictionCache.evict_for_spec / evict_prefill, cache.py:252-265 — move rows
 *   [src_start, src_start+n) to [dst_start, dst_start+n) within each (layer, head) of K and V, with clone semantics
 *   (source is read completely before it is overwritten).
 */
int tf_tail_update(const void* K, const void* V, long long kv_layer_stride, long long kv_head_stride, void* retrK,
                   void* retrV, long long r_layer_stride, long long r_head_stride, int n_layers, int H, int d,
                   int prefill, int budget, int seq_len_host, const int32_t* seq_len_dev, int max_new,
                   tf_stream_t stream);
int tf_window_slide(void* K, void* V, long long layer_stride, long long head_stride, int n_layers, int H, int d,
                    int src_start, int dst_start, int n_rows, tf_stream_t stream);
/* tf_kv_compact: DistributedSimpleCache.gather_kv_incremental, cache.py:333-343 — after a tree verify, the KV rows of the
 *   accepted nodes (src_idx_dev[i], absolute slots) are packed to slots dst_start + i of every (layer, head), clone semantics. */
int tf_kv_compact(void* K, void* V, long long layer_stride, long long head_stride, int n_layers, int H, int d,
                  const int32_t* src_idx_dev, int n, int dst_start, tf_stream_t stream);

/* ---- elementwise glue of the decoder layer (fp16 rounding points of the reference) -----------------------------
 * tf_add_rmsnorm: h = fp16(h + delta) (delta may be NULL); out = fp16(w * fp16(h * rsqrt(mean(h^2) + eps)))
 *   (residual add modeling_llama.py:286,292 + LlamaRMSNorm :138-143).  h [rows][hidden] updated in place; hidden % 8 == 0,
 *   16-byte aligned pointers.
 * tf_silu_mul: out = fp16(fp16(silu(gate)) * up), gate/up = halves of gate_up [rows][2*inter] (LlamaMLP :157).
 */
int tf_add_rmsnorm(void* h, const void* delta, const void* weight, float eps, void* out, int rows, int hidden,
                   tf_stream_t stream);
int tf_silu_mul(const void* gate_up, void* out, int rows, int inter, tf_stream_t stream);

/* ---- decode-time linear layers (SURVEY §8 row f-1) -----------------------------------------------------------------
 * tf_skinny_gemm: y[M,N] = x[M,K] · W[N,K]^T, M <= 16, fp16 in/out, fp32 accumulate — replaces the F.linear / nn.Linear
 *   call sites of the decode path (models/modeling_llama.py:213-215,243,157,408; models/tensor_op.py:143-145,176,353-357)
 *   when only the gamma+1 speculated rows are live.  One CTA owns 16 output columns and the whole K (chunks of 32 dealt
 *   round-robin to its 8 warps); weights stream once from HBM straight into mma.sync B-fragments; the warps' fp32
 *   accumulators are summed in a fixed order (deterministic, no atomics).  K % 32 == 0; row strides in elements;
 *   `workspace` is unused (tf_skinny_gemm_workspace_bytes returns 0; kept for ABI stability).
 */
size_t tf_skinny_gemm_workspace_bytes(int N);
int tf_skinny_gemm(const void* x, long long x_row_stride, const void* W, long long w_row_stride, int M, int N, int K, void* y,
                   long long y_row_stride, void* workspace, size_t workspace_bytes, tf_stream_t stream);

/* tf_stream_linear: every decode-time projection (q|k|v, o_proj, gate|up, down_proj, lm_head) as ONE weight-streaming kernel
 *   built for chains of programmatically dependent launches:  y = epilogue( x · W^T ), 1 <= M <= 24, K % 64 == 0, any N.
 *   Replaces nn.Linear at models/modeling_llama.py:213-215,243,157,408 and models/tensor_op.py:143-145,176,353-357.
 *   w_tensormap: HOST pointer to the 128-byte descriptor of W from tf_weight_tensormap_encode (box_rows = 16, or 8 for
 *     the gate/up pairs of epilogue 1).  Encode once per weight matrix.  x [M][K] fp16, rows of x_row_stride elements.
 *   epilogue 0: y fp16 [M][N].  epilogue 1: W = [gate rows (N/2); up rows (N/2)], y fp16 [M][N/2] =
 *     SiLU(fp16(x·Wg^T)) * fp16(x·Wu^T) — LlamaMLP / TP_MLP (models/tensor_op.py:346-357), bit-identical to tf_silu_mul on the
 *     unfused product.  epilogue 2: y fp32 [M][N] = float(fp16(product)) — lm_head + `.float()` (modeling_llama.py:408-409).
 *   A pipeline stage carries 16 weight rows x 512 k (tensor TMA, SWIZZLE_128B) AND the matching k-slice of the token rows, so
 *   nothing is staged up front and K is unbounded; two ~100 KB CTAs per SM (M <= 8).  The producer lane issues the WEIGHT
 *   boxes of its first ring-full before `griddepcontrol.wait` (weights never depend on the predecessor kernel) and everything
 *   else after it: with tf_set_pdl the ring of kernel n+1 fills while kernel n drains.  The (tile, k-step) axis is cut into
 *   equal contiguous ranges, a tile cut by a boundary is handed between the two neighbouring CTAs through `workspace`
 *   (tf_stream_linear_workspace_bytes() bytes, ZERO-FILLED before first use, left zero; one per stream).  Sums are taken in
 *   a fixed order: results are bit-reproducible.
 */
int tf_weight_tensormap_encode(void* out_128B, const void* W, int N, int K, long long row_stride, int box_rows);
size_t tf_stream_linear_workspace_bytes(void);
int tf_stream_linear(const void* x, long long x_row_stride, const void* w_tensormap, int M, int N, int K, int epilogue, void* y,
                     long long y_row_stride, void* workspace, size_t workspace_bytes, tf_stream_t stream);

/* ---- E4M3 projection weights (opt-in; fp16 stays the default) ------------------------------------------------------
 * A projection matrix W [N][K] (one row per output feature) is stored as
 *   codes     uint8 [N][K] (torch.float8_e4m3fn bits), row-major like the fp16 matrix, row stride in bytes (% 16 == 0);
 *   exponents int8  [N], one per row.
 * Row w: e = max(-15, the smallest integer with max|w| <= 448 * 2^e) (0 for an all-zero row); code = e4m3_rn(w / 2^e), round to
 * nearest even.  The row stands for D = code * 2^e, which is an exact fp16 value (codes are multiples of 2^-9 with at most 4
 * significant bits, and e >= -15): nothing rounds in D.  Rows that are not finite or have max|w| > 61440 = 240 * 2^8 (above
 * which D can round past the fp16 maximum) are refused.
 * tf_weight_quantize_e4m3: W fp16 [N][row_stride elements] -> codes and exponents.  A refused row is left unwritten and counted
 *   into *refused_rows (device int32, may be NULL); the caller reads the count after the stream is synchronised.
 * tf_weight_dequantize_e4m3: codes and exponents -> D fp16 [N][d_row_stride elements] (the GEMM path of > 24-row forwards).
 * tf_weight_tensormap_encode_e4m3: the descriptor of a code matrix for tf_stream_linear_e4m3 (one view for every epilogue).
 * tf_stream_linear_e4m3: tf_stream_linear over E4M3 weights, epilogues 0, 1 and 2 (no TP seams), same M / K / alignment checks,
 *   workspace and PDL bit.  The same kernel with 8 KB code stages: a lane converts the codes of its k slots with
 *   cvt.rn.f16x2.e4m3x2 once for all token blocks, and the epilogue multiplies each row's fp32 sum by its 2^e (the gate and the
 *   up row each by their own) before the fp16 rounding.  As D is exact and power-of-two scaling commutes with the fp32 products
 *   and sums, y is BIT-IDENTICAL to tf_stream_linear on D for every M <= 24 and epilogue.  Exception measured on H100: rows
 *   whose D is almost entirely fp16 subnormals (max|w| around 2^-10 and below) can differ in the last bit of a few small
 *   outputs, because the fp16 kernel's tensor-core sums over subnormal operands are not exactly 2^e times the e4m3 kernel's.
 */
int tf_weight_quantize_e4m3(const void* W, long long row_stride, int N, int K, void* codes, long long codes_row_stride, int8_t* exps,
                            int32_t* refused_rows, tf_stream_t stream);
int tf_weight_dequantize_e4m3(const void* codes, long long codes_row_stride, const int8_t* exps, int N, int K, void* D, long long d_row_stride,
                              tf_stream_t stream);
int tf_weight_tensormap_encode_e4m3(void* out_128B, const void* codes, int N, int K, long long row_stride);
int tf_stream_linear_e4m3(const void* x, long long x_row_stride, const void* w_tensormap, const int8_t* w_exp, int M, int N, int K,
                          int epilogue, void* y, long long y_row_stride, void* workspace, size_t workspace_bytes, tf_stream_t stream);

/* tf_stream_linear_allreduce: the TP seams as ONE kernel — the row-parallel o_proj / down_proj of tf_stream_linear AND the
 *   all-reduce(SUM) that follows it in the reference (models/tensor_op.py:176-179, 357-359): y = sum_r x_r · W_r^T, fp16, identical
 *   bits on every rank.  The reducer warp of each finished [16 features x M tokens] tile stores its fp16 partial into slot `rank`
 *   of every rank's inbox (ONE `multimem.st` through the NVSwitch when `multicast_buffer` != NULL, else one peer store per rank),
 *   raises the tile's flag on every rank, waits for the peers' flags of that tile and adds the copies in rank order in fp32,
 *   while the other warps already stream the next tile.  `peer_buffers[r]` = this process's mapping of rank r's symmetric buffer
 *   of tf_stream_linear_allreduce_buffer_bytes() bytes (zero-filled once); `multicast_buffer` = the NVLS multicast mapping of
 *   the same symmetric allocation or NULL; `epoch_and_counter` int32[2], local, zero-initialised.  N <= 8192, M <= 24,
 *   2 <= world <= 8; every rank must issue the same sequence of calls (a peer that never delivers trips a bounded spin → trap).
 */
size_t tf_stream_linear_allreduce_buffer_bytes(void);
int tf_stream_linear_allreduce(const void* x, long long x_row_stride, const void* w_tensormap, int M, int N, int K, void* y,
                               long long y_row_stride, void* workspace, size_t workspace_bytes, void* const* peer_buffers,
                               void* multicast_buffer, int rank, int world, int32_t* epoch_and_counter, tf_stream_t stream);

/* The LL seam — what the TP engine runs by default on o_proj / down_proj (models/tensor_op.py:176-179, 357-359: row-parallel
 *   linear, dist.all_reduce, then the residual add + RMSNorm of the decoder layer, models/TP_layers.py:177-201) as TWO kernels with
 *   no stand-alone collective between them:
 *   tf_stream_linear_ll_push  = tf_stream_linear whose epilogue pushes every fp16 feature pair as an 8-byte {half2, epoch} slot into
 *     slot-array `rank` of EVERY rank's tf_allreduce_ll inbox (one `multimem.st` through the NVSwitch when `multicast_buffer` != NULL,
 *     else one peer store per rank).  No fence, no flag, nothing waited for; no y is written.
 *   tf_add_rmsnorm_ll         = tf_add_rmsnorm whose `delta` is read from the local inbox: polls the slots of its row until their
 *     flag shows the epoch, adds the `world` copies in rank order in fp32, rounds to fp16 (bit-identical to tf_allreduce_ll followed
 *     by tf_add_rmsnorm, and identical on every rank), then h += delta, RMSNorm.  Its last CTA advances the epoch.
 *   Buffers: the SAME symmetric buffer (tf_allreduce_ll_buffer_bytes(max_message_bytes), zero-filled once) and `epoch_and_counter`
 *   as tf_allreduce_ll — the three calls may be mixed freely on one stream as long as every push is followed by exactly one
 *   tf_add_rmsnorm_ll of the same [M, N] before the next exchange, and every rank issues the same sequence.  M*N*2 <= max_message_bytes.
 */
int tf_stream_linear_ll_push(const void* x, long long x_row_stride, const void* w_tensormap, int M, int N, int K, void* workspace,
                             size_t workspace_bytes, void* const* peer_buffers, void* multicast_buffer, int rank, int world,
                             size_t max_message_bytes, const int32_t* epoch_and_counter, tf_stream_t stream);
int tf_add_rmsnorm_ll(void* h, const void* local_buffer, int world, size_t max_message_bytes, int32_t* epoch_and_counter, const void* weight,
                      float eps, void* out, int rows, int hidden, tf_stream_t stream);

/* tf_skinny_gemm_allreduce: the row-parallel linear AND the all-reduce that follows it in the reference (o_proj:
 *   models/tensor_op.py:176-179; down_proj: :357-359) as ONE kernel over NVLink peer memory: y = sum_r x_r · W_r^T.  Each CTA
 *   pushes its finished [M x 16] tile (fp16) into every rank's inbox with peer stores, publishes a per-tile flag, waits for
 *   the peers' copies of the same tile and adds them in rank order (bit-identical on all ranks).  `peer_buffers[r]` = this
 *   process's mapping of rank r's symmetric buffer of tf_skinny_gemm_allreduce_buffer_bytes() bytes (zero-filled once);
 *   `epoch_and_counter` int32[2], local, zero-initialised.  N % 16 == 0, N <= 8192, M <= 16, 2 <= world <= 8; all ranks must
 *   issue the same sequence of calls.
 */
size_t tf_skinny_gemm_allreduce_buffer_bytes(void);
int tf_skinny_gemm_allreduce(const void* x, long long x_row_stride, const void* W, long long w_row_stride, int M, int N, int K,
                             void* y, long long y_row_stride, void* const* peer_buffers, int rank, int world,
                             int32_t* epoch_and_counter, tf_stream_t stream);

/* ---- whole-loop graph: the draft -> retrieve -> verify iteration as ONE graph launch with a device-side WHILE loop -------------
 * replaces utils/graph_infer.py (GraphInferenceEngine :129-194: gamma+3 draft graphs + 1 verify graph) as driven by
 * utils/decoding.py:163-223 (Middle_Spec: a host synchronisation after every sampled token, :186,193,203) and :70-141 (the outer
 * accept walk).  The caller captures three cudaGraph_t (stream capture of its own forwards): `pre` (tf_loop_begin), `body` (draft
 * forward of gamma rows -> tf_loop_draft_sample -> retrieval-verify forward -> tf_loop_middle_accept) and `post`
 * (tf_loop_prepare_full -> full-KV forward of gamma+2 rows -> tf_loop_verify -> cache maintenance -> result copy);
 * tf_loop_graph_build makes  pre -> WHILE(n < gamma){ body; cudaGraphSetConditional } -> post  out of them.
 * state int32[8]: [0] n, [1] k = ids emitted, [2] last accept, [3] accepted draft tokens, [4] inner iterations.
 * rng: device struct {uint64 seed, uint64 next_draw} — counter-based Philox4x32-10; draw c, element i -> lane i%4 of
 *   Philox(counter = (i/4, c_lo, c_hi, 0), key = seed); uniform = ((x >> 8) + 1/2) * 2^-24 in float32, strictly inside (0,1)
 *   (the one word that rounds to 1.0 gives 1 - 2^-24), exponential = -log(uniform).  Order of draws = the reference's: per inner
 *   iteration exponential / uniform / exponential, per outer iteration a uniform block then (when a token is drawn) one
 *   exponential.  tf_philox_fill(state, kind 0 uniform | 1 exponential) replays one draw into a buffer and advances the
 *   counter — the step-wise loop uses it, which is how both loops are compared event for event.
 * tf_loop_verify: res int32[16]: [0] tokens produced, [1] accepted ids, [2] rejected, [3] gamma2, [4] examined, [5] hit eos,
 *   [6] inner iterations, [7] inner accepts, [8] draft-window shift, [9] new seq_len; it also advances *seq_len_dev by count + 1 and
 *   writes the next first token.  tf_window_slide_dev = tf_window_slide with the source offset read from device memory. */
int tf_philox_fill(void* rng_state, int kind, float* out, int n, tf_stream_t stream);
int tf_loop_begin(int32_t* state, int64_t* verify_tokens, const int64_t* first_token, int gamma, const int32_t* seq_len_dev,
                  int64_t* position_ids, tf_stream_t stream);
int tf_loop_draft_sample(const float* draft_probs, int V, const int32_t* state, void* rng_state, int64_t* verify_tokens,
                         tf_stream_t stream);
int tf_loop_middle_accept(const float* draft_probs, const float* verify_probs, int64_t* verify_tokens, void* rng_state, int gamma,
                          int V, int32_t* state, int64_t* out_ids, float* spec_probs, tf_stream_t stream);
int tf_loop_prepare_full(const int32_t* state, const int64_t* out_ids, const int64_t* first_token, int64_t* full_ids, int rows,
                         tf_stream_t stream);
int tf_loop_verify(const float* p_rows, const float* q_rows, const int64_t* out_ids, const int32_t* state, void* rng_state, int V,
                   int strict_less, int64_t eos, int64_t* first_token, int32_t* res, int64_t* tokens, int64_t* pass_tokens,
                   int pass_len, int32_t* seq_len_dev, tf_stream_t stream);
int tf_window_slide_dev(void* K, void* V, long long layer_stride, long long head_stride, int L, int H, int d, int src_base,
                        const int32_t* shift_dev, int dst_start, int n_rows, tf_stream_t stream);
int tf_loop_graph_build(void* pre_graph, void* body_graph, void* post_graph, const int32_t* state, int gamma, void** exec_out);
int tf_loop_graph_launch(void* exec, tf_stream_t stream);
int tf_loop_graph_destroy(void* exec);

/* ---- TP seam: one-shot all-reduce over NVLink peer memory -----------------------------------------------------------
 * replaces dist.all_reduce(SUM) after the row-parallel o_proj / down_proj (models/tensor_op.py:179,225,271,326,359) for the
 * small decode-time messages ([rows<=32, hidden] fp16).  `peer_buffers[r]` = this process's mapping of rank r's symmetric
 * buffer (tf_allreduce_buffer_bytes(max_message_bytes) bytes, zero-filled once, shared through CUDA IPC / symmetric
 * memory; entry `rank` is the local buffer); `multicast_buffer` = the NVLS multicast mapping of the same allocation, or NULL.
 * PUSH model: every rank stores its slice into slot `rank` on all ranks (one `multimem.st` through the switch, or one peer store
 * per rank), raises a flag per CTA, waits for the peers' flags and adds the `world` LOCAL slots in rank order in fp32 →
 * bit-identical results on all ranks.  `epoch_and_counter`: int32[2] in local device memory, zero-initialised.  Every rank must
 * issue the same sequence of calls with the same n_elements (a peer that never arrives trips a bounded spin → trap).
 * Graph-capturable; never blocks the host; releases its programmatic dependents at entry (tf_set_pdl bit 256).
 */
size_t tf_allreduce_buffer_bytes(size_t max_message_bytes);
/* tf_allreduce_ll: the same all-reduce in "low latency" form — every 8-byte slot carries {half2 payload, epoch}, pushed to all ranks
 * (multimem.st / peer stores) and polled locally: one one-way NVLink latency, no system-scope fence, no flag round trip.  Buffer:
 * tf_allreduce_ll_buffer_bytes(max_message_bytes), zero-filled once; n_elements % 2 == 0.  Default seam exchange of the TP path. */
size_t tf_allreduce_ll_buffer_bytes(size_t max_message_bytes);
int tf_allreduce_ll(void* const* peer_buffers, void* multicast_buffer, int rank, int world, const void* in, void* out,
                    long long n_elements, size_t max_message_bytes, int32_t* epoch_and_counter, tf_stream_t stream);
int tf_allreduce_oneshot(void* const* peer_buffers, void* multicast_buffer, int rank, int world, const void* in, void* out,
                         long long n_elements, size_t max_message_bytes, int32_t* epoch_and_counter, tf_stream_t stream);

/* ---- sampling ------------------------------------------------------------------------------------------------------
 * tf_norm_logits: utils/sampling.py:43-60 (norm_logits) incl. the top-p filter :16-27 — logits/T, descending stable
 *   sort, softmax, cumulative sum, keep the prefix whose exclusive cumulative mass <= top_p (first token always kept),
 *   renormalise.  fp32 in/out, one CTA per row, rows x V with V <= TF_SAMPLING_MAX_VOCAB.  top_p >= 1 keeps everything.
 * tf_sample_argmax: utils/sampling.py:63-65 — torch.multinomial(p, 1) on CUDA is argmax(p / Exp(1)-noise); the noise
 *   is an input so the caller decides the random stream.  Writes an int64 token per row (first index on ties).
 * tf_residual_probs: utils/sampling.py:68-75 (max_fn): out = relu(p-q) / sum(relu(p-q)).
 */
#define TF_SAMPLING_MAX_VOCAB 32768
size_t tf_norm_logits_workspace_bytes(int rows, int V);
int tf_norm_logits(const float* logits, long long row_stride, int rows, int V, float temperature, float top_p,
                   float* probs, void* workspace, size_t workspace_bytes, tf_stream_t stream);
int tf_sample_argmax(const float* probs, long long probs_row_stride, const float* expo, long long expo_row_stride,
                     int rows, int V, int64_t* out_tokens, tf_stream_t stream);
int tf_residual_probs(const float* p, const float* q, int V, float* out, tf_stream_t stream);

/* ---- fused speculative accept/reject (one warp-level walk + one CTA-wide resample) -----------------------------
 * tf_middle_accept: one inner (`Middle_Spec`) decision, utils/decoding.py:192-220.
 *   Device state `st` (int32[8]): st[0] = n (verified-token count so far), st[1] = number of ids emitted so far.
 *   Inputs: draft_probs [V]; verify_probs [gamma+1][V]; verify_tokens int64 [gamma+1] (slot n+1 holds the draft token);
 *   uniform r [1]; expo [V].  accept iff r < min(1, vp[n][t]/sp[t]).  On accept: emit (t, q=vp[n]) and
 *   (t2 ~ vp[n+1], q=vp[n+1]), n += 2; on reject: emit (t2 ~ vp[n], q=vp[n]), n += 1.  t2 is written to
 *   verify_tokens[n] when n <= gamma.  Emitted ids go to out_ids[st[1]..], their proposal rows are copied to
 *   spec_probs[k][V].  st[2] = last accept flag, st[3] += accepted, st[4] += drafted.
 * tf_verify_accept: the outer accept walk, utils/decoding.py:97-121 — for i < g2: accept gen[i] iff
 *   r_i < min(1, p[i][gen[i]] / q[i][gen[i]]) (strict `<`; `<=` when strict_less == 0, the TP variant :354), stop at the
 *   first reject or at an accepted EOS (:108-110).  res int32[4] = {count accepted, rejected?, uniforms examined,
 *   stopped on EOS?}; pass_tokens int64 [g2+2] = {first_token, accepted..., 100...} (decoding.py:94-95,104).
 * tf_verify_resample: the one multinomial that follows (:114 residual `max_fn(p-q)` on reject, :130 bonus from
 *   p[g2] when everything was accepted), driven by `res` ON THE DEVICE: token = argmax(x / expo), written to
 *   out_token[0] and pass_tokens[count+1]; res[0] is incremented for the bonus like :134.  When the walk stopped on an
 *   accepted EOS before the end nothing is sampled and out_token = that EOS (the reference draws nothing there).
 */
/* tf_tree_accept_walk: the Sequoia accept walk, utils/SpecTree_TP.py:147-165 (accept_step) driven by :181-197 (verify),
 *   as one kernel.  target_probs [T][V] (top-p'd softmax of the target), draft_logits [T][V] (MODIFIED in place exactly like the
 *   reference: a rejected token's logit becomes -FLT_MAX), verify_tokens int64 [T], successor lists in CSR form
 *   (succ_off int32 [T+1], succ int32), uniforms consumed one per examined child.  out int32[32]: [0] accepted nodes,
 *   [1] -1 (all children rejected) / -2 (leaf), [2] uniforms consumed, [3] terminal (token 0 or 2 accepted), [4] residual
 *   is NaN, [8..8+max_accept) accepted node ids.  `residual` [V] = the distribution the next token is drawn from.
 */
int tf_tree_accept_walk(const float* target_probs, float* draft_logits, const int64_t* verify_tokens, const int32_t* succ_off,
                        const int32_t* succ, const float* uniforms, float temperature, int V, int max_accept, int32_t* out,
                        float* residual, float* scratch_V, tf_stream_t stream);

int tf_middle_accept(const float* draft_probs, const float* verify_probs, int64_t* verify_tokens, const float* uniform,
                     const float* expo, int gamma, int V, int32_t* st, int64_t* out_ids, float* spec_probs,
                     tf_stream_t stream);
int tf_verify_accept(const float* p_rows, const float* q_rows, const int64_t* gen, int g2, const float* uniforms,
                     int V, int strict_less, int64_t eos_token, int64_t first_token, int32_t* res,
                     int64_t* pass_tokens, tf_stream_t stream);
int tf_verify_resample(const float* p_rows, const float* q_rows, const int64_t* gen, int g2, const float* expo, int V,
                       int32_t* res, int64_t* out_token, int64_t* pass_tokens, tf_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* TRIFORCE_B200_H_ */
