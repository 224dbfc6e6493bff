// Tree (Sequoia) verify attention on the Hopper tensor cores (wgmma): R = 128·k query rows (the 512 tree nodes of BASELINE
// cfg5) against the full KV of one layer — `variant = 2` of tf_verify_attn_tree.  Replaces the SDPA-with-additive-mask call of
// the reference (models/tensor_op.py:230-272 → F.scaled_dot_product_attention with a [512, S+512] fp16 mask, 134 MB at 128K).
// The same kernel in CAUSAL mode is the prefill attention (SURVEY §8 row f-2): the R rows of a prompt chunk against the keys
// written so far, bottom-right causal — the reference's eager 128-token chunks through flash_attn_with_kvcache
// (utils/graph_infer.py:28-37 → models/modeling_llama.py:240); tiles above a block's diagonal are never loaded.
//
// This is the one place in the hot path where the (rows x d) x (d x keys) contraction FILLS a tensor-core tile: each KV byte
// feeds 128 query rows of a CTA (2·128 FLOP per byte; the other row blocks of the same head read it from L2), where the
// mma.sync kernel had to re-read the KV once per 32-row block.
//
// One CTA = (128-row query block, head, KV split), 288 threads:
//   warps 0-7  two consumer warpgroups; warpgroup w owns query rows 64w .. 64w+63 of the block.  Per 128-key tile:
//              S = Q·K^T as 8 x wgmma m64n128k16 (A = Q, B = K, both K-major from shared memory) into 64 fp32 registers per
//              thread, online softmax in registers (quad shuffles for the row maximum, exp2 domain), P packed to fp16 in
//              registers in exactly the A-fragment layout of the next wgmma, O += P·V as 8 x wgmma m64n128k16 with A from
//              registers and B = V MN-major (transposed) from shared memory; the tree mask (ancestor bitmask of the last T
//              columns), the kv_len bound and the causal diagonal are applied to the tiles they touch.
//   warp 8     TMA producer: the Q block once (tensor map over [R][H][d]), then K and V tiles of 128 keys (four 64x64 boxes
//              each, SWIZZLE_128B — exactly the canonical K-major / MN-major wgmma shared-memory layouts) into a ring of single
//              32 KB tiles in the order K0 V0 K1 V1 ...; a slot is released when both warpgroups' wgmmas that read it completed.
//   The two warpgroups are independent: while one runs its softmax, the tensor core serves the other's wgmmas.
// Partials (m, l, unnormalised O) per (block, head, split) go to the workspace; `tree_attn_merge_kernel` combines the splits.
//
// Grouped-query attention (tf_tree_attn_tc_gqa): the grid stays (block, QUERY head, split) and only the producer's K/V head
// coordinate becomes h / grp.  The grp CTAs of a group each stream the same K/V tiles, so KV is read grp times per block
// instead of once.  That is acceptable here: this kernel is bound by the tensor cores (2·128 FLOP per byte), the group's
// CTAs run side by side, and the repeated reads hit L2.
//
// An E4M3 store (tf_tree_attn_tc_e4m3, the format of common.cuh; MHA or GQA): the wgmma takes both B operands from shared
// memory as fp16, so the codes become fp16 tiles there and the consumers run unchanged.  Warps 8-11 (the converter warpgroup,
// 384 threads per CTA) replace the producer warp: thread 0 loads the Q block and the 16 KB code tiles (two 64-key boxes of
// 128-byte rows, SWIZZLE_128B) with their 128 exponents into a ring of kTcCodeSlots; all 128 threads expand each code tile into
// exactly the SWIZZLE_128B fp16 tile TMA would have written from the dequantized store D (common.cuh: D = fp16_rn(code·2^e)),
// then fence.proxy.async (the wgmma reads through the async proxy) and arrive on the slot the consumers wait for.  The output
// is therefore bit-identical to tf_tree_attn_tc over a store holding D.
#include <string.h>

#include "common.cuh"

namespace tf {

constexpr int kTcKeys = 128;           // keys per tile (wgmma N of QK^T, K extent of PV)
constexpr int kTcD = 128;              // head dim
constexpr int kTcBlockRows = 128;      // query rows per CTA: two 64-row warpgroups sharing every K / V tile
constexpr int kTcSlots = 4;            // ring of single 32 KB K / V tiles (two tiles of keys in flight)
constexpr int kTcConsumerWarps = 8;
constexpr int kTcThreads = (kTcConsumerWarps + 1) * 32;
constexpr uint32_t kTcTileBytes = kTcKeys * kTcD * 2;  // 32 KB: one K or V tile, also the Q block
constexpr uint32_t kTcHalfBytes = kTcTileBytes / 2;    // one 64-element (128-byte) column half: 128 rows x 128 B
// E4M3 store: the converter warpgroup and its ring of code tiles (16 KB of codes + 128 exponents each; 4 slots = two tiles of
// keys ahead of the conversion, 226 KB of shared memory in all)
constexpr int kTcConvThreads = 128;
constexpr int kTcThreadsE4m3 = kTcConsumerWarps * 32 + kTcConvThreads;
constexpr int kTcCodeSlots = 4;
constexpr uint32_t kTcCodeBytes = kTcKeys * kTcD;      // 16 KB: one K or V tile of codes

// ---- wgmma wrappers ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

#define TC_ACC8(x, i) "+f"(x[i]), "+f"(x[i + 1]), "+f"(x[i + 2]), "+f"(x[i + 3]), "+f"(x[i + 4]), "+f"(x[i + 5]), "+f"(x[i + 6]), "+f"(x[i + 7])
#define TC_ACC64(x) TC_ACC8(x, 0), TC_ACC8(x, 8), TC_ACC8(x, 16), TC_ACC8(x, 24), TC_ACC8(x, 32), TC_ACC8(x, 40), TC_ACC8(x, 48), TC_ACC8(x, 56)
#define TC_D64 \
  "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,"  \
  "%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}"

// d[64x128] (+)= A[64x16] · B[16x128], A and B from shared memory, both K-major
__device__ __forceinline__ void wg_mma_ss(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 " TC_D64 ", %64, %65, p, 1, 1, 0, 0;\n"
      "}\n"
      : TC_ACC64(d)
      : "l"(adesc), "l"(bdesc), "r"(accumulate)
      : "memory");
}
// d[64x128] += A[64x16] · B[16x128], A from registers (the m64k16 A fragment), B from shared memory MN-major (transposed)
__device__ __forceinline__ void wg_mma_rs_tb(float (&d)[64], const uint32_t* a, uint64_t bdesc) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 " TC_D64 ", {%64,%65,%66,%67}, %68, 1, 1, 1, 1;\n"
      : TC_ACC64(d)
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc)
      : "memory");
}

// wgmma shared-memory descriptor (cute/arch/mma_sm90_desc.hpp: GmmaDescriptor) of a [rows][64 fp16] half tile of 128-byte rows
// under SWIZZLE_128B (8-row atoms of 1024 B), as TMA writes it:
//   K-major (the contraction runs along the 128-byte row): SBO = 1024 B between 8-row groups; a K = 16 step = +32 B;
//   MN-major (the row IS the N extent, contraction across rows): LBO = distance to the next 64-element half (16 KB),
//   SBO = 1024 B between 8-row (= 8-k) groups; a K = 16 step = +16 rows = +2048 B.
__device__ __forceinline__ uint64_t wg_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFFu) >> 4);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32;
  d |= (uint64_t)1 << 62;  // LayoutType::B128 (SWIZZLE_128B)
  return d;
}

__device__ __forceinline__ void tc_tma_3d(uint32_t smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(
                   smem_dst),
               "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}

struct TcArgs {
  int layer, H, R;
  int grp;                    // query heads per KV head: query head h reads K/V head h / grp (1: MHA)
  int kv_len;                 // keys (prefix + tree columns)
  int tree_cols;              // last tree_cols keys follow the bitmask (0: every key below kv_len is visible to every row)
  const uint32_t* tree_mask;  // [R][tree_cols / 32]
  int causal;                 // 1: bottom-right causal mask of R new rows (prefill chunks): row i sees key j iff j <= kv_len - R + i
  float scale_log2;
  int splits, tiles_per_split;
  float* part_o;              // [blocks][H][splits][128][128] unnormalised
  float* part_m;              // [blocks][H][splits][128]   running maximum (log2 domain), -inf when the split saw nothing
  float* part_l;              // [blocks][H][splits][128]
  float* debug_s;             // nullable: scores of the CTA's first tile (block 0, head 0, split 0, rows 0..127) — test hook
  const int8_t* k_exp;        // E4M3 store only: exponents [layer][H / grp][cap]
  const int8_t* v_exp;
  long long cap;
};

// Visibility of the 32 keys key0 .. key0+31 for one query row, as a bit word.  base = key0 - prefix (prefix = kv_len - tree_cols):
// keys below the prefix are visible to everybody, tree column c follows bit c of the row's ancestor mask, keys >= kv_len (columns
// >= tree_cols) are invisible.
__device__ __forceinline__ uint32_t tc_vis_word(const uint32_t* __restrict__ mrow, int words, int base) {
  if (base <= -32) return 0xffffffffu;
  auto mw = [&](int k) -> uint32_t { return (mrow != nullptr && k < words) ? __ldg(mrow + k) : 0u; };
  if (base < 0) {
    const int n = -base;  // 1..31 prefix keys, then tree columns 0..
    return ((1u << n) - 1u) | (mw(0) << n);
  }
  const int w = base >> 5, sh = base & 31;
  uint32_t x = mw(w) >> sh;
  if (sh) x |= mw(w + 1) << (32 - sh);
  return x;
}

__device__ __forceinline__ float tc_ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

__device__ __forceinline__ uint32_t pack_half2(float lo, float hi) {
  const __half2 h = __floats2half2_rn(lo, hi);
  return *reinterpret_cast<const uint32_t*>(&h);
}

// Register fragments (wgmma m64nNk16, per warp of the warpgroup: 16 rows; g = lane / 4, t = lane % 4):
//   accumulator element 4n + e  <->  row g + 8 (e >> 1), column 8n + 2t + (e & 1)
//   A fragment of k-step kk     <->  {row g, keys 16kk + 2t..}, {row g+8, same}, {row g, keys 16kk + 8 + 2t..}, {row g+8, same}
// so the scores of keys 16kk .. 16kk+15 (accumulator elements 8kk .. 8kk+7) are, packed in pairs, the A fragment of PV step kk.
//
// E4M3: converter thread ct expands 16-byte code chunk c = ct & 7 of rows 16 it + ct / 8 (it = 0..7) into the two 16-byte fp16
// chunks 2(c & 3), 2(c & 3) + 1 of column half c / 4.  Loads and stores are whole 128-byte rows per 8-thread phase; threads with
// c >= 4 store their second chunk first, so that each store instruction's phase also hits eight different bank groups.
__device__ __forceinline__ void tc_convert_tile(const uint8_t* __restrict__ codes, const int8_t* __restrict__ exps, uint8_t* __restrict__ dst,
                                                int ct) {
#pragma unroll
  for (int it = 0; it < kTcKeys * kTcD / 16 / kTcConvThreads; ++it) {
    const int idx = it * kTcConvThreads + ct;
    const int r = idx >> 3, c = idx & 7, sw = r & 7;
    const uint4 w = *reinterpret_cast<const uint4*>(codes + r * 128 + ((c ^ sw) << 4));
    __half fa, fb;
    kv_e4m3_factors(exps[r], fa, fb);
    const __half2 a2 = __half2half2(fa), b2 = __half2half2(fb);
    const uint32_t cw[4] = {w.x, w.y, w.z, w.w};
    uint32_t o[8];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const __half2 lo = kv_e4m3_apply(kv_e4m3_codes2((uint16_t)(cw[k] & 0xffffu)), a2, b2);
      const __half2 hi = kv_e4m3_apply(kv_e4m3_codes2((uint16_t)(cw[k] >> 16)), a2, b2);
      o[2 * k] = *reinterpret_cast<const uint32_t*>(&lo);
      o[2 * k + 1] = *reinterpret_cast<const uint32_t*>(&hi);
    }
    const uint4 first = make_uint4(o[0], o[1], o[2], o[3]), second = make_uint4(o[4], o[5], o[6], o[7]);
    uint8_t* row = dst + (c >> 2) * kTcHalfBytes + r * 128;
    const int j0 = 2 * (c & 3);
    const bool swap = c >= 4;
    *reinterpret_cast<uint4*>(row + (((swap ? j0 + 1 : j0) ^ sw) << 4)) = swap ? second : first;
    *reinterpret_cast<uint4*>(row + (((swap ? j0 : j0 + 1) ^ sw) << 4)) = swap ? first : second;
  }
}

template <bool kE4m3>
__global__ void __launch_bounds__(kE4m3 ? kTcThreadsE4m3 : kTcThreads, 1)
    tree_attn_tc_kernel(const __grid_constant__ CUtensorMap qmap, const __grid_constant__ CUtensorMap kmap, const __grid_constant__ CUtensorMap vmap,
                        const TcArgs a) {
  extern __shared__ uint8_t tc_smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(tc_smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* q_s = smem;                      // [2 halves][128 rows][128 B]
  uint8_t* kv_s = q_s + kTcTileBytes;       // [slots] single tiles [2 halves][128 keys][128 B]: K0 V0 K1 V1 ...
  uint8_t* codes_s = kv_s + (size_t)kTcSlots * kTcTileBytes;  // E4M3: [code slots][128 keys][128 B], then [code slots][128] exponents
  int8_t* cexp_s = reinterpret_cast<int8_t*>(codes_s + (size_t)kTcCodeSlots * kTcCodeBytes);
  uint64_t* bars = reinterpret_cast<uint64_t*>(kE4m3 ? reinterpret_cast<uint8_t*>(cexp_s) + kTcCodeSlots * kTcKeys : codes_s);
  uint64_t* q_full = bars;                  // 1
  uint64_t* kv_full = bars + 1;             // [slots]
  uint64_t* kv_empty = kv_full + kTcSlots;  // [slots]
  uint64_t* code_full = kv_empty + kTcSlots;  // E4M3: [code slots]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int qb = blockIdx.x, h = blockIdx.y, sp = blockIdx.z;
  // causal mode: this block's rows see nothing beyond key kv_len - R + (last row of the block) → its tiles end at the diagonal,
  // and its KV splits divide what is left evenly
  const int last_key = a.causal ? min(a.kv_len - 1, a.kv_len - a.R + qb * kTcBlockRows + kTcBlockRows - 1) : a.kv_len - 1;
  const int tiles_total = last_key >= 0 ? last_key / kTcKeys + 1 : 0;
  const int tiles_per_split = a.causal ? (tiles_total + a.splits - 1) / a.splits : a.tiles_per_split;
  const int t_begin = sp * tiles_per_split;
  const int t_end = min(tiles_total, t_begin + tiles_per_split);
  const int n_tiles = t_end - t_begin;  // may be <= 0 for trailing splits: they publish an empty partial

  if (threadIdx.x == 0) {
    mbar_init(q_full, 1);
    for (int s = 0; s < kTcSlots; ++s) { mbar_init(&kv_full[s], kE4m3 ? kTcConvThreads : 1); mbar_init(&kv_empty[s], kTcConsumerWarps); }
    if constexpr (kE4m3)
      for (int s = 0; s < kTcCodeSlots; ++s) mbar_init(&code_full[s], 1);
    fence_mbar_init();
  }
  __syncthreads();

  if constexpr (kE4m3) {
    if (warp >= kTcConsumerWarps) {
      // ================= converter warpgroup (thread 0 also issues the loads) =================
      const int ct = threadIdx.x - kTcConsumerWarps * 32;
      const int hk = h / a.grp;
      const size_t exp_row0 = ((size_t)a.layer * (a.H / a.grp) + hk) * (size_t)a.cap;
      // code tile i (K of key tile i / 2 for even i, V for odd i) into code slot i % kTcCodeSlots.  Its exponents stop at cap
      // (cap and key0 are multiples of 64); a code box beyond cap is zero-filled by TMA, and a zero code is 0 at any exponent.
      auto issue = [&](int i) {
        const uint32_t cs = (uint32_t)i % kTcCodeSlots;
        const int key0 = (t_begin + (i >> 1)) * kTcKeys;
        const CUtensorMap* map = (i & 1) ? &vmap : &kmap;
        const uint32_t ebytes = (uint32_t)min((long long)kTcKeys, a.cap - key0);
        uint8_t* dst = codes_s + (size_t)cs * kTcCodeBytes;
        mbar_expect_tx(&code_full[cs], kTcCodeBytes + ebytes);
        tma_load_4d(dst, map, &code_full[cs], 0, key0, hk, a.layer);
        tma_load_4d(dst + kTcCodeBytes / 2, map, &code_full[cs], 0, key0 + 64, hk, a.layer);
        bulk_load(cexp_s + cs * kTcKeys, ((i & 1) ? a.v_exp : a.k_exp) + exp_row0 + key0, ebytes, &code_full[cs]);
      };
      if (n_tiles > 0) {
        if (ct == 0) {
          prefetch_tensormap(&qmap);
          prefetch_tensormap(&kmap);
          prefetch_tensormap(&vmap);
          mbar_expect_tx(q_full, kTcTileBytes);
          tc_tma_3d(smem_u32(q_s), &qmap, q_full, 0, h, qb * kTcBlockRows);
          tc_tma_3d(smem_u32(q_s) + kTcHalfBytes, &qmap, q_full, 64, h, qb * kTcBlockRows);
          for (int i = 0; i < min(kTcCodeSlots, 2 * n_tiles); ++i) issue(i);
        }
        for (int i = 0; i < 2 * n_tiles; ++i) {
          const uint32_t cs = (uint32_t)i % kTcCodeSlots, cph = ((uint32_t)i / kTcCodeSlots) & 1u;
          const uint32_t s = (uint32_t)i % kTcSlots, ph = ((uint32_t)i / kTcSlots) & 1u;
          mbar_wait(&code_full[cs], cph);
          mbar_wait(&kv_empty[s], ph ^ 1u);
          tc_convert_tile(codes_s + (size_t)cs * kTcCodeBytes, cexp_s + cs * kTcKeys, kv_s + (size_t)s * kTcTileBytes, ct);
          fence_proxy_async();  // the generic-proxy stores above, before the consumers' wgmma reads them through the async proxy
          mbar_arrive(&kv_full[s]);
          asm volatile("bar.sync 1, %0;" ::"n"(kTcConvThreads) : "memory");  // every converter thread is done with code slot cs
          if (ct == 0 && i + kTcCodeSlots < 2 * n_tiles) issue(i + kTcCodeSlots);
        }
      }
      return;
    }
  }

  if (!kE4m3 && warp == kTcConsumerWarps) {
    // ================= TMA producer =================
    if (lane == 0 && n_tiles > 0) {
      prefetch_tensormap(&qmap);
      prefetch_tensormap(&kmap);
      prefetch_tensormap(&vmap);
      mbar_expect_tx(q_full, kTcTileBytes);  // rows beyond R are zero-filled by TMA (their results are never stored)
      tc_tma_3d(smem_u32(q_s), &qmap, q_full, 0, h, qb * kTcBlockRows);
      tc_tma_3d(smem_u32(q_s) + kTcHalfBytes, &qmap, q_full, 64, h, qb * kTcBlockRows);
      for (int i = 0; i < 2 * n_tiles; ++i) {
        const uint32_t s = (uint32_t)i % kTcSlots, ph = ((uint32_t)i / kTcSlots) & 1u;
        mbar_wait(&kv_empty[s], ph ^ 1u);
        mbar_expect_tx(&kv_full[s], kTcTileBytes);
        const int key0 = (t_begin + (i >> 1)) * kTcKeys;
        uint8_t* dst = kv_s + (size_t)s * kTcTileBytes;
        const CUtensorMap* map = (i & 1) ? &vmap : &kmap;
#pragma unroll
        for (int half = 0; half < 2; ++half) {
#pragma unroll
          for (int kb = 0; kb < 2; ++kb)  // the KV tensor maps carry 64-key boxes: two per 128-key tile, stacked row after row
            tma_load_4d(dst + half * kTcHalfBytes + kb * (kTcHalfBytes / 2), map, &kv_full[s], half * 64, key0 + kb * 64, h / a.grp, a.layer);
        }
      }
    }
    return;
  }

  // ================= consumer warpgroups =================
  const int wg = warp >> 2;                         // 64-row half of the block
  const int g = lane >> 2, t = lane & 3;
  const int rb0 = wg * 64 + (warp & 3) * 16 + g;    // rows of this thread within the block: rb0 and rb0 + 8
  const int row0 = qb * kTcBlockRows + rb0;
  const int prefix = a.kv_len - a.tree_cols;
  const int words = a.tree_cols >> 5;
  const uint32_t* mrow[2] = {a.tree_mask != nullptr ? a.tree_mask + (size_t)min(row0, a.R - 1) * words : nullptr,
                             a.tree_mask != nullptr ? a.tree_mask + (size_t)min(row0 + 8, a.R - 1) * words : nullptr};
  const uint32_t q_u = smem_u32(q_s) + (uint32_t)wg * 64u * 128u;
  float o[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};  // running maximum (log2 domain, scaled) and partial denominator

  if (n_tiles > 0) mbar_wait(q_full, 0);
  for (int j = 0; j < n_tiles; ++j) {
    const uint32_t ks = (uint32_t)(2 * j) % kTcSlots, kph = ((uint32_t)(2 * j) / kTcSlots) & 1u;
    const uint32_t vs = (uint32_t)(2 * j + 1) % kTcSlots, vph = ((uint32_t)(2 * j + 1) / kTcSlots) & 1u;
    const int key0 = (t_begin + j) * kTcKeys;
    // ---- S = Q K^T ----
    float s[64];
    mbar_wait(&kv_full[ks], kph);
    const uint32_t k_u = smem_u32(kv_s + (size_t)ks * kTcTileBytes);
    wg_fence();
#pragma unroll
    for (int kk = 0; kk < kTcD / 16; ++kk) {
      const uint32_t off = (uint32_t)(kk >> 2) * kTcHalfBytes + (uint32_t)(kk & 3) * 32u;
      wg_mma_ss(s, wg_desc(q_u + off, 16, 1024), wg_desc(k_u + off, 16, 1024), kk > 0 ? 1u : 0u);
    }
    wg_commit();
    wg_wait_all();
    __syncwarp();
    if (lane == 0) mbar_arrive(&kv_empty[ks]);
    if (a.debug_s != nullptr && j == 0 && qb == 0 && h == 0 && sp == 0) {  // test hook: the raw score tile
#pragma unroll
      for (int i = 0; i < 64; ++i) a.debug_s[(size_t)(rb0 + 8 * ((i >> 1) & 1)) * 128 + 8 * (i >> 2) + 2 * t + (i & 1)] = s[i];
    }
    // does this tile touch tree columns / the end of the keys / (causal) the diagonal of this block?  (uniform per CTA)
    const bool masked_tile = a.causal ? key0 + kTcKeys - 1 > a.kv_len - a.R + qb * kTcBlockRows : key0 + kTcKeys > prefix;
    if (masked_tile) {
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        uint32_t vis[4];
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          if (a.causal) {  // keys key0+32c .. : visible up to lim = min(kv_len - 1, kv_len - R + row)
            const int nvis = min(a.kv_len - 1, a.kv_len - a.R + row0 + 8 * hr) - (key0 + c * 32) + 1;
            vis[c] = nvis >= 32 ? 0xffffffffu : (nvis <= 0 ? 0u : ((1u << nvis) - 1u));
          } else {
            vis[c] = tc_vis_word(mrow[hr], words, key0 + c * 32 - prefix);
          }
        }
#pragma unroll
        for (int n = 0; n < 16; ++n)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int col = 8 * n + 2 * t + e;
            if (!((vis[col >> 5] >> (col & 31)) & 1u)) s[4 * n + 2 * hr + e] = -INFINITY;
          }
      }
    }
    // ---- online softmax of the two rows (the four threads of a quad share a row) ----
    float mref[2];
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      float tmax = -INFINITY;
#pragma unroll
      for (int n = 0; n < 16; ++n) tmax = fmaxf(tmax, fmaxf(s[4 * n + 2 * hr], s[4 * n + 2 * hr + 1]));
      tmax = fmaxf(tmax, __shfl_xor_sync(0xffffffffu, tmax, 1));
      tmax = fmaxf(tmax, __shfl_xor_sync(0xffffffffu, tmax, 2));
      const float m_new = fmaxf(m_run[hr], tmax * a.scale_log2);  // -inf stays -inf
      const float alpha = (m_run[hr] == -INFINITY) ? 0.f : tc_ex2(m_run[hr] - m_new);
      l_run[hr] *= alpha;
#pragma unroll
      for (int n = 0; n < 16; ++n) {
        o[4 * n + 2 * hr] *= alpha;
        o[4 * n + 2 * hr + 1] *= alpha;
      }
      m_run[hr] = m_new;
      mref[hr] = (m_new == -INFINITY) ? 0.f : m_new;
    }
    // ---- p = exp2(s*scale - m), denominator, fp16 pack straight into the A fragments of PV ----
    uint32_t pa[32];
#pragma unroll
    for (int n = 0; n < 16; ++n)
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        const float p0 = tc_ex2(fmaf(s[4 * n + 2 * hr], a.scale_log2, -mref[hr]));
        const float p1 = tc_ex2(fmaf(s[4 * n + 2 * hr + 1], a.scale_log2, -mref[hr]));
        l_run[hr] += p0 + p1;
        pa[4 * (n >> 1) + 2 * (n & 1) + hr] = pack_half2(p0, p1);
      }
    // ---- O += P V ----
    mbar_wait(&kv_full[vs], vph);
    const uint32_t v_u = smem_u32(kv_s + (size_t)vs * kTcTileBytes);
    wg_fence();
#pragma unroll
    for (int kk = 0; kk < kTcKeys / 16; ++kk)  // B = V [128 keys][128 d] MN-major: 16 keys = 16 rows of 128 B; d halves 16 KB apart
      wg_mma_rs_tb(o, &pa[4 * kk], wg_desc(v_u + (uint32_t)kk * 16u * 128u, kTcHalfBytes, 1024));
    wg_commit();
    wg_wait_all();
    __syncwarp();
    if (lane == 0) mbar_arrive(&kv_empty[vs]);
  }
  // ---- publish the partial of this (block, head, split) ----
  const size_t slot = ((size_t)qb * a.H + h) * a.splits + sp;
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    const int rb = rb0 + 8 * hr;
    float l = l_run[hr];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    if (n_tiles > 0) {
      float* po = a.part_o + (slot * kTcBlockRows + rb) * kTcD;
#pragma unroll
      for (int n = 0; n < 16; ++n) *reinterpret_cast<float2*>(po + 8 * n + 2 * t) = make_float2(o[4 * n + 2 * hr], o[4 * n + 2 * hr + 1]);
    }
    if (t == 0) {
      a.part_m[slot * kTcBlockRows + rb] = n_tiles > 0 ? m_run[hr] : -INFINITY;
      a.part_l[slot * kTcBlockRows + rb] = n_tiles > 0 ? l : 0.f;
    }
  }
}

// out[row][h][:] = sum_s 2^(m_s - m) O_s / sum_s 2^(m_s - m) l_s over the KV splits (fixed order → deterministic)
__global__ void __launch_bounds__(128) tree_attn_merge_kernel(const float* __restrict__ part_o, const float* __restrict__ part_m,
                                                            const float* __restrict__ part_l, int H, int R, int splits, __half* __restrict__ out) {
  const int row = blockIdx.x, h = blockIdx.y;
  if (row >= R) return;
  const int qb = row / kTcBlockRows, r = row % kTcBlockRows;
  const size_t slot0 = ((size_t)qb * H + h) * splits;
  float m = -INFINITY;
  for (int s = 0; s < splits; ++s) m = fmaxf(m, part_m[(slot0 + s) * kTcBlockRows + r]);
  float den = 0.f, acc = 0.f;
  const int c = threadIdx.x;
  for (int s = 0; s < splits; ++s) {
    const float ms = part_m[(slot0 + s) * kTcBlockRows + r];
    if (ms == -INFINITY) continue;
    const float w = exp2f(ms - m);
    den = fmaf(w, part_l[(slot0 + s) * kTcBlockRows + r], den);
    acc = fmaf(w, part_o[((slot0 + s) * kTcBlockRows + r) * kTcD + c], acc);
  }
  out[((size_t)row * H + h) * kTcD + c] = __float2half_rn(den > 0.f ? acc / den : 0.f);
}

typedef CUresult (*PFN_encodeTiledTC)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                      const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                      CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static int tc_plan_splits(int blocks, int H, int tiles_total) {
  int sms = sm_count();
  if (sms <= 0) sms = 132;
  // enough CTAs for >= ~8 waves of one-CTA-per-SM work items, but never fewer than 16 tiles per split
  int splits = (8 * sms + blocks * H - 1) / (blocks * H);
  const int max_splits = tiles_total / 16 > 0 ? tiles_total / 16 : 1;
  if (splits > max_splits) splits = max_splits;
  if (splits < 1) splits = 1;
  return splits;
}

}  // namespace tf

extern "C" {

size_t tf_tree_attn_tc_workspace_bytes(int R, int H, int kv_len_max) {
  using namespace tf;
  if (R <= 0 || H <= 0 || kv_len_max <= 0) return 0;
  const int blocks = (R + kTcBlockRows - 1) / kTcBlockRows;
  const int splits = tc_plan_splits(blocks, H, (kv_len_max + kTcKeys - 1) / kTcKeys);
  const size_t slots = (size_t)blocks * H * splits;
  return slots * kTcBlockRows * (kTcD + 2) * sizeof(float) + 256;
}

// q fp16 [R][H][128] contiguous; out fp16 [R][H][128]; H query heads over H / grp KV heads.  debug_scores: nullable, fp32 [128][128].
// k_exp / v_exp non-NULL: the tensor maps are over the codes of an E4M3 store of `cap` slots (the checks on them are the caller's).
static int tree_attn_tc_impl(const void* q, const void* k_tensormap, const void* v_tensormap, int layer, int kv_len, int R, int H,
                             int grp, int d, float scale, const uint32_t* tree_mask, int tree_cols, int causal, void* out,
                             void* workspace, size_t workspace_bytes, float* debug_scores, tf_stream_t stream_,
                             const int8_t* k_exp = nullptr, const int8_t* v_exp = nullptr, long long cap = 0) {
  using namespace tf;
  cudaStream_t stream = (cudaStream_t)stream_;
  TF_CHECK_ARG(q && k_tensormap && v_tensormap && out && workspace, "tf_tree_attn_tc: NULL pointer");
  TF_CHECK_SUPPORTED(d == kTcD, "tf_tree_attn_tc: head_dim %d (only 128)", d);
  TF_CHECK_ARG(R >= 1 && R <= 65536, "tf_tree_attn_tc: R=%d outside [1,65536]", R);
  TF_CHECK_ARG(causal == 0 || (causal == 1 && tree_cols == 0 && kv_len >= R), "tf_tree_attn_tc: causal mode takes no tree mask and needs kv_len >= R");
  TF_CHECK_ARG(H >= 1 && layer >= 0 && kv_len >= 1, "tf_tree_attn_tc: bad H / layer / kv_len");
  TF_CHECK_ARG(tree_cols >= 0 && tree_cols % 32 == 0 && tree_cols <= kv_len && (tree_cols == 0 || tree_mask != nullptr),
               "tf_tree_attn_tc: tree_cols must be a multiple of 32 within kv_len, with a mask when > 0");
  TF_CHECK_ARG(workspace_bytes >= tf_tree_attn_tc_workspace_bytes(R, H, kv_len) && ((uintptr_t)workspace & 15) == 0, "tf_tree_attn_tc: workspace too small or misaligned");
  TF_CHECK_ARG(((uintptr_t)q & 15) == 0, "tf_tree_attn_tc: q must be 16-byte aligned");
  static PFN_encodeTiledTC encode = nullptr;
  if (!encode) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
    if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || !fn) {
      set_error("cuTensorMapEncodeTiled not available from the driver (%s)", cudaGetErrorString(e));
      return TF_ERR_CUDA;
    }
    encode = (PFN_encodeTiledTC)fn;
  }
  // q [R][H][128] as (d, head, row): box = 64 elements x 1 head x 128 rows → a [128 rows][128 B] half block, SWIZZLE_128B
  CUtensorMap qmap, kmap, vmap;
  {
    cuuint64_t gdim[3] = {(cuuint64_t)d, (cuuint64_t)H, (cuuint64_t)R};
    cuuint64_t gstride[2] = {(cuuint64_t)d * 2, (cuuint64_t)H * d * 2};
    cuuint32_t box[3] = {64, 1, (cuuint32_t)kTcBlockRows};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = encode(&qmap, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, const_cast<void*>(q), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
      set_error("cuTensorMapEncodeTiled (q) failed with CUresult %d", (int)r);
      return TF_ERR_CUDA;
    }
  }
  memcpy(&kmap, k_tensormap, sizeof(kmap));
  memcpy(&vmap, v_tensormap, sizeof(vmap));
  const int blocks = (R + kTcBlockRows - 1) / kTcBlockRows;
  const int tiles_total = (kv_len + kTcKeys - 1) / kTcKeys;
  const int splits = tc_plan_splits(blocks, H, tiles_total);
  TcArgs a;
  a.layer = layer; a.H = H; a.R = R; a.grp = grp; a.kv_len = kv_len; a.tree_cols = tree_cols; a.tree_mask = tree_cols > 0 ? tree_mask : nullptr;
  a.causal = causal;
  a.scale_log2 = scale * 1.4426950408889634f;
  a.splits = splits;
  a.tiles_per_split = (tiles_total + splits - 1) / splits;
  const size_t slots = (size_t)blocks * H * splits;
  a.part_o = (float*)workspace;
  a.part_m = a.part_o + slots * kTcBlockRows * kTcD;
  a.part_l = a.part_m + slots * kTcBlockRows;
  a.debug_s = debug_scores;
  a.k_exp = k_exp;
  a.v_exp = v_exp;
  a.cap = cap;
  if (k_exp != nullptr) {
    const size_t smem = 1024 + (size_t)(1 + kTcSlots) * kTcTileBytes + (size_t)kTcCodeSlots * (kTcCodeBytes + kTcKeys) + 256;
    TF_ENSURE_DYNAMIC_SMEM(tree_attn_tc_kernel<true>, smem);
    tree_attn_tc_kernel<true><<<dim3(blocks, H, splits), kTcThreadsE4m3, smem, stream>>>(qmap, kmap, vmap, a);
  } else {
    const size_t smem = 1024 + (size_t)(1 + kTcSlots) * kTcTileBytes + 256;
    TF_ENSURE_DYNAMIC_SMEM(tree_attn_tc_kernel<false>, smem);
    tree_attn_tc_kernel<false><<<dim3(blocks, H, splits), kTcThreads, smem, stream>>>(qmap, kmap, vmap, a);
  }
  TF_CHECK_LAUNCH();
  tree_attn_merge_kernel<<<dim3(R, H), 128, 0, stream>>>(a.part_o, a.part_m, a.part_l, H, R, splits, (__half*)out);
  TF_CHECK_LAUNCH();
  return TF_OK;
}

int tf_tree_attn_tc(const void* q, const void* k_tensormap, const void* v_tensormap, int layer, int kv_len, int R, int H, int d, float scale,
                    const uint32_t* tree_mask, int tree_cols, int causal, void* out, void* workspace, size_t workspace_bytes,
                    float* debug_scores, tf_stream_t stream) {
  return tree_attn_tc_impl(q, k_tensormap, v_tensormap, layer, kv_len, R, H, 1, d, scale, tree_mask, tree_cols, causal, out, workspace,
                           workspace_bytes, debug_scores, stream);
}

int tf_tree_attn_tc_gqa(const void* q, const void* k_tensormap, const void* v_tensormap, int layer, int kv_len, int R, int Hq, int Hkv,
                        int d, float scale, const uint32_t* tree_mask, int tree_cols, int causal, void* out, void* workspace,
                        size_t workspace_bytes, tf_stream_t stream) {
  if (Hkv <= 0 || Hq <= 0 || Hq % Hkv != 0) {
    tf::set_error("tf_tree_attn_tc_gqa: Hq (%d) must be a positive multiple of Hkv (%d)", Hq, Hkv);
    return TF_ERR_INVALID;
  }
  return tree_attn_tc_impl(q, k_tensormap, v_tensormap, layer, kv_len, R, Hq, Hq / Hkv, d, scale, tree_mask, tree_cols, causal, out,
                           workspace, workspace_bytes, nullptr, stream);
}

// The store arguments of the two E4M3 entries (the converter warpgroup's loads need them; the rest is tree_attn_tc_impl's)
static int tree_attn_tc_e4m3_checks(const char* name, const int8_t* k_exp, const int8_t* v_exp, long long cap, int kv_len, int Hq,
                                    int Hkv) {
  if (Hkv <= 0 || Hq <= 0 || Hq % Hkv != 0) {
    tf::set_error("%s: Hq (%d) must be a positive multiple of Hkv (%d)", name, Hq, Hkv);
    return TF_ERR_INVALID;
  }
  TF_CHECK_ARG(k_exp && v_exp, "%s: NULL exponent pointer", name);
  TF_CHECK_ARG((((uintptr_t)k_exp | (uintptr_t)v_exp) & 15) == 0, "%s: exponents must be 16-byte aligned", name);
  TF_CHECK_ARG(cap > 0 && cap % TF_VERIFY_BOX_KEYS == 0, "%s: cap (%lld) must be a positive multiple of %d", name, cap,
               TF_VERIFY_BOX_KEYS);
  TF_CHECK_ARG(kv_len <= cap, "%s: kv_len (%d) exceeds cap %lld", name, kv_len, cap);
  return TF_OK;
}

int tf_tree_attn_tc_e4m3(const void* q, const void* k_tensormap, const void* v_tensormap, const int8_t* k_exp, const int8_t* v_exp,
                         long long cap, int layer, int kv_len, int R, int Hq, int Hkv, int d, float scale, const uint32_t* tree_mask,
                         int tree_cols, void* out, void* workspace, size_t workspace_bytes, tf_stream_t stream) {
  const int rc = tree_attn_tc_e4m3_checks("tf_tree_attn_tc_e4m3", k_exp, v_exp, cap, kv_len, Hq, Hkv);
  if (rc != TF_OK) return rc;
  return tree_attn_tc_impl(q, k_tensormap, v_tensormap, layer, kv_len, R, Hq, Hq / Hkv, d, scale, tree_mask, tree_cols, 0, out,
                           workspace, workspace_bytes, nullptr, stream, k_exp, v_exp, cap);
}

// The causal tile bound (last_key, and the split's tile count) is computed once per CTA before the roles part, so the converter
// warpgroup loads and converts exactly the tiles the consumers read.
int tf_tree_attn_tc_causal_e4m3(const void* q, const void* k_tensormap, const void* v_tensormap, const int8_t* k_exp,
                                const int8_t* v_exp, long long cap, int layer, int kv_len, int R, int Hq, int Hkv, int d, float scale,
                                void* out, void* workspace, size_t workspace_bytes, tf_stream_t stream) {
  const int rc = tree_attn_tc_e4m3_checks("tf_tree_attn_tc_causal_e4m3", k_exp, v_exp, cap, kv_len, Hq, Hkv);
  if (rc != TF_OK) return rc;
  return tree_attn_tc_impl(q, k_tensormap, v_tensormap, layer, kv_len, R, Hq, Hq / Hkv, d, scale, nullptr, 0, 1, out, workspace,
                           workspace_bytes, nullptr, stream, k_exp, v_exp, cap);
}

}  // extern "C"
