// (iii) Verify attention: R <= 32 query rows (the gamma+1 speculated tokens, or 1 for autoregressive decode) against
// kv_len keys of one layer — the retrieval budget (4K) or the full 128K KV.  Replaces flash_attn_with_kvcache at
// models/modeling_llama.py:240 / tensor_op.py:166-168,316 of the reference.
//
// HBM-bound: every K/V byte is read exactly once; algorithmic bytes per launch = kv_len * H * d * 2 (K+V) * 2 B.
// Design:
//   * stream-K split: the (head, 64-key tile) work units of the launch are laid on one axis and cut into G equal
//     contiguous ranges, G = resident CTA slots (SMs x CTAs/SM) — one wave, perfectly balanced for any kv_len, which is
//     read from device memory so a captured CUDA graph follows kv_cache.seq_len;
//   * a producer warp streams 64x128 fp16 K and V tiles with TMA (cp.async.bulk.tensor, SWIZZLE_128B) into an mbarrier
//     ring; four consumer warps each own a 16-key slice of every tile (or 32 keys x one of two 16-row blocks when
//     R > 16): S = Q K^T with mma.sync m16n8k16 (fp32 accumulate), online softmax in the exp2 domain with quad shuffles,
//     O += P V.  The contraction is only 2*R FLOP per KV byte, far below the tensor roofline — tensor cores are used to
//     keep the FP32 pipe out of the way, not because the problem is compute bound;
//   * per-(CTA, head) partials (m, l, O) go to a small workspace; the LAST CTA to deliver a partial of a head (an
//     arrival counter per head, self-resetting) merges that head's <= G/H + 2 partials — no second launch;
//   * grouped-query attention (tf_verify_attn_gqa: Hq query heads over Hkv KV heads, group size grp = Hq / Hkv, query
//     head h reads KV head h / grp): the work units are (KV head, tile) and a CTA computes the R * grp packed rows of
//     all query heads of a group against every tile it loads, so each K/V byte is still read once per launch.
//     "Head" below means KV head; MHA is grp = 1 and runs the same code.
//   * an E4M3 store (tf_verify_attn_e4m3, the format of common.cuh): the same kernel with KV = __nv_fp8_e4m3.  A stage carries
//     the 64-key code tiles (TMA) and the tiles' 64 + 64 exponents (bulk copy); twice the stages keep the fp16 ring's bytes in
//     flight.  No calibrated split, L2 prefetch or tree mode.  Over an E4M3 retrieval cache (tf_verify_attn_e4m3_clean) the
//     producer fills the ring with code tiles and exponents of the clean region before pdl_wait, as the fp16 kernel does.
//   * the split is equal by default.  SMs need not all pull the same HBM bandwidth (GPC-level sharing; per-CTA
//     %globaltimer stamps show it, tools/attn_timing.py), so under an equal split the kernel waits on the slowest GPCs.
//     tf_verify_attn_calibrate
//     measures the per-CTA streaming time of this very kernel and stores a cumulative split table (fractions of the tile
//     axis per blockIdx) in the workspace; launches with the same grid then cut the axis in proportion to the measured
//     per-CTA rate.  The table only moves segment boundaries: per-(CTA, head) partials and their merge order stay a pure
//     function of (table, kv_len), so results are deterministic for a given table.
// Numerics follow FlashAttention-2: fp16 operands, fp32 scores/softmax/accumulators, P rounded to fp16 for the PV MMA.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include <cuda_fp8.h>

#include "common.cuh"

namespace tf {

constexpr int BN = TF_VERIFY_BOX_KEYS;  // keys per pipeline stage
constexpr int kConsumerWarps = 4;
constexpr int kThreadsAttn = (kConsumerWarps + 1) * 32;
constexpr float kLog2e = 1.4426950408889634f;

__device__ __forceinline__ void ldmatrix_x4(uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3, uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}
__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3, uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}
__device__ __forceinline__ void mma_16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t pack_half2(float lo, float hi) {
  __half2 h = __floats2half2_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&h);
}
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

#ifdef TF_ATTN_TIMING
// Profiling build only (TF_EXTRA_NVCC_FLAGS=-DTF_ATTN_TIMING): thread 0 of every CTA stamps %globaltimer at the phase
// boundaries of the kernel into g_attn_timing[blockIdx.x][8]; tools/attn_timing.py reads them.
__device__ unsigned long long* g_attn_timing = nullptr;
__device__ __forceinline__ void stamp(int slot) {
  if (g_attn_timing != nullptr && threadIdx.x == 0) {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    g_attn_timing[(size_t)blockIdx.x * 8 + slot] = t;
  }
}
#define TF_STAMP(slot) stamp(slot)
#else
#define TF_STAMP(slot)
#endif

struct SplitInfo {
  uint32_t tph;    // tiles per head
  uint32_t total;  // H * tph
};
// first tile of CTA b: equal split, or the calibrated cumulative table (u32 fixed-point fractions, tab[0] == 0)
__device__ __forceinline__ uint32_t split_start(uint32_t b, uint32_t total, uint32_t G, const uint32_t* __restrict__ tab) {
  if (b >= G) return total;
  if (tab != nullptr) return (uint32_t)(((uint64_t)__ldg(tab + b) * total) >> 32);
  return (uint32_t)(((uint64_t)b * total) / G);
}
__device__ __forceinline__ unsigned long long global_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
constexpr int kSplitHdr = 4;  // u32 header words of a split table: {G the table was calibrated for, 0, 0, 0}

struct AttnSmemLayout {
  // dynamic shared memory: [STAGES][K tile | V tile] (1024-aligned) | e4m3 only: [STAGES][K exponents | V exponents] |
  // Osh | msh | lsh | barriers
  static __host__ __device__ size_t tile_bytes(int D, int eb) { return (size_t)BN * D * eb; }
  static __host__ __device__ size_t exp_bytes(int eb) { return eb == 1 ? (size_t)2 * BN : 0; }
  static __host__ __device__ size_t bytes(int D, int MT, int stages, int eb) {
    return 1024 /*align slack*/ + (size_t)stages * (2 * tile_bytes(D, eb) + exp_bytes(eb)) + (size_t)16 * MT * D * 4 + 2 * 4 * 32 * 4 +
           2 * 8 * stages + 64;
  }
};

__device__ __forceinline__ uint32_t lds32(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr));
  return v;
}
__device__ __forceinline__ uint32_t prmt(uint32_t a, uint32_t b, uint32_t sel) {
  uint32_t r;
  asm("prmt.b32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(sel));
  return r;
}
__device__ __forceinline__ uint32_t h2u(__half2 h) { return *reinterpret_cast<uint32_t*>(&h); }

constexpr int kPfChunk = 4096;  // bytes per L2 prefetch request (tf_verify_attn_prefetch)

// KV = __half: the fp16 store.  KV = __nv_fp8_e4m3: the E4M3 store of common.cuh, codes through kmap / vmap and exponents
// [layer][H][cap] in k_exp / v_exp.  sm_90 has no 8-bit ldmatrix, so the e4m3 fragments are built from 32-bit shared loads:
//   K: a thread's word holds d elements 4tq..4tq+3 of one key and stands for the mma's k positions {2tq, 2tq+1, 2tq+8, 2tq+9};
//      the Q fragment is loaded in the same order, so the dot product is unchanged.  K exponents scale the score columns:
//      (q·code)·2^e equals q·D unless D itself rounds (e < -15, or a ±65504 row whose D is ±inf; see the header).
//   V: words of key rows (k, k+1) are interleaved byte-wise (prmt) into e4m3 pairs along the mma's k axis; a thread's word holds
//      4 d columns, so n-block 4j+i carries columns 32j + 4n + i at mma column n, and O is written back in that order.  V is
//      dequantized exactly to D (kv_e4m3_apply) before the PV mma.
template <typename KV, int D, int MT, int STAGES>
__global__ void __launch_bounds__(kThreadsAttn, (MT == 1 ? 2 : 1)) verify_attn_mma_kernel(
    const __grid_constant__ CUtensorMap kmap, const __grid_constant__ CUtensorMap vmap, const __half* __restrict__ q,
    int layer, int kv_len_host, const int32_t* __restrict__ kv_len_dev, int R, int H, int grp, float scale_log2,
    float* __restrict__ part_m, float* __restrict__ part_l, float* __restrict__ part_o, int* __restrict__ head_counters,
    __half* __restrict__ out, const uint32_t* __restrict__ tree_mask, int tree_cols,
    const uint32_t* __restrict__ split_table, uint32_t* __restrict__ cta_ns, int clean_keys, const uint8_t* __restrict__ pf_ptr,
    uint32_t pf_chunks, const int8_t* __restrict__ k_exp, const int8_t* __restrict__ v_exp, long long cap) {
  constexpr bool kE4m3 = sizeof(KV) == 1;
  constexpr int NKW = kConsumerWarps / MT;  // warps along the key axis
  constexpr int KW = BN / NKW;              // keys per warp per tile (16 or 32)
  constexpr int NB = KW / 8;                // score n-blocks per warp
  constexpr int KS = KW / 16;               // PV k-steps per warp
  constexpr int DK = D / 16;                // QK k-steps
  constexpr int DN = D / 8;                 // output n-blocks
  constexpr int SUBS = D / 64;              // 64-element (128 B) swizzle spans per row
  constexpr uint32_t TILE_BYTES = BN * D * sizeof(KV);
  constexpr uint32_t SUB_BYTES = BN * 128;
  constexpr uint32_t EXP_BYTES = kE4m3 ? 2 * BN : 0;  // per stage: K then V exponents of the tile's keys
  constexpr uint32_t ROW_BYTES = D * sizeof(KV);

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* tiles = smem;
  int8_t* exps = reinterpret_cast<int8_t*>(tiles + (size_t)STAGES * 2 * TILE_BYTES);
  float* Osh = reinterpret_cast<float*>(tiles + (size_t)STAGES * (2 * TILE_BYTES + EXP_BYTES));  // [16*MT][D]
  float* msh = Osh + 16 * MT * D;                                                 // [NKW][16*MT]  (<= 4*32)
  float* lsh = msh + 4 * 32;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(lsh + 4 * 32);
  uint64_t* empty_bar = full_bar + STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t b = blockIdx.x;
  // Programmatic dependent launch: the next kernel may start.  Nothing the previous kernel wrote (q, the new K/V rows,
  // kv_len_dev) is touched before pdl_wait().  With a host-side length and `clean_keys` > 0 — keys [0, clean_keys) are NOT
  // written by the predecessor (the retrieval budget below the gamma+1 fresh slots) — the producer lane fills its ring
  // with tiles of that region BEFORE the dependency resolves, so the stream is already running when q arrives.
  pdl_launch_dependents();
  if (threadIdx.x == 0) {
    prefetch_tensormap(&kmap);
    prefetch_tensormap(&vmap);
  }
  const bool early = kv_len_dev == nullptr && clean_keys >= BN;
  if (!early) pdl_wait();
  TF_STAMP(0);
#ifdef TF_ATTN_TIMING
  if (g_attn_timing != nullptr && threadIdx.x == 0) {
    unsigned int smid;
    asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
    g_attn_timing[(size_t)blockIdx.x * 8 + 6] = smid;
  }
#endif
  const int kv_len = kv_len_host + (kv_len_dev ? *kv_len_dev : 0);
  const uint32_t tph = kv_len > 0 ? (uint32_t)((kv_len + BN - 1) / BN) : 0u;
  const uint32_t total = tph * (uint32_t)H;
  const uint32_t G = min(gridDim.x, total);  // effective split: every participating CTA owns >= 1 tile
  if (b >= G) return;
  // calibrated split: only for the grid it was measured on, and only when every CTA still owns tiles (weights are
  // clamped to [1/2, 2] x equal by tf_verify_attn_calibrate, so total >= 4 G keeps begin strictly increasing)
  const uint32_t* tab = nullptr;
  if (split_table != nullptr && G == gridDim.x && total >= 4u * G && __ldg(split_table) == G) tab = split_table + kSplitHdr;
  const uint32_t begin = split_start(b, total, G, tab), end = split_start(b + 1, total, G, tab);
  __shared__ int s_is_last, s_bfirst, s_blast;
  const unsigned long long t_entry = cta_ns != nullptr ? global_ns() : 0ull;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], kConsumerWarps); }
    fence_mbar_init();
  }
  __syncthreads();
  if (begin >= end) return;

  if (warp == kConsumerWarps) {
    // ================= producer warp: one elected lane issues the TMA loads =================
    if (lane == 0) {
      uint32_t it = 0;
      uint32_t gt = begin;
      auto issue = [&](uint32_t gt_, uint32_t s) {
        const int h = (int)(gt_ / tph);
        const int key0 = (int)(gt_ % tph) * BN;
        mbar_expect_tx(&full_bar[s], 2 * TILE_BYTES + EXP_BYTES);
        uint8_t* kt = tiles + (size_t)s * 2 * TILE_BYTES;
        uint8_t* vt = kt + TILE_BYTES;
        if constexpr (kE4m3) {
          tma_load_4d(kt, &kmap, &full_bar[s], 0, key0, h, layer);
          tma_load_4d(vt, &vmap, &full_bar[s], 0, key0, h, layer);
          const size_t e0 = ((size_t)layer * H + h) * (size_t)cap + key0;
          bulk_load(exps + (size_t)s * EXP_BYTES, k_exp + e0, BN, &full_bar[s]);
          bulk_load(exps + (size_t)s * EXP_BYTES + BN, v_exp + e0, BN, &full_bar[s]);
        } else {
#pragma unroll
          for (int sub = 0; sub < SUBS; ++sub) {
            tma_load_4d(kt + sub * SUB_BYTES, &kmap, &full_bar[s], sub * 64, key0, h, layer);
            tma_load_4d(vt + sub * SUB_BYTES, &vmap, &full_bar[s], sub * 64, key0, h, layer);
          }
        }
      };
      // L2 prefetch of the weights the NEXT kernel streams (o_proj after a short-store attention, which is latency-bound and
      // leaves HBM idle): chunk c of kPfChunk bytes belongs to CTA c % gridDim.x, which issues its chunks a few per tile so that
      // they queue BEHIND its own K/V loads.  Weights are constants, so this needs no ordering against pdl_wait.
      uint32_t pf_next = b;
      const uint32_t pf_mine = pf_ptr != nullptr && pf_chunks > b ? (pf_chunks - b + gridDim.x - 1) / gridDim.x : 0u;
      const uint32_t pf_per_tile = pf_mine ? (pf_mine + (end - begin) - 1) / (end - begin) : 0u;
      auto pf_step = [&]() {
        for (uint32_t k = 0; k < pf_per_tile && pf_next < pf_chunks; ++k, pf_next += gridDim.x)
          asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(pf_ptr + (size_t)pf_next * kPfChunk), "n"(kPfChunk) : "memory");
      };
      if (early) {
        // the first ring-full, as long as the tiles lie entirely inside the clean region (all stages are still free)
        for (; gt < end && it < (uint32_t)STAGES; ++gt, ++it) {
          if ((int)((gt % tph) + 1) * BN > clean_keys) break;
          issue(gt, it);
          pf_step();
        }
        pdl_wait();
      }
      for (; gt < end; ++gt, ++it) {
        const uint32_t s = it % STAGES, ph = (it / STAGES) & 1u;
        mbar_wait(&empty_bar[s], ph ^ 1u);
        issue(gt, s);
        pf_step();
      }
    }
    return;
  }

  // ================= consumer warps =================
  if (early) pdl_wait();  // q (and the fresh K/V rows the last tiles carry) come from the predecessor
  const int g = lane >> 2, tq = lane & 3;
  const int mtile = warp % MT, kslice = warp / MT;
  const int row0 = mtile * 16 + g, row1 = row0 + 8;  // packed query rows owned by this thread
  // Packed row i is token row i / grp of query head h * grp + i % grp (grp = 1: MHA, packed row = token row).
  const int rows = R * grp, Hq = H * grp;
  const int tr0 = row0 / grp, tr1 = row1 / grp;
  const int kbase = kslice * KW;

  uint32_t it = 0;
  uint32_t gt = begin;
  while (gt < end) {
    const int h = (int)(gt / tph);
    const uint32_t t0 = gt % tph;
    const uint32_t t1 = min(tph, t0 + (end - gt));

    // ---- Q fragments of this head (A operand, rows >= R are zero) ----
    uint32_t qa[DK][4];
    {
      const __half* q0 = q + ((size_t)tr0 * Hq + h * grp + row0 % grp) * D;
      const __half* q1 = q + ((size_t)tr1 * Hq + h * grp + row1 % grp) * D;
#pragma unroll
      for (int kk = 0; kk < DK; ++kk) {
        // mma k positions (2tq, 2tq+1 | 2tq+8, 2tq+9) hold d (c, c+1 | c2, c2+1): in order, or as the e4m3 K word lays them out
        const int c = kk * 16 + (kE4m3 ? 4 * tq : 2 * tq);
        const int c2 = kE4m3 ? c + 2 : c + 8;
        qa[kk][0] = row0 < rows ? *reinterpret_cast<const uint32_t*>(q0 + c) : 0u;
        qa[kk][1] = row1 < rows ? *reinterpret_cast<const uint32_t*>(q1 + c) : 0u;
        qa[kk][2] = row0 < rows ? *reinterpret_cast<const uint32_t*>(q0 + c2) : 0u;
        qa[kk][3] = row1 < rows ? *reinterpret_cast<const uint32_t*>(q1 + c2) : 0u;
      }
    }
    // ---- which CTAs deliver partials of head h: the owners of its first and last tile ----
    const uint32_t lo_t = (uint32_t)h * tph, hi_t = lo_t + tph;
    if (tab != nullptr) {
      for (uint32_t c = threadIdx.x; c < G; c += kConsumerWarps * 32) {
        const uint32_t cs = split_start(c, total, G, tab), ce = split_start(c + 1, total, G, tab);
        if (cs <= lo_t && lo_t < ce) s_bfirst = (int)c;
        if (cs <= hi_t - 1 && hi_t - 1 < ce) s_blast = (int)c;
      }
    } else if (threadIdx.x == 0) {
      s_bfirst = (int)((((uint64_t)lo_t + 1) * G - 1) / total);
      s_blast = (int)(((uint64_t)hi_t * G - 1) / total);
    }
    float o[DN][4];
#pragma unroll
    for (int n = 0; n < DN; ++n) { o[n][0] = o[n][1] = o[n][2] = o[n][3] = 0.f; }
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;

    for (uint32_t t = t0; t < t1; ++t, ++it) {
      const uint32_t s = it % STAGES, ph = (it / STAGES) & 1u;
      mbar_wait(&full_bar[s], ph);
      if (it == 0) TF_STAMP(1);
      const uint32_t kt = smem_u32(tiles + (size_t)s * 2 * TILE_BYTES);
      const uint32_t vt = kt + TILE_BYTES;
      const int8_t* kx = exps + (size_t)s * EXP_BYTES;  // e4m3: exponents of the tile's keys
      const int8_t* vx = kx + BN;
      // byte offset of 16-byte chunk `chunk` of e4m3 key row `row` (SWIZZLE_128B rows of 128 B, SWIZZLE_64B rows of 64 B)
      auto e4m3_chunk = [&](int row, int chunk) -> uint32_t {
        return (uint32_t)(row * ROW_BYTES + ((chunk ^ (D == 128 ? (row & 7) : ((row >> 1) & 3))) << 4));
      };

      // ---- S = Q K^T for this warp's KW keys ----
      float sc[NB][4];
#pragma unroll
      for (int n = 0; n < NB; ++n) { sc[n][0] = sc[n][1] = sc[n][2] = sc[n][3] = 0.f; }
#pragma unroll
      for (int kk = 0; kk < DK; ++kk) {
        if constexpr (kE4m3) {
#pragma unroll
          for (int n = 0; n < NB; ++n) {
            const uint32_t w = lds32(kt + e4m3_chunk(kbase + n * 8 + g, kk) + 4 * tq);
            mma_16816(sc[n], qa[kk], h2u(kv_e4m3_codes2((uint16_t)(w & 0xffffu))), h2u(kv_e4m3_codes2((uint16_t)(w >> 16))));
          }
        } else {
#pragma unroll
          for (int np = 0; np < NB / 2; ++np) {
            const int mat = lane >> 3;
            const int krow = kbase + (np * 2 + (mat >> 1)) * 8 + (lane & 7);
            const int chunk = 2 * kk + (mat & 1);
            const uint32_t addr = kt + (chunk >> 3) * SUB_BYTES + krow * 128 + (((chunk & 7) ^ (krow & 7)) << 4);
            uint32_t b0, b1, b2, b3;
            ldmatrix_x4(b0, b1, b2, b3, addr);
            mma_16816(sc[np * 2], qa[kk], b0, b1);
            mma_16816(sc[np * 2 + 1], qa[kk], b2, b3);
          }
        }
      }
      if constexpr (kE4m3) {  // score column j = (q . code_j) * 2^e_j
#pragma unroll
        for (int n = 0; n < NB; ++n) {
          const int j = kbase + n * 8 + 2 * tq;
          const float s0 = kv_e4m3_pow2(kx[j]), s1 = kv_e4m3_pow2(kx[j + 1]);
          sc[n][0] *= s0; sc[n][2] *= s0;
          sc[n][1] *= s1; sc[n][3] *= s1;
        }
      }

      // ---- mask.  Causal (bottom-right): token row r sees key j iff j <= kv_len - R + r.  Tree (Sequoia) mode: the first
      //      kv_len - T keys are visible to every row, the last T columns follow the token row's bitmask (ancestors of the
      //      node).  Both take the TOKEN row of a packed row, never the packed row. ----
      const int key_tile0 = (int)t * BN + kbase;
      if (tree_mask == nullptr) {
        if (key_tile0 + KW - 1 > kv_len - R) {
          const int lim0 = kv_len - R + tr0, lim1 = kv_len - R + tr1;
#pragma unroll
          for (int n = 0; n < NB; ++n) {
            const int j = key_tile0 + n * 8 + 2 * tq;
            if (j > lim0) sc[n][0] = -INFINITY;
            if (j + 1 > lim0) sc[n][1] = -INFINITY;
            if (j > lim1) sc[n][2] = -INFINITY;
            if (j + 1 > lim1) sc[n][3] = -INFINITY;
          }
        }
      } else {
        const int prefix = kv_len - tree_cols;
        if (key_tile0 + KW - 1 >= prefix) {
          const int words = tree_cols >> 5;
          const uint32_t* m0p = tree_mask + (size_t)min(tr0, R - 1) * words;
          const uint32_t* m1p = tree_mask + (size_t)min(tr1, R - 1) * words;
#pragma unroll
          for (int n = 0; n < NB; ++n) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int j = key_tile0 + n * 8 + 2 * tq + e;
              const int c = j - prefix;
              bool v0 = true, v1 = true;
              if (j >= kv_len) { v0 = v1 = false; }
              else if (c >= 0) {
                v0 = (__ldg(m0p + (c >> 5)) >> (c & 31)) & 1u;
                v1 = (__ldg(m1p + (c >> 5)) >> (c & 31)) & 1u;
              }
              if (!v0) sc[n][e] = -INFINITY;
              if (!v1) sc[n][2 + e] = -INFINITY;
            }
          }
        }
      }

      // ---- online softmax (exp2 domain) ----
      float tm0 = -INFINITY, tm1 = -INFINITY;
#pragma unroll
      for (int n = 0; n < NB; ++n) {
        tm0 = fmaxf(tm0, fmaxf(sc[n][0], sc[n][1]));
        tm1 = fmaxf(tm1, fmaxf(sc[n][2], sc[n][3]));
      }
      tm0 = fmaxf(tm0, __shfl_xor_sync(0xffffffffu, tm0, 1));
      tm0 = fmaxf(tm0, __shfl_xor_sync(0xffffffffu, tm0, 2));
      tm1 = fmaxf(tm1, __shfl_xor_sync(0xffffffffu, tm1, 1));
      tm1 = fmaxf(tm1, __shfl_xor_sync(0xffffffffu, tm1, 2));
      const float mn0 = fmaxf(m0, tm0), mn1 = fmaxf(m1, tm1);
      const float mu0 = (mn0 == -INFINITY) ? 0.f : mn0 * scale_log2;
      const float mu1 = (mn1 == -INFINITY) ? 0.f : mn1 * scale_log2;
      const bool grew = (mn0 > m0) || (mn1 > m1);
      if (__any_sync(0xffffffffu, grew)) {
        const float a0 = exp2f(m0 * scale_log2 - mu0), a1 = exp2f(m1 * scale_log2 - mu1);
        l0 *= a0;
        l1 *= a1;
#pragma unroll
        for (int n = 0; n < DN; ++n) { o[n][0] *= a0; o[n][1] *= a0; o[n][2] *= a1; o[n][3] *= a1; }
      }
      m0 = mn0;
      m1 = mn1;
      uint32_t pa[KS][4];
#pragma unroll
      for (int n = 0; n < NB; ++n) {
        const float p0 = exp2f(fmaf(sc[n][0], scale_log2, -mu0));
        const float p1 = exp2f(fmaf(sc[n][1], scale_log2, -mu0));
        const float p2 = exp2f(fmaf(sc[n][2], scale_log2, -mu1));
        const float p3 = exp2f(fmaf(sc[n][3], scale_log2, -mu1));
        l0 += p0 + p1;
        l1 += p2 + p3;
        pa[n >> 1][(n & 1) * 2 + 0] = pack_half2(p0, p1);
        pa[n >> 1][(n & 1) * 2 + 1] = pack_half2(p2, p3);
      }

      // ---- O += P V ----
#pragma unroll
      for (int ks = 0; ks < KS; ++ks) {
        if constexpr (kE4m3) {
          // b0 = keys (k, k+1), b1 = keys (k+8, k+9) of column 32j + 4g + i, scaled per key to D
          const int k = kbase + ks * 16 + 2 * tq;
          __half a0, a1, a8, a9, m0_, m1_, m8_, m9_;
          kv_e4m3_factors(vx[k], a0, m0_);
          kv_e4m3_factors(vx[k + 1], a1, m1_);
          kv_e4m3_factors(vx[k + 8], a8, m8_);
          kv_e4m3_factors(vx[k + 9], a9, m9_);
          const __half2 fa0 = __halves2half2(a0, a1), fb0 = __halves2half2(m0_, m1_);
          const __half2 fa1 = __halves2half2(a8, a9), fb1 = __halves2half2(m8_, m9_);
#pragma unroll
          for (int j = 0; j < DN / 4; ++j) {
            const int chunk = 2 * j + (g >> 2), off = (g & 3) * 4;
            const uint32_t w0 = lds32(vt + e4m3_chunk(k, chunk) + off), w1 = lds32(vt + e4m3_chunk(k + 1, chunk) + off);
            const uint32_t w8 = lds32(vt + e4m3_chunk(k + 8, chunk) + off), w9 = lds32(vt + e4m3_chunk(k + 9, chunk) + off);
            const uint32_t lo01 = prmt(w0, w1, 0x5140), hi01 = prmt(w0, w1, 0x7362);
            const uint32_t lo89 = prmt(w8, w9, 0x5140), hi89 = prmt(w8, w9, 0x7362);
            const uint32_t p0[4] = {lo01 & 0xffffu, lo01 >> 16, hi01 & 0xffffu, hi01 >> 16};
            const uint32_t p8[4] = {lo89 & 0xffffu, lo89 >> 16, hi89 & 0xffffu, hi89 >> 16};
#pragma unroll
            for (int i = 0; i < 4; ++i)
              mma_16816(o[4 * j + i], pa[ks], h2u(kv_e4m3_apply(kv_e4m3_codes2((uint16_t)p0[i]), fa0, fb0)),
                        h2u(kv_e4m3_apply(kv_e4m3_codes2((uint16_t)p8[i]), fa1, fb1)));
          }
        } else {
#pragma unroll
          for (int nd = 0; nd < DN; nd += 2) {
            const int mat = lane >> 3;
            const int krow = kbase + ks * 16 + (mat & 1) * 8 + (lane & 7);
            const int chunk = nd + (mat >> 1);
            const uint32_t addr = vt + (chunk >> 3) * SUB_BYTES + krow * 128 + (((chunk & 7) ^ (krow & 7)) << 4);
            uint32_t b0, b1, b2, b3;
            ldmatrix_x4_trans(b0, b1, b2, b3, addr);
            mma_16816(o[nd], pa[ks], b0, b1);
            mma_16816(o[nd + 1], pa[ks], b2, b3);
          }
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[s]);
    }

    if (cta_ns != nullptr && threadIdx.x == 0 && t1 - t0 == end - gt) cta_ns[b] = (uint32_t)(global_ns() - t_entry);
    // ---- merge the warps of this CTA and write the (CTA, head) partial ----
    TF_STAMP(2);
    l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
    l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
    if (tq == 0) {
      msh[kslice * 16 * MT + row0] = m0;
      msh[kslice * 16 * MT + row1] = m1;
      lsh[kslice * 16 * MT + row0] = l0;
      lsh[kslice * 16 * MT + row1] = l1;
    }
    named_bar_sync(1, kConsumerWarps * 32);
    float mc0 = -INFINITY, mc1 = -INFINITY;
#pragma unroll
    for (int w = 0; w < NKW; ++w) {
      mc0 = fmaxf(mc0, msh[w * 16 * MT + row0]);
      mc1 = fmaxf(mc1, msh[w * 16 * MT + row1]);
    }
    const float mcu0 = (mc0 == -INFINITY) ? 0.f : mc0 * scale_log2;
    const float mcu1 = (mc1 == -INFINITY) ? 0.f : mc1 * scale_log2;
    {
      // deterministic merge: the key-slice warps add their rescaled accumulators in slice order (no atomics)
      const float a0 = exp2f(m0 * scale_log2 - mcu0), a1 = exp2f(m1 * scale_log2 - mcu1);
#pragma unroll 1
      for (int w = 0; w < NKW; ++w) {
        if (kslice == w) {
#pragma unroll
          for (int n = 0; n < DN; ++n) {
            if constexpr (kE4m3) {  // mma columns (2tq, 2tq+1) of n-block n are d columns c and c + 4
              const int c = 32 * (n >> 2) + 8 * tq + (n & 3);
              float* p0 = Osh + row0 * D + c;
              float* p1 = Osh + row1 * D + c;
              const float v00 = o[n][0] * a0, v01 = o[n][1] * a0, v10 = o[n][2] * a1, v11 = o[n][3] * a1;
              p0[0] = w > 0 ? p0[0] + v00 : v00;
              p0[4] = w > 0 ? p0[4] + v01 : v01;
              p1[0] = w > 0 ? p1[0] + v10 : v10;
              p1[4] = w > 0 ? p1[4] + v11 : v11;
            } else {
              const int c = n * 8 + 2 * tq;
              float2* p0 = reinterpret_cast<float2*>(&Osh[row0 * D + c]);
              float2* p1 = reinterpret_cast<float2*>(&Osh[row1 * D + c]);
              float2 v0 = make_float2(o[n][0] * a0, o[n][1] * a0), v1 = make_float2(o[n][2] * a1, o[n][3] * a1);
              if (w > 0) {
                const float2 u0 = *p0, u1 = *p1;
                v0.x += u0.x; v0.y += u0.y; v1.x += u1.x; v1.y += u1.y;
              }
              *p0 = v0;
              *p1 = v1;
            }
          }
        }
        named_bar_sync(1, kConsumerWarps * 32);
      }
    }
    const size_t slot = (size_t)b + (size_t)h;
    for (int i = threadIdx.x; i < rows * D; i += kConsumerWarps * 32) part_o[slot * (size_t)(TF_VERIFY_MAX_ROWS * D) + i] = Osh[i];
    for (int r = threadIdx.x; r < rows; r += kConsumerWarps * 32) {
      float mc = -INFINITY;
      for (int w = 0; w < NKW; ++w) mc = fmaxf(mc, msh[w * 16 * MT + r]);
      const float mcu = (mc == -INFINITY) ? 0.f : mc * scale_log2;
      float lc = 0.f;
      for (int w = 0; w < NKW; ++w) lc += lsh[w * 16 * MT + r] * exp2f(msh[w * 16 * MT + r] * scale_log2 - mcu);
      part_m[slot * TF_VERIFY_MAX_ROWS + r] = mc;
      part_l[slot * TF_VERIFY_MAX_ROWS + r] = lc;
    }
    // ---- fused combine: the LAST CTA to deliver a partial of head h merges all of them (no second launch).
    //      Publication = CTA barrier (orders every consumer thread's partial stores before thread 0) + ONE acq_rel
    //      gpu-scope atomic by thread 0 (release is cumulative over what the barrier ordered; the last arriver's acquire
    //      plus the barrier below makes all partials of the head visible to its threads). ----
    named_bar_sync(1, kConsumerWarps * 32);
    const uint32_t b_first = (uint32_t)s_bfirst, b_last = (uint32_t)s_blast;
    if (threadIdx.x == 0) {
      int prev;
      asm volatile("atom.acq_rel.gpu.global.add.s32 %0, [%1], 1;" : "=r"(prev) : "l"(head_counters + h) : "memory");
      const int last = (prev == (int)(b_last - b_first));
      if (last) head_counters[h] = 0;  // self-cleaning: ready for the next launch / graph replay
      s_is_last = last;
    }
    TF_STAMP(3);
    named_bar_sync(1, kConsumerWarps * 32);
    if (s_is_last) {
      TF_STAMP(5);
      // Every thread merges the P partials of its own outputs online (running max / denominator per row, fixed order
      // p = 0..P-1): no shared memory, no barriers, and all loads of a batch are independent (one L2 round trip each).
      const int P = (int)(b_last - b_first) + 1;
      constexpr int F4R = D / 4;                                      // float4 per output row
      constexpr int KF = (16 * MT * F4R) / (kConsumerWarps * 32);     // float4 outputs per thread
      constexpr int PB = MT == 1 ? 4 : 2;                             // partials per batch
      // Head-sharded long stores leave one head dozens of partials (4 heads on 296 CTAs: 74).  With R <= 8 rows the upper half of a
      // thread's output slots is idle (rows 8..15), so it runs a SECOND independent partial stream there: twice the loads in flight,
      // half the dependent L2 round trips; the two streams are merged at the end.  Only for P > 16, i.e. never on unsharded or
      // parity-sized launches, whose merge order stays exactly as it was.
      const bool dual = (KF == 4) && (MT == 1) && (rows <= 8) && (P > 16);
      const int pstep = dual ? 2 * PB : PB;
      float4 acc[KF];
      float mr[KF], den[KF];
#pragma unroll
      for (int k = 0; k < KF; ++k) { acc[k] = make_float4(0.f, 0.f, 0.f, 0.f); mr[k] = -INFINITY; den[k] = 0.f; }
      for (int p0 = 0; p0 < P; p0 += pstep) {
        float4 v[PB][KF];
        float pm_[PB][KF], pl_[PB][KF];
#pragma unroll
        for (int pp = 0; pp < PB; ++pp) {
#pragma unroll
          for (int k = 0; k < KF; ++k) {
            const int kk = dual ? (k & 1) : k;
            const int pidx = p0 + pp + (dual ? (k >> 1) * PB : 0);
            const int f = threadIdx.x + kk * (kConsumerWarps * 32);
            const int r = f / F4R;
            const bool ok = (pidx < P) && (r < rows);
            const size_t sl = (size_t)b_first + (size_t)(ok ? pidx : 0) + (size_t)h;
            v[pp][k] = ok ? __ldcg(reinterpret_cast<const float4*>(part_o + sl * (size_t)(TF_VERIFY_MAX_ROWS * D)) + f) : make_float4(0.f, 0.f, 0.f, 0.f);
            pm_[pp][k] = ok ? __ldcg(&part_m[sl * TF_VERIFY_MAX_ROWS + r]) : -INFINITY;
            pl_[pp][k] = ok ? __ldcg(&part_l[sl * TF_VERIFY_MAX_ROWS + r]) : 0.f;
          }
        }
#pragma unroll
        for (int pp = 0; pp < PB; ++pp) {
#pragma unroll
          for (int k = 0; k < KF; ++k) {
            const float mn = fmaxf(mr[k], pm_[pp][k]);
            const float mnu = (mn == -INFINITY) ? 0.f : mn * scale_log2;
            const float a = exp2f(mr[k] * scale_log2 - mnu), w = exp2f(pm_[pp][k] * scale_log2 - mnu);
            acc[k].x = fmaf(w, v[pp][k].x, acc[k].x * a);
            acc[k].y = fmaf(w, v[pp][k].y, acc[k].y * a);
            acc[k].z = fmaf(w, v[pp][k].z, acc[k].z * a);
            acc[k].w = fmaf(w, v[pp][k].w, acc[k].w * a);
            den[k] = fmaf(w, pl_[pp][k], den[k] * a);
            mr[k] = mn;
          }
        }
      }
      if (dual) {  // fold stream B (slots 2, 3) into stream A (slots 0, 1)
#pragma unroll
        for (int k = 0; k < KF / 2; ++k) {
          const int kb = k + KF / 2;
          const float mn = fmaxf(mr[k], mr[kb]);
          const float mnu = (mn == -INFINITY) ? 0.f : mn * scale_log2;
          const float a = exp2f(mr[k] * scale_log2 - mnu), w = exp2f(mr[kb] * scale_log2 - mnu);
          acc[k].x = fmaf(w, acc[kb].x, acc[k].x * a);
          acc[k].y = fmaf(w, acc[kb].y, acc[k].y * a);
          acc[k].z = fmaf(w, acc[kb].z, acc[k].z * a);
          acc[k].w = fmaf(w, acc[kb].w, acc[k].w * a);
          den[k] = fmaf(w, den[kb], den[k] * a);
          mr[k] = mn;
        }
      }
#pragma unroll
      for (int k = 0; k < KF; ++k) {
        if (dual && k >= KF / 2) continue;
        const int f = threadIdx.x + k * (kConsumerWarps * 32);
        const int r = f / F4R, c4 = f % F4R;
        if (r < rows) {
          const float inv = 1.f / den[k];
          uint2 pk;
          pk.x = pack_half2(acc[k].x * inv, acc[k].y * inv);
          pk.y = pack_half2(acc[k].z * inv, acc[k].w * inv);
          *reinterpret_cast<uint2*>(out + ((size_t)(r / grp) * Hq + h * grp + r % grp) * D + c4 * 4) = pk;
        }
      }
    }
    TF_STAMP(4);
    named_bar_sync(1, kConsumerWarps * 32);  // Osh/msh/lsh/s_is_last are reused by the next segment
    gt += (t1 - t0);
  }
}

static int g_max_slots() {
  int sms = sm_count();
  if (sms <= 0) sms = 132;
  return sms * 2;
}

template <typename KV, int D, int MT, int STAGES>
static int launch_mma(const CUtensorMap& kmap, const CUtensorMap& vmap, const __half* q, int layer, int kv_len_host,
                      const int32_t* kv_len_dev, int R, int H, int grp, float scale_log2, float* pm, float* pl, float* po, int* counters,
                      __half* out, int G, const uint32_t* tree_mask, int tree_cols, const uint32_t* split_table, uint32_t* cta_ns,
                      int clean_keys, bool allow_pdl, cudaStream_t stream, const uint8_t* pf_ptr, uint32_t pf_chunks,
                      const int8_t* k_exp, const int8_t* v_exp, long long cap) {
  auto kern = verify_attn_mma_kernel<KV, D, MT, STAGES>;
  const size_t smem = AttnSmemLayout::bytes(D, MT, STAGES, (int)sizeof(KV));
  int dev = 0;
  TF_CHECK_CUDA(cudaGetDevice(&dev));
  static bool attr_done[64] = {false};  // the attribute is per (function, device)
  const bool attr_set = dev < 64 && attr_done[dev];
  if (!attr_set) {
    TF_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    // ask for the largest shared-memory carve-out so that two ~109 KB CTAs are resident per SM (ncu showed the default
    // carve-out leaving room for one)
    TF_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    if (dev < 64) attr_done[dev] = true;
  }
  // Programmatic launch only for short stores: the long (full-KV) launches use the calibrated per-CTA split, which assumes the
  // block placement of a launch onto an EMPTY GPU — an early launch next to a draining predecessor changes it, which
  // can cost more than the overlap gains.  They still trigger their own dependents early.
  TF_CHECK_CUDA(launch_kernel(allow_pdl ? kPdlVerifyAttn : 0, kern, G, kThreadsAttn, smem, stream, kmap, vmap, q, layer, kv_len_host, kv_len_dev, R, H, grp, scale_log2, pm, pl, po, counters,
                              out, tree_mask, tree_cols, split_table, cta_ns, clean_keys, pf_ptr, pf_chunks, k_exp, v_exp, cap));
  TF_CHECK_LAUNCH();
  return TF_OK;
}

}  // namespace tf

extern "C" {

#ifdef TF_ATTN_TIMING
int tf_debug_attn_timing(void* buf) {
  unsigned long long* p = (unsigned long long*)buf;
  return cudaMemcpyToSymbol(tf::g_attn_timing, &p, sizeof(p)) == cudaSuccess ? 0 : -1;
}
#endif

// workspace = [per-head arrival counters (ZERO on first use; the kernel leaves them zero)] [m] [l] [O]
//             [split table 0 (grid = 2 CTAs/SM)] [split table 1 (grid = 1 CTA/SM)] [per-CTA streaming time, ns]
struct AttnWorkspace {
  int* counters;
  float *pm, *pl, *po;
  uint32_t* table[2];
  uint32_t* cta_ns;
  size_t bytes;
};
static AttnWorkspace attn_workspace(void* base, int H, int d) {
  const size_t slots_max = (size_t)tf::g_max_slots();
  const size_t slots = slots_max + (size_t)H;
  AttnWorkspace w;
  uintptr_t p = ((uintptr_t)base + 255) & ~(uintptr_t)255;
  w.counters = (int*)p;
  p = (p + (size_t)H * sizeof(int) + 255) & ~(uintptr_t)255;
  w.pm = (float*)p;
  w.pl = w.pm + slots * TF_VERIFY_MAX_ROWS;
  w.po = w.pl + slots * TF_VERIFY_MAX_ROWS;
  p = ((uintptr_t)(w.po + slots * (size_t)TF_VERIFY_MAX_ROWS * d) + 255) & ~(uintptr_t)255;
  const size_t tab_words = (size_t)tf::kSplitHdr + slots_max + 4;
  w.table[0] = (uint32_t*)p;
  w.table[1] = w.table[0] + tab_words;
  w.cta_ns = w.table[1] + tab_words;
  w.bytes = (size_t)((uintptr_t)(w.cta_ns + slots_max) - (uintptr_t)base);
  return w;
}

size_t tf_verify_attn_workspace_bytes(int R, int H, int d) {
  (void)R;
  if (H <= 0 || d <= 0) return 0;
  return attn_workspace((void*)0, H, d).bytes + 256;  // + worst-case alignment of the caller's base pointer
}

// partials, counters and split tables are per KV head: the MHA workspace of Hkv heads
size_t tf_verify_attn_gqa_workspace_bytes(int R, int Hq, int Hkv, int d) {
  if (Hkv <= 0 || Hq <= 0 || Hq % Hkv != 0) return 0;
  return tf_verify_attn_workspace_bytes(R, Hkv, d);
}

struct AttnPlan {
  int G;          // grid
  int table_idx;  // which split table this grid uses
};
static AttnPlan attn_plan(int R, int H, int d, int kv_len_max) {
  const int slots_max = tf::g_max_slots();
  // grid: one wave of resident CTAs, but never more CTAs than the longest possible input has tiles / min tiles per CTA.
  // Head-sharded short stores (<= 8 local heads over a retrieval budget: TP 4 / 8 of a 32-head model) get >= 8 tiles per CTA:
  // measured with the per-GPU head counts of 8 / 4 GPUs on one device (tools/bench_kernels.py --tp-shapes, 4 103 keys, in a graph):
  // 4 heads 30.2 us -> 18.3 (4 tiles per CTA) -> 13.2 (8); 8 heads 22.6 -> 19.0 -> 18.5 — one-tile CTAs leave the last CTA of a
  // head dozens of partials to merge.  Unsharded shapes (and every parity-sized model with > 8 heads) keep 1; env
  // TF_ATTN_MIN_TILES overrides everywhere.
  static const long long kEnvMinTiles = getenv("TF_ATTN_MIN_TILES") ? (atoll(getenv("TF_ATTN_MIN_TILES")) > 0 ? atoll(getenv("TF_ATTN_MIN_TILES")) : 1) : 0;
  // (stores below 2 048 keys — the parity-sized models — keep their split: the golden traces pin it to the last bit)
  const long long kMinTilesPerCta = kEnvMinTiles > 0 ? kEnvMinTiles : ((H <= 8 && kv_len_max >= 2048 && kv_len_max < 16384) ? 8 : 1);
  const long long max_tiles = (long long)H * ((kv_len_max + tf::BN - 1) / tf::BN);
  AttnPlan p{slots_max, 0};
  if (d == 128 && R > 16) { p.G = slots_max / 2 > 0 ? slots_max / 2 : 1; p.table_idx = 1; }  // 6-stage ring: one CTA per SM
  if ((long long)p.G > max_tiles / kMinTilesPerCta) p.G = (int)(max_tiles / kMinTilesPerCta);
  if (p.G < 1) p.G = 1;
  return p;
}

// H = KV heads, grp = query heads per KV head (1: MHA); q / out are [R][H * grp][d]
static int verify_attn_impl(const void* q, const void* k_tensormap, const void* v_tensormap, int layer, int kv_len_host,
                            const int32_t* kv_len_dev, int kv_len_max, int R, int H, int grp, int d, float scale, void* out,
                            void* workspace, size_t workspace_bytes, int variant, const uint32_t* tree_mask, int tree_cols,
                            bool record_cta_ns, int clean_keys, tf_stream_t stream_, const void* next_weights = nullptr,
                            size_t next_weight_bytes = 0, const int8_t* k_exp = nullptr, const int8_t* v_exp = nullptr,
                            long long cap = 0) {
  using namespace tf;
  cudaStream_t stream = (cudaStream_t)stream_;
  TF_CHECK_ARG(q && k_tensormap && v_tensormap && out && workspace, "tf_verify_attn: NULL pointer");
  TF_CHECK_ARG(R >= 1 && R <= TF_VERIFY_MAX_ROWS, "tf_verify_attn: R=%d outside [1,%d]", R, TF_VERIFY_MAX_ROWS);
  TF_CHECK_ARG(grp >= 1 && R * grp <= TF_VERIFY_MAX_ROWS,
               "tf_verify_attn_gqa: R=%d rows x %d query heads per KV head exceed %d packed rows", R, grp, TF_VERIFY_MAX_ROWS);
  TF_CHECK_SUPPORTED(d == 64 || d == 128, "tf_verify_attn: head_dim %d not in {64,128}", d);
  TF_CHECK_ARG(H >= 1 && layer >= 0, "tf_verify_attn: bad H/layer");
  TF_CHECK_ARG(kv_len_dev || kv_len_host >= R, "tf_verify_attn: kv_len (%d) must include the %d new rows", kv_len_host, R);
  TF_CHECK_ARG(kv_len_max >= R, "tf_verify_attn: kv_len_max < R");
  TF_CHECK_ARG(workspace_bytes >= tf_verify_attn_workspace_bytes(R, H, d), "tf_verify_attn: workspace too small");
  TF_CHECK_SUPPORTED(variant == 0 || variant == 1, "tf_verify_attn: variant %d not built", variant);
  TF_CHECK_ARG(((uintptr_t)q & 3) == 0 && ((uintptr_t)out & 7) == 0, "tf_verify_attn: q must be 4-byte and out 8-byte aligned");

  CUtensorMap kmap, vmap;
  memcpy(&kmap, k_tensormap, sizeof(kmap));
  memcpy(&vmap, v_tensormap, sizeof(vmap));

  const int rows = R * grp;  // packed rows of one CTA (the launch instance is chosen on these)
  const AttnPlan plan = attn_plan(rows, H, d, kv_len_max);
  const AttnWorkspace w = attn_workspace(workspace, H, d);
  const int G = plan.G;
  const bool e4m3 = k_exp != nullptr;
  const uint32_t* tab = e4m3 ? nullptr : w.table[plan.table_idx];  // e4m3 launches have no calibrated split
  uint32_t* cta_ns = record_cta_ns ? w.cta_ns : nullptr;
  const float scale_log2 = scale * kLog2e;
  const __half* qh = (const __half*)q;
  const bool allow_pdl = kv_len_max < 16384;
  if (clean_keys < 0 || tree_mask != nullptr) clean_keys = 0;
  // L2 prefetch of the next projection's weights: only behind a short (latency-bound) store — a full-KV launch needs all of HBM
  const uint8_t* pf_ptr = allow_pdl ? (const uint8_t*)next_weights : nullptr;
  const uint32_t pf_chunks = pf_ptr ? (uint32_t)(next_weight_bytes / kPfChunk) : 0u;

#define TF_LAUNCH_MMA(KV_, D_, MT_, ST_)                                                                                            \
  launch_mma<KV_, D_, MT_, ST_>(kmap, vmap, qh, layer, kv_len_host, kv_len_dev, R, H, grp, scale_log2, w.pm, w.pl, w.po, w.counters, \
                                (__half*)out, G, tree_mask, tree_cols, tab, cta_ns, clean_keys, allow_pdl, stream, pf_ptr, pf_chunks, \
                                k_exp, v_exp, cap)
  // e4m3 tiles are half the bytes: twice the stages keep the same bytes in flight as the fp16 ring
  if (e4m3) {
    if (d == 128) return rows <= 16 ? TF_LAUNCH_MMA(__nv_fp8_e4m3, 128, 1, 6) : TF_LAUNCH_MMA(__nv_fp8_e4m3, 128, 2, 12);
    return rows <= 16 ? TF_LAUNCH_MMA(__nv_fp8_e4m3, 64, 1, 8) : TF_LAUNCH_MMA(__nv_fp8_e4m3, 64, 2, 8);
  }
  if (d == 128) return rows <= 16 ? TF_LAUNCH_MMA(__half, 128, 1, 3) : TF_LAUNCH_MMA(__half, 128, 2, 6);
  return rows <= 16 ? TF_LAUNCH_MMA(__half, 64, 1, 4) : TF_LAUNCH_MMA(__half, 64, 2, 4);
#undef TF_LAUNCH_MMA
}

// Measures the per-CTA streaming time of this very kernel on the caller's KV store and installs a split table
// proportional to the measured per-CTA rate (see the header comment).  Synchronises `stream` (calibration is an init-time
// call, never captured).  report (host, nullable): {max/min per-CTA time before, after, median ns before, after}.
int tf_verify_attn_calibrate(const void* q, const void* k_tensormap, const void* v_tensormap, int layer, int kv_len, int R,
                             int H, int d, float scale, void* out, void* workspace, size_t workspace_bytes, int rounds,
                             double* report, tf_stream_t stream_) {
  using namespace tf;
  cudaStream_t stream = (cudaStream_t)stream_;
  TF_CHECK_ARG(rounds >= 0 && rounds <= 16, "tf_verify_attn_calibrate: rounds=%d outside [0,16]", rounds);
  TF_CHECK_ARG(workspace && workspace_bytes >= tf_verify_attn_workspace_bytes(R, H, d), "tf_verify_attn_calibrate: workspace too small");
  TF_CHECK_SUPPORTED(d == 64 || d == 128, "tf_verify_attn_calibrate: head_dim %d not in {64,128}", d);
  const AttnPlan plan = attn_plan(R, H, d, kv_len);
  const AttnWorkspace w = attn_workspace(workspace, H, d);
  const int G = plan.G;
  const long long total = (long long)H * ((kv_len + BN - 1) / BN);
  uint32_t* tab_dev = w.table[plan.table_idx];
  std::vector<uint32_t> tab((size_t)kSplitHdr + G, 0u);
  if (rounds == 0 || total < 16ll * G) {  // too little work to measure: back to the equal split
    TF_CHECK_CUDA(cudaMemsetAsync(tab_dev, 0, kSplitHdr * sizeof(uint32_t), stream));
    TF_CHECK_CUDA(cudaStreamSynchronize(stream));
    if (report) report[0] = report[1] = report[2] = report[3] = 0.0;
    return TF_OK;
  }
  std::vector<double> wgt((size_t)G, 1.0 / G);
  std::vector<uint32_t> ns((size_t)G);
  auto install = [&]() -> int {
    double cum = 0.0;
    for (int b = 0; b < G; ++b) {
      double f = cum * 4294967296.0;
      if (f > 4294967295.0) f = 4294967295.0;
      tab[(size_t)kSplitHdr + b] = b == 0 ? 0u : (uint32_t)f;
      cum += wgt[(size_t)b];
    }
    tab[0] = (uint32_t)G;
    TF_CHECK_CUDA(cudaMemcpyAsync(tab_dev, tab.data(), tab.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, stream));
    TF_CHECK_CUDA(cudaStreamSynchronize(stream));
    return TF_OK;
  };
  std::vector<uint32_t> samples((size_t)G * 3);
  auto measure = [&](double* spread, double* median) -> int {
    // per-CTA median of three launches (after one warm-up launch under the new table)
    for (int rep = 0; rep < 4; ++rep) {
      TF_CHECK_CUDA(cudaMemsetAsync(w.cta_ns, 0, (size_t)G * sizeof(uint32_t), stream));
      const int rc = verify_attn_impl(q, k_tensormap, v_tensormap, layer, kv_len, nullptr, kv_len, R, H, 1, d, scale, out, workspace,
                                      workspace_bytes, 0, nullptr, 0, true, 0, stream_);
      if (rc != TF_OK) return rc;
      if (rep > 0) {
        TF_CHECK_CUDA(cudaMemcpyAsync(samples.data() + (size_t)(rep - 1) * G, w.cta_ns, (size_t)G * sizeof(uint32_t), cudaMemcpyDeviceToHost, stream));
        TF_CHECK_CUDA(cudaStreamSynchronize(stream));
      }
    }
    for (int b = 0; b < G; ++b) {
      uint32_t x[3] = {samples[(size_t)b], samples[(size_t)G + b], samples[(size_t)2 * G + b]};
      std::sort(x, x + 3);
      ns[(size_t)b] = x[1];
    }
    std::vector<uint32_t> sorted(ns);
    std::sort(sorted.begin(), sorted.end());
    if (sorted.front() == 0) { set_error("tf_verify_attn_calibrate: a CTA reported no streaming time"); return TF_ERR_CUDA; }
    *spread = (double)sorted.back() / (double)sorted.front();
    *median = (double)sorted[sorted.size() / 2];
    if (getenv("TF_CALIBRATE_DEBUG"))
      fprintf(stderr, "[tf_verify_attn_calibrate] G=%d min %u med %u max %u ns\n", G, sorted.front(), sorted[sorted.size() / 2], sorted.back());
    return TF_OK;
  };
  // start from the equal split
  int rc = install();
  if (rc != TF_OK) return rc;
  double spread0 = 0, med0 = 0, spread = 0, med = 0;
  for (int round = 0; round < rounds; ++round) {
    rc = measure(&spread, &med);
    if (rc != TF_OK) return rc;
    if (round == 0) { spread0 = spread; med0 = med; }
    // tiles_b proportional to rate_b = share_b / time_b, clamped to [1/2, 2] x equal
    double sum = 0.0;
    for (int b = 0; b < G; ++b) { wgt[(size_t)b] = wgt[(size_t)b] / (double)ns[(size_t)b]; sum += wgt[(size_t)b]; }
    for (int b = 0; b < G; ++b) {
      double x = wgt[(size_t)b] / sum * G;
      x = x < 0.5 ? 0.5 : (x > 2.0 ? 2.0 : x);
      wgt[(size_t)b] = x;
    }
    sum = 0.0;
    for (int b = 0; b < G; ++b) sum += wgt[(size_t)b];
    for (int b = 0; b < G; ++b) wgt[(size_t)b] /= sum;
    rc = install();
    if (rc != TF_OK) return rc;
  }
  rc = measure(&spread, &med);
  if (rc != TF_OK) return rc;
  if (report) { report[0] = spread0; report[1] = spread; report[2] = med0; report[3] = med; }
  return TF_OK;
}

int tf_verify_attn(const void* q, const void* k_tensormap, const void* v_tensormap, int layer, int kv_len_host,
                   const int32_t* kv_len_dev, int kv_len_max, int R, int H, int d, float scale, void* out,
                   void* workspace, size_t workspace_bytes, int variant, int clean_keys, tf_stream_t stream) {
  return verify_attn_impl(q, k_tensormap, v_tensormap, layer, kv_len_host, kv_len_dev, kv_len_max, R, H, 1, d, scale, out, workspace,
                          workspace_bytes, variant, nullptr, 0, false, clean_keys, stream);
}

static int gqa_group(int Hq, int Hkv, const char* what) {
  if (Hkv <= 0 || Hq <= 0 || Hq % Hkv != 0) {
    tf::set_error("%s: Hq (%d) must be a positive multiple of Hkv (%d)", what, Hq, Hkv);
    return 0;
  }
  return Hq / Hkv;
}

int tf_verify_attn_gqa(const void* q, const void* k_tensormap, const void* v_tensormap, int layer, int kv_len_host,
                       const int32_t* kv_len_dev, int kv_len_max, int R, int Hq, int Hkv, int d, float scale, void* out,
                       void* workspace, size_t workspace_bytes, int variant, int clean_keys, tf_stream_t stream) {
  const int grp = gqa_group(Hq, Hkv, "tf_verify_attn_gqa");
  if (grp == 0) return TF_ERR_INVALID;
  return verify_attn_impl(q, k_tensormap, v_tensormap, layer, kv_len_host, kv_len_dev, kv_len_max, R, Hkv, grp, d, scale, out,
                          workspace, workspace_bytes, variant, nullptr, 0, false, clean_keys, stream);
}

static int verify_attn_e4m3_impl(const void* q, const void* k_tensormap, const void* v_tensormap, const int8_t* k_exp,
                                 const int8_t* v_exp, long long cap, int layer, int kv_len_host, const int32_t* kv_len_dev, int kv_len_max,
                                 int R, int Hq, int Hkv, int d, float scale, void* out, void* workspace, size_t workspace_bytes,
                                 int clean_keys, tf_stream_t stream) {
  const int grp = gqa_group(Hq, Hkv, "tf_verify_attn_e4m3");
  if (grp == 0) return TF_ERR_INVALID;
  TF_CHECK_ARG(k_exp && v_exp, "tf_verify_attn_e4m3: NULL exponent pointer");
  TF_CHECK_ARG(cap > 0 && cap % TF_VERIFY_BOX_KEYS == 0, "tf_verify_attn_e4m3: cap (%lld) must be a positive multiple of %d", cap,
               TF_VERIFY_BOX_KEYS);
  TF_CHECK_ARG((((uintptr_t)k_exp | (uintptr_t)v_exp) & 15) == 0, "tf_verify_attn_e4m3: exponents must be 16-byte aligned");
  TF_CHECK_ARG(kv_len_max <= cap && (kv_len_dev || kv_len_host <= cap), "tf_verify_attn_e4m3: kv_len (%d, max %d) exceeds cap %lld",
               kv_len_host, kv_len_max, cap);
  return verify_attn_impl(q, k_tensormap, v_tensormap, layer, kv_len_host, kv_len_dev, kv_len_max, R, Hkv, grp, d, scale, out,
                          workspace, workspace_bytes, 0, nullptr, 0, false, clean_keys, stream, nullptr, 0, k_exp, v_exp, cap);
}

int tf_verify_attn_e4m3(const void* q, const void* k_tensormap, const void* v_tensormap, const int8_t* k_exp, const int8_t* v_exp,
                        long long cap, int layer, int kv_len_host, const int32_t* kv_len_dev, int kv_len_max, int R, int Hq, int Hkv,
                        int d, float scale, void* out, void* workspace, size_t workspace_bytes, tf_stream_t stream) {
  return verify_attn_e4m3_impl(q, k_tensormap, v_tensormap, k_exp, v_exp, cap, layer, kv_len_host, kv_len_dev, kv_len_max, R, Hq, Hkv, d,
                               scale, out, workspace, workspace_bytes, 0, stream);
}

int tf_verify_attn_e4m3_clean(const void* q, const void* k_tensormap, const void* v_tensormap, const int8_t* k_exp, const int8_t* v_exp,
                              long long cap, int layer, int kv_len_host, const int32_t* kv_len_dev, int kv_len_max, int R, int Hq,
                              int Hkv, int d, float scale, void* out, void* workspace, size_t workspace_bytes, int clean_keys,
                              tf_stream_t stream) {
  TF_CHECK_ARG(clean_keys >= 0 && clean_keys <= cap, "tf_verify_attn_e4m3_clean: clean_keys (%d) outside [0, cap %lld]", clean_keys, cap);
  return verify_attn_e4m3_impl(q, k_tensormap, v_tensormap, k_exp, v_exp, cap, layer, kv_len_host, kv_len_dev, kv_len_max, R, Hq, Hkv, d,
                               scale, out, workspace, workspace_bytes, clean_keys, stream);
}

int tf_verify_attn_prefetch(const void* q, const void* k_tensormap, const void* v_tensormap, int layer, int kv_len_host,
                            const int32_t* kv_len_dev, int kv_len_max, int R, int H, int d, float scale, void* out, void* workspace,
                            size_t workspace_bytes, int variant, int clean_keys, const void* next_weights, size_t next_weight_bytes,
                            tf_stream_t stream) {
  if (next_weights != nullptr && (((uintptr_t)next_weights & 15) != 0)) {
    tf::set_error("tf_verify_attn_prefetch: next_weights must be 16-byte aligned");
    return TF_ERR_INVALID;
  }
  return verify_attn_impl(q, k_tensormap, v_tensormap, layer, kv_len_host, kv_len_dev, kv_len_max, R, H, 1, d, scale, out, workspace,
                          workspace_bytes, variant, nullptr, 0, false, clean_keys, stream, next_weights, next_weight_bytes);
}

static int verify_attn_tree_impl(const void* q, const void* k_tensormap, const void* v_tensormap, int layer, int kv_len_host,
                                 const int32_t* kv_len_dev, int kv_len_max, int R, int H, int grp, int d, float scale,
                                 const uint32_t* tree_mask, int tree_cols, void* out, void* workspace, size_t workspace_bytes,
                                 tf_stream_t stream) {
  if (!tree_mask || tree_cols <= 0 || tree_cols % 32 != 0) {
    tf::set_error("tf_verify_attn_tree: tree_mask must be non-NULL and tree_cols a positive multiple of 32 (got %d)", tree_cols);
    return TF_ERR_INVALID;
  }
  if (!kv_len_dev && kv_len_host < tree_cols) {
    tf::set_error("tf_verify_attn_tree: kv_len (%d) must include the %d tree columns", kv_len_host, tree_cols);
    return TF_ERR_INVALID;
  }
  return verify_attn_impl(q, k_tensormap, v_tensormap, layer, kv_len_host, kv_len_dev, kv_len_max, R, H, grp, d, scale, out, workspace,
                          workspace_bytes, 0, tree_mask, tree_cols, false, 0, stream);
}

int tf_verify_attn_tree(const void* q, const void* k_tensormap, const void* v_tensormap, int layer, int kv_len_host,
                        const int32_t* kv_len_dev, int kv_len_max, int R, int H, int d, float scale, const uint32_t* tree_mask,
                        int tree_cols, void* out, void* workspace, size_t workspace_bytes, tf_stream_t stream) {
  return verify_attn_tree_impl(q, k_tensormap, v_tensormap, layer, kv_len_host, kv_len_dev, kv_len_max, R, H, 1, d, scale, tree_mask,
                               tree_cols, out, workspace, workspace_bytes, stream);
}

int tf_verify_attn_tree_gqa(const void* q, const void* k_tensormap, const void* v_tensormap, int layer, int kv_len_host,
                            const int32_t* kv_len_dev, int kv_len_max, int R, int Hq, int Hkv, int d, float scale,
                            const uint32_t* tree_mask, int tree_cols, void* out, void* workspace, size_t workspace_bytes,
                            tf_stream_t stream) {
  const int grp = gqa_group(Hq, Hkv, "tf_verify_attn_tree_gqa");
  if (grp == 0) return TF_ERR_INVALID;
  return verify_attn_tree_impl(q, k_tensormap, v_tensormap, layer, kv_len_host, kv_len_dev, kv_len_max, R, Hkv, grp, d, scale,
                               tree_mask, tree_cols, out, workspace, workspace_bytes, stream);
}

}  // extern "C"
