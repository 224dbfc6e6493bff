// Decode-time projections (q|k|v, o_proj, gate|up, down_proj, lm_head) as ONE weight-streaming kernel that is built to sit in
// a chain of programmatically dependent launches:
//     y[M, N] = epilogue( x[M, K] · W[N, K]^T ),   M <= 24 rows (the gamma+1 speculated tokens; gamma = 16 on BASELINE cfg4)
//   epilogue 0: fp16 store;  1: SiLU(gate)·up of LlamaMLP / TP_MLP (tensor_op.py:346-357) with W = [gate rows; up rows];
//            2: fp32 store of the fp16-rounded value (lm_head: the reference computes fp16 logits and calls .float(),
//               modeling_llama.py:408-409);
//            3: TP seam — the row-parallel o_proj / down_proj AND the all-reduce that follows it in the reference
//               (tensor_op.py:176-179, 357-359) in this one kernel, over NVLink peer memory (see "fused all-reduce" below).
// Replaces the `nn.Linear` call sites modeling_llama.py:213-215,243,157,408 (TP: tensor_op.py:143-145,176,353-357) — SURVEY §8
// row f-1: 13.5 GB of weights are 85 % of the bytes of a retrieval-verify step.
//
// HBM-bound: algorithmic bytes = N*K*2 per launch (weights read once; x is L2-resident).  What bounds a 5-45 us launch of this
// kind is not the streaming rate but the fixed cost around it (launch, pipeline ramp, x staging, tail), so the design removes
// the fixed cost from the critical path instead of polishing the steady state:
//   * NOTHING of x is staged up front.  A pipeline stage carries 16 weight rows x 512 k (16 KB, two tensor-TMA boxes) AND the
//     matching 512-k slice of the <= 8 x MT token rows (8 KB per token block, from L2) — so there is no prologue, no limit on
//     K (down_proj, K = 11008, runs on the same kernel), and a CTA needs ~100 KB: two CTAs per SM.
//   * Programmatic dependent launch: every CTA signals `launch_dependents` at entry, and its producer lane issues the WEIGHT
//     boxes of the first ring-full of stages BEFORE `griddepcontrol.wait` — weights do not depend on the predecessor — and the
//     x boxes of those stages after it.  With 2 CTAs/SM of ~100 KB, a CTA of the next kernel becomes resident the moment a CTA
//     of this one retires and fills its ring while the rest of this kernel drains: HBM never idles across the kernel
//     boundary, and the dependent's exposed latency is one L2 read of x.
//   * persistent-style grid (2 CTAs per SM): the (tile of 16 weight rows, 512-wide k-step) units lie on one tile-major axis
//     cut into one contiguous range per CTA (no tile quantisation).  A tile cut by a range boundary is finished by the CTA
//     that holds its first k-steps; the neighbour computes the rest FIRST thing and hands it over through a small global
//     buffer + release/acquire flag.  Sums are taken in k order → deterministic, bit-reproducible.
//   * the weight matrix is described to TMA as [rows][K/64][64 elements]: ONE box [64, 4, 16] = 16 rows x 256 k lands as
//     128-byte lines under SWIZZLE_128B, consecutive rows on different swizzle keys → conflict-free LDS.128 fragment loads
//     without padding; x uses the same view with 8-row boxes.  Out-of-range rows / k are zero-filled by TMA.
//   * eight consumer warps split every stage along k; the 16 weight rows are the A operand of mma.sync m16n8k16, the <= 8
//     tokens of a block the B operand (nothing wasted on an empty half tile); fp32 accumulate; per tile the eight partial
//     accumulators are summed in warp order by a rotating reducer warp that also runs the epilogue.
//
// Fused all-reduce (epilogue 3).  Every rank owns one symmetric buffer [flags | inbox], mapped into all peers (and, where the
// fabric offers it, into one NVLS MULTICAST address that reaches all ranks with a single store):
//   the reducer warp of a finished tile rounds its [16 features x M tokens] partial to fp16 (the reference's per-rank partial
//   is an fp16 tensor), gathers each feature's tokens into one 16-byte vector (warp shuffles) and stores it into slot `rank` of
//   EVERY rank's inbox — one `multimem.st` through the switch, or one peer store per rank; fences (system scope), raises the
//   tile's flag on every rank, waits for the peers' flags of the same tile, adds the `world` inbox copies in rank order in fp32
//   (bit-identical on all ranks — the replicated sampling of the TP loop relies on it) and writes y.  Meanwhile the other seven
//   warps stream the next tile: the exchange of tile t hides behind the weights of tile t+1, there is no second launch, no
//   staging copy and no trailing barrier (inboxes are double-buffered by launch parity: nobody can be two launches ahead of a
//   rank that is still reading).  A peer that never shows up (diverged launch sequence, dead rank) trips a bounded spin and
//   traps instead of hanging the GPU.
//
// LL seam (epilogue 4) — the form the TP engine uses.  The reducer warp rounds its tile to fp16, pairs neighbouring features of
// one token (one shuffle) and PUSHES each pair as an 8-byte {half2, epoch} slot into slot-array `rank` of every rank's
// tf_allreduce_ll inbox (one `multimem.st` through the switch, or one peer store per rank) and moves on: data and flag travel in
// the same store, so there is no fence, no flag round trip and nothing to wait for inside the projection.  The CONSUMER of the
// seam (tf_add_rmsnorm_ll, allreduce.cu) polls its local slots, adds the `world` copies in rank order in fp32, rounds to fp16
// (bit-identical to all-reduce-then-add) and goes on with the residual add and the RMSNorm; it also advances the epoch.
#include <string.h>

#include <type_traits>

#include <cuda_fp8.h>

#include "common.cuh"

namespace tf {

constexpr int kSlMaxRanks = 8;
constexpr int kSlArMaxN = 8192;                      // output features of a fused-all-reduce launch
constexpr int kSlArMaxTiles = kSlArMaxN / 16;
constexpr int kSlArTok = 24;                         // token slots per feature in an inbox
constexpr size_t kSlArFlagBytes = (size_t)kSlArMaxTiles * kSlMaxRanks * sizeof(int);
constexpr size_t kSlArInboxBytes = (size_t)kSlArMaxN * kSlArTok * sizeof(__half);  // one source rank, one parity

struct StreamPeers {
  void* ptr[kSlMaxRanks];   // every rank's symmetric buffer as mapped into THIS process (entry `rank` = the local one)
  void* mc;                 // NVLS multicast mapping of the same buffer, or nullptr
  int rank, world;
  int* epoch;               // local int32[2]: launch epoch, CTA-done counter (zero-initialised)
  size_t ll_slots_per_src;  // epilogue 4: slots of one source rank in the tf_allreduce_ll inbox (its capacity in bytes / 4)
};

constexpr int kSlWarps = 8;
constexpr int kSlConsumers = kSlWarps * 32;
constexpr int kSlThreads = kSlConsumers + 32;
constexpr int kSlRows = 16;                               // weight rows (output features) per tile
constexpr int kSlKC = 512;                                // k elements per stage
constexpr uint32_t kSlWBytes = kSlRows * kSlKC * 2;       // 16 KB of weights per stage
constexpr uint32_t kSlXBytes = 8 * kSlKC * 2;             // 8 KB of x per token block per stage
constexpr int kSlMaxStages = 8;
// E4M3 weights (stream_linear_kernel<MT, __nv_fp8_e4m3>): a stage carries the codes of the same 16 rows x 512 k, 8 KB, and the
// ring may hold more stages in the same shared memory
constexpr uint32_t kSlWBytesE4 = kSlRows * kSlKC;
constexpr int kSlMaxStagesE4 = 12;
template <typename WT> struct SlW {
  static constexpr bool kE4 = std::is_same<WT, __nv_fp8_e4m3>::value;
  static constexpr uint32_t kBytes = kE4 ? kSlWBytesE4 : kSlWBytes;
  static constexpr int kMaxStages = kE4 ? kSlMaxStagesE4 : kSlMaxStages;
};
constexpr size_t kSlSmemTwoPerSM = 233472 / 2 - 1024;     // dynamic shared memory that still lets two CTAs share an SM
constexpr size_t kSlSmemOnePerSM = 232448;                // 227 KB opt-in maximum

__device__ __forceinline__ void sl_tma_3d(uint32_t smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(
                   smem_dst),
               "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
__device__ __forceinline__ uint4 sl_lds128(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
  return v;
}
__device__ __forceinline__ void sl_mma(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void sl_consumer_bar() { asm volatile("bar.sync 2, %0;" ::"n"(kSlConsumers) : "memory"); }

struct StreamArgs {
  int M, N, K;
  int epilogue;             // 0 fp16 | 1 SiLU(gate)*up (N = 2*inter weight rows, y[M][N/2]) | 2 fp32 | 3 fused all-reduce | 4 LL push
  void* y;
  long long y_row_stride;   // elements
  int stages;
  float4* part;             // [grid][MT][32 lanes]: the k-steps of a cut tile computed by the right-hand neighbour
  int* flags;               // [grid]: part[b] published (zero between launches)
  StreamPeers peers;        // epilogue 3 only
  const int8_t* wexp;       // E4M3 weights: one exponent per weight row (stream_linear_kernel<MT, __nv_fp8_e4m3> only)
};

__device__ __forceinline__ void sl_st_release_sys(int* p, int v) { asm volatile("st.release.sys.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
__device__ __forceinline__ int sl_ld_acquire_sys(const int* p) {
  int v;
  asm volatile("ld.acquire.sys.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint4 sl_ld_volatile_v4(const void* p) {
  uint4 r;  // never served from a stale L1 line of an earlier launch
  asm volatile("ld.volatile.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p) : "memory");
  return r;
}
__device__ __forceinline__ void sl_st_v4(void* p, uint4 v) {
  asm volatile("st.relaxed.sys.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ void sl_multimem_st_v4(void* mc, uint4 v) {  // one store, delivered to every rank by the switch
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(mc), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

// MT = token blocks of 8 rows (1: M <= 8, 2: M <= 16, 3: M <= 24).  WT = the weight element: __half, or __nv_fp8_e4m3 for
// E4M3 weights (codes through wmap, exponents a.wexp; see "E4M3 weights" at tf_stream_linear_e4m3).
template <int MT, typename WT = __half>
__global__ void __launch_bounds__(kSlThreads, MT == 1 ? 2 : 1)
    stream_linear_kernel(const __grid_constant__ CUtensorMap wmap, const __grid_constant__ CUtensorMap xmap, const StreamArgs a) {
  extern __shared__ uint8_t sl_smem_raw[];
  constexpr bool kE4 = SlW<WT>::kE4;
  constexpr uint32_t kWBytes = SlW<WT>::kBytes;
  constexpr uint32_t kStage = kWBytes + MT * kSlXBytes;
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(sl_smem_raw) + 1023) & ~(uintptr_t)1023);
  const int stages = a.stages;
  uint8_t* ring = smem;                                                              // [stages][W 16 KB | x MT * 8 KB]
  float4* red = reinterpret_cast<float4*>(ring + (size_t)stages * kStage);           // [2][MT][8 warps][32 lanes]
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(red + 2 * MT * kSlWarps * 32);
  uint64_t* empty_bar = full_bar + SlW<WT>::kMaxStages;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles = a.epilogue == 1 ? (a.N / 2 + 7) / 8 : (a.N + kSlRows - 1) / kSlRows;
  const int ksteps = (a.K + kSlKC - 1) / kSlKC;
  const int inter = a.N / 2;
  // this CTA's contiguous range of (tile, k-step) units; gridDim.x <= tiles, so a range holds >= ksteps units and a tile is
  // shared by at most two CTAs
  const long long units = (long long)tiles * ksteps;
  const int u0 = (int)(units * blockIdx.x / gridDim.x), u1 = (int)(units * (blockIdx.x + 1) / gridDim.x);

  pdl_launch_dependents();  // the next kernel on the stream may become resident as soon as SM slots free up
  if (threadIdx.x == 0) {
    for (int s = 0; s < stages; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], kSlWarps); }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == kSlWarps) {
    // ================= producer: one elected lane issues the tensor loads =================
    if (lane == 0) {
      prefetch_tensormap(&wmap);
      prefetch_tensormap(&xmap);
      const uint32_t ring_u = smem_u32(ring);
      auto load_w = [&](int u, uint32_t s) {
        const int tile = u / ksteps, ks = u - tile * ksteps;
        const uint32_t dst = ring_u + s * kStage;
        if constexpr (kE4) {
          // codes seen as (32 bytes, rows, K/32): a box [32, 8, 8] is 8 rows x 256 k, laid out [k-block of 32][row][32 bytes]
          const int kq0 = ks * (kSlKC / 32);
#pragma unroll
          for (int half = 0; half < 2; ++half)
#pragma unroll
            for (int rg = 0; rg < 2; ++rg) {
              const int row0 = a.epilogue == 1 ? (rg == 0 ? tile * 8 : inter + tile * 8) : tile * kSlRows + rg * 8;
              sl_tma_3d(dst + half * (kWBytes / 2) + rg * (kWBytes / 4), &wmap, &full_bar[s], 0, row0, kq0 + half * 8);
            }
          return;
        }
        const int kb0 = ks * (kSlKC / 64);
#pragma unroll
        for (int half = 0; half < 2; ++half) {
          const uint32_t d = dst + half * (kSlWBytes / 2);
          if (a.epilogue == 1) {  // 8 gate rows, then the 8 matching up rows (the map's box is 8 rows high)
            sl_tma_3d(d, &wmap, &full_bar[s], 0, kb0 + half * 4, tile * 8);
            sl_tma_3d(d + kSlWBytes / 4, &wmap, &full_bar[s], 0, kb0 + half * 4, inter + tile * 8);
          } else {
            sl_tma_3d(d, &wmap, &full_bar[s], 0, kb0 + half * 4, tile * kSlRows);
          }
        }
      };
      auto load_x = [&](int u, uint32_t s) {
        const int tile = u / ksteps, ks = u - tile * ksteps;
        const uint32_t dst = ring_u + s * kStage + kWBytes;
        const int kb0 = ks * (kSlKC / 64);
#pragma unroll
        for (int b = 0; b < MT; ++b)
#pragma unroll
          for (int half = 0; half < 2; ++half) sl_tma_3d(dst + (b * 2 + half) * (kSlXBytes / 2), &xmap, &full_bar[s], 0, kb0 + half * 4, b * 8);
      };
      const int n_units = u1 - u0;
      const int pre = n_units < stages ? n_units : stages;
      // weights of the first ring-full: independent of the predecessor kernel → issued before the dependency resolves
      for (int i = 0; i < pre; ++i) {
        mbar_expect_tx(&full_bar[i], kStage);
        load_w(u0 + i, (uint32_t)i);
      }
      pdl_wait();  // x (and everything else the predecessor wrote) is visible from here on
      for (int i = 0; i < pre; ++i) load_x(u0 + i, (uint32_t)i);
      uint32_t it = (uint32_t)pre;
      for (int u = u0 + pre; u < u1; ++u, ++it) {
        const uint32_t s = it % (uint32_t)stages, ph = (it / (uint32_t)stages) & 1u;
        mbar_wait(&empty_bar[s], ph ^ 1u);
        mbar_expect_tx(&full_bar[s], kStage);
        load_w(u, s);
        load_x(u, s);
      }
    }
    return;
  }

  // ================= consumer warps =================
  pdl_wait();  // consumers touch global memory (y, the hand-over buffer) only after the predecessor has completed
  const int g = lane >> 2, t = lane & 3;
  // fused all-reduce: the launch epoch.  It only advances when the LAST CTA of a launch retires, so every CTA of this launch
  // reads the same value; read after pdl_wait (the previous fused launch on the stream has completed).
  const int ar_epoch = a.epilogue >= 3 ? *reinterpret_cast<volatile int*>(a.peers.epoch) + 1 : 0;
  const uint32_t ring_u = smem_u32(ring);
  uint32_t it = 0;
  int ordinal = 0;
  int u = u0;
  while (u < u1) {
    // ---- one segment = the k-steps of one tile that fall into this CTA's range ----
    const int tile = u / ksteps;
    const int ks_begin = u - tile * ksteps;
    const int ks_end = min(ksteps, ks_begin + (u1 - u));  // exclusive
    float acc[MT][4];
#pragma unroll
    for (int b = 0; b < MT; ++b) { acc[b][0] = acc[b][1] = acc[b][2] = acc[b][3] = 0.f; }
    for (int ks = ks_begin; ks < ks_end; ++ks, ++it) {
      const uint32_t s = it % (uint32_t)stages, ph = (it / (uint32_t)stages) & 1u;
      mbar_wait(&full_bar[s], ph);
      const uint32_t wst = ring_u + s * kStage;
      const uint32_t xst = wst + kWBytes;
#pragma unroll
      for (int cc = 0; cc < 2; ++cc) {
        if constexpr (kE4) {
          // the same chunk and k slots as below; lane (g, t) takes the 8 code bytes k = 32c + 8t .. +7 of rows g and g+8
          // from [half 4 KB][row group 2 KB][k-block c & 7][row & 7][32 bytes]: the 16 lanes of a half warp read 128
          // consecutive bytes (conflict-free LDS.64), and each code is converted once for all MT token blocks
          const int c = warp + cc * kSlWarps;
          const uint32_t half = (uint32_t)c >> 3, kq = (uint32_t)c & 7u;
          const uint32_t wa_addr = wst + half * (kWBytes / 2) + (kq * 8u + (uint32_t)g) * 32u + (uint32_t)t * 8u;
          uint2 ca, cb;
          asm volatile("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(ca.x), "=r"(ca.y) : "r"(wa_addr));
          asm volatile("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(cb.x), "=r"(cb.y) : "r"(wa_addr + kWBytes / 4));
          uint4 wa, wb;
          {
            __half2 h;
            h = kv_e4m3_codes2((uint16_t)(ca.x & 0xffffu)); wa.x = *reinterpret_cast<uint32_t*>(&h);
            h = kv_e4m3_codes2((uint16_t)(ca.x >> 16));     wa.y = *reinterpret_cast<uint32_t*>(&h);
            h = kv_e4m3_codes2((uint16_t)(ca.y & 0xffffu)); wa.z = *reinterpret_cast<uint32_t*>(&h);
            h = kv_e4m3_codes2((uint16_t)(ca.y >> 16));     wa.w = *reinterpret_cast<uint32_t*>(&h);
            h = kv_e4m3_codes2((uint16_t)(cb.x & 0xffffu)); wb.x = *reinterpret_cast<uint32_t*>(&h);
            h = kv_e4m3_codes2((uint16_t)(cb.x >> 16));     wb.y = *reinterpret_cast<uint32_t*>(&h);
            h = kv_e4m3_codes2((uint16_t)(cb.y & 0xffffu)); wb.z = *reinterpret_cast<uint32_t*>(&h);
            h = kv_e4m3_codes2((uint16_t)(cb.y >> 16));     wb.w = *reinterpret_cast<uint32_t*>(&h);
          }
          // x keeps the fp16 layout of the fp16 kernel (the same line / swizzle arithmetic)
          const uint32_t kb = ((uint32_t)c & 7u) >> 1, j = (((uint32_t)c & 1u) << 2) + (uint32_t)t;
          const uint32_t la = 4u * (uint32_t)g + kb;
#pragma unroll
          for (int b = 0; b < MT; ++b) {
            const uint4 xa = sl_lds128(xst + (uint32_t)(b * 2 + (int)half) * (kSlXBytes / 2) + la * 128u + ((j ^ (la & 7u)) << 4));
            sl_mma(acc[b], wa.x, wb.x, wa.y, wb.y, xa.x, xa.y);
            sl_mma(acc[b], wa.z, wb.z, wa.w, wb.w, xa.z, xa.w);
          }
          continue;
        }
        // chunk c of the stage = 32 k; lane (g, t) takes the 16 bytes k = 32c + 8t .. +7 of weight rows g and g+8 and of token
        // row g.  Inside a box the 128-byte line of (row r, k-block kb) is line L = 4r + kb, its 16-byte piece j at j ^ (L & 7).
        const int c = warp + cc * kSlWarps;
        const uint32_t half = (uint32_t)c >> 3, kb = ((uint32_t)c & 7u) >> 1, j = (((uint32_t)c & 1u) << 2) + (uint32_t)t;
        const uint32_t la = 4u * (uint32_t)g + kb, lb = la + 32u;
        const uint32_t wbase = wst + half * (kSlWBytes / 2);
        const uint4 wa = sl_lds128(wbase + la * 128u + ((j ^ (la & 7u)) << 4));
        const uint4 wb = sl_lds128(wbase + lb * 128u + ((j ^ (lb & 7u)) << 4));
#pragma unroll
        for (int b = 0; b < MT; ++b) {
          const uint4 xa = sl_lds128(xst + (uint32_t)(b * 2 + (int)half) * (kSlXBytes / 2) + la * 128u + ((j ^ (la & 7u)) << 4));
          // k-step 1 uses halfs 0..3 of each lane's 8, k-step 2 halfs 4..7 — the same permutation of k on A and B
          sl_mma(acc[b], wa.x, wb.x, wa.y, wb.y, xa.x, xa.y);
          sl_mma(acc[b], wa.z, wb.z, wa.w, wb.w, xa.z, xa.w);
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[s]);
    }
    // ---- cross-warp sum in warp order by a rotating reducer; everyone else moves on to the next segment.  red is double
    //      buffered by segment parity: a warp that writes buffer p again (two segments later) has passed the barrier of the
    //      segment in between, which the previous reducer of p only reaches after it finished reading. ----
    float4* rbuf = red + (size_t)(ordinal & 1) * MT * kSlWarps * 32;
#pragma unroll
    for (int b = 0; b < MT; ++b) rbuf[(b * kSlWarps + warp) * 32 + lane] = make_float4(acc[b][0], acc[b][1], acc[b][2], acc[b][3]);
    sl_consumer_bar();
    if (warp == (ordinal & (kSlWarps - 1))) {
      const bool second_half = ks_begin > 0;     // the tile's first k-steps belong to CTA b-1, which finishes the tile
      const bool first_half = ks_end < ksteps;   // the remaining k-steps belong to CTA b+1, which hands them over
      if (first_half) {
        if (lane == 0) {
          int ready;
          unsigned spins = 0;
          do {
            asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(ready) : "l"(a.flags + blockIdx.x + 1) : "memory");
            if (ready == 0 && ++spins > (1u << 26)) asm volatile("trap;");  // the neighbour CTA never ran: fail loudly, do not hang
          } while (ready == 0);
        }
        __syncwarp();
      }
      float4 sums[MT];
#pragma unroll
      for (int b = 0; b < MT; ++b) {
        float4 sum = rbuf[(b * kSlWarps) * 32 + lane];
#pragma unroll
        for (int w = 1; w < kSlWarps; ++w) {
          const float4 v = rbuf[(b * kSlWarps + w) * 32 + lane];
          sum.x += v.x; sum.y += v.y; sum.z += v.z; sum.w += v.w;
        }
        if (second_half) {
          a.part[((size_t)blockIdx.x * MT + b) * 32 + lane] = sum;
        } else if (first_half) {
          const float4 v = __ldcg(a.part + ((size_t)(blockIdx.x + 1) * MT + b) * 32 + lane);
          sum.x += v.x; sum.y += v.y; sum.z += v.z; sum.w += v.w;
        }
        sums[b] = sum;
      }
      if (!second_half && a.epilogue == 3) {
        // ---- fused all-reduce of this tile over NVLink peer memory (see the header) ----
        const StreamPeers& P = a.peers;
        const size_t inbox0 = kSlArFlagBytes + (size_t)(ar_epoch & 1) * kSlMaxRanks * kSlArInboxBytes;
        const int n_feat = tile * kSlRows + (t == 0 ? g : g + 8);  // lanes t = 0 / 1 carry feature g / g+8, all 8 tokens of a block
        const uint32_t quad = (uint32_t)lane & ~3u;
#pragma unroll
        for (int b = 0; b < MT; ++b) {
          const __half2 lo = __floats2half2_rn(sums[b].x, sums[b].y), hi = __floats2half2_rn(sums[b].z, sums[b].w);
          const uint32_t lo_u = *reinterpret_cast<const uint32_t*>(&lo), hi_u = *reinterpret_cast<const uint32_t*>(&hi);
          uint4 va, vb;
          va.x = __shfl_sync(0xffffffffu, lo_u, quad + 0); va.y = __shfl_sync(0xffffffffu, lo_u, quad + 1);
          va.z = __shfl_sync(0xffffffffu, lo_u, quad + 2); va.w = __shfl_sync(0xffffffffu, lo_u, quad + 3);
          vb.x = __shfl_sync(0xffffffffu, hi_u, quad + 0); vb.y = __shfl_sync(0xffffffffu, hi_u, quad + 1);
          vb.z = __shfl_sync(0xffffffffu, hi_u, quad + 2); vb.w = __shfl_sync(0xffffffffu, hi_u, quad + 3);
          if (t < 2 && n_feat < a.N) {
            const size_t off = inbox0 + (size_t)P.rank * kSlArInboxBytes + ((size_t)n_feat * kSlArTok + (size_t)b * 8) * sizeof(__half);
            const uint4 v = t == 0 ? va : vb;
            if (P.mc != nullptr) {
              sl_multimem_st_v4(reinterpret_cast<uint8_t*>(P.mc) + off, v);
            } else {
              for (int p = 0; p < P.world; ++p) sl_st_v4(reinterpret_cast<uint8_t*>(P.ptr[p]) + off, v);
            }
          }
        }
        __threadfence_system();
        __syncwarp();
        if (lane < P.world) {
          sl_st_release_sys(reinterpret_cast<int*>(P.ptr[lane]) + tile * kSlMaxRanks + P.rank, ar_epoch);
          const int* mine = reinterpret_cast<const int*>(P.ptr[P.rank]) + tile * kSlMaxRanks + lane;
          unsigned spins = 0;
          while (sl_ld_acquire_sys(mine) < ar_epoch) {
            if (++spins > (1u << 25)) asm volatile("trap;");  // a peer never delivered this tile: fail loudly instead of hanging
          }
        }
        __syncwarp();
        if (t < 2 && n_feat < a.N) {
          __half* y = reinterpret_cast<__half*>(a.y);
#pragma unroll
          for (int b = 0; b < MT; ++b) {
            float acc[8];
#pragma unroll
            for (int k = 0; k < 8; ++k) acc[k] = 0.f;
            for (int p = 0; p < P.world; ++p) {  // rank order → bit-identical sums on every rank
              const uint4 v = sl_ld_volatile_v4(reinterpret_cast<const uint8_t*>(P.ptr[P.rank]) + inbox0 + (size_t)p * kSlArInboxBytes +
                                                ((size_t)n_feat * kSlArTok + (size_t)b * 8) * sizeof(__half));
              const __half2* h2 = reinterpret_cast<const __half2*>(&v);
#pragma unroll
              for (int k = 0; k < 4; ++k) {
                const float2 f = __half22float2(h2[k]);
                acc[2 * k] += f.x;
                acc[2 * k + 1] += f.y;
              }
            }
#pragma unroll
            for (int k = 0; k < 8; ++k)
              if (b * 8 + k < a.M) y[(size_t)(b * 8 + k) * a.y_row_stride + n_feat] = __float2half_rn(acc[k]);
          }
        }
      }
      if (!second_half && a.epilogue == 4) {
        // ---- LL push of this tile (see the header): lane (g, t) holds features g / g+8 of tokens 2t, 2t+1; after one exchange
        //      with lane (g^1, t) an even-g lane owns {features g, g+1} of token 2t, an odd-g lane {g-1, g} of token 2t+1 ----
        const StreamPeers& P = a.peers;
        const size_t my_off = ((size_t)(ar_epoch & 1) * kSlMaxRanks + (size_t)P.rank) * P.ll_slots_per_src * 8;
        const bool odd = (g & 1) != 0;
#pragma unroll
        for (int b = 0; b < MT; ++b) {
          const float send_lo = odd ? sums[b].x : sums[b].y, send_hi = odd ? sums[b].z : sums[b].w;  // what the partner needs
          const float got_lo = __shfl_xor_sync(0xffffffffu, send_lo, 4), got_hi = __shfl_xor_sync(0xffffffffu, send_hi, 4);
          const int tok = b * 8 + 2 * t + (odd ? 1 : 0);
          const int n0 = tile * kSlRows + (g & ~1);
          const __half2 lo = odd ? __floats2half2_rn(got_lo, sums[b].y) : __floats2half2_rn(sums[b].x, got_lo);
          const __half2 hi = odd ? __floats2half2_rn(got_hi, sums[b].w) : __floats2half2_rn(sums[b].z, got_hi);
          if (tok < a.M) {
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
              const int n = n0 + hh * 8;
              if (n >= a.N) continue;
              const uint32_t v = hh == 0 ? *reinterpret_cast<const uint32_t*>(&lo) : *reinterpret_cast<const uint32_t*>(&hi);
              const size_t off = my_off + (((size_t)tok * a.N + n) >> 1) * 8;
              if (P.mc != nullptr) {
                asm volatile("multimem.st.relaxed.sys.global.v2.f32 [%0], {%1,%2};" ::"l"(reinterpret_cast<uint8_t*>(P.mc) + off), "r"(v),
                             "r"((uint32_t)ar_epoch)
                             : "memory");
              } else {
                for (int p = 0; p < P.world; ++p)
                  asm volatile("st.relaxed.sys.global.v2.u32 [%0], {%1,%2};" ::"l"(reinterpret_cast<uint8_t*>(P.ptr[p]) + off), "r"(v),
                               "r"((uint32_t)ar_epoch)
                               : "memory");
              }
            }
          }
        }
      }
#pragma unroll
      for (int b = 0; b < MT; ++b) {
        if (second_half || a.epilogue >= 3) continue;
        float4 sum = sums[b];
        if constexpr (kE4) {
          // the row's 2^e on the whole sum (the neighbour's partial included), before the fp16 rounding of the fp16 kernel:
          // code * 2^e is D exactly and power-of-two scaling commutes with the fp32 products and sums, so y is the fp16
          // kernel's y on D bit for bit (except rows whose D is almost all fp16 subnormals, see tf_stream_linear_e4m3)
          const int r_lo = a.epilogue == 1 ? tile * 8 + g : tile * kSlRows + g;
          const int r_hi = a.epilogue == 1 ? inter + tile * 8 + g : r_lo + 8;
          const float s_lo = kv_e4m3_pow2(r_lo < (a.epilogue == 1 ? inter : a.N) ? (int)a.wexp[r_lo] : 0);
          const float s_hi = kv_e4m3_pow2(r_hi < a.N && (a.epilogue != 1 || tile * 8 + g < inter) ? (int)a.wexp[r_hi] : 0);
          sum.x *= s_lo; sum.y *= s_lo; sum.z *= s_hi; sum.w *= s_hi;
        }
        // accumulator layout: (x, y) = weight row g, tokens 2t, 2t+1; (z, w) = weight row g+8, same tokens
        const int tok0 = b * 8 + 2 * t, tok1 = tok0 + 1;
        if (a.epilogue == 1) {
          const int jj = tile * 8 + g;
          if (jj < inter) {
            // gate and up are rounded to fp16 first (they are fp16 tensors in the reference), then SiLU·mul as tf_silu_mul
            __half* y = reinterpret_cast<__half*>(a.y);
            const float g0 = __half2float(__float2half_rn(sum.x)), g1 = __half2float(__float2half_rn(sum.y));
            const __half2 sl = __floats2half2_rn(g0 / (1.f + expf(-g0)), g1 / (1.f + expf(-g1)));
            const __half2 r = __hmul2_rn(sl, __floats2half2_rn(sum.z, sum.w));
            if (tok0 < a.M) y[(size_t)tok0 * a.y_row_stride + jj] = __low2half(r);
            if (tok1 < a.M) y[(size_t)tok1 * a.y_row_stride + jj] = __high2half(r);
          }
        } else {
          const int n_lo = tile * kSlRows + g, n_hi = n_lo + 8;
          const __half h00 = __float2half_rn(sum.x), h01 = __float2half_rn(sum.y), h10 = __float2half_rn(sum.z), h11 = __float2half_rn(sum.w);
          if (a.epilogue == 2) {
            float* y = reinterpret_cast<float*>(a.y);
            if (tok0 < a.M) {
              if (n_lo < a.N) y[(size_t)tok0 * a.y_row_stride + n_lo] = __half2float(h00);
              if (n_hi < a.N) y[(size_t)tok0 * a.y_row_stride + n_hi] = __half2float(h10);
            }
            if (tok1 < a.M) {
              if (n_lo < a.N) y[(size_t)tok1 * a.y_row_stride + n_lo] = __half2float(h01);
              if (n_hi < a.N) y[(size_t)tok1 * a.y_row_stride + n_hi] = __half2float(h11);
            }
          } else {
            __half* y = reinterpret_cast<__half*>(a.y);
            if (tok0 < a.M) {
              if (n_lo < a.N) y[(size_t)tok0 * a.y_row_stride + n_lo] = h00;
              if (n_hi < a.N) y[(size_t)tok0 * a.y_row_stride + n_hi] = h10;
            }
            if (tok1 < a.M) {
              if (n_lo < a.N) y[(size_t)tok1 * a.y_row_stride + n_lo] = h01;
              if (n_hi < a.N) y[(size_t)tok1 * a.y_row_stride + n_hi] = h11;
            }
          }
        }
      }
      if (second_half) {  // publish: the warp's stores, then a cumulative release by lane 0
        __syncwarp();
        if (lane == 0) asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(a.flags + blockIdx.x), "r"(1) : "memory");
      }
      if (first_half && lane == 0) a.flags[blockIdx.x + 1] = 0;  // consumed: ready for the next launch on this stream
    }
    u += ks_end - ks_begin;
    ++ordinal;
  }
  if (a.epilogue == 3) {  // the last CTA of the launch advances the epoch (the next launch on this stream starts after this one)
    sl_consumer_bar();
    if (threadIdx.x == 0) {
      __threadfence();
      const int prev = atomicAdd(a.peers.epoch + 1, 1);
      if (prev == (int)gridDim.x - 1) {
        a.peers.epoch[1] = 0;
        *reinterpret_cast<volatile int*>(a.peers.epoch) = ar_epoch;
      }
    }
  }
}

struct StreamPlan {
  int stages, ctas_per_sm;
  size_t smem;
};
template <typename WT = __half>
static StreamPlan stream_plan(int MT) {
  const size_t stage = SlW<WT>::kBytes + (size_t)MT * kSlXBytes;
  const size_t fixed = 1024 + (size_t)2 * MT * kSlWarps * 32 * sizeof(float4) + 2 * SlW<WT>::kMaxStages * sizeof(uint64_t);
  StreamPlan p;
  p.ctas_per_sm = 2;
  int s = (int)((kSlSmemTwoPerSM - fixed) / stage);
  if (MT > 1 || s < 3) {  // wider token blocks: one CTA per SM with a deeper ring
    p.ctas_per_sm = 1;
    s = (int)((kSlSmemOnePerSM - fixed) / stage);
  }
  if (s > SlW<WT>::kMaxStages) s = SlW<WT>::kMaxStages;
  p.stages = s;
  p.smem = fixed + (size_t)s * stage;
  return p;
}

typedef CUresult (*PFN_encodeTiledSL)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                      const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                      CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiledSL sl_encoder() {
  static PFN_encodeTiledSL encode = nullptr;
  if (!encode) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
    if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || !fn) {
      set_error("cuTensorMapEncodeTiled not available from the driver (%s)", cudaGetErrorString(e));
      return nullptr;
    }
    encode = (PFN_encodeTiledSL)fn;
  }
  return encode;
}

// [rows][K] fp16 seen as (64 elements, K/64 k-blocks, rows), fastest first; box = 64 x 4 x box_rows = box_rows rows x 256 k
static int sl_encode(CUtensorMap* map, const void* base, int rows, int K, long long row_stride, int box_rows, bool weights) {
  PFN_encodeTiledSL encode = sl_encoder();
  if (!encode) return TF_ERR_CUDA;
  cuuint64_t gdim[3] = {64, (cuuint64_t)(K / 64), (cuuint64_t)rows};
  cuuint64_t gstride[2] = {128, (cuuint64_t)row_stride * 2};
  cuuint32_t box[3] = {64, 4, (cuuint32_t)box_rows};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = encode(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, const_cast<void*>(base), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                      CU_TENSOR_MAP_SWIZZLE_128B, weights ? CU_TENSOR_MAP_L2_PROMOTION_L2_256B : CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                      CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled (%s) failed with CUresult %d", weights ? "weights" : "x", (int)r);
    return TF_ERR_CUDA;
  }
  return TF_OK;
}

template <int MT, typename WT = __half>
static int launch_stream(const CUtensorMap& wmap, const CUtensorMap& xmap, const StreamArgs& a, size_t smem, int grid, cudaStream_t stream) {
  auto kern = stream_linear_kernel<MT, WT>;
  int dev = 0;
  TF_CHECK_CUDA(cudaGetDevice(&dev));
  static size_t configured[64] = {0};  // per device: the attribute is per (function, device)
  if (dev < 64 && smem > configured[dev]) {
    TF_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    TF_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    configured[dev] = smem;
  }
  TF_CHECK_CUDA(launch_kernel(kPdlStream, kern, dim3(grid), dim3(kSlThreads), smem, stream, wmap, xmap, a));
  TF_CHECK_LAUNCH();
  return TF_OK;
}

// ---- E4M3 weights: per-row quantization and dequantization (the rule of common.cuh with e clamped at -15) ----------------
constexpr int kWqThreads = 256;
constexpr uint32_t kWqRefuseAbove = 0x7b80u;  // fp16 bits of 61440 = 240 * 2^8

__device__ __forceinline__ int weight_e4m3_exponent(float amax) {
  const int e = kv_e4m3_exponent(amax);
  return e < -15 ? -15 : e;  // code * 2^e stays an exact fp16 value (codes are multiples of 2^-9 with <= 4 significant bits)
}

// one CTA per row: max |w| over K as the largest fp16 magnitude bit pattern (NaN / inf compare above every finite value),
// then the codes of 8 elements per thread and step
__global__ void __launch_bounds__(kWqThreads) weight_quantize_e4m3_kernel(const __half* __restrict__ W, long long row_stride, int K,
                                                                         uint8_t* __restrict__ codes, long long codes_row_stride,
                                                                         int8_t* __restrict__ exps, int32_t* refused) {
  __shared__ uint32_t red[kWqThreads / 32];
  const int row = blockIdx.x;
  const __half* w = W + (size_t)row * row_stride;
  uint32_t m = 0;
  for (int k = threadIdx.x * 8; k < K; k += kWqThreads * 8) {
    const uint4 v = *reinterpret_cast<const uint4*>(w + k);
    const uint32_t u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) m = max(m, max(u[i] & 0x7fffu, (u[i] >> 16) & 0x7fffu));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  m = red[0];
#pragma unroll
  for (int i = 1; i < kWqThreads / 32; ++i) m = max(m, red[i]);
  if (m > kWqRefuseAbove) {  // non-finite, or large enough for D to round past the fp16 maximum: counted, row left alone
    if (threadIdx.x == 0 && refused) atomicAdd(refused, 1);
    return;
  }
  const int e = weight_e4m3_exponent(__half2float(__ushort_as_half((unsigned short)m)));
  if (threadIdx.x == 0) exps[row] = (int8_t)e;
  uint8_t* c = codes + (size_t)row * codes_row_stride;
  for (int k = threadIdx.x * 8; k < K; k += kWqThreads * 8) {
    const uint4 v = *reinterpret_cast<const uint4*>(w + k);
    const __half2* h = reinterpret_cast<const __half2*>(&v);
    uint2 o;
    uint32_t q[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 f = __half22float2(h[i]);
      q[i] = kv_e4m3_quantize2(f.x, f.y, e);
    }
    o.x = q[0] | (q[1] << 16);
    o.y = q[2] | (q[3] << 16);
    *reinterpret_cast<uint2*>(c + k) = o;
  }
}

__global__ void __launch_bounds__(kWqThreads) weight_dequantize_e4m3_kernel(const uint8_t* __restrict__ codes, long long codes_row_stride,
                                                                           const int8_t* __restrict__ exps, int K, __half* __restrict__ D,
                                                                           long long d_row_stride) {
  const int row = blockIdx.x;
  const int e = exps[row];
  const uint8_t* c = codes + (size_t)row * codes_row_stride;
  __half* d = D + (size_t)row * d_row_stride;
  for (int k = threadIdx.x * 8; k < K; k += kWqThreads * 8)
    *reinterpret_cast<uint4*>(d + k) = kv_e4m3_dequant8(*reinterpret_cast<const uint2*>(c + k), e);
}

// codes [rows][row_stride bytes] seen as (32 bytes, rows, K/32), fastest first; box = 32 x 8 rows x 8 = 8 rows x 256 k, no swizzle
static int sl_encode_e4m3(CUtensorMap* map, const void* base, int rows, int K, long long row_stride) {
  PFN_encodeTiledSL encode = sl_encoder();
  if (!encode) return TF_ERR_CUDA;
  cuuint64_t gdim[3] = {32, (cuuint64_t)rows, (cuuint64_t)(K / 32)};
  cuuint64_t gstride[2] = {(cuuint64_t)row_stride, 32};
  cuuint32_t box[3] = {32, 8, 8};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = encode(map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, const_cast<void*>(base), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                      CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled (e4m3 weights) failed with CUresult %d", (int)r);
    return TF_ERR_CUDA;
  }
  return TF_OK;
}

}  // namespace tf

extern "C" {

int tf_weight_tensormap_encode(void* out, const void* W, int N, int K, long long row_stride, int box_rows) {
  using namespace tf;
  TF_CHECK_ARG(out && W, "tf_weight_tensormap_encode: NULL pointer");
  TF_CHECK_ARG(N >= 1 && K >= 64 && K % 64 == 0, "tf_weight_tensormap_encode: need N >= 1 and K a positive multiple of 64 (N=%d, K=%d)", N, K);
  TF_CHECK_ARG(box_rows == 8 || box_rows == 16, "tf_weight_tensormap_encode: box_rows %d not in {8 (gate/up pairs), 16}", box_rows);
  TF_CHECK_ARG(((uintptr_t)W & 15) == 0 && row_stride >= K && (row_stride * 2) % 16 == 0, "tf_weight_tensormap_encode: W / row_stride must keep 16-byte alignment");
  CUtensorMap map;
  int rc = sl_encode(&map, W, N, K, row_stride, box_rows, true);
  if (rc != TF_OK) return rc;
  memcpy(out, &map, sizeof(map));
  return TF_OK;
}

size_t tf_stream_linear_workspace_bytes(void) {
  int sms = tf::sm_count();
  if (sms <= 0) sms = 132;
  return (size_t)(2 * sms + 1) * (3 * 32 * sizeof(float4) + sizeof(int)) + 256;
}

static int stream_linear_impl(const void* x, long long x_row_stride, const void* w_tensormap, int M, int N, int K, int epilogue, void* y,
                              long long y_row_stride, void* workspace, size_t workspace_bytes, const tf::StreamPeers* peers,
                              tf_stream_t stream_, const int8_t* wexp = nullptr) {
  using namespace tf;
  TF_CHECK_ARG(x && w_tensormap && (y || epilogue == 4) && workspace, "tf_stream_linear: NULL pointer");
  TF_CHECK_ARG(workspace_bytes >= tf_stream_linear_workspace_bytes() && ((uintptr_t)workspace & 15) == 0, "tf_stream_linear: workspace too small or misaligned");
  TF_CHECK_ARG(M >= 1 && M <= 24, "tf_stream_linear: M=%d outside [1,24]", M);
  TF_CHECK_ARG(N >= 1 && K >= 64 && K % 64 == 0, "tf_stream_linear: need N >= 1 and K a positive multiple of 64 (N=%d, K=%d)", N, K);
  TF_CHECK_ARG(epilogue >= 0 && epilogue <= 4 && (epilogue >= 3) == (peers != nullptr), "tf_stream_linear: epilogue %d not in {0 fp16, 1 silu*up, 2 fp32}", epilogue);
  TF_CHECK_ARG(epilogue != 1 || (N % 2 == 0), "tf_stream_linear: the SiLU epilogue needs N = 2*inter");
  TF_CHECK_ARG(((uintptr_t)x & 15) == 0 && x_row_stride >= K && x_row_stride % 8 == 0, "tf_stream_linear: x / x_row_stride must keep 16-byte alignment");
  const int MT = (M + 7) / 8;
  const StreamPlan plan = wexp ? stream_plan<__nv_fp8_e4m3>(MT) : stream_plan(MT);
  CUtensorMap wmap, xmap;
  memcpy(&wmap, w_tensormap, sizeof(wmap));
  int rc = sl_encode(&xmap, x, M, K, x_row_stride, 8, false);
  if (rc != TF_OK) return rc;
  StreamArgs a;
  a.M = M; a.N = N; a.K = K; a.epilogue = epilogue; a.y = y; a.y_row_stride = y_row_stride; a.stages = plan.stages;
  memset(&a.peers, 0, sizeof(a.peers));
  if (peers) a.peers = *peers;
  a.wexp = wexp;
  const int tiles = epilogue == 1 ? (N / 2 + 7) / 8 : (N + kSlRows - 1) / kSlRows;
  int sms = sm_count();
  if (sms <= 0) sms = 132;
  const int want = plan.ctas_per_sm * sms;
  const int grid = tiles < want ? tiles : want;
  a.part = (float4*)workspace;
  a.flags = (int*)((uint8_t*)workspace + (size_t)(2 * sms + 1) * 3 * 32 * sizeof(float4));
  cudaStream_t stream = (cudaStream_t)stream_;
  if (wexp) {
    switch (MT) {
      case 1: return launch_stream<1, __nv_fp8_e4m3>(wmap, xmap, a, plan.smem, grid, stream);
      case 2: return launch_stream<2, __nv_fp8_e4m3>(wmap, xmap, a, plan.smem, grid, stream);
      default: return launch_stream<3, __nv_fp8_e4m3>(wmap, xmap, a, plan.smem, grid, stream);
    }
  }
  switch (MT) {
    case 1: return launch_stream<1>(wmap, xmap, a, plan.smem, grid, stream);
    case 2: return launch_stream<2>(wmap, xmap, a, plan.smem, grid, stream);
    default: return launch_stream<3>(wmap, xmap, a, plan.smem, grid, stream);
  }
}

int tf_stream_linear(const void* x, long long x_row_stride, const void* w_tensormap, int M, int N, int K, int epilogue, void* y,
                     long long y_row_stride, void* workspace, size_t workspace_bytes, tf_stream_t stream) {
  if (epilogue >= 3) {
    tf::set_error("tf_stream_linear: epilogues 3 / 4 go through tf_stream_linear_allreduce / tf_stream_linear_ll_push");
    return TF_ERR_INVALID;
  }
  return stream_linear_impl(x, x_row_stride, w_tensormap, M, N, K, epilogue, y, y_row_stride, workspace, workspace_bytes, nullptr, stream);
}

size_t tf_stream_linear_allreduce_buffer_bytes(void) {
  return tf::kSlArFlagBytes + 2 * (size_t)tf::kSlMaxRanks * tf::kSlArInboxBytes;
}

int tf_stream_linear_allreduce(const void* x, long long x_row_stride, const void* w_tensormap, int M, int N, int K, void* y,
                               long long y_row_stride, void* workspace, size_t workspace_bytes, void* const* peer_buffers,
                               void* multicast_buffer, int rank, int world, int32_t* epoch_and_counter, tf_stream_t stream) {
  using namespace tf;
  TF_CHECK_ARG(peer_buffers && epoch_and_counter, "tf_stream_linear_allreduce: NULL pointer");
  TF_CHECK_ARG(world >= 2 && world <= kSlMaxRanks && rank >= 0 && rank < world, "tf_stream_linear_allreduce: bad rank/world (%d/%d)", rank, world);
  TF_CHECK_ARG(N >= 1 && N <= kSlArMaxN, "tf_stream_linear_allreduce: N=%d outside [1,%d]", N, kSlArMaxN);
  StreamPeers peers;
  memset(&peers, 0, sizeof(peers));
  for (int p = 0; p < world; ++p) {
    TF_CHECK_ARG(peer_buffers[p] != nullptr && ((uintptr_t)peer_buffers[p] & 15) == 0, "tf_stream_linear_allreduce: peer buffer %d is NULL or misaligned", p);
    peers.ptr[p] = peer_buffers[p];
  }
  peers.mc = multicast_buffer;
  peers.rank = rank;
  peers.world = world;
  peers.epoch = epoch_and_counter;
  return stream_linear_impl(x, x_row_stride, w_tensormap, M, N, K, 3, y, y_row_stride, workspace, workspace_bytes, &peers, stream);
}


int tf_stream_linear_ll_push(const void* x, long long x_row_stride, const void* w_tensormap, int M, int N, int K, void* workspace,
                             size_t workspace_bytes, void* const* peer_buffers, void* multicast_buffer, int rank, int world,
                             size_t max_message_bytes, const int32_t* epoch_and_counter, tf_stream_t stream) {
  using namespace tf;
  TF_CHECK_ARG(peer_buffers && epoch_and_counter, "tf_stream_linear_ll_push: NULL pointer");
  TF_CHECK_ARG(world >= 2 && world <= kSlMaxRanks && rank >= 0 && rank < world, "tf_stream_linear_ll_push: bad rank/world (%d/%d)", rank, world);
  TF_CHECK_ARG(N >= 2 && N % 2 == 0, "tf_stream_linear_ll_push: N=%d must be even", N);
  const size_t cap = (max_message_bytes + 255) / 256 * 256;  // as tf_allreduce_ll_buffer_bytes lays the inbox out
  TF_CHECK_ARG((size_t)M * (size_t)N * 2 <= cap, "tf_stream_linear_ll_push: message of %zu B exceeds the inbox (%zu B)", (size_t)M * N * 2, cap);
  StreamPeers peers;
  memset(&peers, 0, sizeof(peers));
  for (int p = 0; p < world; ++p) {
    TF_CHECK_ARG(peer_buffers[p] != nullptr && ((uintptr_t)peer_buffers[p] & 15) == 0, "tf_stream_linear_ll_push: peer buffer %d is NULL or misaligned", p);
    peers.ptr[p] = peer_buffers[p];
  }
  peers.mc = multicast_buffer;
  peers.rank = rank;
  peers.world = world;
  peers.epoch = const_cast<int32_t*>(epoch_and_counter);  // read only: the consumer (tf_add_rmsnorm_ll) advances it
  peers.ll_slots_per_src = cap / 4;
  return stream_linear_impl(x, x_row_stride, w_tensormap, M, N, K, 4, nullptr, 0, workspace, workspace_bytes, &peers, stream);
}

int tf_weight_quantize_e4m3(const void* W, long long row_stride, int N, int K, void* codes, long long codes_row_stride, int8_t* exps,
                            int32_t* refused_rows, tf_stream_t stream) {
  using namespace tf;
  TF_CHECK_ARG(W && codes && exps, "tf_weight_quantize_e4m3: NULL pointer");
  TF_CHECK_ARG(N >= 1 && K >= 64 && K % 64 == 0, "tf_weight_quantize_e4m3: need N >= 1 and K a positive multiple of 64 (N=%d, K=%d)", N, K);
  TF_CHECK_ARG(((uintptr_t)W & 15) == 0 && row_stride >= K && row_stride % 8 == 0, "tf_weight_quantize_e4m3: W / row_stride must keep 16-byte alignment");
  TF_CHECK_ARG(((uintptr_t)codes & 15) == 0 && codes_row_stride >= K && codes_row_stride % 16 == 0, "tf_weight_quantize_e4m3: codes / codes_row_stride must keep 16-byte alignment");
  weight_quantize_e4m3_kernel<<<N, kWqThreads, 0, (cudaStream_t)stream>>>((const __half*)W, row_stride, K, (uint8_t*)codes, codes_row_stride, exps,
                                                                         refused_rows);
  TF_CHECK_LAUNCH();
  return TF_OK;
}

int tf_weight_dequantize_e4m3(const void* codes, long long codes_row_stride, const int8_t* exps, int N, int K, void* D, long long d_row_stride,
                              tf_stream_t stream) {
  using namespace tf;
  TF_CHECK_ARG(codes && exps && D, "tf_weight_dequantize_e4m3: NULL pointer");
  TF_CHECK_ARG(N >= 1 && K >= 64 && K % 64 == 0, "tf_weight_dequantize_e4m3: need N >= 1 and K a positive multiple of 64 (N=%d, K=%d)", N, K);
  TF_CHECK_ARG(((uintptr_t)codes & 15) == 0 && codes_row_stride >= K && codes_row_stride % 16 == 0, "tf_weight_dequantize_e4m3: codes / codes_row_stride must keep 16-byte alignment");
  TF_CHECK_ARG(((uintptr_t)D & 15) == 0 && d_row_stride >= K && d_row_stride % 8 == 0, "tf_weight_dequantize_e4m3: D / d_row_stride must keep 16-byte alignment");
  weight_dequantize_e4m3_kernel<<<N, kWqThreads, 0, (cudaStream_t)stream>>>((const uint8_t*)codes, codes_row_stride, exps, K, (__half*)D, d_row_stride);
  TF_CHECK_LAUNCH();
  return TF_OK;
}

int tf_weight_tensormap_encode_e4m3(void* out, const void* codes, int N, int K, long long row_stride) {
  using namespace tf;
  TF_CHECK_ARG(out && codes, "tf_weight_tensormap_encode_e4m3: NULL pointer");
  TF_CHECK_ARG(N >= 1 && K >= 64 && K % 64 == 0, "tf_weight_tensormap_encode_e4m3: need N >= 1 and K a positive multiple of 64 (N=%d, K=%d)", N, K);
  TF_CHECK_ARG(((uintptr_t)codes & 15) == 0 && row_stride >= K && row_stride % 16 == 0, "tf_weight_tensormap_encode_e4m3: codes / row_stride must keep 16-byte alignment");
  CUtensorMap map;
  int rc = sl_encode_e4m3(&map, codes, N, K, row_stride);
  if (rc != TF_OK) return rc;
  memcpy(out, &map, sizeof(map));
  return TF_OK;
}

int tf_stream_linear_e4m3(const void* x, long long x_row_stride, const void* w_tensormap, const int8_t* w_exp, int M, int N, int K,
                          int epilogue, void* y, long long y_row_stride, void* workspace, size_t workspace_bytes, tf_stream_t stream) {
  if (epilogue >= 3) {
    tf::set_error("tf_stream_linear_e4m3: epilogue %d not in {0 fp16, 1 silu*up, 2 fp32} (no TP seams over E4M3 weights)", epilogue);
    return TF_ERR_INVALID;
  }
  if (!w_exp) {
    tf::set_error("tf_stream_linear_e4m3: NULL exponents");
    return TF_ERR_INVALID;
  }
  return stream_linear_impl(x, x_row_stride, w_tensormap, M, N, K, epilogue, y, y_row_stride, workspace, workspace_bytes, nullptr, stream,
                            w_exp);
}

}  // extern "C"
