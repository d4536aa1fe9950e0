// Weight-streaming GEMM for decode-sized batches (5 <= T <= 128 tokens):  C[T, N] = A[T, K] * W[N, K]^T, bound by HBM.
//
// At these sizes the step reads every weight byte once and does ~2T flop per byte: the kernel's only job is to keep all 132 SMs
// pulling their share of W at the HBM rate.  Two facts shape it:
//   * tile width: a W stage of [128 rows x 64] = 16 KB streams at the full HBM rate (lm head: 1.34 GB in 205 us), [64 x 64] gets
//     ~40 % and [32 x 64] ~26 %: per stage the one-thread TMA producer and the one-thread MMA issuer each spend a few hundred
//     cycles, so a stage must carry >= 16 KB.  Tiles are therefore always 128 wide;
//   * N / 128 tiles do not divide over 132 SMs (wo of Nemo: 40 tiles; gate/up: 224 = 1.7 rounds), so the work is cut stream-K
//     style instead: the (tile, k-block) units of the whole problem are one sequence, and CTA c takes the c-th contiguous 1/G of
//     it -- every SM streams the same number of bytes (+- one 16 KB stage) in one pass, whatever N and K are.
// A CTA's range covers the tail of one tile, some whole tiles and the head of another (or, when tiles are longer than ranges,
// a piece from the middle of one).  Partial tiles are reduced deterministically: a contributor that does not hold the tile's
// first k-block writes its fp32 accumulator to its own slot of the workspace and raises its flag -- always as the FIRST segment
// of its range; the owner of the first k-block -- always as the LAST segment of its range -- waits for the flags, sums the slots
// in ascending k order (all 128 epilogue threads, up to four contributors per L2 round trip), adds its own accumulator and runs
// the epilogue.  No atomics on data, no host-visible state: flags are consumed (reset) by their single reader.  The partition
// and the flag protocol are model-checked on the CPU in tests/test_streamk_protocol.py; scripts/trace_streamk.py (tracing build)
// prints the time line of a chain of launches.
//
// Structure per CTA is that of gemm_wgmma.cuh: warp 0 TMA producer ([TA x 64] A box + [128 x 64] W box per stage, deep ring),
// one consumer warpgroup per 64 rows of the A box issuing wgmma (M = 64 -- rows >= TA read past a 32-row box and are never
// stored --, N = 128, fp32 accumulators in registers) and running the pair epilogues of epilogue.cuh on its fragment.  GROUPED: the mixture-of-experts variant -- m
// tiles (expert segments of <= TA rows) come from the device-side plan of csrc/moe.cuh, each with its own weight tensor map.
#pragma once
#include <type_traits>

#include "gemm_wgmma.cuh"
#include "workspace.cuh"

namespace mb200 {

constexpr int SK_BN = 128;
static_assert(SK_PARTIAL_BYTES == (size_t)SK_MAX_CTAS * 128 * SK_BN * sizeof(float), "one [128 x SK_BN] fp32 slot per CTA");

// -DMB200_SK_TRACE: every CTA of the dense kernel stamps %globaltimer / %clock64 at eight points of its life into a device ring
// (scripts/trace_streamk.py reads it through mb200_debug_sk_trace) -- how the microseconds between dependent launches are spent.
#ifdef MB200_SK_TRACE
constexpr int SK_TRACE_LAUNCHES = 64, SK_TRACE_POINTS = 8;
__device__ unsigned long long sk_trace_buf[SK_TRACE_LAUNCHES][SK_MAX_CTAS][SK_TRACE_POINTS][2];
__device__ unsigned sk_trace_count;
__device__ __forceinline__ void sk_stamp(unsigned launch, int point) {
  unsigned long long g, c;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(g));
  asm volatile("mov.u64 %0, %%clock64;" : "=l"(c));
  sk_trace_buf[launch % SK_TRACE_LAUNCHES][blockIdx.x][point][0] = g;
  sk_trace_buf[launch % SK_TRACE_LAUNCHES][blockIdx.x][point][1] = c;
}
#define SK_STAMP(point) sk_stamp(*trace_launch, point)
#else
#define SK_STAMP(point) ((void)0)
#endif

struct SkParams {
  int T, N, K;
  EpiParams epi;
  float* partials;  // [gridDim][TA][128] fp32
  unsigned* flags;  // [gridDim], zero between launches
};

// W4 stages.  A 64-wide k-block of a 128-row INT4 tile is 4 KB of codes, and a weight stage must carry 16 KB to stream at the HBM
// rate (above).  So the codes do not travel with the stages: one TMA brings a CHUNK of up to four consecutive k-blocks of one tile
// ([128 rows x 128 B] = 16 KB) into a ring of its own, and warps 1-3 convert it k-block by k-block into the bf16 W' tiles of the
// ordinary stages.  A chunk starts at the first unit of a CTA's range, at the first k-block of a tile, or after four k-blocks; a
// chunk cut short by the range end reads up to three k-blocks it does not use (past K they read as zero).  The units, their
// partition over the CTAs and every tile's k order stay the bf16 kernel's.
constexpr int SK_W4_CHUNK_KB = 4, SK_W4_CHUNK_BYTES = SK_BN * SK_W4_CHUNK_KB * TG_BK / 2, SK_W4_SLOTS = 4;
template <int TA>
struct SkW4Cfg {  // the bf16 stage (A + W' tile) and, after the stages, the chunk ring
  using B = TgCfg<SK_BN, TA>;
  static constexpr int kABytes = B::kABytes, kBBytes = B::kBBytes, kStageBytes = B::kStageBytes, kSlack = B::kSlack;
  static constexpr int kWG = B::kWG, kThreads = B::kThreads, kRawBytes = 0;
  static constexpr int kRing = SK_W4_SLOTS * SK_W4_CHUNK_BYTES;
  static constexpr int kFit = (227 * 1024 - 1024 - 512 - kSlack - kRing) / kStageBytes;
  static constexpr int kStages = B::kStages < kFit ? B::kStages : kFit;
  static constexpr int kSmem = kStages * kStageBytes + kSlack + kRing + 1024 + 512;
  static_assert(kStages >= 3 && kSmem <= 227 * 1024, "W4 stream-K shared memory plan");
};
__device__ __forceinline__ bool mbar_test_wait(uint64_t* bar, uint32_t parity) {  // non-blocking probe
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}

// W8: FP8 weights, converted per stage by warps 1-3 exactly as in tc_gemm_body (gemm_wgmma.cuh): the experts' W' tiles (grouped)
// or the exact q tiles of a dense Linear, whose row scales the epilogue applies (MODE carries EPI_WSCALE).  The partition into
// (tile, k-block) units is the bf16 kernel's, so an FP8 call splits and sums every tile the same way.
// W4: INT4 weights, the packed codes arriving in 16 KB chunks (SkW4Cfg above) and converted to the bf16 W' tile of each stage
// by warps 1-3 (convert_w4_tile; group scales gscale when dense, gscales->s[expert] of the tile's expert when grouped); same
// partition, same k-blocks, same split-tile sums as the bf16 kernel, so the result is the bf16 kernel's on W'.  A chunk never
// crosses a tile, so each chunk belongs to one expert.
template <int MODE, int TA, bool GROUPED, bool W8 = false, bool W4 = false>
__device__ __forceinline__ void sk_gemm_body(const CUtensorMap& map_a, const CUtensorMap* map_w_base, const SkParams& p, const int32_t* plan,
                                             const MoeWeightScales* scales = nullptr, const uint16_t* gscale = nullptr,
                                             const MoeWeightGroupScales* gscales = nullptr) {
  static_assert(!W8 || GROUPED || (MODE & EPI_WSCALE) != 0, "FP8 dense weights: the epilogue applies the row scales");
  static_assert(!W4 || (MODE & EPI_WSCALE) == 0, "INT4 weights: bf16 epilogue");
  constexpr bool RAW = W8 || W4;
  using Cfg = std::conditional_t<W4, SkW4Cfg<TA>, TgCfg<SK_BN, TA, W8>>;
  constexpr int STAGES = Cfg::kStages, STAGE_BYTES = Cfg::kStageBytes, A_BYTES = Cfg::kABytes, NCONS = 128 * Cfg::kWG;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* chunks = smem + STAGES * STAGE_BYTES + Cfg::kSlack;  // W4: the chunk ring
  uint64_t* full = reinterpret_cast<uint64_t*>(chunks + (W4 ? SK_W4_SLOTS * SK_W4_CHUNK_BYTES : 0));
  uint64_t* empty = full + STAGES;
  uint64_t* raw = empty + STAGES;  // W8: per stage; W4: chunk landed [SLOTS], chunk converted [SLOTS]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int G = (int)gridDim.x, cta = (int)blockIdx.x;
  if (GROUPED) pdl_wait();  // the routing plan (m tiles) is the preceding kernels' output
  const int num_m = GROUPED ? plan[0] : 1, num_n = p.N / SK_BN, num_k = p.K / TG_BK;
  const int32_t* tile_expert = GROUPED ? plan + MOE_PLAN_HEADER : nullptr;
  const int32_t* tile_row0 = GROUPED ? plan + MOE_PLAN_HEADER + plan[2] : nullptr;
  // unit u = (tile, k-block) = (u / num_k, u % num_k); CTA c owns units [first(c), first(c + 1))
  const long long total = (long long)num_m * num_n * num_k;
  const long long per = total / G, rem = total % G;
  auto first = [&](int c) { return (long long)c * per + (c < rem ? c : rem); };
  const long long u_begin = first(cta), u_end = first(cta + 1);

  if (threadIdx.x == 0) {
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full[i], RAW ? 1 + W8_CONVERTERS : 1);
      mbar_init(&empty[i], Cfg::kWG);
      if (W8) mbar_init(&raw[i], 1);
    }
    if (W4) {
      for (int i = 0; i < SK_W4_SLOTS; ++i) {
        mbar_init(&raw[i], 1);
        mbar_init(&raw[SK_W4_SLOTS + i], W8_CONVERTERS);
      }
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_a) : "memory");
  }
#ifdef MB200_SK_TRACE
  __shared__ unsigned trace_launch_slot;
  if (threadIdx.x == 32) trace_launch_slot = atomicAdd(&sk_trace_count, 1u) / gridDim.x;  // all CTAs of a launch start before any of the next
  volatile unsigned* trace_launch = &trace_launch_slot;
#endif
  __syncthreads();
  if (threadIdx.x == 0) {
    SK_STAMP(0);  // CTA set up
    pdl_trigger();
  }

  if (warp == 0) {
    // ================= TMA producer =================
    // Iteration `it` handles unit u_begin + it.  Weights are never written by any kernel: the W tiles of the first ring are
    // requested BEFORE the programmatic-dependent-launch wait (they stream in while the previous kernel drains); the A tiles of
    // those stages, which the previous kernel produced, follow after it.  Grouped: the tile list (and with it every weight
    // address) is the previous kernel's output, so nothing is requested before the wait at the top of the body.
    if (W4 && lane == 0) {
      const uint32_t n_it = (uint32_t)(u_end - u_begin);
      uint32_t issued = 0, next_it = 0;  // chunks requested; the first iteration of the next chunk
      auto issue_chunk = [&]() {
        const uint32_t u = (uint32_t)u_begin + next_it, slot = issued % SK_W4_SLOTS;
        const int tile = (int)(u / (uint32_t)num_k), kb = (int)(u % (uint32_t)num_k);
        mbar_arrive_expect_tx(&raw[slot], SK_W4_CHUNK_BYTES);
        if constexpr (GROUPED)
          tma_load_2d(chunks + slot * SK_W4_CHUNK_BYTES, map_w_base + tile_expert[tile % num_m], &raw[slot], kb * (TG_BK / 2),
                      (tile / num_m) * SK_BN);
        else
          tma_load_2d(chunks + slot * SK_W4_CHUNK_BYTES, map_w_base, &raw[slot], kb * (TG_BK / 2), tile * SK_BN);
        next_it += (uint32_t)min(min(SK_W4_CHUNK_KB, num_k - kb), (int)(n_it - next_it));
        ++issued;
      };
      auto chunk_free = [&](bool block) {  // slot of chunk `issued`: converted from its previous chunk
        uint64_t* bar = &raw[SK_W4_SLOTS + issued % SK_W4_SLOTS];
        const uint32_t par = ((issued / SK_W4_SLOTS) & 1) ^ 1;
        if (!block) return mbar_test_wait(bar, par);
        mbar_wait_quiet(bar, par);
        return true;
      };
      while (issued < (uint32_t)SK_W4_SLOTS && next_it < n_it) issue_chunk();  // weights: before the programmatic-dependent wait
      pdl_wait();
      SK_STAMP(1);
      for (uint32_t it = 0; it < n_it; ++it) {
        // the chunk holding unit `it` must be requested before this thread blocks on a stage (its slot's previous chunk only needs
        // units before `it`); later chunks as soon as their slots are free
        while (next_it <= it) {
          chunk_free(true);
          issue_chunk();
        }
        while (next_it < n_it && chunk_free(false)) issue_chunk();
        const uint32_t s = it % STAGES, par = (it / STAGES) & 1;
        mbar_wait_quiet(&empty[s], par ^ 1);
        mbar_arrive_expect_tx(&full[s], A_BYTES);
        const uint32_t u = (uint32_t)u_begin + it;
        tma_load_2d(smem + s * STAGE_BYTES, &map_a, &full[s], (int)(u % (uint32_t)num_k) * TG_BK,
                    GROUPED ? tile_row0[(u / (uint32_t)num_k) % (uint32_t)num_m] : 0);
      }
      SK_STAMP(3);
    } else if (lane == 0) {
      const uint32_t n_it = (uint32_t)(u_end - u_begin);
      auto issue = [&](uint32_t it, bool do_a, bool do_w) {
        const uint32_t u = (uint32_t)u_begin + it;
        const int tile = (int)(u / (uint32_t)num_k), kb = (int)(u % (uint32_t)num_k);
        const uint32_t s = it % STAGES;
        uint8_t* sa = smem + s * STAGE_BYTES;
        if (do_w) {
          const int n0 = (tile / num_m) * SK_BN;
          const CUtensorMap* wmap = GROUPED ? map_w_base + tile_expert[tile % num_m] : map_w_base;
          if (RAW) {
            mbar_arrive_expect_tx(&raw[s], Cfg::kRawBytes);
            tma_load_2d(sa + A_BYTES + Cfg::kBBytes, wmap, &raw[s], kb * (W4 ? TG_BK / 2 : TG_BK), n0);
          } else {
            tma_load_2d(sa + A_BYTES, wmap, &full[s], kb * TG_BK, n0);
          }
        }
        if (do_a) tma_load_2d(sa, &map_a, &full[s], kb * TG_BK, GROUPED ? tile_row0[tile % num_m] : 0);
      };
      const uint32_t head = GROUPED ? 0u : (n_it < (uint32_t)STAGES ? n_it : (uint32_t)STAGES);  // (grouped: the tile list itself is the previous kernel's output)
      for (uint32_t it = 0; it < head; ++it) {
        mbar_arrive_expect_tx(&full[it % STAGES], RAW ? A_BYTES : STAGE_BYTES);  // first lap: every slot is free
        issue(it, false, true);
      }
      pdl_wait();
      SK_STAMP(1);  // predecessor complete: A tiles may be requested
      for (uint32_t it = 0; it < head; ++it) issue(it, true, false);
      for (uint32_t it = head; it < n_it; ++it) {
        const uint32_t s = it % STAGES, par = (it / STAGES) & 1;
        mbar_wait_quiet(&empty[s], par ^ 1);
        mbar_arrive_expect_tx(&full[s], RAW ? A_BYTES : STAGE_BYTES);
        issue(it, true, true);
      }
      SK_STAMP(3);  // last tile requested
    }
  } else if (W4 && warp < 4) {
    // ================= INT4: the chunks' k-blocks -> the bf16 W' tile of every stage, in the producer's order =================
    const int ct = (int)threadIdx.x - 32, G = p.K / kInt4Group;
    const uint32_t n_it = (uint32_t)(u_end - u_begin);
    uint32_t chunk = 0, slot = 0;
    int pos = SK_W4_CHUNK_KB;
    for (uint32_t it = 0; it < n_it; ++it) {
      const uint32_t u = (uint32_t)u_begin + it;
      const int tile = (int)(u / (uint32_t)num_k), kb = (int)(u % (uint32_t)num_k);
      if (kb == 0 || pos == SK_W4_CHUNK_KB || it == 0) {  // the chunk boundaries of the producer's issue_chunk
        if (it != 0) mbar_arrive(&raw[SK_W4_SLOTS + slot]);
        slot = chunk % SK_W4_SLOTS;
        mbar_wait_quiet(&raw[slot], (chunk / SK_W4_SLOTS) & 1);
        ++chunk;
        pos = 0;
      }
      const uint32_t s = it % STAGES, par = (it / STAGES) & 1;
      mbar_wait_quiet(&empty[s], par ^ 1);  // the stage's previous W' tile has been read
      const uint16_t* gs = GROUPED ? gscales->s[tile_expert[tile % num_m]] + (int64_t)(tile / num_m) * SK_BN * G : gscale + (int64_t)tile * SK_BN * G;
      convert_w4_tile<SK_BN, SK_W4_CHUNK_KB * TG_BK / 2>(chunks + slot * SK_W4_CHUNK_BYTES + pos * (TG_BK / 2), smem + s * STAGE_BYTES + A_BYTES,
                                                         gs + kb / 2, G, ct);
      mbar_arrive(&full[s]);
      ++pos;
    }
  } else if (W8 && warp < 4) {
    // ================= FP8: e4m3 -> bf16 W' tile of every stage, in the producer's order =================
    const int ct = (int)threadIdx.x - 32;
    const uint32_t n_it = (uint32_t)(u_end - u_begin);
    for (uint32_t it = 0; it < n_it; ++it) {
      const int tile = (int)(((uint32_t)u_begin + it) / (uint32_t)num_k);
      const uint32_t s = it % STAGES, par = (it / STAGES) & 1;
      mbar_wait_quiet(&raw[s], par);
      uint8_t* sa = smem + s * STAGE_BYTES;
      if constexpr (GROUPED)
        convert_w8_tile<SK_BN>(sa + A_BYTES + Cfg::kBBytes, sa + A_BYTES, scales->s[tile_expert[tile % num_m]] + (tile / num_m) * SK_BN, ct);
      else
        convert_w8_tile<SK_BN, true>(sa + A_BYTES + Cfg::kBBytes, sa + A_BYTES, nullptr, ct);
      mbar_arrive(&full[s]);
    }
  } else if (warp >= 4) {
    // ================= consumer warpgroups: rows 64 * wg .. + 63 of the [TA x 128] tile =================
    if (!GROUPED) pdl_wait();  // stores below must not pass the predecessor's reads of the same buffers (returns at once when it is done)
    const int wg = (warp >> 2) - 1, wt = (int)threadIdx.x & 127, ct = (int)threadIdx.x - 128;  // ct: 0 .. NCONS-1
    const int r0 = wg * 64 + ((warp & 3) << 4) + (lane >> 2), c0 = 2 * (lane & 3);  // fragment rows r0, r0 + 8; columns c0 + 8j (+1)
    const bool row0_ok = r0 < TA, row1_ok = r0 + 8 < TA;  // accumulator rows >= TA come from beyond the short A box
    uint32_t it = 0;
    float acc[SK_BN / 2];
    for (long long u = u_begin; u < u_end;) {
      const int tile = (int)(u / num_k), kb0 = (int)(u % num_k);
      const int kb1 = (int)min((long long)num_k, kb0 + (u_end - u));
      const int m0 = GROUPED ? tile_row0[tile % num_m] : 0, n0 = (tile / num_m) * SK_BN;
      for (int kb = kb0; kb < kb1; ++kb, ++it) {
        const uint32_t s = it % STAGES, par = (it / STAGES) & 1;
        mbar_wait_quiet(&full[s], par);
#ifdef MB200_SK_TRACE
        if (it == 0 && ct == 0) SK_STAMP(2);  // first stage landed: first MMA
#endif
        const uint32_t a_addr = smem_u32(smem + s * STAGE_BYTES);
        wgmma_kblock<SK_BN>(acc, a_addr + wg * 64 * TG_BK * 2, a_addr + A_BYTES, kb == kb0);
        if (kb > kb0) {
          wgmma_wait<1>();
          if (wt == 0) mbar_arrive(&empty[(it - 1) % STAGES]);
        }
      }
      wgmma_wait<0>();
      wgmma_fence_acc(acc);
      if (wt == 0) mbar_arrive(&empty[(it - 1) % STAGES]);
#ifdef MB200_SK_TRACE
      if (ct == 0 && u + (kb1 - kb0) >= u_end) SK_STAMP(5);  // last accumulator complete
#endif
      // Split tiles.  A contributor that does not own the tile's first k-block parks its fp32 accumulator in its workspace slot;
      // the owner adds the slots in ascending k order, then its own accumulator, and runs the epilogue.
      const bool owner = kb0 == 0 && kb1 != num_k;
      if (kb0 != 0) {
        // ---- contributor: park the fp32 accumulator in this CTA's slot, then raise the flag ----
        float* mine = p.partials + (size_t)cta * TA * SK_BN;
#pragma unroll
        for (int j = 0; j < SK_BN / 8; ++j) {
          if (row0_ok) *reinterpret_cast<float2*>(mine + r0 * SK_BN + c0 + 8 * j) = make_float2(acc[4 * j], acc[4 * j + 1]);
          if (row1_ok) *reinterpret_cast<float2*>(mine + (r0 + 8) * SK_BN + c0 + 8 * j) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
        }
        __threadfence();
        asm volatile("bar.sync 2, %0;" ::"n"(NCONS) : "memory");
        if (ct == 0) st_release_u32(p.flags + cta, 1u);
      } else {
        if (owner) {
          // Contributors holding the tile's tail did it FIRST in their ranges; those whose whole range lies inside this tile
          // finish together with this CTA.  The flags are polled in parallel (one thread per contributor); then every thread adds
          // the contributors' slots to its fragment, one round trip to L2 per contributor.
          const long long tile_end = (long long)(tile + 1) * num_k;
          int last = cta;
          while (last + 1 < G && first(last + 1) < tile_end) ++last;
          for (int c = cta + 1 + ct; c <= last; c += NCONS) {
            unsigned spins = 0;
            while (ld_acquire_u32(p.flags + c) == 0u) {
              if (++spins == MB200_WATCHDOG_SPINS) __trap();  // no printf: see mbar_wait_quiet
            }
          }
          asm volatile("bar.sync 2, %0;" ::"n"(NCONS) : "memory");
#pragma unroll 1
          for (int c = cta + 1; c <= last; ++c) {  // ascending k order
            const float* slot = p.partials + (size_t)c * TA * SK_BN;
#pragma unroll
            for (int j = 0; j < SK_BN / 8; ++j) {
              if (row0_ok) {
                const float2 v = __ldcg(reinterpret_cast<const float2*>(slot + r0 * SK_BN + c0 + 8 * j));
                acc[4 * j] += v.x, acc[4 * j + 1] += v.y;
              }
              if (row1_ok) {
                const float2 v = __ldcg(reinterpret_cast<const float2*>(slot + (r0 + 8) * SK_BN + c0 + 8 * j));
                acc[4 * j + 2] += v.x, acc[4 * j + 3] += v.y;
              }
            }
          }
          asm volatile("bar.sync 2, %0;" ::"n"(NCONS) : "memory");
          if (ct == 0)
            for (int c = cta + 1; c <= last; ++c) p.flags[c] = 0u;  // consumed: ready for the next launch
        }
        // ---- the whole tile is in this accumulator: epilogue ----
        epi_fragment<MODE, SK_BN>(p.epi, acc, m0 + r0, n0, lane, min(p.T, m0 + TA));
      }
      u += kb1 - kb0;
    }
#ifdef MB200_SK_TRACE
    if (ct == 0) SK_STAMP(6);  // epilogues done
#endif
  }
#ifdef MB200_SK_TRACE
  __syncthreads();
  if (threadIdx.x == 0) SK_STAMP(7);  // exit
#endif
}

template <int MODE, int TA>
__global__ void __launch_bounds__(TgCfg<SK_BN, TA>::kThreads, 1)
    gemm_streamk_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_w, const SkParams p) {
  sk_gemm_body<MODE, TA, false>(map_a, &map_w, p, nullptr);
}

template <int MODE, int TA>
__global__ void __launch_bounds__(TgCfg<SK_BN, TA>::kThreads, 1)
    gemm_streamk_grouped_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ MoeWeightMaps maps_w, const SkParams p,
                                const int32_t* __restrict__ plan) {
  sk_gemm_body<MODE, TA, true>(map_a, maps_w.m, p, plan);
}

template <int MODE, int TA>
__global__ void __launch_bounds__(TgCfg<SK_BN, TA, true>::kThreads, 1)
    gemm_streamk_fp8_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_w, const SkParams p) {
  sk_gemm_body<MODE, TA, false, true>(map_a, &map_w, p, nullptr);
}

template <int MODE, int TA>
__global__ void __launch_bounds__(TgCfg<SK_BN, TA, false, true>::kThreads, 1)
    gemm_streamk_int4_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_w, const SkParams p,
                             const uint16_t* __restrict__ gscale) {
  sk_gemm_body<MODE, TA, false, false, true>(map_a, &map_w, p, nullptr, nullptr, gscale);
}

template <int MODE, int TA>
__global__ void __launch_bounds__(TgCfg<SK_BN, TA, true>::kThreads, 1)
    gemm_streamk_grouped_fp8_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ MoeWeightMaps maps_w,
                                    const __grid_constant__ MoeWeightScales scales, const SkParams p, const int32_t* __restrict__ plan) {
  sk_gemm_body<MODE, TA, true, true>(map_a, maps_w.m, p, plan, &scales);
}

// INT4 expert weights: maps_w are the experts' code matrices as uint8 [N, K/2] (box [128 x 128] bytes: one chunk), gscales their
// bf16 group scales [N, K/128].
template <int MODE, int TA>
__global__ void __launch_bounds__(TgCfg<SK_BN, TA, false, true>::kThreads, 1)
    gemm_streamk_grouped_int4_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ MoeWeightMaps maps_w,
                                     const __grid_constant__ MoeWeightGroupScales gscales, const SkParams p, const int32_t* __restrict__ plan) {
  sk_gemm_body<MODE, TA, true, false, true>(map_a, maps_w.m, p, plan, nullptr, nullptr, &gscales);
}

inline bool streamk_eligible(int64_t T, int64_t N, int64_t K) {
  const char* e = getenv("MB200_STREAMK");
  if (e != nullptr && e[0] == '0') return false;
  return T >= 1 && T <= 128 && N % SK_BN == 0 && K % TG_BK == 0;
}

// workspace: partial slots and flags where workspace.cuh puts them (both overlap scratch of other, stream-ordered entry points)
template <int MODE, int TA>
int launch_streamk_ta(const GemmParams& g, void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  using Cfg = TgCfg<SK_BN, TA>;
  int dev = 0, sms = 0;
  MB_CHECK_CUDA(cudaGetDevice(&dev));
  MB_CHECK_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  if (sms > SK_MAX_CTAS) sms = SK_MAX_CTAS;
  if (workspace == nullptr || workspace_bytes < kWsSkPartials.end()) return fail(MB200_E_WORKSPACE, "stream-K gemm: workspace %zu < %zu", workspace_bytes, kWsSkPartials.end());
  CUtensorMap map_a, map_w;
  int rc = make_tensor_map_2d(&map_a, g.a, g.T, g.K, TA);
  if (rc) return rc;
  rc = make_tensor_map_2d(&map_w, g.w, g.N, g.K, SK_BN);
  if (rc) return rc;
  SkParams p;
  p.T = g.T;
  p.N = g.N;
  p.K = g.K;
  p.epi = g.epi;
  p.partials = reinterpret_cast<float*>((uint8_t*)workspace + kWsSkPartials.offset);
  p.flags = reinterpret_cast<unsigned*>((uint8_t*)workspace + kWsSkFlags.offset);
  const long long units = (long long)(g.N / SK_BN) * (g.K / TG_BK);
  const int grid = (int)(units < sms ? units : sms);
  MB_CHECK_CUDA(cudaFuncSetAttribute(gemm_streamk_kernel<MODE, TA>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmem));
  MB_CHECK_CUDA(launch_pdl(gemm_streamk_kernel<MODE, TA>, dim3((unsigned)grid), dim3(Cfg::kThreads), (size_t)Cfg::kSmem, stream, map_a, map_w, p));
  note_launch("gemm_streamk_kernel<%d, %d>", MODE, TA);
  return MB200_OK;
}

template <int MODE>
int launch_streamk(const GemmParams& g, void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  if (g.T <= 32) return launch_streamk_ta<MODE, 32>(g, workspace, workspace_bytes, stream);
  if (g.T <= 64) return launch_streamk_ta<MODE, 64>(g, workspace, workspace_bytes, stream);
  return launch_streamk_ta<MODE, 128>(g, workspace, workspace_bytes, stream);
}

// FP8 dense weights (MODE carries EPI_WSCALE): the bf16 launcher's partition and workspace, an e4m3 weight map
template <int MODE, int TA>
int launch_streamk_fp8_ta(const GemmParams& g, void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  using Cfg = TgCfg<SK_BN, TA, true>;
  int dev = 0, sms = 0;
  MB_CHECK_CUDA(cudaGetDevice(&dev));
  MB_CHECK_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  if (sms > SK_MAX_CTAS) sms = SK_MAX_CTAS;
  if (workspace == nullptr || workspace_bytes < kWsSkPartials.end()) return fail(MB200_E_WORKSPACE, "stream-K gemm (fp8): workspace %zu < %zu", workspace_bytes, kWsSkPartials.end());
  CUtensorMap map_a, map_w;
  int rc = make_tensor_map_2d(&map_a, g.a, g.T, g.K, TA);
  if (rc) return rc;
  rc = make_tensor_map_e4m3(&map_w, g.w, g.N, g.K, SK_BN);
  if (rc) return rc;
  SkParams p;
  p.T = g.T;
  p.N = g.N;
  p.K = g.K;
  p.epi = g.epi;
  p.partials = reinterpret_cast<float*>((uint8_t*)workspace + kWsSkPartials.offset);
  p.flags = reinterpret_cast<unsigned*>((uint8_t*)workspace + kWsSkFlags.offset);
  const long long units = (long long)(g.N / SK_BN) * (g.K / TG_BK);
  const int grid = (int)(units < sms ? units : sms);
  MB_CHECK_CUDA(cudaFuncSetAttribute(gemm_streamk_fp8_kernel<MODE, TA>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmem));
  MB_CHECK_CUDA(launch_pdl(gemm_streamk_fp8_kernel<MODE, TA>, dim3((unsigned)grid), dim3(Cfg::kThreads), (size_t)Cfg::kSmem, stream, map_a, map_w, p));
  note_launch("gemm_streamk_fp8_kernel<%d, %d>", MODE, TA);
  return MB200_OK;
}

template <int MODE>
int launch_streamk_fp8(const GemmParams& g, void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  if (g.T <= 32) return launch_streamk_fp8_ta<MODE, 32>(g, workspace, workspace_bytes, stream);
  if (g.T <= 64) return launch_streamk_fp8_ta<MODE, 64>(g, workspace, workspace_bytes, stream);
  return launch_streamk_fp8_ta<MODE, 128>(g, workspace, workspace_bytes, stream);
}

// INT4 dense weights: the bf16 launcher's partition and workspace, a packed code map with chunk-wide boxes and the group scales
template <int MODE, int TA>
int launch_streamk_int4_ta(const GemmParams& g, const uint16_t* gscale, void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  using Cfg = SkW4Cfg<TA>;
  int dev = 0, sms = 0;
  MB_CHECK_CUDA(cudaGetDevice(&dev));
  MB_CHECK_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  if (sms > SK_MAX_CTAS) sms = SK_MAX_CTAS;
  if (workspace == nullptr || workspace_bytes < kWsSkPartials.end()) return fail(MB200_E_WORKSPACE, "stream-K gemm (int4): workspace %zu < %zu", workspace_bytes, kWsSkPartials.end());
  CUtensorMap map_a, map_w;
  int rc = make_tensor_map_2d(&map_a, g.a, g.T, g.K, TA);
  if (rc) return rc;
  rc = make_tensor_map_int4(&map_w, g.w, g.N, g.K, SK_BN, SK_W4_CHUNK_KB * TG_BK / 2);
  if (rc) return rc;
  SkParams p;
  p.T = g.T;
  p.N = g.N;
  p.K = g.K;
  p.epi = g.epi;
  p.partials = reinterpret_cast<float*>((uint8_t*)workspace + kWsSkPartials.offset);
  p.flags = reinterpret_cast<unsigned*>((uint8_t*)workspace + kWsSkFlags.offset);
  const long long units = (long long)(g.N / SK_BN) * (g.K / TG_BK);
  const int grid = (int)(units < sms ? units : sms);
  MB_CHECK_CUDA(cudaFuncSetAttribute(gemm_streamk_int4_kernel<MODE, TA>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmem));
  MB_CHECK_CUDA(launch_pdl(gemm_streamk_int4_kernel<MODE, TA>, dim3((unsigned)grid), dim3(Cfg::kThreads), (size_t)Cfg::kSmem, stream, map_a, map_w, p,
                           gscale));
  note_launch("gemm_streamk_int4_kernel<%d, %d>", MODE, TA);
  return MB200_OK;
}

template <int MODE>
int launch_streamk_int4(const GemmParams& g, const uint16_t* gscale, void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  if (g.T <= 32) return launch_streamk_int4_ta<MODE, 32>(g, gscale, workspace, workspace_bytes, stream);
  if (g.T <= 64) return launch_streamk_int4_ta<MODE, 64>(g, gscale, workspace, workspace_bytes, stream);
  return launch_streamk_int4_ta<MODE, 128>(g, gscale, workspace, workspace_bytes, stream);
}

}  // namespace mb200
