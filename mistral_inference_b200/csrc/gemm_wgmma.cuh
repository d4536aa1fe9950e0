// C[T, N] = A[T, K] * W[N, K]^T on the Hopper tensor cores: wgmma.mma_async with register accumulators, TMA-fed.
//
// Roofline: tensor pipe (2*T*N*K flops).  Persistent, warp-specialised kernel, one CTA per SM:
//   warpgroup 0     TMA producer (one thread): cp.async.bulk.tensor (128B-swizzled [TA x 64] A tile + [BN x 64] W tile per stage)
//                   -> 4- or 6-stage ring.  For T >= 512 the CTAs run as clusters of two on vertically adjacent tiles and each
//                   fetches half of the shared W tile, multicast into both shared memories (2/3 of the L2 -> SM traffic of the
//                   single-CTA kernel)
//   warpgroups 1-2  consumers: each issues wgmma (M = 64 rows of the tile, N = BN, K = 16 x 4 per stage) straight from the
//                   shared-memory stage, releases the stage once the next stage's MMAs are in flight, and after the last k-block
//                   runs the pair epilogues of epilogue.cuh (bf16 rounding, then RoPE + ring scatter / SiLU*mul / residual add /
//                   fp32 logits) on its register fragment.  Small-batch tiles (TA <= 64) have one consumer warpgroup.
// Both operands are K-major ([rows, K] row-major): the canonical TN GEMM, no transposes anywhere.
// Tiles are walked m-fastest so that the CTAs that share a W tile run together and hit it in L2.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_fp8.h>

#include <cstdlib>

#include "decode_megakernel.cuh"  // mbarrier helpers with the watchdog
#include "epilogue.cuh"
#include "gemm_mma.cuh"
#include "int4.cuh"
#include "wgmma.cuh"

namespace mb200 {

constexpr int TG_BM = 128, TG_BN = 256, TG_BK = 64;
// The tile width BN is 256 (4 stages of 48 KB), 192 (4 stages of 40 KB) or 128 (6 stages of 32 KB).  256 has the least W traffic
// per flop; 128 is chosen by the launcher for problems too small to give every SM a 256-wide tile (and for N that is a multiple
// of 128 only); 192 only for N that is a multiple of 192 but not of 128.
// TA = rows of the A (token) box.  128 for prefill.  For small batches (decode with 5..64 tokens) the box is 32 or 64 rows:
// the wgmma still has M = 64 and reads 8 KB from the A tile's base, i.e. with a 32-row box it runs into the W tile that follows
// it in the stage -- accumulator row i depends on A row i only, and rows >= TA are never stored.  The stage shrinks to
// (TA + BN) * 128 bytes, so the ring gets deep enough to keep a whole SM's share of HBM bandwidth in flight: those launches are
// weight-streaming GEMMs, bound by HBM, with BN chosen by the launcher to give every SM at most one (equal) tile per round.
// W8 (FP8 expert weights, csrc/moe.cuh): a stage also holds the e4m3 [BN x 64] W tile as TMA delivered it (kRawBytes, unswizzled)
// next to the bf16 tile the MMAs read, which the producer warpgroup's three idle warps write from it (convert_w8_tile).
// W4 (INT4 dense and expert weights): the same arrangement with the packed [BN x 32-byte] code tile as the raw area (convert_w4_tile).
template <int BN, int TA = 128, bool W8 = false, bool W4 = false>
struct TgCfg {
  static_assert(!(W8 && W4), "one weight format per stage");
  static constexpr int kABytes = TA * TG_BK * 2;
  static constexpr int kBBytes = BN * TG_BK * 2;
  static constexpr int kRawBytes = W8 ? BN * TG_BK : (W4 ? BN * TG_BK / 2 : 0);
  static constexpr int kStageBytes = kABytes + kBBytes + kRawBytes;
  static constexpr int kWG = TA > 64 ? 2 : 1;  // consumer warpgroups: 64 accumulator rows each
  static constexpr int kThreads = 128 * (1 + kWG);
  // A wgmma reads 64 rows (8 KB) from a stage's A base; in the LAST stage that must not run past the ring
  static constexpr int kSlack = kStageBytes < 64 * TG_BK * 2 ? 64 * TG_BK * 2 - kStageBytes : 0;
  static constexpr int kMaxStages = (227 * 1024 - 1024 - 512 - kSlack) / kStageBytes;
  // decode-sized variants: a ring of ~100 KB (80 KB of weights in flight per CTA, above the bandwidth-delay product of one SM's
  // share of HBM) instead of the whole 227 KB: a successor's CTA, which starts when the predecessor's CTA on its SM exits, has its
  // first ring filled sooner, and other decode kernels' CTAs fit beside it.  W8: an e4m3 stage carries half the HBM bytes of a
  // bf16 one and needs the bf16 tile beside it, so its ring is twice as long to keep the same bytes in flight.
  static constexpr int kShortRingStages = ((W8 || W4 ? 200 : 100) * 1024) / kStageBytes;
  static constexpr int kStages = (TA < 128 || BN < 128) ? (kShortRingStages < 3 ? 3 : (kShortRingStages > kMaxStages ? kMaxStages : kShortRingStages))
                                                        : (W8 || W4) ? kMaxStages : (BN == 128 ? 6 : 4);
  static constexpr int kSmem = kStages * kStageBytes + kSlack + 1024 /*align*/ + 512 /*barriers*/;
  static_assert(kSmem <= 227 * 1024, "shared memory plan exceeds the 227 KB of an sm_90 block");
};

struct TcGemmParams {
  int T, N, K;
  EpiParams epi;
};

// ---- PTX wrappers ---------------------------------------------------------------------------------
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(smem_u32(smem_dst)),
               "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
               : "memory");
}
// Same, delivered to the same shared-memory offset (and signalled on the same barrier offset) of every CTA in cta_mask.
__device__ __forceinline__ void tma_load_2d_multicast(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, uint16_t cta_mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, %4}], [%2], %5;" ::"r"(
          smem_u32(smem_dst)),
      "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "h"(cta_mask)
      : "memory");
}
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// arrive on the barrier at this shared-memory offset in CTA `cta` of the cluster
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t* bar, uint32_t cta) {
  uint32_t remote;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(smem_u32(bar)), "r"(cta));
  asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(remote) : "memory");
}

// ---- FP8 expert weights: e4m3 tile -> the bf16 W' tile of the stage ----------------------------------------------------------
// W'[n, k] = bf16_rn(fp32(float(q[n, k]) * s[n])): e4m3 -> f16 is exact (cvt.rn.f16x2.e4m3x2), f16 -> f32 exact, one IEEE fp32
// multiply, one bf16 rounding -- the same bits as the CPU restatement in oracle/fp8.py.  The bf16 tile is written in the 128B-swizzled
// layout TMA gives the bf16 kernels (16-byte chunk c of row r at chunk c ^ (r & 7)), so the wgmma descriptors are unchanged.
// Thread ct of W8_CONVERTERS takes 16-byte e4m3 chunks ct, ct + W8_CONVERTERS, ...: consecutive threads read consecutive 16 bytes,
// and each quarter warp's 16-byte stores hit 8 distinct chunk columns of two rows (no bank conflicts).
// DENSE (FP8 dense weights, include/mistral_b200.h): the tile is q itself, converted exactly (e4m3x2_to_float2, then a bf16 pack
// that cannot round: no multiply); the row scale is applied to the accumulator in the epilogue (EPI_WSCALE) and scale_rows is unused.
constexpr int W8_CONVERTERS = 96;  // warps 1-3 of the producer warpgroup
template <int BN, bool DENSE = false>
__device__ __forceinline__ void convert_w8_tile(const uint8_t* raw, uint8_t* wtile, const float* __restrict__ scale_rows, int ct) {
#pragma unroll 2
  for (int q = ct; q < BN * (TG_BK / 16); q += W8_CONVERTERS) {
    const int row = q >> 2, c = q & 3;
    const uint4 v = *reinterpret_cast<const uint4*>(raw + row * TG_BK + c * 16);
    const uint32_t in[4] = {v.x, v.y, v.z, v.w};
    uint32_t o[8];
    if constexpr (DENSE) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float2 f = e4m3x2_to_float2(in[j >> 1] >> (16 * (j & 1)));
        o[j] = pack2_rn(f.x, f.y);
      }
    } else {
    const float s = __ldg(scale_rows + row);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const __half2_raw hr = __nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)(in[j >> 1] >> (16 * (j & 1))), __NV_E4M3);
      const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&hr));
      const __nv_bfloat162 b = __floats2bfloat162_rn(__fmul_rn(f.x, s), __fmul_rn(f.y, s));
      o[j] = *reinterpret_cast<const uint32_t*>(&b);
    }
    }
    uint8_t* dst = wtile + row * (TG_BK * 2);
    *reinterpret_cast<uint4*>(dst + (((2 * c) ^ (row & 7)) << 4)) = make_uint4(o[0], o[1], o[2], o[3]);
    *reinterpret_cast<uint4*>(dst + (((2 * c + 1) ^ (row & 7)) << 4)) = make_uint4(o[4], o[5], o[6], o[7]);
  }
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy stores -> the wgmma (async proxy) reads
}

// ---- INT4 dense weights: packed code tile -> the bf16 W' tile of the stage -----------------------------------------------------
// raw = [BN rows x 32 bytes] (64 codes of k-block kb per row, as stored; rows RS bytes apart: 32 for a one-k-block tile, 128 for a
// k-block inside stream-K's four-k-block chunk), gs = the scale of row 0's group of this k-block, row r's at gs[r * G].  W' comes from int4x8_to_bf16x2 (int4.cuh), so the tile holds exactly the bf16 weights the contract names and the MMAs,
// descriptors and epilogue are the bf16 kernel's.  Thread ct takes 16-byte code chunks ct, ct + W8_CONVERTERS, ... (32 codes: four
// swizzled 16-byte bf16 chunks of one row); a quarter warp's stores hit 8 distinct chunk columns of four rows.
template <int BN, int RS = TG_BK / 2>
__device__ __forceinline__ void convert_w4_tile(const uint8_t* raw, uint8_t* wtile, const uint16_t* __restrict__ gs, int G, int ct) {
#pragma unroll 2
  for (int q = ct; q < BN * 2; q += W8_CONVERTERS) {
    const int row = q >> 1, c = q & 1;
    const uint4 v = *reinterpret_cast<const uint4*>(raw + row * RS + c * 16);
    const uint32_t s2 = (uint32_t)__ldg(gs + (int64_t)row * G) * 0x10001u;
    const uint32_t in[4] = {v.x, v.y, v.z, v.w};
    uint8_t* dst = wtile + row * (TG_BK * 2);
#pragma unroll
    for (int h = 0; h < 4; ++h) {
      uint32_t o[4];
      int4x8_to_bf16x2<true>(in[h], s2, o);
      *reinterpret_cast<uint4*>(dst + (((4 * c + h) ^ (row & 7)) << 4)) = make_uint4(o[0], o[1], o[2], o[3]);
    }
  }
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy stores -> the wgmma (async proxy) reads
}

// One consumer warpgroup's share of a k-block: the 64 tile rows starting at a_addr against the whole [BN x 64] W tile.
template <int BN>
__device__ __forceinline__ void wgmma_kblock(float (&acc)[BN / 2], uint32_t a_addr, uint32_t b_addr, bool first) {
  const uint64_t adesc = wgmma_desc_sw128(a_addr), bdesc = wgmma_desc_sw128(b_addr);
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < TG_BK / 16; ++k)  // +32 bytes (= 2 in 16-byte units) per K = 16 step inside the 128-byte swizzled row
    wgmma_ss(acc, adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k), (first && k == 0) ? 0u : 1u);
  wgmma_commit();
}

// Pair epilogues on a consumer's accumulator fragment (rows r0 and r0 + 8 of the tile, see wgmma.cuh); rows >= limit are not stored.
template <int MODE, int BN>
__device__ __forceinline__ void epi_fragment(const EpiParams& epi, const float (&acc)[BN / 2], int t0, int n0, int lane, int limit) {
  const int nc = n0 + 2 * (lane & 3);
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    if (t0 < limit) epi_pair<MODE>(epi, t0, nc + 8 * j, acc[4 * j], acc[4 * j + 1]);
    if (t0 + 8 < limit) epi_pair<MODE>(epi, t0 + 8, nc + 8 * j, acc[4 * j + 2], acc[4 * j + 3]);
  }
}

// Tile order of the persistent GEMMs.  The persistent CTAs take tiles t = cta, cta + n_cta, ...: at any moment ~n_cta consecutive
// tile ids are in flight, in lock step through K.  With few m units the walk is m-fastest: the CTAs that share a W tile run together.
// With many (a 32 x 1024-token prefill: A = 335 MB; a Mixtral prefill: hundreds of MB of gathered rows, far beyond the 50 MB L2)
// m-fastest makes every CTA stream its own A tile from DRAM once per n tile.  There the in-flight set is shaped as a GM x GN block
// instead (GM m units share each W tile, GN n tiles share each A tile): DRAM traffic per tile drops ~4x.
template <int kGM, int kGN>
__device__ __forceinline__ void tile_walk_mn(int tile, int num_m, int num_n, int& mu, int& nt) {
  if (num_m <= 16) {
    mu = tile % num_m;
    nt = tile / num_m;
    return;
  }
  const int per_row = kGN * num_m, rows_full = num_n / kGN;  // an "n-block row": all m units x kGN n tiles
  int nb, r, gn;
  if (tile < rows_full * per_row) {
    nb = tile / per_row;
    r = tile % per_row;
    gn = kGN;
  } else {
    nb = rows_full;
    r = tile - rows_full * per_row;
    gn = num_n - rows_full * kGN;
  }
  const int blk = kGM * gn, mb_full = num_m / kGM;
  int mblk, q, gm;
  if (r < mb_full * blk) {
    mblk = r / blk;
    q = r % blk;
    gm = kGM;
  } else {
    mblk = mb_full;
    q = r - mb_full * blk;
    gm = num_m - mb_full * kGM;
  }
  mu = mblk * kGM + q % gm;
  nt = nb * kGN + q / gm;
}

// CL = 2: thread-block clusters of two CTAs that work on vertically adjacent tiles (same W columns, consecutive 128-row blocks).
// Each CTA fetches HALF of the shared [256 x 64] W tile and TMA-multicasts it into both shared memories, so the L2 -> SM traffic
// per CTA and k-block drops from 48 KB to 32 KB.  A stage may be refilled only when BOTH CTAs' consumers have read it: the empty
// barriers count one arrival per consumer warpgroup of the pair.
//
// GROUPED = true (mixture of experts, csrc/moe.cuh): the A rows are the (token, expert) pairs sorted by expert, every expert's
// segment padded to a multiple of TA rows; m tile i covers rows plan.tile_row0[i] .. + TA of expert plan.tile_expert[i], whose
// weight matrix has its own tensor map (map_w[expert]).  The number of m tiles is DEVICE data (no host sync after routing).
constexpr int MOE_PLAN_HEADER = 64;  // int32 words: [0] m tiles of this rank, [1] padded rows in total, [2] tile capacity, [6] tile pairs, [8..] segment starts
// after the header: tile_expert[cap], tile_row0[cap], pair_expert[cap], pair_info[cap] (cap = plan[2]).  A PAIR is two vertically
// adjacent m tiles of ONE expert (or a single last tile: bit 30 of pair_info clear), the unit of the 2-CTA cluster variant.
constexpr int MOE_PAIR_SECOND = 1 << 30;
constexpr int MOE_MAX_EXPERTS = 16;  // tensor maps travel as kernel parameters (128 B each)
struct MoeWeightMaps {
  CUtensorMap m[MOE_MAX_EXPERTS];
};
struct MoeWeightScales {  // W8: per-row fp32 scales of each expert's matrix (null for experts of other ranks)
  const float* s[MOE_MAX_EXPERTS];
};
struct MoeWeightGroupScales {  // W4: bf16 group scales [N, K/128] of each expert's code matrix (null for experts of other ranks)
  const uint16_t* s[MOE_MAX_EXPERTS];
};

// W8 (single CTA only): the producer thread loads the e4m3 W tile into the stage's raw area on raw[s]; warps 1-3 wait on raw[s],
// write the bf16 tile and arrive on full[s] (W8_CONVERTERS arrivals next to the producer's expect_tx for the A tile).  Grouped:
// the experts' W' tiles (§3.9); dense: the exact q tiles, the row scales applied by the epilogue (MODE carries EPI_WSCALE).
// W4 (single CTA only): the same with the packed INT4 code tile and its group scales (bf16 bits [N, K/128]: gscale when dense,
// gscales->s[expert] of the tile's expert when grouped); the converter warps write W' itself, so the epilogue is the bf16 kernel's.
template <int MODE, int CL, int BN, int TA, bool GROUPED, bool W8 = false, bool W4 = false>
__device__ __forceinline__ void tc_gemm_body(const CUtensorMap& map_a, const CUtensorMap* map_w_base, const TcGemmParams& p, const int32_t* plan,
                                             const MoeWeightScales* scales = nullptr, const uint16_t* gscale = nullptr,
                                             const MoeWeightGroupScales* gscales = nullptr) {
  static_assert(TA == 128 || CL == 1, "small-batch variant is single-CTA");
  static_assert(!W8 || CL == 1, "FP8 weights: single-CTA variant only");
  static_assert(!W8 || GROUPED || (MODE & EPI_WSCALE) != 0, "FP8 dense weights: the epilogue applies the row scales");
  static_assert(!W4 || (CL == 1 && (MODE & EPI_WSCALE) == 0), "INT4 weights: single-CTA variant, bf16 epilogue");
  constexpr bool RAW = W8 || W4;  // W tiles land in the raw area and are converted by warps 1-3
  using Cfg = TgCfg<BN, TA, W8, W4>;
  constexpr int STAGES = Cfg::kStages, B_BYTES = Cfg::kBBytes, STAGE_BYTES = Cfg::kStageBytes, A_BYTES = Cfg::kABytes;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);  // SW128 wants 1024-B tiles
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES + Cfg::kSlack);
  uint64_t* empty = full + STAGES;
  uint64_t* raw = empty + STAGES;  // W8 / W4 only

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int rank = CL > 1 ? (int)cluster_ctarank() : 0;
  const int cta = (int)blockIdx.x / CL, n_cta = (int)gridDim.x / CL;  // cluster index / clusters in the grid
  // a cluster walks "super tiles" of CL vertically adjacent tiles; rows past T read as zeros (TMA) and are never stored
  // grouped: m units are the plan's tiles (single CTA) or tile pairs (cluster of two)
  const int num_m = GROUPED ? (CL > 1 ? plan[6] : plan[0]) : ((p.T + TG_BM - 1) / TG_BM + CL - 1) / CL;
  const int num_n = p.N / BN, num_tiles = num_m * num_n, num_k = p.K / TG_BK;
  const int32_t* tile_expert = GROUPED ? plan + MOE_PLAN_HEADER + (CL > 1 ? 2 * plan[2] : 0) : nullptr;
  const int32_t* tile_row0 = GROUPED ? tile_expert + plan[2] : nullptr;
  constexpr int kGM = CL > 1 ? 8 : 12, kGN = CL > 1 ? 9 : 12;
  auto tile_mn = [&](int tile, int& mu, int& nt) { tile_walk_mn<kGM, kGN>(tile, num_m, num_n, mu, nt); };
  // first row of this CTA's m tile of unit `u` (cluster rank 1 takes the pair's second tile; a missing second tile is recomputed
  // from the first one's rows and not stored)
  auto grouped_m0 = [&](int u, bool& store) {
    const int info = tile_row0[u];
    store = true;
    if (CL == 1) return info;
    const int row0 = info & (MOE_PAIR_SECOND - 1);
    if (rank == 0) return row0;
    store = (info & MOE_PAIR_SECOND) != 0;
    return store ? row0 + TG_BM : row0;
  };
  const CUtensorMap& map_w = *map_w_base;

  if (threadIdx.x == 0) {
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full[i], RAW ? 1 + W8_CONVERTERS : 1);
      mbar_init(&empty[i], CL * Cfg::kWG);
      if (RAW) mbar_init(&raw[i], 1);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_a) : "memory");
    if (!GROUPED) asm volatile("prefetch.tensormap [%0];" ::"l"(&map_w) : "memory");
  }
  if (CL > 1)
    cluster_sync_all();  // the peer's barriers must be initialised before any multicast copy or remote arrival reaches them
  else
    __syncthreads();

  if (warp == 0) {
    // ================= TMA producer =================
    if (lane == 0) {
      uint32_t it = 0;
      for (int tile = cta; tile < num_tiles; tile += n_cta) {
        bool store_unused;
        int mu, nt;
        tile_mn(tile, mu, nt);
        const int m0 = GROUPED ? grouped_m0(mu, store_unused) : (mu * CL + rank) * TG_BM, n0 = nt * BN;
        const CUtensorMap* wmap = GROUPED ? map_w_base + tile_expert[mu] : map_w_base;
        for (int kb = 0; kb < num_k; ++kb, ++it) {
          const uint32_t s = it % STAGES, par = (it / STAGES) & 1;
          mbar_wait_quiet(&empty[s], par ^ 1);
          uint8_t* sa = smem + s * STAGE_BYTES;
          if constexpr (RAW) {
            mbar_arrive_expect_tx(&full[s], A_BYTES);
            tma_load_2d(sa, &map_a, &full[s], kb * TG_BK, m0);
            mbar_arrive_expect_tx(&raw[s], Cfg::kRawBytes);
            tma_load_2d(sa + A_BYTES + B_BYTES, wmap, &raw[s], kb * (W4 ? TG_BK / 2 : TG_BK), n0);
            continue;
          }
          mbar_arrive_expect_tx(&full[s], STAGE_BYTES);  // A + both halves of W (the peer's half may land first: tx-count goes negative)
          tma_load_2d(sa, &map_a, &full[s], kb * TG_BK, m0);
          if (CL > 1)
            tma_load_2d_multicast(sa + A_BYTES + rank * (B_BYTES / CL), wmap, &full[s], kb * TG_BK, n0 + rank * (BN / CL),
                                  (uint16_t)((1u << CL) - 1));
          else
            tma_load_2d(sa + A_BYTES, wmap, &full[s], kb * TG_BK, n0);
        }
      }
    }
  } else if (RAW && warp < 4) {
    // ================= FP8 / INT4: raw W tile -> bf16 tile of every stage, in the producer's order =================
    const int ct = (int)threadIdx.x - 32;
    uint32_t it = 0;
    for (int tile = cta; tile < num_tiles; tile += n_cta) {
      int mu, nt;
      tile_mn(tile, mu, nt);
      const float* srows = GROUPED && W8 ? scales->s[tile_expert[mu]] + nt * BN : nullptr;
      for (int kb = 0; kb < num_k; ++kb, ++it) {
        const uint32_t s = it % STAGES, par = (it / STAGES) & 1;
        mbar_wait_quiet(&raw[s], par);
        uint8_t* sa = smem + s * STAGE_BYTES;
        if constexpr (W4 && GROUPED) {
          const int G = p.K / kInt4Group;
          convert_w4_tile<BN>(sa + A_BYTES + B_BYTES, sa + A_BYTES, gscales->s[tile_expert[mu]] + (int64_t)nt * BN * G + kb / 2, G, ct);
        } else if constexpr (W4) {
          const int G = p.K / kInt4Group;
          convert_w4_tile<BN>(sa + A_BYTES + B_BYTES, sa + A_BYTES, gscale + (int64_t)nt * BN * G + kb / 2, G, ct);
        } else {
          convert_w8_tile<BN, !GROUPED>(sa + A_BYTES + B_BYTES, sa + A_BYTES, srows, ct);
        }
        mbar_arrive(&full[s]);
      }
    }
  } else if (warp >= 4) {
    // ================= consumer warpgroups: rows 64 * wg .. + 63 of the tile =================
    const int wg = (warp >> 2) - 1, wt = (int)threadIdx.x & 127;
    const int row_in_tile = wg * 64 + ((warp & 3) << 4) + (lane >> 2);  // fragment rows row_in_tile and row_in_tile + 8
    auto release = [&](uint32_t s) {
      if (wt == 0) {
        if (CL > 1) {
          for (uint32_t c = 0; c < (uint32_t)CL; ++c) mbar_arrive_cluster(&empty[s], c);
        } else {
          mbar_arrive(&empty[s]);
        }
      }
    };
    uint32_t it = 0;
    float acc[BN / 2];
    for (int tile = cta; tile < num_tiles; tile += n_cta) {
      bool store = true;
      int mu, nt;
      tile_mn(tile, mu, nt);
      const int m0 = GROUPED ? grouped_m0(mu, store) : (mu * CL + rank) * TG_BM, n0 = nt * BN;
      for (int kb = 0; kb < num_k; ++kb, ++it) {
        const uint32_t s = it % STAGES, par = (it / STAGES) & 1;
        mbar_wait_quiet(&full[s], par);
        const uint32_t a_addr = smem_u32(smem + s * STAGE_BYTES) + wg * 64 * TG_BK * 2;
        wgmma_kblock<BN>(acc, a_addr, smem_u32(smem + s * STAGE_BYTES) + A_BYTES, kb == 0);
        if (kb > 0) {  // the previous k-block's MMAs have read their stage
          wgmma_wait<1>();
          release((it - 1) % STAGES);
        }
      }
      wgmma_wait<0>();
      wgmma_fence_acc(acc);
      release((it - 1) % STAGES);
      // accumulator rows >= TA were computed from whatever follows the short A box in shared memory: never stored
      const int limit = store ? min(p.T, m0 + TA) : 0;
      epi_fragment<MODE, BN>(p.epi, acc, m0 + row_in_tile, n0, lane, limit);
    }
  }
  if (CL > 1) cluster_sync_all();  // the peer's last remote arrivals still reach this CTA's barriers
}

template <int MODE, int CL, int BN, int TA = 128>
__global__ void __launch_bounds__(TgCfg<BN, TA>::kThreads, 1)
    gemm_wgmma_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_w, const TcGemmParams p) {
  tc_gemm_body<MODE, CL, BN, TA, false>(map_a, &map_w, p, nullptr);
}

template <int MODE, int CL, int BN, int TA>
__global__ void __launch_bounds__(TgCfg<BN, TA>::kThreads, 1)
    gemm_wgmma_grouped_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ MoeWeightMaps maps_w, const TcGemmParams p,
                              const int32_t* __restrict__ plan) {
  tc_gemm_body<MODE, CL, BN, TA, true>(map_a, maps_w.m, p, plan);
}

// FP8 dense weights: map_w is an e4m3 [N, K] map (box [BN x 64] bytes, no swizzle); MODE carries EPI_WSCALE.
template <int MODE, int BN, int TA>
__global__ void __launch_bounds__(TgCfg<BN, TA, true>::kThreads, 1)
    gemm_wgmma_fp8_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_w, const TcGemmParams p) {
  tc_gemm_body<MODE, 1, BN, TA, false, true>(map_a, &map_w, p, nullptr);
}

// INT4 dense weights: map_w is the packed code matrix as uint8 [N, K/2] (box [BN x 32] bytes, no swizzle), gscale its group scales.
template <int MODE, int BN, int TA>
__global__ void __launch_bounds__(TgCfg<BN, TA, false, true>::kThreads, 1)
    gemm_wgmma_int4_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_w, const TcGemmParams p,
                           const uint16_t* __restrict__ gscale) {
  tc_gemm_body<MODE, 1, BN, TA, false, false, true>(map_a, &map_w, p, nullptr, nullptr, gscale);
}

// FP8 expert weights: maps_w are e4m3 [N, K] maps (box [BN x 64] bytes, no swizzle), scales the per-row fp32 scales.
template <int MODE, int BN, int TA>
__global__ void __launch_bounds__(TgCfg<BN, TA, true>::kThreads, 1)
    gemm_wgmma_grouped_fp8_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ MoeWeightMaps maps_w,
                                  const __grid_constant__ MoeWeightScales scales, const TcGemmParams p, const int32_t* __restrict__ plan) {
  tc_gemm_body<MODE, 1, BN, TA, true, true>(map_a, maps_w.m, p, plan, &scales);
}

// INT4 expert weights: maps_w are the experts' packed code matrices as uint8 [N, K/2] (box [BN x 32] bytes, no swizzle), gscales
// their bf16 group scales [N, K/128].
template <int MODE, int BN, int TA>
__global__ void __launch_bounds__(TgCfg<BN, TA, false, true>::kThreads, 1)
    gemm_wgmma_grouped_int4_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ MoeWeightMaps maps_w,
                                   const __grid_constant__ MoeWeightGroupScales gscales, const TcGemmParams p, const int32_t* __restrict__ plan) {
  tc_gemm_body<MODE, 1, BN, TA, true, false, true>(map_a, maps_w.m, p, plan, nullptr, nullptr, &gscales);
}

// ---- host: tensor maps (driver API through the runtime's entry-point lookup, no libcuda link dependency) ----
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                    const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline PFN_encodeTiled get_encode_tiled() {
  static PFN_encodeTiled fn = nullptr;
  if (fn == nullptr) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess && qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(ptr);
  }
  return fn;
}

// [rows, K] bf16 row-major, box = [box_rows x 64] elements, 128-byte swizzle, out-of-range rows read as zero
inline int make_tensor_map_2d(CUtensorMap* map, const void* base, int64_t rows, int64_t K, int box_rows) {
  PFN_encodeTiled enc = get_encode_tiled();
  if (enc == nullptr) return fail(MB200_E_CUDA, "cuTensorMapEncodeTiled entry point not available");
  const cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)rows};
  const cuuint64_t strides[1] = {(cuuint64_t)K * 2};
  const cuuint32_t box[2] = {(cuuint32_t)TG_BK, (cuuint32_t)box_rows};
  const cuuint32_t estr[2] = {1, 1};
  const CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                         CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(MB200_E_CUDA, "cuTensorMapEncodeTiled failed (%d) rows=%lld K=%lld", (int)r, (long long)rows, (long long)K);
  return MB200_OK;
}

// [rows, K] e4m3 (one byte per element), box = [box_rows x 64] bytes, unswizzled: the raw tile that convert_w8_tile reads
inline int make_tensor_map_e4m3(CUtensorMap* map, const void* base, int64_t rows, int64_t K, int box_rows) {
  PFN_encodeTiled enc = get_encode_tiled();
  if (enc == nullptr) return fail(MB200_E_CUDA, "cuTensorMapEncodeTiled entry point not available");
  const cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)rows};
  const cuuint64_t strides[1] = {(cuuint64_t)K};
  const cuuint32_t box[2] = {(cuuint32_t)TG_BK, (cuuint32_t)box_rows};
  const cuuint32_t estr[2] = {1, 1};
  const CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                         CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(MB200_E_CUDA, "cuTensorMapEncodeTiled (e4m3) failed (%d) rows=%lld K=%lld", (int)r, (long long)rows, (long long)K);
  return MB200_OK;
}

// INT4 codes as uint8 [rows, K/2], box = [box_rows x box_bytes] (32: one k-block of 64 codes; 128: stream-K's chunk of four),
// unswizzled: the raw tile that convert_w4_tile reads; columns past K/2 read as zero
inline int make_tensor_map_int4(CUtensorMap* map, const void* base, int64_t rows, int64_t K, int box_rows, int box_bytes = TG_BK / 2) {
  PFN_encodeTiled enc = get_encode_tiled();
  if (enc == nullptr) return fail(MB200_E_CUDA, "cuTensorMapEncodeTiled entry point not available");
  const cuuint64_t dims[2] = {(cuuint64_t)(K / 2), (cuuint64_t)rows};
  const cuuint64_t strides[1] = {(cuuint64_t)(K / 2)};
  const cuuint32_t box[2] = {(cuuint32_t)box_bytes, (cuuint32_t)box_rows};
  const cuuint32_t estr[2] = {1, 1};
  const CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                         CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(MB200_E_CUDA, "cuTensorMapEncodeTiled (int4) failed (%d) rows=%lld K=%lld", (int)r, (long long)rows, (long long)K);
  return MB200_OK;
}

inline bool wgmma_gemm_eligible(int64_t T, int64_t N, int64_t K) {
  if (K % TG_BK != 0) return false;
  if (T >= TG_BM) return N % 128 == 0 || N % 192 == 0;
  return N % 32 == 0;  // small-batch weight-streaming variant (T <= 64 uses short A boxes; 65..127 the 128-row box)
}

// MB200_GEMM_CLUSTER=0 forces the single-CTA kernel; MB200_GEMM_BN=128|192|256 forces the tile width.  Read at every launch
// (a getenv is ~100 ns) so the tests can switch variants inside one process.
inline bool wgmma_cluster_enabled() {
  const char* e = getenv("MB200_GEMM_CLUSTER");
  return !(e != nullptr && e[0] == '0');
}
inline int wgmma_forced_bn() {
  const char* e = getenv("MB200_GEMM_BN");
  return e != nullptr ? atoi(e) : 0;
}

// The prefill tile width (T >= 128) for every weight format: the quantised launchers run single CTAs where bf16 runs clusters of
// two (pair), but take the BN that bf16 takes, so each tile sums the same k-blocks in the same order.  128-wide tiles only when
// 256-wide ones cannot fill the machine once (small T or N): per flop a narrow tile pulls 1.5x the bytes out of L2.  192-wide
// tiles are used for N that is a multiple of 192 only (and by the tests).  MB200_GEMM_BN overrides when it divides N.
inline int wgmma_prefill_bn(int T, int N, bool pair, int sms) {
  const int units = pair ? sms / 2 : sms, m_units = pair ? ceil_div(ceil_div(T, TG_BM), 2) : ceil_div(T, TG_BM);
  int bn = 256;
  if (N % 256 != 0 || (int64_t)m_units * (N / 256) < units) {
    bn = N % 128 == 0 ? 128 : 192;
  }
  const int forced = wgmma_forced_bn();
  if ((forced == 128 || forced == 192 || forced == 256) && N % forced == 0) bn = forced;
  return bn;
}

template <int MODE, int BN>
int launch_gemm_wgmma_bn(const GemmParams& g, bool pair, int sms, cudaStream_t stream) {
  using Cfg = TgCfg<BN>;
  CUtensorMap map_a, map_w;
  int rc = make_tensor_map_2d(&map_a, g.a, g.T, g.K, TG_BM);
  if (rc) return rc;
  rc = make_tensor_map_2d(&map_w, g.w, g.N, g.K, pair ? BN / 2 : BN);
  if (rc) return rc;
  TcGemmParams p;
  p.T = g.T;
  p.N = g.N;
  p.K = g.K;
  p.epi = g.epi;
  if (pair) {
    const int supers = ceil_div(ceil_div(g.T, TG_BM), 2) * (g.N / BN), pairs = sms / 2;
    MB_CHECK_CUDA(cudaFuncSetAttribute(gemm_wgmma_kernel<MODE, 2, BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmem));
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(2u * (unsigned)(supers < pairs ? supers : pairs));
    cfg.blockDim = dim3(Cfg::kThreads);
    cfg.dynamicSmemBytes = Cfg::kSmem;
    cfg.stream = stream;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = 2;
    at[0].val.clusterDim.y = 1;
    at[0].val.clusterDim.z = 1;
    cfg.attrs = at;
    cfg.numAttrs = 1;
    MB_CHECK_CUDA(cudaLaunchKernelEx(&cfg, gemm_wgmma_kernel<MODE, 2, BN>, map_a, map_w, p));
    note_launch("gemm_wgmma_kernel<%d, 2, %d, %d>", MODE, BN, TG_BM);
    MB_CHECK_LAUNCH("gemm_wgmma_kernel<cluster 2>");
    return MB200_OK;
  }
  const int tiles = ceil_div(g.T, TG_BM) * (g.N / BN);
  MB_CHECK_CUDA(cudaFuncSetAttribute(gemm_wgmma_kernel<MODE, 1, BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmem));
  gemm_wgmma_kernel<MODE, 1, BN><<<tiles < sms ? tiles : sms, Cfg::kThreads, Cfg::kSmem, stream>>>(map_a, map_w, p);
  note_launch("gemm_wgmma_kernel<%d, 1, %d, %d>", MODE, BN, TG_BM);
  MB_CHECK_LAUNCH("gemm_wgmma_kernel");
  return MB200_OK;
}

// ---- small-batch (decode, T < 128) launcher: weight-streaming, HBM-bound ------------------------------------------------------
// One M tile; the N tiles are dealt to persistent CTAs.  BN is chosen so that the rounds of the persistent schedule are as full
// as possible (every CTA streams the same number of weight rows), preferring wider tiles (bigger TMA boxes) on ties.
inline int wgmma_small_bn(int64_t N, int sms) {
  const int forced = wgmma_forced_bn();
  if ((forced == 32 || forced == 64 || forced == 128 || forced == 256) && N % forced == 0) return forced;
  int best = 0;
  double best_score = -1.0;
  const int cand[4] = {256, 128, 64, 32};
  for (int i = 0; i < 4; ++i) {
    const int bn = cand[i];
    if (N % bn != 0) continue;
    const int64_t tiles = N / bn, rounds = (tiles + sms - 1) / sms;
    double score = (double)tiles / (double)(rounds * sms);
    if (tiles < sms / 2) score *= 0.5;  // too few SMs pulling: per-SM ingest, not HBM, would bind
    if (score > best_score + 1e-9) {
      best_score = score;
      best = bn;
    }
  }
  return best;
}

template <int MODE, int BN, int TA>
int launch_gemm_wgmma_small_bn(const GemmParams& g, int sms, cudaStream_t stream) {
  using Cfg = TgCfg<BN, TA>;
  CUtensorMap map_a, map_w;
  int rc = make_tensor_map_2d(&map_a, g.a, g.T, g.K, TA);
  if (rc) return rc;
  rc = make_tensor_map_2d(&map_w, g.w, g.N, g.K, BN);
  if (rc) return rc;
  TcGemmParams p;
  p.T = g.T;
  p.N = g.N;
  p.K = g.K;
  p.epi = g.epi;
  const int tiles = g.N / BN;
  MB_CHECK_CUDA(cudaFuncSetAttribute(gemm_wgmma_kernel<MODE, 1, BN, TA>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmem));
  gemm_wgmma_kernel<MODE, 1, BN, TA><<<tiles < sms ? tiles : sms, Cfg::kThreads, Cfg::kSmem, stream>>>(map_a, map_w, p);
  note_launch("gemm_wgmma_kernel<%d, 1, %d, %d>", MODE, BN, TA);
  MB_CHECK_LAUNCH("gemm_wgmma_kernel<small batch>");
  return MB200_OK;
}

template <int MODE, int TA>
int launch_gemm_wgmma_small_ta(const GemmParams& g, int sms, cudaStream_t stream) {
  switch (wgmma_small_bn(g.N, sms)) {
    case 256: return launch_gemm_wgmma_small_bn<MODE, 256, TA>(g, sms, stream);
    case 128: return launch_gemm_wgmma_small_bn<MODE, 128, TA>(g, sms, stream);
    case 64: return launch_gemm_wgmma_small_bn<MODE, 64, TA>(g, sms, stream);
    case 32: return launch_gemm_wgmma_small_bn<MODE, 32, TA>(g, sms, stream);
    default: return fail(MB200_E_INVALID, "small-batch GEMM: N=%d is not a multiple of 32", g.N);
  }
}

template <int MODE>
int launch_gemm_wgmma(const GemmParams& g, cudaStream_t stream) {
  const bool pair = wgmma_cluster_enabled() && g.T >= 4 * TG_BM;
  int dev = 0, sms = 0;
  MB_CHECK_CUDA(cudaGetDevice(&dev));
  MB_CHECK_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  if (g.T <= 32) return launch_gemm_wgmma_small_ta<MODE, 32>(g, sms, stream);
  if (g.T <= 64) return launch_gemm_wgmma_small_ta<MODE, 64>(g, sms, stream);
  if (g.T < TG_BM) return launch_gemm_wgmma_small_ta<MODE, 128>(g, sms, stream);
  const int bn = wgmma_prefill_bn(g.T, g.N, pair, sms);
  if (bn == 192) return launch_gemm_wgmma_bn<MODE, 192>(g, pair, sms, stream);
  const bool narrow = bn == 128;
  return narrow ? launch_gemm_wgmma_bn<MODE, 128>(g, pair, sms, stream) : launch_gemm_wgmma_bn<MODE, 256>(g, pair, sms, stream);
}

// ---- FP8 dense weights: the same tile choices as launch_gemm_wgmma, single CTA only ------------------------------------------
// A shape that the bf16 launcher runs as 2-CTA clusters (T >= 512) runs as single CTAs at the same BN: the W8 stage holds the
// e4m3 tile next to the bf16 tile its converter warps write, and the multicast halves of the cluster variant have no such pair.
template <int MODE, int BN, int TA>
int launch_gemm_wgmma_fp8_bn(const GemmParams& g, int sms, cudaStream_t stream) {
  using Cfg = TgCfg<BN, TA, true>;
  CUtensorMap map_a, map_w;
  int rc = make_tensor_map_2d(&map_a, g.a, g.T, g.K, TA);
  if (rc) return rc;
  rc = make_tensor_map_e4m3(&map_w, g.w, g.N, g.K, BN);
  if (rc) return rc;
  TcGemmParams p;
  p.T = g.T;
  p.N = g.N;
  p.K = g.K;
  p.epi = g.epi;
  const int tiles = ceil_div(g.T, TG_BM) * (g.N / BN);
  MB_CHECK_CUDA(cudaFuncSetAttribute(gemm_wgmma_fp8_kernel<MODE, BN, TA>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmem));
  gemm_wgmma_fp8_kernel<MODE, BN, TA><<<tiles < sms ? tiles : sms, Cfg::kThreads, Cfg::kSmem, stream>>>(map_a, map_w, p);
  note_launch("gemm_wgmma_fp8_kernel<%d, %d, %d>", MODE, BN, TA);
  MB_CHECK_LAUNCH("gemm_wgmma_fp8_kernel");
  return MB200_OK;
}

template <int MODE, int TA>
int launch_gemm_wgmma_fp8_small_ta(const GemmParams& g, int sms, cudaStream_t stream) {
  switch (wgmma_small_bn(g.N, sms)) {
    case 256: return launch_gemm_wgmma_fp8_bn<MODE, 256, TA>(g, sms, stream);
    case 128: return launch_gemm_wgmma_fp8_bn<MODE, 128, TA>(g, sms, stream);
    case 64: return launch_gemm_wgmma_fp8_bn<MODE, 64, TA>(g, sms, stream);
    case 32: return launch_gemm_wgmma_fp8_bn<MODE, 32, TA>(g, sms, stream);
    default: return fail(MB200_E_INVALID, "small-batch GEMM (fp8): N=%d is not a multiple of 32", g.N);
  }
}

template <int MODE>
int launch_gemm_wgmma_fp8(const GemmParams& g, cudaStream_t stream) {
  int dev = 0, sms = 0;
  MB_CHECK_CUDA(cudaGetDevice(&dev));
  MB_CHECK_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  if (g.T <= 32) return launch_gemm_wgmma_fp8_small_ta<MODE, 32>(g, sms, stream);
  if (g.T <= 64) return launch_gemm_wgmma_fp8_small_ta<MODE, 64>(g, sms, stream);
  if (g.T < TG_BM) return launch_gemm_wgmma_fp8_small_ta<MODE, 128>(g, sms, stream);
  // the bf16 launcher's BN, with the m units it would have used (clusters of two for T >= 512 unless switched off)
  const int bn = wgmma_prefill_bn(g.T, g.N, wgmma_cluster_enabled() && g.T >= 4 * TG_BM, sms);
  if (bn == 192) return launch_gemm_wgmma_fp8_bn<MODE, 192, TG_BM>(g, sms, stream);
  return bn == 128 ? launch_gemm_wgmma_fp8_bn<MODE, 128, TG_BM>(g, sms, stream) : launch_gemm_wgmma_fp8_bn<MODE, 256, TG_BM>(g, sms, stream);
}

// ---- INT4 dense weights: the tile choices of launch_gemm_wgmma_fp8 (single CTAs where bf16 runs clusters, same BN) ------------
// Each tile's k order is the bf16 kernel's and its bf16 tile is W', so from 128 tokens on the result equals the bf16 launcher on W'.
template <int MODE, int BN, int TA>
int launch_gemm_wgmma_int4_bn(const GemmParams& g, const uint16_t* gscale, int sms, cudaStream_t stream) {
  using Cfg = TgCfg<BN, TA, false, true>;
  CUtensorMap map_a, map_w;
  int rc = make_tensor_map_2d(&map_a, g.a, g.T, g.K, TA);
  if (rc) return rc;
  rc = make_tensor_map_int4(&map_w, g.w, g.N, g.K, BN);
  if (rc) return rc;
  TcGemmParams p;
  p.T = g.T;
  p.N = g.N;
  p.K = g.K;
  p.epi = g.epi;
  const int tiles = ceil_div(g.T, TG_BM) * (g.N / BN);
  MB_CHECK_CUDA(cudaFuncSetAttribute(gemm_wgmma_int4_kernel<MODE, BN, TA>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmem));
  gemm_wgmma_int4_kernel<MODE, BN, TA><<<tiles < sms ? tiles : sms, Cfg::kThreads, Cfg::kSmem, stream>>>(map_a, map_w, p, gscale);
  note_launch("gemm_wgmma_int4_kernel<%d, %d, %d>", MODE, BN, TA);
  MB_CHECK_LAUNCH("gemm_wgmma_int4_kernel");
  return MB200_OK;
}

template <int MODE, int TA>
int launch_gemm_wgmma_int4_small_ta(const GemmParams& g, const uint16_t* gscale, int sms, cudaStream_t stream) {
  switch (wgmma_small_bn(g.N, sms)) {
    case 256: return launch_gemm_wgmma_int4_bn<MODE, 256, TA>(g, gscale, sms, stream);
    case 128: return launch_gemm_wgmma_int4_bn<MODE, 128, TA>(g, gscale, sms, stream);
    case 64: return launch_gemm_wgmma_int4_bn<MODE, 64, TA>(g, gscale, sms, stream);
    case 32: return launch_gemm_wgmma_int4_bn<MODE, 32, TA>(g, gscale, sms, stream);
    default: return fail(MB200_E_INVALID, "small-batch GEMM (int4): N=%d is not a multiple of 32", g.N);
  }
}

template <int MODE>
int launch_gemm_wgmma_int4(const GemmParams& g, const uint16_t* gscale, cudaStream_t stream) {
  int dev = 0, sms = 0;
  MB_CHECK_CUDA(cudaGetDevice(&dev));
  MB_CHECK_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  if (g.T <= 32) return launch_gemm_wgmma_int4_small_ta<MODE, 32>(g, gscale, sms, stream);
  if (g.T <= 64) return launch_gemm_wgmma_int4_small_ta<MODE, 64>(g, gscale, sms, stream);
  if (g.T < TG_BM) return launch_gemm_wgmma_int4_small_ta<MODE, 128>(g, gscale, sms, stream);
  const int bn = wgmma_prefill_bn(g.T, g.N, wgmma_cluster_enabled() && g.T >= 4 * TG_BM, sms);
  if (bn == 192) return launch_gemm_wgmma_int4_bn<MODE, 192, TG_BM>(g, gscale, sms, stream);
  return bn == 128 ? launch_gemm_wgmma_int4_bn<MODE, 128, TG_BM>(g, gscale, sms, stream)
                   : launch_gemm_wgmma_int4_bn<MODE, 256, TG_BM>(g, gscale, sms, stream);
}

}  // namespace mb200
