// Mixture of experts for T > 1 tokens (prefill and batched decode): device-side router + grouped tensor-core expert GEMMs.
// Replaces MoeLayer.forward (moe.py:24-32) -- gate Linear, torch.topk, softmax, and the per-expert `torch.where` / index /
// FeedForward / weighted `+=` loop with its host synchronisations -- by five launches with NO host round trip:
//
//   moe_route_kernel    logits = bf16(hn . gate^T); top-k on the bf16 logits (ties: lower expert index first); fp32 softmax over
//                       the k selected -> bf16 weights (moe.py:25-27); the k (expert, weight) pairs of a token are stored in
//                       ASCENDING expert index: the order the reference's `results[idx] += w * expert(x)` loop visits them.
//   moe_plan_kernel     one CTA: per-expert row counts, segment starts (each expert's segment padded to a multiple of the GEMM's
//                       m-tile), a DETERMINISTIC slot for every (token, expert) pair (token order inside a segment: identical on
//                       every rank of an expert-parallel group, which is what lets ranks write each other's rows), and the list
//                       of m tiles of the experts this rank owns.
//   moe_gather_kernel   xs[slot] = hn[token], row_w[slot] = routing weight  (rows of local experts only)
//   gemm_wgmma_grouped_kernel x2 (gemm_wgmma.cuh): g = silu(xs W1_e^T) * (xs W3_e^T);  yw = bf16(w * bf16(g W2_e^T)), the
//                       second one storing every row on ALL ranks of the group (peer stores over NVLink) -- the exchange step of
//                       expert parallelism is the epilogue of the down projection, an all-gather of rows with no reduction.
//   moe_combine_kernel  (expert parallel: signal the peers / wait for theirs) out[t] = bf16(h[t] + sum_j yw[slot(t, j)]) with the
//                       sum taken in ascending expert index, each step rounded to bf16 like `results +=` -- bit-identical to the
//                       reference for any k and any number of ranks.
// Roofline: tensor pipe for prefill (2 * rows * 3 * dim * hidden flop), HBM for decode (every touched expert's weights once).
#pragma once
#include "gemm_streamk.cuh"
#include "gemm_wgmma.cuh"

namespace mb200 {

constexpr int MOE_MAX_TOPK = 8;

// ---- router: one warp per token (WIDE = false: prefill) or one CTA per token with the 8 warps splitting the row (WIDE = true:
// decode-sized batches, where a single warp walking 4096 dims x 8 experts is pure load latency: 36 us measured for 8 tokens) ------
template <int E, bool WIDE>
__global__ void __launch_bounds__(256) moe_route_kernel(const bf16* __restrict__ hn, const bf16* __restrict__ gate_w, int T, int dim, int k,
                                                        int32_t* __restrict__ sel, bf16* __restrict__ wts) {
  pdl_trigger();
  pdl_wait();  // hn is the preceding RMSNorm's output
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int t = WIDE ? (int)blockIdx.x : (int)blockIdx.x * 8 + warp;
  if (t >= T) return;
  const int kc = dim >> 3;
  const uint4* xr = reinterpret_cast<const uint4*>(hn + (int64_t)t * dim);
  float acc[E];
#pragma unroll
  for (int e = 0; e < E; ++e) acc[e] = 0.f;
#pragma unroll 2
  for (int c = WIDE ? (int)threadIdx.x : lane; c < kc; c += WIDE ? 256 : 32) {
    const uint4 xv = xr[c];
    const uint32_t xw[4] = {xv.x, xv.y, xv.z, xv.w};
#pragma unroll
    for (int e = 0; e < E; ++e) {
      const uint4 gv = __ldg(reinterpret_cast<const uint4*>(gate_w + (int64_t)e * dim) + c);
      const uint32_t gw[4] = {gv.x, gv.y, gv.z, gv.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        acc[e] = fmaf(bf16lo(gw[j]), bf16lo(xw[j]), acc[e]);
        acc[e] = fmaf(bf16hi(gw[j]), bf16hi(xw[j]), acc[e]);
      }
    }
  }
  if constexpr (WIDE) {  // fold the 8 warps' partial sums in a fixed order
    __shared__ float part[8][E];
#pragma unroll
    for (int e = 0; e < E; ++e) {
      const float v = warp_sum(acc[e]);
      if (lane == 0) part[warp][e] = v;
    }
    __syncthreads();
    if (warp != 0) return;
#pragma unroll
    for (int e = 0; e < E; ++e) {
      float v = 0.f;
#pragma unroll
      for (int w = 0; w < 8; ++w) v += part[w][e];
      acc[e] = round_bf16(v);  // the router Linear's bf16 output (moe.py:25)
    }
  } else {
#pragma unroll
    for (int e = 0; e < E; ++e) acc[e] = round_bf16(warp_sum(acc[e]));  // the router Linear's bf16 output (moe.py:25)
  }
  if (lane != 0) return;
  int se[MOE_MAX_TOPK];
  float sv[MOE_MAX_TOPK];
  unsigned taken = 0u;
  for (int j = 0; j < k; ++j) {  // top-k on the bf16 logits, ties -> lower index
    int best = -1;
    float bv = 0.f;
#pragma unroll
    for (int e = 0; e < E; ++e)
      if (!((taken >> e) & 1u) && (best < 0 || acc[e] > bv)) {
        best = e;
        bv = acc[e];
      }
    taken |= 1u << best;
    se[j] = best;
    sv[j] = bv;
  }
  float den = 0.f, ex[MOE_MAX_TOPK];
  for (int j = 0; j < k; ++j) {
    ex[j] = expf(sv[j] - sv[0]);  // sv[0] is the maximum
    den += ex[j];
  }
  for (int j = 0; j < k; ++j) sv[j] = round_bf16(ex[j] / den);  // softmax in fp32, then .to(bf16) (moe.py:27)
  for (int a = 1; a < k; ++a)  // ascending expert index, weights travelling with their experts
    for (int b = a; b > 0 && se[b] < se[b - 1]; --b) {
      const int ts = se[b];
      se[b] = se[b - 1];
      se[b - 1] = ts;
      const float tv = sv[b];
      sv[b] = sv[b - 1];
      sv[b - 1] = tv;
    }
  for (int j = 0; j < k; ++j) {
    sel[(int64_t)t * k + j] = se[j];
    wts[(int64_t)t * k + j] = __float2bfloat16_rn(sv[j]);
  }
}

// ---- plan: one CTA ---------------------------------------------------------------------------------------------------------
// plan layout (int32): [0] m tiles owned by this rank, [1] padded rows in total, [2] tile capacity, [3] pairs, [4]/[5] statistics, [8 + e] start of
// expert e's segment (e = 0..E), then tile_expert[capacity], tile_row0[capacity] from word MOE_PLAN_HEADER.
constexpr int MP_THREADS = 1024;
__global__ void __launch_bounds__(MP_THREADS) moe_plan_kernel(const int32_t* __restrict__ sel, int pairs, int E, int tile_rows, int shard_rank,
                                                              int shard_world, int tile_cap, int32_t* __restrict__ slot, int32_t* __restrict__ plan) {
  extern __shared__ int32_t sm[];  // cnt[E][MP_THREADS], then seg[E + 1], total[E]
  int32_t* cnt = sm;
  int32_t* seg = sm + E * MP_THREADS;
  int32_t* total = seg + E + 1;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (pairs <= 512) {
    // decode-sized batch: thread e walks the whole (short) pair list for expert e -- same deterministic plan, a few hundred cycles
    if (tid < E) {
      int n = 0;
      for (int i = 0; i < pairs; ++i)
        if (sel[i] == tid) slot[i] = n++;  // position inside the expert's segment; the segment start is added below
      total[tid] = n;
    }
    __syncthreads();
    if (tid == 0) {
      int rows = 0, n = 0, touched = 0;
      for (int e = 0; e < E; ++e) {
        seg[e] = rows;
        plan[8 + e] = rows;
        const int m_tiles = (total[e] + tile_rows - 1) / tile_rows;
        touched += total[e] > 0;
        if (e % shard_world == shard_rank)
          for (int m = 0; m < m_tiles && n < tile_cap; ++m, ++n) {
            plan[MOE_PLAN_HEADER + n] = e;
            plan[MOE_PLAN_HEADER + tile_cap + n] = rows + m * tile_rows;
          }
        rows += m_tiles * tile_rows;
      }
      plan[8 + E] = rows;
      plan[0] = n;
      plan[1] = rows;
      plan[2] = tile_cap;
      plan[3] = pairs;
      plan[4] += touched;
      plan[5] += 1;
      plan[6] = 0;  // decode-sized calls never take the cluster variant
    }
    __syncthreads();
    for (int i = tid; i < pairs; i += MP_THREADS) slot[i] += seg[sel[i]];
    return;
  }
  const int per = (pairs + MP_THREADS - 1) / MP_THREADS;
  const int p0 = min(tid * per, pairs), p1 = min(p0 + per, pairs);
  for (int e = 0; e < E; ++e) cnt[e * MP_THREADS + tid] = 0;
  for (int i = p0; i < p1; ++i) cnt[sel[i] * MP_THREADS + tid] += 1;
  __syncthreads();
  // exclusive scan of every expert's 1024 counts: warp w takes experts w, w + 32, ...; lane l scans entries [32 l, 32 l + 32)
  for (int e = warp; e < E; e += MP_THREADS / 32) {
    int32_t* c = cnt + e * MP_THREADS + lane * 32;
    int run = 0;
    for (int i = 0; i < 32; ++i) {
      const int v = c[i];
      c[i] = run;
      run += v;
    }
    int incl = run;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int up = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += up;
    }
    const int base = incl - run;
    for (int i = 0; i < 32; ++i) c[i] += base;
    if (lane == 31) total[e] = incl;
  }
  __syncthreads();
  if (tid == 0) {
    int rows = 0, n = 0, np = 0;
    for (int e = 0; e < E; ++e) {
      seg[e] = rows;
      plan[8 + e] = rows;
      const int m_tiles = (total[e] + tile_rows - 1) / tile_rows;
      if (e % shard_world == shard_rank) {
        for (int m = 0; m < m_tiles && n < tile_cap; ++m, ++n) {
          plan[MOE_PLAN_HEADER + n] = e;
          plan[MOE_PLAN_HEADER + tile_cap + n] = rows + m * tile_rows;
        }
        for (int m = 0; m < m_tiles && np < tile_cap; m += 2, ++np) {  // pairs of vertically adjacent tiles for the 2-CTA cluster GEMM
          plan[MOE_PLAN_HEADER + 2 * tile_cap + np] = e;
          plan[MOE_PLAN_HEADER + 3 * tile_cap + np] = (rows + m * tile_rows) | (m + 1 < m_tiles ? MOE_PAIR_SECOND : 0);
        }
      }
      rows += m_tiles * tile_rows;
    }
    plan[6] = np;
    seg[E] = rows;
    plan[8 + E] = rows;
    plan[0] = n;
    plan[1] = rows;
    plan[2] = tile_cap;
    plan[3] = pairs;
    int touched = 0;
    for (int e = 0; e < E; ++e) touched += total[e] > 0;
    plan[4] += touched;  // statistics (never reset by the kernel): experts with at least one row, summed over calls ...
    plan[5] += 1;        // ... and the number of calls: the measured "distinct experts per layer" of bench.py
  }
  __syncthreads();
  int run[MOE_MAX_EXPERTS];
#pragma unroll
  for (int e = 0; e < MOE_MAX_EXPERTS; ++e) run[e] = 0;
  for (int i = p0; i < p1; ++i) {
    const int e = sel[i];
    int r = 0;
#pragma unroll
    for (int q = 0; q < MOE_MAX_EXPERTS; ++q)  // static indexing keeps `run` in registers
      if (q == e) r = run[q]++;
    slot[i] = seg[e] + cnt[e * MP_THREADS + tid] + r;
  }
}

// ---- gather: one warp per (token, expert) pair ------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) moe_gather_kernel(const uint4* __restrict__ hn, const int32_t* __restrict__ sel, const bf16* __restrict__ wts,
                                                         const int32_t* __restrict__ slot, int pairs, int k, int row_chunks, int shard_rank,
                                                         int shard_world, uint4* __restrict__ xs, bf16* __restrict__ row_w) {
  const int pair = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (pair >= pairs) return;
  if (sel[pair] % shard_world != shard_rank) return;  // another rank's expert
  const int t = pair / k, s = slot[pair];
  if (lane == 0) row_w[s] = wts[pair];
  const uint4* src = hn + (int64_t)t * row_chunks;
  uint4* dst = xs + (int64_t)s * row_chunks;
  for (int c = lane; c < row_chunks; c += 32) dst[c] = src[c];
}

// ---- combine (+ the expert-parallel handshake) --------------------------------------------------------------------------------
struct MoeCombineParams {
  const uint4* yw;        // [rows, dim] weighted expert outputs (all ranks' rows once the handshake is through)
  const int32_t* slot;    // [T, k]
  const uint4* residual;  // h [T, dim] or null
  uint4* out;             // [T, dim]
  int T, k, row_chunks;
  // expert parallel (n_ranks > 1): flags[r] of THIS rank is written by rank r when all its rows of this call have landed here
  int n_ranks, my_rank;
  unsigned* my_flags;               // [n_ranks] in this rank's comm buffer
  unsigned* peer_flags[kMaxPeers];  // the same array on the other ranks (mapped)
  unsigned* epoch;                  // local device word: completed calls on this buffer
  int* done_counter;                // local, self-resetting
};
__device__ __forceinline__ unsigned ld_acquire_sys_u32(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys_u32(unsigned* p, unsigned v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

__global__ void __launch_bounds__(128) moe_combine_kernel(const MoeCombineParams p) {
  const int t = blockIdx.x;
  if (p.n_ranks > 1) {
    // This kernel starts after this rank's down projection has finished (stream order), i.e. after its peer stores were issued
    // and completed.  Block 0 tells every peer; every block then waits until every peer has told this rank.
    __shared__ unsigned target;
    if (threadIdx.x == 0) {
      const unsigned e = *reinterpret_cast<volatile unsigned*>(p.epoch) + 1u;
      target = e;
      if (blockIdx.x == 0) {
        __threadfence_system();
        for (int r = 0; r < p.n_ranks - 1; ++r) st_release_sys_u32(p.peer_flags[r] + p.my_rank, e);
        st_release_sys_u32(p.my_flags + p.my_rank, e);
      }
      for (int r = 0; r < p.n_ranks; ++r) {
        unsigned long long spins = 0;
        while ((int)(ld_acquire_sys_u32(p.my_flags + r) - e) < 0) {
          if (++spins == (1ull << 26)) {
            printf("[mb200 watchdog] rank %d block %d: no signal from rank %d for MoE exchange %u (have %u)\n", p.my_rank, (int)blockIdx.x, r, e,
                   ld_acquire_sys_u32(p.my_flags + r));
            __trap();
          }
        }
      }
    }
    __syncthreads();
    (void)target;
  }
  const int32_t* sl = p.slot + (int64_t)t * p.k;
  for (int c = threadIdx.x; c < p.row_chunks; c += 128) {
    float r[8];
    {
      const uint4 v = p.yw[(int64_t)sl[0] * p.row_chunks + c];
      const uint32_t u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        r[2 * j] = bf16lo(u[j]);  // results starts at zero: bf16(0 + t) == t
        r[2 * j + 1] = bf16hi(u[j]);
      }
    }
    for (int q = 1; q < p.k; ++q) {
      const uint4 v = p.yw[(int64_t)sl[q] * p.row_chunks + c];
      const uint32_t u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        r[2 * j] = round_bf16(r[2 * j] + bf16lo(u[j]));  // results[idx] += ... in bf16 (moe.py:31)
        r[2 * j + 1] = round_bf16(r[2 * j + 1] + bf16hi(u[j]));
      }
    }
    uint32_t o[4];
    if (p.residual != nullptr) {
      const uint4 h = p.residual[(int64_t)t * p.row_chunks + c];
      const uint32_t hu[4] = {h.x, h.y, h.z, h.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) o[j] = pack_bf16x2(bf16lo(hu[j]) + r[2 * j], bf16hi(hu[j]) + r[2 * j + 1]);  // h + r (transformer_layers.py:168)
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j) o[j] = pack_bf16x2(r[2 * j], r[2 * j + 1]);
    }
    p.out[(int64_t)t * p.row_chunks + c] = make_uint4(o[0], o[1], o[2], o[3]);
  }
  if (p.n_ranks > 1) {  // the last block to finish publishes the epoch for the next call on this buffer
    __syncthreads();
    if (threadIdx.x == 0) {
      __threadfence();
      const int prev = atomicAdd(p.done_counter, 1);
      if (prev == (int)gridDim.x - 1) {
        *p.done_counter = 0;
        __threadfence();
        *reinterpret_cast<volatile unsigned*>(p.epoch) = *reinterpret_cast<volatile unsigned*>(p.epoch) + 1u;
      }
    }
  }
}

// ---- FP8 expert weights: row-wise e4m3 quantiser, one CTA per row ----------------------------------------------------------------
// s[n] = fp32(amax[n] / 448) (1 for an all-zero row), q[n, k] = e4m3_rn_satfinite(fp32(W[n, k] / s[n])): IEEE divisions (the library
// is built without fast math), cvt.rn.satfinite.e4m3x2.f32 clamps to +-448 like the contract's clamp.  q rows land q_stride bytes
// apart and scales scale_stride floats apart, so w1 / w3 fill the interleaved rows of the packed gate/up matrix directly.
__global__ void __launch_bounds__(256) quantize_e4m3_rows_kernel(const uint4* __restrict__ w, int K, uint8_t* __restrict__ q, int64_t q_stride,
                                                                 float* __restrict__ scale, int64_t scale_stride) {
  const int n = blockIdx.x, chunks = K >> 3;
  const uint4* row = w + (int64_t)n * chunks;
  float amax = 0.f;
  for (int c = threadIdx.x; c < chunks; c += 256) {
    const uint4 v = row[c];
    const uint32_t u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) amax = fmaxf(amax, fmaxf(fabsf(bf16lo(u[j])), fabsf(bf16hi(u[j]))));
  }
  __shared__ float part[8];
  amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 16));
  amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 8));
  amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 4));
  amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 2));
  amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 1));
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = amax;
  __syncthreads();
  amax = part[0];
#pragma unroll
  for (int i = 1; i < 8; ++i) amax = fmaxf(amax, part[i]);
  const float s = amax == 0.f ? 1.f : __fdiv_rn(amax, 448.f);
  if (threadIdx.x == 0) scale[(int64_t)n * scale_stride] = s;
  uint2* qrow = reinterpret_cast<uint2*>(q + (int64_t)n * q_stride);
  for (int c = threadIdx.x; c < chunks; c += 256) {
    const uint4 v = row[c];
    const uint32_t u[4] = {v.x, v.y, v.z, v.w};
    uint32_t o[2] = {0u, 0u};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = make_float2(__fdiv_rn(bf16lo(u[j]), s), __fdiv_rn(bf16hi(u[j]), s));
      o[j >> 1] |= (uint32_t)__nv_cvt_float2_to_fp8x2(f, __NV_SATFINITE, __NV_E4M3) << (16 * (j & 1));
    }
    qrow[c] = make_uint2(o[0], o[1]);
  }
}

// ---- host side -------------------------------------------------------------------------------------------------------------
inline int moe_tile_rows(int64_t T) { return T <= 32 ? 32 : (T <= 64 ? 64 : 128); }  // an expert gets at most one row per token: decode batches fit ONE short m tile
inline int64_t moe_tile_cap(int64_t pairs, int64_t E, int tile_rows) { return (pairs + tile_rows - 1) / tile_rows + E; }
inline int64_t moe_plan_words(int64_t pairs, int64_t E, int tile_rows) { return MOE_PLAN_HEADER + 4 * moe_tile_cap(pairs, E, tile_rows); }
inline int64_t moe_row_cap(int64_t pairs, int64_t E, int tile_rows) { return moe_tile_cap(pairs, E, tile_rows) * tile_rows; }

// Weight format of a grouped call's experts.  FP8: `scales` holds E per-row fp32 scale arrays; INT4: E bf16 group-scale arrays.
enum class MoeFmt { BF16, FP8, INT4 };

// The weight formats a grouped MODE is built for.  The un-merged LoRA stages of FP8 experts add two: the up-projection (EPI_STORE)
// reads bf16 B tables, and the LoRA-combining base GEMMs (EPI_LORA) read e4m3 experts.  Every other mode is built for all three.
template <int MODE>
constexpr bool grouped_fmt_built(MoeFmt f) {
  return MODE == EPI_STORE ? f == MoeFmt::BF16 : ((MODE & EPI_LORA) != 0 ? f == MoeFmt::FP8 : true);
}

// Tensor maps of the experts' weights (bf16, e4m3, or INT4 codes with boxes of int4_box_bytes) and their scale tables; an expert
// of another rank (NULL) gets a placeholder that this rank's tiles never reference.
inline int moe_weight_maps(MoeWeightMaps* maps, MoeWeightScales* sc, MoeWeightGroupScales* gsc, const CUtensorMap& placeholder,
                           const void* const* w_host, MoeFmt fmt, const void* const* scales, int E, int64_t N, int64_t K, int box_rows,
                           int int4_box_bytes = TG_BK / 2) {
  for (int e = 0; e < MOE_MAX_EXPERTS; ++e) {
    const void* w = e < E && w_host[e] != nullptr ? w_host[e] : nullptr;
    const void* s = w != nullptr && fmt != MoeFmt::BF16 ? scales[e] : nullptr;
    sc->s[e] = fmt == MoeFmt::FP8 ? static_cast<const float*>(s) : nullptr;
    gsc->s[e] = fmt == MoeFmt::INT4 ? static_cast<const uint16_t*>(s) : nullptr;
    if (w == nullptr) {
      maps->m[e] = placeholder;
      continue;
    }
    if (fmt != MoeFmt::BF16 && s == nullptr) return fail(MB200_E_INVALID, "grouped gemm: expert %d has quantised weights but no scales", e);
    if (fmt == MoeFmt::INT4 && (((uintptr_t)w & 15) != 0 || ((uintptr_t)s & 1) != 0))
      return fail(MB200_E_INVALID, "grouped gemm (int4): expert %d: misaligned codes or scales", e);
    const int rc = fmt == MoeFmt::FP8    ? make_tensor_map_e4m3(&maps->m[e], w, N, K, box_rows)
                   : fmt == MoeFmt::INT4 ? make_tensor_map_int4(&maps->m[e], w, N, K, box_rows, int4_box_bytes)
                                         : make_tensor_map_2d(&maps->m[e], w, N, K, box_rows);
    if (rc) return rc;
  }
  return MB200_OK;
}

// FP8 and INT4: gemm_wgmma_grouped_fp8_kernel / gemm_wgmma_grouped_int4_kernel, always one CTA per tile (CL = 1): in a cluster pair
// each CTA would have to convert the whole multicast tile, and the quantised tile already cuts the L2 -> SM bytes that the
// multicast saves a third of.  The tile's k order is the bf16 kernel's at the same BN, so the result is too.
template <int MODE, int BN, int TA, int CL = 1>
int launch_grouped_bn(const void* a, int64_t rows_cap, int64_t K, int64_t N, const void* const* w_host, int E, const int32_t* plan, const EpiParams& epi,
                      int sms, cudaStream_t stream, MoeFmt fmt, const void* const* scales) {
  using Cfg = TgCfg<BN, TA>;
  CUtensorMap map_a;
  MoeWeightMaps maps;
  MoeWeightScales sc;
  MoeWeightGroupScales gsc;
  int rc = make_tensor_map_2d(&map_a, a, rows_cap, K, TA);
  if (rc) return rc;
  // cluster pairs: each CTA fetches half of the W tile and multicasts it
  rc = moe_weight_maps(&maps, &sc, &gsc, map_a, w_host, fmt, scales, E, N, K, fmt != MoeFmt::BF16 ? BN : BN / CL);
  if (rc) return rc;
  TcGemmParams p;
  p.T = (int)rows_cap;
  p.N = (int)N;
  p.K = (int)K;
  p.epi = epi;
  if constexpr (grouped_fmt_built<MODE>(MoeFmt::FP8)) {
    if (fmt == MoeFmt::FP8) {
      using Cfg8 = TgCfg<BN, TA, true>;
      MB_CHECK_CUDA(cudaFuncSetAttribute(gemm_wgmma_grouped_fp8_kernel<MODE, BN, TA>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg8::kSmem));
      gemm_wgmma_grouped_fp8_kernel<MODE, BN, TA><<<sms, Cfg8::kThreads, Cfg8::kSmem, stream>>>(map_a, maps, sc, p, plan);
      MB_CHECK_LAUNCH("gemm_wgmma_grouped_fp8_kernel");
      note_launch("gemm_wgmma_grouped_fp8_kernel<%d, 1, %d, %d>", MODE, BN, TA);
      return MB200_OK;
    }
  }
  if constexpr (grouped_fmt_built<MODE>(MoeFmt::INT4)) {
    if (fmt == MoeFmt::INT4) {
      using Cfg4 = TgCfg<BN, TA, false, true>;
      MB_CHECK_CUDA(cudaFuncSetAttribute(gemm_wgmma_grouped_int4_kernel<MODE, BN, TA>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg4::kSmem));
      gemm_wgmma_grouped_int4_kernel<MODE, BN, TA><<<sms, Cfg4::kThreads, Cfg4::kSmem, stream>>>(map_a, maps, gsc, p, plan);
      MB_CHECK_LAUNCH("gemm_wgmma_grouped_int4_kernel");
      note_launch("gemm_wgmma_grouped_int4_kernel<%d, %d, %d>", MODE, BN, TA);
      return MB200_OK;
    }
  }
  if constexpr (!grouped_fmt_built<MODE>(MoeFmt::BF16)) {
    return fail(MB200_E_INVALID, "grouped gemm: epilogue mode %d has no variant for these weights", MODE);
  } else {
    MB_CHECK_CUDA(cudaFuncSetAttribute(gemm_wgmma_grouped_kernel<MODE, CL, BN, TA>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmem));
    if (CL == 1) {
      gemm_wgmma_grouped_kernel<MODE, CL, BN, TA><<<sms, Cfg::kThreads, Cfg::kSmem, stream>>>(map_a, maps, p, plan);
      MB_CHECK_LAUNCH("gemm_wgmma_grouped_kernel");
      note_launch("gemm_wgmma_grouped_kernel<%d, %d, %d, %d>", MODE, CL, BN, TA);
      return MB200_OK;
    }
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(2u * (unsigned)(sms / 2));
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
    MB_CHECK_CUDA(cudaLaunchKernelEx(&cfg, gemm_wgmma_grouped_kernel<MODE, CL, BN, TA>, map_a, maps, p, plan));
    MB_CHECK_LAUNCH("gemm_wgmma_grouped_kernel<cluster 2>");
    note_launch("gemm_wgmma_grouped_kernel<%d, %d, %d, %d>", MODE, CL, BN, TA);
    return MB200_OK;
  }
}

// tile width: prefill (128-row tiles) takes the widest tile that divides N; decode-sized calls (32-row tiles, HBM-bound) pick the
// width that fills the rounds of the persistent schedule best for the EXPECTED number of touched experts
// decode-sized calls: the stream-K weight-streaming kernel over (expert segment, n tile, k block) units
template <int MODE, int TA>
int launch_grouped_streamk(const void* a, int64_t rows_cap, int64_t K, int64_t N, const void* const* w_host, int E, const int32_t* plan,
                           const EpiParams& epi, void* workspace, size_t workspace_bytes, int sms, cudaStream_t stream, MoeFmt fmt,
                           const void* const* scales) {
  using Cfg = TgCfg<SK_BN, TA>;
  if (sms > SK_MAX_CTAS) sms = SK_MAX_CTAS;
  if (workspace == nullptr || workspace_bytes < kWsSkPartials.end()) return fail(MB200_E_WORKSPACE, "grouped stream-K gemm: workspace %zu < %zu", workspace_bytes, kWsSkPartials.end());
  CUtensorMap map_a;
  MoeWeightMaps maps;
  MoeWeightScales sc;
  MoeWeightGroupScales gsc;
  int rc = make_tensor_map_2d(&map_a, a, rows_cap, K, TA);
  if (rc) return rc;
  rc = moe_weight_maps(&maps, &sc, &gsc, map_a, w_host, fmt, scales, E, N, K, SK_BN, SK_W4_CHUNK_KB * TG_BK / 2);
  if (rc) return rc;
  SkParams p;
  p.T = (int)rows_cap;
  p.N = (int)N;
  p.K = (int)K;
  p.epi = epi;
  p.partials = reinterpret_cast<float*>((uint8_t*)workspace + kWsSkPartials.offset);
  p.flags = reinterpret_cast<unsigned*>((uint8_t*)workspace + kWsSkFlags.offset);
  if constexpr (grouped_fmt_built<MODE>(MoeFmt::FP8)) {
    if (fmt == MoeFmt::FP8) {
      using Cfg8 = TgCfg<SK_BN, TA, true>;
      MB_CHECK_CUDA(cudaFuncSetAttribute(gemm_streamk_grouped_fp8_kernel<MODE, TA>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg8::kSmem));
      MB_CHECK_CUDA(launch_pdl(gemm_streamk_grouped_fp8_kernel<MODE, TA>, dim3((unsigned)sms), dim3(Cfg8::kThreads), (size_t)Cfg8::kSmem, stream, map_a,
                               maps, sc, p, plan));
      note_launch("gemm_streamk_grouped_fp8_kernel<%d, %d>", MODE, TA);
      return MB200_OK;
    }
  }
  if constexpr (grouped_fmt_built<MODE>(MoeFmt::INT4)) {
    if (fmt == MoeFmt::INT4) {  // (the grouped body waits for the plan before it requests any chunk)
      using Cfg4 = SkW4Cfg<TA>;
      MB_CHECK_CUDA(cudaFuncSetAttribute(gemm_streamk_grouped_int4_kernel<MODE, TA>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg4::kSmem));
      MB_CHECK_CUDA(launch_pdl(gemm_streamk_grouped_int4_kernel<MODE, TA>, dim3((unsigned)sms), dim3(Cfg4::kThreads), (size_t)Cfg4::kSmem, stream, map_a,
                               maps, gsc, p, plan));
      note_launch("gemm_streamk_grouped_int4_kernel<%d, %d>", MODE, TA);
      return MB200_OK;
    }
  }
  if constexpr (!grouped_fmt_built<MODE>(MoeFmt::BF16)) {
    return fail(MB200_E_INVALID, "grouped stream-K gemm: epilogue mode %d has no variant for these weights", MODE);
  } else {
    MB_CHECK_CUDA(cudaFuncSetAttribute(gemm_streamk_grouped_kernel<MODE, TA>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmem));
    MB_CHECK_CUDA(launch_pdl(gemm_streamk_grouped_kernel<MODE, TA>, dim3((unsigned)sms), dim3(Cfg::kThreads), (size_t)Cfg::kSmem, stream, map_a, maps, p,
                             plan));
    note_launch("gemm_streamk_grouped_kernel<%d, %d>", MODE, TA);
    return MB200_OK;
  }
}

template <int MODE>
int launch_grouped(const void* a, int64_t rows_cap, int64_t K, int64_t N, const void* const* w_host, int E, int est_mtiles, int tile_rows,
                   const int32_t* plan, const EpiParams& epi, void* workspace, size_t workspace_bytes, cudaStream_t stream, MoeFmt fmt,
                   const void* const* scales) {
  int dev = 0, sms = 0;
  MB_CHECK_CUDA(cudaGetDevice(&dev));
  MB_CHECK_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  MB_CHECK_ARG(K % TG_BK == 0 && N % 32 == 0, "grouped gemm: K=%lld must be a multiple of 64, N=%lld of 32", (long long)K, (long long)N);
  MB_CHECK_ARG(fmt != MoeFmt::INT4 || K % kInt4Group == 0, "grouped gemm (int4): K=%lld must be a multiple of 128", (long long)K);
  MB_CHECK_ARG(grouped_fmt_built<MODE>(fmt), "grouped gemm: epilogue mode %d has no variant for these weights", MODE);
  if (tile_rows < 128 && streamk_eligible(tile_rows, N, K)) {
    if (tile_rows == 32) return launch_grouped_streamk<MODE, 32>(a, rows_cap, K, N, w_host, E, plan, epi, workspace, workspace_bytes, sms, stream, fmt, scales);
    return launch_grouped_streamk<MODE, 64>(a, rows_cap, K, N, w_host, E, plan, epi, workspace, workspace_bytes, sms, stream, fmt, scales);
  }
  if (tile_rows == 128) {
    // enough rows per expert for vertically adjacent tile pairs: the 2-CTA cluster kernel (W tile multicast, 2/3 of the L2 -> SM traffic)
    if (N % 256 == 0 && fmt == MoeFmt::BF16 && wgmma_cluster_enabled() && rows_cap >= (int64_t)E * 512)
      return launch_grouped_bn<MODE, 256, 128, 2>(a, rows_cap, K, N, w_host, E, plan, epi, sms, stream, fmt, scales);
    if (N % 256 == 0) return launch_grouped_bn<MODE, 256, 128>(a, rows_cap, K, N, w_host, E, plan, epi, sms, stream, fmt, scales);
    if (N % 128 == 0) return launch_grouped_bn<MODE, 128, 128>(a, rows_cap, K, N, w_host, E, plan, epi, sms, stream, fmt, scales);
    if (N % 64 == 0) return launch_grouped_bn<MODE, 64, 128>(a, rows_cap, K, N, w_host, E, plan, epi, sms, stream, fmt, scales);
    return launch_grouped_bn<MODE, 32, 128>(a, rows_cap, K, N, w_host, E, plan, epi, sms, stream, fmt, scales);
  }
  int best = 32;
  double best_score = -1.0;
  const int forced = wgmma_forced_bn();
  const int cand[4] = {256, 128, 64, 32};
  for (int i = 0; i < 4; ++i) {
    const int bn = cand[i];
    if (N % bn != 0) continue;
    if (forced == bn) {
      best = bn;
      break;
    }
    const int64_t tiles = (int64_t)est_mtiles * (N / bn), rounds = (tiles + sms - 1) / sms;
    const double score = (double)tiles / (double)(rounds * sms);
    if (score > best_score + 0.02) {  // wider tiles (bigger TMA boxes) unless a narrower one fills the rounds clearly better
      best_score = score;
      best = bn;
    }
  }
  if (tile_rows == 64) {
    switch (best) {
      case 256: return launch_grouped_bn<MODE, 256, 64>(a, rows_cap, K, N, w_host, E, plan, epi, sms, stream, fmt, scales);
      case 128: return launch_grouped_bn<MODE, 128, 64>(a, rows_cap, K, N, w_host, E, plan, epi, sms, stream, fmt, scales);
      case 64: return launch_grouped_bn<MODE, 64, 64>(a, rows_cap, K, N, w_host, E, plan, epi, sms, stream, fmt, scales);
      default: return launch_grouped_bn<MODE, 32, 64>(a, rows_cap, K, N, w_host, E, plan, epi, sms, stream, fmt, scales);
    }
  }
  switch (best) {
    case 256: return launch_grouped_bn<MODE, 256, 32>(a, rows_cap, K, N, w_host, E, plan, epi, sms, stream, fmt, scales);
    case 128: return launch_grouped_bn<MODE, 128, 32>(a, rows_cap, K, N, w_host, E, plan, epi, sms, stream, fmt, scales);
    case 64: return launch_grouped_bn<MODE, 64, 32>(a, rows_cap, K, N, w_host, E, plan, epi, sms, stream, fmt, scales);
    default: return launch_grouped_bn<MODE, 32, 32>(a, rows_cap, K, N, w_host, E, plan, epi, sms, stream, fmt, scales);
  }
}

}  // namespace mb200
