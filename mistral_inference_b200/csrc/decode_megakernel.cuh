// Persistent decode step: ONE cooperative kernel per generated token (batch 1).
//
// Why: a batch-1 decode step streams ~14.2 GB of weights through ~160 dependent matrix-vector products of
// 5-36 us each.  As separate kernels every boundary drains the memory pipe (launch + ramp-up + tail is of the
// same order as the kernels themselves), which is what caps the per-op path near 50 % of the HBM roofline.
// Here one CTA per SM lives for the whole token:
//   * a PRODUCER warp walks the CTA's static weight schedule for the whole model (every layer's QKV / wo /
//     gate-up / down slice and the lm-head slice are contiguous row ranges known up front) and streams it with
//     cp.async.bulk (TMA bulk copies, completion on mbarriers) through a shared-memory ring (12 x 16 KB on an H100).
//     Weights do not depend on activations, so the producer never waits for a phase boundary: while the consumers sit
//     in a grid barrier the ring keeps filling, and HBM stays busy across all ~190 dependencies.
//   * 8 CONSUMER warps do the math out of shared memory (fp32 FMA on bf16 pairs; batch 1 is ~0.1 flop/byte, far
//     below the CUDA-core roof, tensor cores would not help), with the same fused prologues/epilogues as the
//     per-op kernels (RMSNorm, RoPE + ring scatter, SiLU*mul, residual adds) and the same rounding points as the
//     reference (SURVEY.md Appendix A).
//   * phases are separated by a grid barrier on monotonic counters (6 per layer, see grid_barrier).
// Row pairs (2 rows = one RoPE pair / one gate-up pair) are dealt to CTAs as contiguous ranges:
// CTA c owns pairs [c*P/G, (c+1)*P/G) of each matrix, so its slice of every weight matrix is one contiguous byte
// range and load imbalance is at most one pair.
// Attention (phases 2a/2b) is flash-decoding split by POSITION: CTA c owns ring slots [c*C, (c+1)*C) of the sequence for ALL
// kv heads, which is one contiguous byte range of the [W, KV, hd] ring for K and one for V -- so it streams through the same
// shared-memory ring as the weights (large bulk copies, issued by the producer long before phase 1 ends; DRAM-friendly, unlike
// per-head 256-byte rows at a 2 KB stride).  Warp w serves kv head w (its H/KV query heads) over the slice, so no cross-warp merge
// is needed; every slice publishes (m, l, acc) per head and phase 2b merges the slices with all loads in flight at once.
// Only the row of the token being decoded (written in phase 1 by other CTAs) is read from global memory after the barrier.
#pragma once
#include "common.cuh"
#include "gemm_mma.cuh"

namespace mb200 {

constexpr int MK_CONSUMER_WARPS = 8;
constexpr int MK_CONSUMERS = MK_CONSUMER_WARPS * 32;
constexpr int MK_PRODUCER_WARPS = 2;  // one issuing thread each, stages dealt round-robin (a single thread is ~700 cycles per stage: the stage period)
constexpr int MK_THREADS = MK_CONSUMERS + 32 * MK_PRODUCER_WARPS;
constexpr int MK_WEIGHT_STAGE_BYTES = 16 * 1024;   // a weight stage: 2 rows x KC elements x 2 B
constexpr int MK_MAX_KC = MK_WEIGHT_STAGE_BYTES / 4;  // elements per row chunk
constexpr int MK_MAX_KC8 = MK_WEIGHT_STAGE_BYTES / 2;  // elements per row chunk of an e4m3 matrix (FP8 dense weights)
constexpr int MK_KV_PAD = 16;                      // K/V position rows are laid out with a 16-byte pad (ldmatrix bank spread)
constexpr int MK_STAGE_BYTES = 16 * 1024 + 16 * MK_KV_PAD;  // ring slot stride: also fits 8 padded 2 KB K/V position rows
constexpr int MK_MAX_STAGES = 12;
constexpr int MK_MAX_SPLITS = 32;

struct MkLayer {  // 64 bytes, device array prepared by the caller (include/mistral_b200.h: mb200_layer_desc)
  const bf16* wqkv;
  const bf16* wo;
  const bf16* w13;
  const bf16* w2;
  const bf16* attn_norm;
  const bf16* ffn_norm;
  bf16* cache_k;  // [max_batch, W, KV, hd]
  bf16* cache_v;
};

// FP8 dense weights (include/mistral_b200.h: mb200_layer_desc_fp8): wqkv / wo / w13 / w2 of `w` point to e4m3 [N, K] matrices,
// s_* to their fp32 row scales.  The norms, the K/V ring and the lm head stay bf16.
struct MkLayerFp8 {
  MkLayer w;
  const float* s_qkv;
  const float* s_o;
  const float* s_13;
  const float* s_2;
};

struct MkParams {
  const MkLayer* layers;  // W8: an MkLayerFp8 array
  const int32_t* windows;  // [n_layers] ring size per layer
  // Mixture of experts (moe.py:16-32): n_experts == 0 -> dense FeedForward (layers[l].w13 / w2)
  int n_experts, top_k;
  const bf16* const* moe_gate;  // [n_layers]              router weight [E, dim]
  const bf16* const* moe_w13;   // [n_layers * n_experts]  expert gate/up, packed like w13
  const bf16* const* moe_w2;    // [n_layers * n_experts]  expert down
  int n_layers;
  const bf16* emb;         // [V, dim]
  const bf16* final_norm;  // [dim]
  const bf16* w_out;       // [V, dim]
  const float* rope;       // [n_pos, 64, 2]
  const int64_t* token;    // device scalar: the token to embed
  int pos;                 // absolute position of that token
  int batch_row;           // which row of the cache this sequence uses
  float* logits;           // [V] fp32
  long long* next_token;   // optional: greedy argmax of the logits (first index on ties, like torch.argmax), or null
  unsigned long long* argmax_slots;  // [gridDim] per-CTA (value, index) keys
  int* argmax_counter;     // self-resetting
  int dim, hidden, H, KV, vocab;
  float eps;
  int n_stages, xs_bytes;
  // scratch (global)
  unsigned* bar_flags;  // grid barrier counter (monotonic, never reset)
  unsigned* bar_epoch;  // device word: number of barriers completed by previous launches (published by the last CTA to finish)
  int* done_counter;    // self-resetting: CTAs that have finished this launch
  bf16* xbuf;           // [2][dim] residual stream ping-pong
  bf16* hbuf;           // [dim]
  bf16* qbuf;           // [H*hd]
  bf16* abuf;           // [H*hd] attention output
  bf16* gbuf;           // [hidden]
  float* partial;       // [KV][splits][REP][hd+2]
  unsigned long long* prof_bar;  // optional [gridDim][n_layers][6][2] arrive/leave %globaltimer of every CTA at every barrier
  unsigned long long* prof;  // optional [8][n_layers][MK_PROF_WORDS] debug timeline of 8 sampled CTAs (see mk_stamp), or null
};

// Debug timeline of 8 sampled CTAs (every 21st): prof[sample][layer][MK_PROF_WORDS] uint64.
//   words 0..15   %globaltimer when consumer thread 0 passes a phase boundary (mk_stamp; 12..15: inside attention)
//   words 16..21  ns the producers spent blocked in the stages of that layer (the lm head counts to the last layer), ADDED
//                 to the buffer, which the caller zero-fills: 16 + producer = waiting for a free slot (ring full),
//                 18 + producer = waiting on the in-flight cap, 20 + producer = the ring-full waits of MK_PROF_LONG_NS or
//                 more: the ring stayed full through a consumer stall, so the SM's share of HBM went idle
//   words 22..23  unused
constexpr int MK_PROF_STAMPS = 16;
constexpr int MK_PROF_WORDS = 24;
constexpr unsigned long long MK_PROF_LONG_NS = 1000;
__device__ __forceinline__ void mk_stamp(const MkParams& p, int tid, int layer, int idx) {
  if (p.prof != nullptr && tid == 0 && blockIdx.x % 21 == 0) {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    p.prof[((blockIdx.x / 21) * p.n_layers + layer) * MK_PROF_WORDS + idx] = t;
  }
}

// ---- PTX: mbarrier + bulk copy ------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_n(uint64_t* bar, uint32_t n) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(n) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// Watchdog: a protocol bug in a persistent cooperative kernel is a GPU hang; every spin loop therefore gives up after
// ~seconds, prints what it was waiting for and traps, which turns the hang into a reportable launch failure.
#ifndef MB200_WATCHDOG_SPINS
#define MB200_WATCHDOG_SPINS (1u << 22)
#endif
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity, int tag = 0, uint32_t it = 0) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins == MB200_WATCHDOG_SPINS) {
      printf("[mb200 watchdog] block %d thread %d stuck in mbarrier wait tag=%d it=%u parity=%u\n", (int)blockIdx.x, (int)threadIdx.x, tag, it,
             parity);
      __trap();
    }
  }
}
// The same wait for kernels that issue wgmma: it traps without the printf, because a function call anywhere in such a kernel
// makes ptxas serialize the whole wgmma pipeline.
__device__ __forceinline__ void mbar_wait_quiet(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins == MB200_WATCHDOG_SPINS) __trap();
  }
}
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)),
               "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void consumer_sync() { asm volatile("bar.sync 1, %0;" ::"n"(MK_CONSUMERS) : "memory"); }

__device__ __forceinline__ uint4 ldcg16(const void* p) { return __ldcg(reinterpret_cast<const uint4*>(p)); }
__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

// Grid barrier among the consumer threads of all CTAs: ONE monotonically increasing counter, never reset.  Thread 0 of each
// CTA arrives with a single release atomic; it alone polls the word with acquire loads.  The k-th barrier of a launch is
// complete when the counter reaches base + k * gridDim, where `base` comes from the host (launch count x barriers per launch
// x gridDim), so nothing has to be read or reset on the device.
// (Measured alternatives on 148 CTAs: counter + generation word with fences 5 us; one flag per CTA polled by 148 threads of
// every CTA 1.5 us when arrivals are spread out but 4-5 us when all CTAs arrive together -- 22 K simultaneous polls.)
// Arrivals are spread over MK_BAR_WORDS counters on different 128-byte lines (bar_word_of below): when all CTAs arrive
// within ~0.5 us (after the short wo / down phases) 148 same-address atomics serialise at one L2 slice (~3 us measured).
constexpr int MK_BAR_WORDS = 8;
__device__ __forceinline__ void st_release_u32(unsigned* p, unsigned v) {
  asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void red_add_release_u32(unsigned* p, unsigned v) {
  asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void bar_stamp(const MkParams& p, int tid, int layer, int which, int leave) {
  if (p.prof_bar != nullptr && tid == 0) {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    p.prof_bar[(((int64_t)blockIdx.x * p.n_layers + layer) * 6 + which) * 2 + leave] = t;
  }
}
// Word j collects the arrivals of a CONTIGUOUS range of CTAs (c -> c * 8 / gridDim).  Waiting for one range only, so that a
// phase could start on the input chunks of the CTAs that have finished, was tried and dropped (see the down projection).
__device__ __forceinline__ int bar_word_of(int cta) { return (cta * MK_BAR_WORDS) / (int)gridDim.x; }
__device__ __forceinline__ unsigned bar_word_count(int j) {  // number of CTAs mapping to word j
  const int G = (int)gridDim.x;
  // first cta with c*8/G >= j  is ceil(j*G/8)
  const int lo = (j * G + MK_BAR_WORDS - 1) / MK_BAR_WORDS, hi = ((j + 1) * G + MK_BAR_WORDS - 1) / MK_BAR_WORDS;
  return (unsigned)(hi - lo);
}
__device__ __forceinline__ void grid_barrier(const MkParams& p, int tid, unsigned& epoch, int layer, int which) {
  ++epoch;  // number of barriers completed once this one is
  bar_stamp(p, tid, layer, which, 0);
  consumer_sync();  // every consumer thread's global writes of this phase happen-before thread 0's release below
  if (tid == 0) red_add_release_u32(p.bar_flags + bar_word_of(blockIdx.x) * 32, 1u);
  // thread j < 8 waits until every CTA of word j has arrived at barrier number `epoch`
  if (tid < MK_BAR_WORDS) {
    const unsigned target = epoch * bar_word_count(tid);
    unsigned spins = 0;
    while ((int)(ld_acquire_u32(p.bar_flags + tid * 32) - target) < 0) {
      if (++spins == MB200_WATCHDOG_SPINS) {
        printf("[mb200 watchdog] block %d stuck in grid barrier word %d target=%u counter=%u\n", (int)blockIdx.x, tid, target,
               ld_acquire_u32(p.bar_flags + tid * 32));
        __trap();
      }
    }
  }
  consumer_sync();
  bar_stamp(p, tid, layer, which, 1);
}

// How a [N, K] matrix is cut for the ring: pairs of rows, K in `nch` chunks of `kc` elements.
// An e4m3 matrix (w8) is cut with twice the elements per chunk: a stage carries at most the same 16 KB (7B's dim-4096 rows: 8 KB).
struct MatCut {
  int pairs, nch, kc, p0, p1;
};
__device__ __forceinline__ MatCut cut_matrix(int N, int K, bool w8 = false) {
  MatCut c;
  c.pairs = N >> 1;
  const int max_kc = w8 ? MK_MAX_KC8 : MK_MAX_KC;
  c.nch = (K + max_kc - 1) / max_kc;
  c.kc = K / c.nch;
  c.p0 = (int)(((long long)blockIdx.x * c.pairs) / gridDim.x);
  c.p1 = (int)(((long long)(blockIdx.x + 1) * c.pairs) / gridDim.x);
  return c;
}

// FP8 dense weights: an e4m3 matrix whose rows are at most 4 KB (7B's dim-4096 rows) carries TWO pairs per stage, so that a stage
// stays at 16 KB (the bytes in flight of the bf16 ring, the same per-stage cost for the producers).  Warps 2i and 2i + 1 of a group
// read stage i (the two pairs are four contiguous rows); each arrives MK_CONSUMER_WARPS / 2 times on its empty barrier, or
// MK_CONSUMER_WARPS when its pair is alone in the stage (the last pair of an odd group).  A group of g pairs has (g + 1) / 2 stages,
// so a warp's stages stay within one lap of the ring (tests/test_fp8_dense_cpu.py model-checks the order).
__device__ __forceinline__ bool two_pairs_per_stage(const MatCut& c, bool w8) { return w8 && c.nch == 1 && 4 * c.kc <= MK_WEIGHT_STAGE_BYTES; }
__device__ __forceinline__ int matrix_stages(const MatCut& c, bool w8) {
  const int P = c.p1 - c.p0;
  return two_pairs_per_stage(c, w8) ? (P / MK_CONSUMER_WARPS) * (MK_CONSUMER_WARPS / 2) + ((P % MK_CONSUMER_WARPS) + 1) / 2 : P * c.nch;
}

// routing decision of one MoE layer (moe.py:24-32), produced on every CTA by moe_route
constexpr int MK_MAX_TOPK = 4;
struct MoeRoute {
  int e[MK_MAX_TOPK];    // selected experts in ASCENDING expert index (the order `results +=` runs in, moe.py:29-31)
  float w[MK_MAX_TOPK];  // their routing weights (bf16 values)
};

struct RingState {
  uint32_t it;  // running stage counter (same sequence in producer and consumers)
};

// Stage order inside a matrix (same in producer and consumers): the CTA's pairs are taken in GROUPS of up to 8 (one pair
// per consumer warp); inside a group the stages are chunk-major: (pair g0+0, ch 0) ... (pair g0+g-1, ch 0), (pair g0+0, ch 1) ...
// So warp w touches stages base + ch*g + w: never more than 8 apart, i.e. always within one lap of the (>= 9-stage) ring --
// which is what makes parity-based mbarrier waits safe (a waiter two laps ahead would alias and pass early).

constexpr float kMaskedScore = -1.0e30f;

// ---- attention slice of this CTA (same arithmetic in producer and consumers) ---------------------------------
struct AttnSlice {
  int C, k_begin, k_end, n_kvst, pps, n_slices;  // positions per CTA, my range, my K (= V) stage count, positions per stage
};
__device__ __forceinline__ AttnSlice attn_slice(const MkParams& p, int W) {
  AttnSlice a;
  const int len = min(p.pos + 1, W);
  a.C = (len + (int)gridDim.x - 1) / (int)gridDim.x;
  a.n_slices = (len + a.C - 1) / a.C;
  a.k_begin = min((int)blockIdx.x * a.C, len);
  a.k_end = min(a.k_begin + a.C, len);
  a.pps = min(16, (MK_STAGE_BYTES / (p.KV * kHeadDim * 2 + MK_KV_PAD)) & ~7);  // 8 or 16 positions per stage (one MMA key block)
  a.n_kvst = (a.k_end - a.k_begin + a.pps - 1) / a.pps;
  return a;
}

// ---- producer (one thread per producer warp) ---------------------------------------------------------------------------
// The CTA's whole schedule (every layer: QKV slice, K/V slice, wo, gate/up, down slices; then the lm-head slice) is a pure
// function of (blockIdx, shapes, pos) and, on MoE layers, of the layer's routing decision.  A `Walk` is a position in it: the
// producer steps it once per stage and blocks only on free ring slots, the in-flight cap and MoE route gates.
// Per-stage budget: a 16 KB stage lasts ~1,300 cycles at one SM's share of HBM on an H100 (~25 GB/s; ~2,600 cycles per issuing
// thread), so a few integer divisions per stage are free.  Measured on an H100 80GB HBM3 at a 400 W power limit (Mistral-7B,
// batch 1, 4k context): this walk decodes at 172.6-173.0 tok/s where the nested loops it replaced ran at 168.5-168.9 (on a
// B200, at ~350 cycles per stage, a schedule iterator had cost 5 %).
// Experiment on record: an L2 look-ahead -- a second Walk issuing cp.async.bulk.prefetch.L2 for the stages up to D past the
// copy cursor while the producer is blocked, so that HBM keeps streaming when a consumer stall outlasts the ring -- measured
// slower on the same H100: 171.3-171.8 tok/s at D = 8, 16 or 24 stages, 170.2-171.6 with an evict-first hint on the
// prefetches (on a B200 the prefetched lines did not survive until the copy), although the debug timeline shows the ring
// staying full through consumer stalls for ~9.5 us of a 167 us layer (DESIGN.md section 3.1): the prefetches are issued by
// the same producer threads through the same bulk-copy path as the copies, and cost more than the idle time they cover.
// Each stage is one or more bulk copies that land in the stage's ring slot: `count` pieces of `bytes`, `src_step` elements
// apart in global memory and `dst_step` bytes apart in the slot.
struct StageCopy {
  const bf16* src;
  int64_t src_step;
  uint32_t bytes, dst_step;
  int count;
};

enum : int { SEG_QKV, SEG_KV, SEG_WO, SEG_UP, SEG_DOWN };  // segments of a layer, in stream order (SEG_UP once per expert)

template <bool W8 = false>
struct Walk {
  uint32_t it;              // running stage number (the consumers' RingState::it of the same stage)
  int layer, seg, e, s, n;  // layer (n_layers: the lm head), segment, gate/up expert of a MoE layer, stage s of the segment's n
  MatCut c;                 // matrix: its cut (row length c.kc * c.nch)
  bool w8;                  // W8: the matrix is e4m3 (every layer matrix; not the lm head)
  int k_begin, k_end, pps;  // K/V slice: positions and positions per stage (attn_slice)
  const bf16* W;            // matrix (unused in a MoE down segment: one per routed expert), or the K rows of the K/V slice
  const bf16* V;            // V rows of the K/V slice

  __device__ __forceinline__ bool done(const MkParams& p) const { return layer > p.n_layers; }
  // the gate/up segment of a MoE layer whose routing decision the producer does not hold yet: expert weights are unknown
  __device__ __forceinline__ bool gated(const MkParams& p, int routed) const {
    return p.n_experts != 0 && layer < p.n_layers && seg == SEG_UP && e == 0 && routed != layer;
  }
  __device__ __forceinline__ void matrix(const bf16* w, int N, int K, bool e4m3 = false) {
    W = w;
    w8 = e4m3;
    c = cut_matrix(N, K, e4m3);
    n = matrix_stages(c, e4m3);
  }
  // experts interleaved per group of pairs: the routed ones in the down segment of a MoE layer, else 1
  __device__ __forceinline__ int experts(const MkParams& p) const { return (seg == SEG_DOWN && p.n_experts) ? p.top_k : 1; }
  // shape of the current segment; `sel` packs the routed experts of the current MoE layer, 8 bits each, ascending
  __device__ __forceinline__ void setup(const MkParams& p, uint32_t sel) {
    const int q_dim = p.H * kHeadDim, kv_dim = p.KV * kHeadDim;
    s = 0;
    if (layer == p.n_layers) {
      matrix(p.w_out, p.vocab, p.dim);
      return;
    }
    const MkLayer& L = W8 ? reinterpret_cast<const MkLayerFp8*>(p.layers)[layer].w : p.layers[layer];
    if (seg == SEG_QKV) {
      matrix(L.wqkv, q_dim + 2 * kv_dim, p.dim, W8);
    } else if (seg == SEG_KV) {
      const int win = p.windows[layer];
      const AttnSlice a = attn_slice(p, win);
      k_begin = a.k_begin;
      k_end = a.k_end;
      pps = a.pps;
      n = 2 * a.n_kvst;  // alternating K / V stages
      W = L.cache_k + ((int64_t)p.batch_row * win) * kv_dim;
      V = L.cache_v + ((int64_t)p.batch_row * win) * kv_dim;
    } else if (seg == SEG_WO) {
      matrix(L.wo, p.dim, q_dim, W8);
    } else if (seg == SEG_UP) {
      matrix(p.n_experts ? p.moe_w13[layer * p.n_experts + ((sel >> (8 * e)) & 0xff)] : L.w13, 2 * p.hidden, p.dim, W8);
    } else {
      matrix(L.w2, p.dim, p.hidden, W8);
      n *= experts(p);
    }
  }
  __device__ __forceinline__ void next_segment(const MkParams& p) {
    if (layer == p.n_layers) {
      ++layer;
      return;
    }
    if (seg == SEG_UP && ++e < (p.n_experts ? p.top_k : 1)) return;
    e = 0;
    if (++seg > SEG_DOWN) {
      seg = SEG_QKV;
      ++layer;
    }
  }
  // moves to the first stage at or after the current segment (skipping segments with no stage on this CTA); stops with n = 0
  // at the end of the schedule or at a route gate
  __device__ __forceinline__ void settle(const MkParams& p, uint32_t sel, int routed) {
    for (;;) {
      n = 0;
      if (done(p) || gated(p, routed)) return;
      setup(p, sel);
      if (n > 0) return;
      next_segment(p);
    }
  }
  __device__ __forceinline__ void next(const MkParams& p, uint32_t sel, int routed) {
    ++it;
    if (++s < n) return;
    next_segment(p);
    settle(p, sel, routed);
  }

  // the copies of stage s, in the order the consumers expect: a matrix slice in groups of up to 8 pairs, inside a group
  // expert-major, then chunk-major (stage (j, ch, w) holds K-chunk ch of pair g0 + w of expert j); the K/V slice alternates
  // K and V stages of `pps` position rows, one copy per row so that rows sit (row bytes + MK_KV_PAD) apart in the slot
  // (8 consecutive rows then cover all 32 banks for ldmatrix)
  __device__ __forceinline__ StageCopy stage(const MkParams& p, uint32_t sel) const {
    StageCopy sc;
    if (seg == SEG_KV) {
      const int64_t row_elems = (int64_t)p.KV * kHeadDim;
      const int k0 = k_begin + (s >> 1) * pps;
      sc.src = ((s & 1) ? V : W) + (int64_t)k0 * row_elems;
      sc.src_step = row_elems;
      sc.bytes = (uint32_t)row_elems * 2;
      sc.dst_step = sc.bytes + MK_KV_PAD;
      sc.count = min(pps, k_end - k0);
      return sc;
    }
    const int ne = experts(p), K = c.kc * c.nch;
    const int per_group = MK_CONSUMER_WARPS * c.nch * ne;
    const int gi = s / per_group, r = s - gi * per_group;
    const int g0 = c.p0 + gi * MK_CONSUMER_WARPS, g = min(MK_CONSUMER_WARPS, c.p1 - g0);
    const int j = r / (c.nch * g), r2 = r - j * (c.nch * g);
    const int ch = r2 / g, w = r2 - ch * g;
    const bf16* m = (seg == SEG_DOWN && p.n_experts) ? p.moe_w2[layer * p.n_experts + ((sel >> (8 * j)) & 0xff)] : W;
    if (W8 && w8 && two_pairs_per_stage(c, true)) {  // e4m3, two pairs (four contiguous rows) per stage
      constexpr int kStagesPerGroup = MK_CONSUMER_WARPS / 2;
      const int g0 = c.p0 + (s / kStagesPerGroup) * MK_CONSUMER_WARPS, first = g0 + 2 * (s % kStagesPerGroup);
      sc.src = m + (int64_t)first * K;  // K bytes per row, in bf16 units: pair p starts at row 2p
      sc.src_step = 0;
      sc.bytes = (uint32_t)(min(2, c.p1 - first) * 2 * c.kc);
      sc.dst_step = 0;
      sc.count = 1;
      return sc;
    }
    if (W8 && w8) {  // e4m3: K bytes per row, in bf16 units (K and kc are multiples of 16)
      const bf16* r8 = m + (int64_t)(g0 + w) * K;
      sc.bytes = (uint32_t)c.kc;
      sc.src = r8 + ((c.nch == 1) ? 0 : ch * (c.kc >> 1));
      sc.src_step = K >> 1;
      sc.dst_step = sc.bytes;
      sc.count = 2;
      if (c.nch == 1) {  // the two rows are contiguous
        sc.bytes *= 2;
        sc.count = 1;
      }
      return sc;
    }
    const bf16* r0 = m + (int64_t)(2 * (g0 + w)) * K;
    sc.bytes = (uint32_t)c.kc * 2;
    if (c.nch == 1) {  // the two rows are contiguous
      sc.src = r0;
      sc.src_step = 0;
      sc.bytes *= 2;
      sc.dst_step = 0;
      sc.count = 1;
    } else {
      sc.src = r0 + ch * c.kc;
      sc.src_step = K;
      sc.dst_step = sc.bytes;
      sc.count = 2;
    }
    return sc;
  }
};

__device__ __forceinline__ void bulk_g2s_hint(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar, uint64_t policy) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(
                   smem_u32(smem_dst)),
               "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
               : "memory");
}
__device__ __forceinline__ unsigned long long globaltimer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}

// In-flight cap: stage `it` is only issued once stage it - cap has LANDED.  All n_stages slots still buffer data through the
// phase boundaries, but the SM never has more than `cap` stages of copies queued: right after a short phase the
// consumers have drained the whole ring, and an uncapped producer then fires 12 x 16 KB at once -- the grid barrier's own
// atomic / polls queue behind that burst in the SM's memory request path (measured: barrier latency 4 us after the wo
// phase vs 1.5 us in steady state).  The bandwidth-delay product of one SM's HBM share is only ~3 stages.  The cap applies to
// every stage, K/V slice stages included.
constexpr int MK_INFLIGHT_CAP = 5;
static_assert(MK_INFLIGHT_CAP <= MK_CONSUMER_WARPS, "below the smallest ring decode_plan accepts (n_stages > MK_CONSUMER_WARPS)");
template <bool W8 = false>
struct Producer {
  uint8_t* ring;
  uint64_t* full;
  uint64_t* empty;
  int n_stages;
  uint64_t policy;  // L2 evict-first: weights and old K/V rows are read exactly once per token
  int me;                  // this producer issues the stages with it % MK_PRODUCER_WARPS == me
  uint32_t slot, par;      // ring slot / parity of the copy cursor's stage, kept incrementally (no division in the issue loop)
  uint32_t cslot, cpar;    // same for stage it - MK_INFLIGHT_CAP
  uint32_t sel;            // routed experts of MoE layer `routed`, 8 bits each (ascending)
  int routed;
  unsigned long long* prof;  // this CTA's rows of the debug timeline, or null

  __device__ __forceinline__ bool owns(uint32_t it) const { return (int)(it % (uint32_t)MK_PRODUCER_WARPS) == me; }
  __device__ __forceinline__ void advance(uint32_t it) {  // ring position of stage it + 1 (`it` = the stage just passed)
    if (++slot == (uint32_t)n_stages) {
      slot = 0;
      par ^= 1;
    }
    if (it + 1 > (uint32_t)MK_INFLIGHT_CAP && ++cslot == (uint32_t)n_stages) {
      cslot = 0;
      cpar ^= 1;
    }
  }

  // fills the ring slot of the copy cursor's stage once stage it - cap has landed (its slot cannot have been refilled yet) and
  // the slot is free.  With the timeline on, the time blocked on either condition is added to the producer's words of the
  // copy cursor's layer.
  __device__ __forceinline__ void copy(const MkParams& p, const Walk<W8>& cp) {
    bool landed = cp.it < (uint32_t)MK_INFLIGHT_CAP || mbar_try_wait(&full[cslot], cpar);
    if (!landed || !mbar_try_wait(&empty[slot], par ^ 1)) {
      const unsigned long long t0 = prof != nullptr ? globaltimer() : 0ull;
      unsigned long long t_landed = t0;
      for (uint32_t spins = 0;;) {
        if (!landed && mbar_try_wait(&full[cslot], cpar)) {
          landed = true;
          if (prof != nullptr) t_landed = globaltimer();
        }
        if (landed && mbar_try_wait(&empty[slot], par ^ 1)) break;
        // the watchdog traps without the printf: a call in this loop makes ptxas spill around it (+256 B of spill loads); a
        // stuck producer still shows as consumers stuck on `full` in their own watchdog reports
        if (++spins == MB200_WATCHDOG_SPINS) __trap();
      }
      if (prof != nullptr) {
        const unsigned long long full_ns = globaltimer() - t_landed;
        unsigned long long* row = prof + (int64_t)min(cp.layer, p.n_layers - 1) * MK_PROF_WORDS + MK_PROF_STAMPS;
        row[me] += full_ns;
        row[2 + me] += t_landed - t0;
        if (full_ns >= MK_PROF_LONG_NS) row[4 + me] += full_ns;
      }
    }
    const StageCopy sc = cp.stage(p, sel);
    uint64_t* bar = &full[slot];
    mbar_arrive_expect_tx(bar, sc.bytes * (uint32_t)sc.count);
    uint8_t* dst = ring + (size_t)slot * MK_STAGE_BYTES;
    for (int r = 0; r < sc.count; ++r) bulk_g2s_hint(dst + r * sc.dst_step, sc.src + r * sc.src_step, sc.bytes, bar, policy);
  }
};

template <bool W8 = false>
__device__ __forceinline__ void producer_main(const MkParams& p, uint8_t* ring, uint64_t* full, uint64_t* empty, int me, const MoeRoute* route,
                                              uint64_t* route_bar) {
  Producer<W8> pr;
  pr.ring = ring;
  pr.full = full;
  pr.empty = empty;
  pr.n_stages = p.n_stages;
  pr.me = me;
  pr.slot = pr.par = pr.cslot = pr.cpar = 0;
  pr.sel = 0;
  pr.routed = -1;
  pr.prof = (p.prof != nullptr && blockIdx.x % 21 == 0) ? p.prof + (int64_t)(blockIdx.x / 21) * p.n_layers * MK_PROF_WORDS : nullptr;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pr.policy));
  Walk<W8> cp;
  cp.it = 0;
  cp.layer = cp.seg = cp.e = 0;
  cp.settle(p, pr.sel, pr.routed);
  while (!cp.done(p)) {
    if (cp.n == 0) {
      // a MoE layer's route gate: expert weights are data dependent, so wait for the layer's routing decision (the only
      // point where the weight stream cannot run ahead of the activations)
      mbar_wait(route_bar, (uint32_t)(cp.layer & 1), 8, (uint32_t)cp.layer);
      uint32_t sel = 0;
      for (int j = 0; j < p.top_k; ++j) sel |= (uint32_t)route->e[j] << (8 * j);
      pr.sel = sel;
      pr.routed = cp.layer;
      cp.settle(p, pr.sel, pr.routed);
      continue;
    }
    if (pr.owns(cp.it)) pr.copy(p, cp);
    pr.advance(cp.it);
    cp.next(p, pr.sel, pr.routed);
  }
}

// ---- consumers: one weight stage of a pair -----------------------------------------------------------------------------
// Waits for ring stage `it`, adds this lane's share of (row 0 . xc) to a0 and of (row 1 . xc) to a1 (kc8 16-byte chunks per row,
// 32 lanes x 16 B per step, unrolled -> plenty of ILP) and releases the slot: the calling warp is its only reader (empty
// barriers count MK_CONSUMER_WARPS arrivals, all from that warp).
__device__ __forceinline__ void consume_pair_stage(const uint8_t* ring, uint64_t* full, uint64_t* empty, int n_stages, uint32_t it,
                                                   const uint4* xc, int kc8, int lane, float& a0, float& a1) {
  const uint32_t slot = it % n_stages, par = (it / n_stages) & 1;
  // Guard (tests/test_megakernel_protocol.py): bulk copies land out of order, so this warp may get here before the
  // slot's PREVIOUS fill (owned by another warp) has landed; `full` would then still be one phase behind and a
  // parity wait would alias and pass early.  Waiting first until that previous fill has been CONSUMED (same
  // condition the producer waits for before refilling) pins `full` to phase {r, r+1} when it is tested.
  mbar_wait(&empty[slot], par ^ 1, 2, it);
  mbar_wait(&full[slot], par, 3, it);
  const uint4* w0 = reinterpret_cast<const uint4*>(ring + (size_t)slot * MK_STAGE_BYTES);
  const uint4* w1 = w0 + kc8;
#pragma unroll 4
  for (int i = lane; i < kc8; i += 32) {
    const uint4 a = w0[i], b = w1[i], x = xc[i];
    const uint32_t aw[4] = {a.x, a.y, a.z, a.w}, bw[4] = {b.x, b.y, b.z, b.w}, xw[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float xl = bf16lo(xw[j]), xh = bf16hi(xw[j]);
      a0 = fmaf(bf16lo(aw[j]), xl, a0);
      a0 = fmaf(bf16hi(aw[j]), xh, a0);
      a1 = fmaf(bf16lo(bw[j]), xl, a1);
      a1 = fmaf(bf16hi(bw[j]), xh, a1);
    }
  }
  __syncwarp();
  if (lane == 0) mbar_arrive_n(&empty[slot], MK_CONSUMER_WARPS);
}

// The same for a stage of an e4m3 pair (FP8 dense weights): kq 16-byte chunks per row, each 16 weights converted exactly
// (e4m3x2_to_float2) and FMA'd against x chunks 2i, 2i + 1 in the bf16 path's element order.
// The pair's rows start `row0` 16-byte chunks into the stage; the warp arrives `arrivals` times on the empty barrier.
__device__ __forceinline__ void consume_pair_stage_w8(const uint8_t* ring, uint64_t* full, uint64_t* empty, int n_stages, uint32_t it,
                                                      const uint4* xc, int kq, int row0, uint32_t arrivals, int lane, float& a0, float& a1) {
  const uint32_t slot = it % n_stages, par = (it / n_stages) & 1;
  mbar_wait(&empty[slot], par ^ 1, 2, it);  // see consume_pair_stage
  mbar_wait(&full[slot], par, 3, it);
  const uint4* w0 = reinterpret_cast<const uint4*>(ring + (size_t)slot * MK_STAGE_BYTES) + row0;
  const uint4* w1 = w0 + kq;
#pragma unroll 2
  for (int i = lane; i < kq; i += 32) {
    const uint4 a = w0[i], b = w1[i];
    const uint32_t aq[4] = {a.x, a.y, a.z, a.w}, bq[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const uint4 x = xc[2 * i + h];
      const uint32_t xw[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 af = e4m3x2_to_float2(aq[2 * h + (j >> 1)] >> (16 * (j & 1)));
        const float2 bf = e4m3x2_to_float2(bq[2 * h + (j >> 1)] >> (16 * (j & 1)));
        const float xl = bf16lo(xw[j]), xh = bf16hi(xw[j]);
        a0 = fmaf(af.x, xl, a0);
        a0 = fmaf(af.y, xh, a0);
        a1 = fmaf(bf.x, xl, a1);
        a1 = fmaf(bf.y, xh, a1);
      }
    }
  }
  __syncwarp();
  if (lane == 0) mbar_arrive_n(&empty[slot], arrivals);
}

// ---- consumers: y[pair] = W[pair rows] . xs, epilogue(pair, acc0, acc1) on one lane ----------------
// Warp-per-pair inside a group: warp w owns pair g0+w and consumes its `nch` stages by itself.  One block barrier per GROUP
// keeps all warps within a group of each other (see the stage-order note above).
// `pre(n)` runs on the finishing lane BEFORE the pair's stages are consumed and its result is handed to `epi`: loads the
// epilogue needs (the residual) are then off the critical path of the phase's last pair (an L2 round trip right before the
// barrier's release store: measured 3.2-4.2 us barrier latency after wo / down vs 1.75 us after gate/up, which loads nothing).
// W8: an e4m3 matrix with fp32 row scales `wscale`; the finishing lane loads the pair's scales with `pre` and hands
// epi fp32(s * acc), the one product of the FP8 definition, in place of acc.
template <bool W8 = false, class Pre, class Epi>
__device__ __forceinline__ void consume_matrix(int N, int K, const uint8_t* ring, uint64_t* full, uint64_t* empty, int n_stages, RingState& rs,
                                               const uint4* xs, int tid, Pre pre, Epi epi, const float* wscale = nullptr) {
  const MatCut c = cut_matrix(N, K, W8);
  const bool two = two_pairs_per_stage(c, W8);
  const int lane = tid & 31, warp = tid >> 5;
  const int kc8 = c.kc >> 3;  // 16-byte chunks per row chunk
  for (int g0 = c.p0; g0 < c.p1; g0 += MK_CONSUMER_WARPS) {
    const int g = min(MK_CONSUMER_WARPS, c.p1 - g0);
    const int g_stages = two ? (g + 1) >> 1 : g * c.nch;
    if (warp < g) {
      uint2 prefetched = make_uint2(0u, 0u);
      float2 ws = make_float2(1.f, 1.f);
      if (lane == 0) {
        prefetched = pre(2 * (g0 + warp));
        if constexpr (W8) ws = __ldg(reinterpret_cast<const float2*>(wscale + 2 * (g0 + warp)));
      }
      float a0 = 0.f, a1 = 0.f;
      for (int ch = 0; ch < c.nch; ++ch) {
        if constexpr (W8) {
          if (two)
            consume_pair_stage_w8(ring, full, empty, n_stages, rs.it + (uint32_t)(warp >> 1), xs, c.kc >> 4, (warp & 1) * (c.kc >> 3),
                                  (warp == g - 1 && (g & 1)) ? MK_CONSUMER_WARPS : MK_CONSUMER_WARPS / 2, lane, a0, a1);
          else
            consume_pair_stage_w8(ring, full, empty, n_stages, rs.it + (uint32_t)(ch * g + warp), xs + ch * kc8, c.kc >> 4, 0, MK_CONSUMER_WARPS,
                                  lane, a0, a1);
        } else
          consume_pair_stage(ring, full, empty, n_stages, rs.it + (uint32_t)(ch * g + warp), xs + ch * kc8, kc8, lane, a0, a1);
      }
      a0 = warp_sum(a0);
      a1 = warp_sum(a1);
      if constexpr (W8) {
        a0 = __fmul_rn(ws.x, a0);
        a1 = __fmul_rn(ws.y, a1);
      }
      if (lane == 0) epi(2 * (g0 + warp), a0, a1, prefetched);
    }
    rs.it += (uint32_t)g_stages;
    consumer_sync();
  }
}

// ---- consumers: stage an activation vector (written by other CTAs: L2 loads) and optionally RMS-normalise it ----
__device__ __forceinline__ void stage_x(uint4* xs, const bf16* src, const bf16* norm_w, int K, float eps, float* red, int tid) {
  const int kc = K >> 3;
#pragma unroll 4
  for (int i = tid; i < kc; i += MK_CONSUMERS) xs[i] = ldcg16(reinterpret_cast<const uint4*>(src) + i);
  consumer_sync();
  if (norm_w == nullptr) return;
  const int lane = tid & 31, warp = tid >> 5;
  float ss = 0.f;
  for (int i = tid; i < kc; i += MK_CONSUMERS) {
    const uint4 v = xs[i];
    const uint32_t u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float a = bf16lo(u[j]), b = bf16hi(u[j]);
      ss = fmaf(a, a, ss);
      ss = fmaf(b, b, ss);
    }
  }
  ss = warp_sum(ss);
  if (lane == 0) red[warp] = ss;
  consumer_sync();
  float tot = 0.f;
#pragma unroll
  for (int w = 0; w < MK_CONSUMER_WARPS; ++w) tot += red[w];
  const float r = ref_rsqrt(tot / (float)K + eps);
  const uint4* wn = reinterpret_cast<const uint4*>(norm_w);
  for (int i = tid; i < kc; i += MK_CONSUMERS) {
    const uint4 v = xs[i], g = wn[i];
    const uint32_t u[4] = {v.x, v.y, v.z, v.w}, gw[4] = {g.x, g.y, g.z, g.w};
    uint32_t o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j)
      o[j] = pack_bf16x2(round_bf16(bf16lo(u[j]) * r) * bf16lo(gw[j]), round_bf16(bf16hi(u[j]) * r) * bf16hi(gw[j]));
    xs[i] = make_uint4(o[0], o[1], o[2], o[3]);
  }
  consumer_sync();
}

__device__ __forceinline__ uint32_t ldcg_u32(const void* p) { return __ldcg(reinterpret_cast<const unsigned int*>(p)); }

// ---- phase 2a: partial attention of this CTA's position slice, all heads, out of the ring, on tensor cores --------------
// Warp w serves kv head w.  Per K/V stage pair (PPS = 8 or 16 positions = one key block) it computes
//   S[16 x PPS] = Q[16 x 128] K^T   with the REP query heads of the group as MMA rows 0..REP-1 (the other rows are zero),
//   online softmax on the accumulator fragments (fp32), P rounded to bf16 as the A operand, O[16 x 128] += P V.
// A CUDA-core version of the same loop (half a warp per key, shuffle-reduced dot products) is ISSUE bound: ~48 instructions
// per (key, head), 5.6 us per layer at kv_len 4096; this form is ~25x fewer instructions.  mma.sync (not wgmma): the tiles
// are tiny and the softmax lives in registers; the tensor pipe is idle otherwise.
// All 8 warps wait for (and release) every K/V stage; a warp touches only its own head's 256-byte segment of each row, so the
// fresh row of the token being decoded and the zero-fill of rows past the slice are patched per warp, without block syncs.
template <int REP, int PPS>
__device__ __forceinline__ void mk_attention_slice(const MkParams& p, const MkLayer& L, int W, uint8_t* ring, uint64_t* full, uint64_t* empty,
                                                   int n_stages, RingState& rs, int tid, int layer) {
  static_assert(REP <= 8, "query heads of a group are MMA rows 0..7");
  const AttnSlice a = attn_slice(p, W);
  if (a.n_kvst == 0) return;
  const int lane = tid & 31, warp = tid >> 5;
  const bool has_head = warp < p.KV;
  const int g = has_head ? warp : 0;
  const int row = lane >> 2, cq = lane & 3;  // accumulator fragment: row = lane/4, column pair = lane%4
  const float sl2 = 0.08838834764831845f * kLog2e;  // scores are scaled by hd^-0.5; softmax in the exp2 domain
  const int64_t row_elems = (int64_t)p.KV * kHeadDim;
  const uint32_t row_stride = (uint32_t)row_elems * 2 + MK_KV_PAD;  // bytes between position rows in a stage

  // Q as A fragments: a0 = (row, k..k+1), a2 = (row, k+8..k+9); rows >= REP and the row+8 halves are zero
  uint32_t qa[8][4];
#pragma unroll
  for (int ks = 0; ks < 8; ++ks) {
    qa[ks][0] = qa[ks][1] = qa[ks][2] = qa[ks][3] = 0u;
    if (row < REP) {
      const bf16* qp = p.qbuf + (g * REP + row) * kHeadDim + ks * 16 + cq * 2;
      qa[ks][0] = ldcg_u32(qp);
      qa[ks][2] = ldcg_u32(qp + 8);
    }
  }
  // the row of the token being decoded was written in phase 1: lanes 0-15 hold its K segment, lanes 16-31 its V segment
  const int cur = p.pos % W;
  uint4 cur_kv = make_uint4(0, 0, 0, 0);
  if (cur >= a.k_begin && cur < a.k_end) {
    const bf16* base = (lane < 16 ? L.cache_k : L.cache_v);
    cur_kv = ldcg16(base + ((int64_t)p.batch_row * W + cur) * row_elems + (int64_t)g * kHeadDim + (lane & 15) * 8);
  }
  float o[16][4];
#pragma unroll
  for (int n = 0; n < 16; ++n) o[n][0] = o[n][1] = o[n][2] = o[n][3] = 0.f;
  float m_run = kMaskedScore, l_run = 0.f;  // state of row `row` (this lane's share of l; reduced over the 4 lanes at the end)

  for (int j = 0; j < a.n_kvst; ++j) {
    const uint32_t itk = rs.it + 2u * j, itv = itk + 1;
    const uint32_t sk = itk % n_stages, pk = (itk / n_stages) & 1, sv = itv % n_stages, pv = (itv / n_stages) & 1;
    mbar_wait(&full[sk], pk, 5, itk);  // every warp visits every K/V stage in order: never more than one lap from the barrier
    mbar_wait(&full[sv], pv, 6, itv);
    if (j == 0) mk_stamp(p, tid, layer, 14);
    if (j == a.n_kvst - 1) mk_stamp(p, tid, layer, 15);
    if (has_head) {
      const int k0 = a.k_begin + j * PPS;
      const int nk = min(PPS, a.k_end - k0);
      uint8_t* kst = ring + (size_t)sk * MK_STAGE_BYTES + g * (kHeadDim * 2);
      uint8_t* vst = ring + (size_t)sv * MK_STAGE_BYTES + g * (kHeadDim * 2);
      // patches (own 256-byte segments only): fresh current-token row; zero the V rows past the slice (P = 0 there, but 0 * NaN)
      if (cur >= k0 && cur < k0 + nk)
        *reinterpret_cast<uint4*>((lane < 16 ? kst : vst) + (size_t)(cur - k0) * row_stride + (lane & 15) * 16) = cur_kv;
      if (nk < PPS)
        for (int r = nk + (lane >> 4); r < PPS; r += 2) *reinterpret_cast<uint4*>(vst + (size_t)r * row_stride + (lane & 15) * 16) = make_uint4(0, 0, 0, 0);
      // generic-proxy writes to a slot that the producer will refill through the async proxy (TMA): order them
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      __syncwarp();

      // ---- S = Q K^T: PPS/8 key tiles x 8 k-steps; one ldmatrix.x4 = the B fragments of 2 k-steps for one key tile
      float sc[PPS / 8][4];
#pragma unroll
      for (int t = 0; t < PPS / 8; ++t) {
        sc[t][0] = sc[t][1] = sc[t][2] = sc[t][3] = 0.f;
        const uint32_t kaddr = smem_u32(kst) + (uint32_t)(t * 8 + (lane & 7)) * row_stride + (uint32_t)(lane >> 3) * 16;
#pragma unroll
        for (int k2 = 0; k2 < 4; ++k2) {
          uint32_t b0, b1, b2, b3;
          ldmatrix_x4(kaddr + k2 * 64, b0, b1, b2, b3);
          mma_bf16_16816(sc[t], qa[2 * k2], b0, b1);
          mma_bf16_16816(sc[t], qa[2 * k2 + 1], b2, b3);
        }
      }
      // ---- online softmax for row `row` (values c0, c1 of each key tile); keys >= nk are masked
      float mx = m_run;
#pragma unroll
      for (int t = 0; t < PPS / 8; ++t) {
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          const int key = t * 8 + cq * 2 + c;
          sc[t][c] = key < nk ? sc[t][c] * sl2 : kMaskedScore;
          mx = fmaxf(mx, sc[t][c]);
        }
      }
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float corr = exp2f(m_run - mx);
      m_run = mx;
      l_run *= corr;
      uint32_t pa[4] = {0u, 0u, 0u, 0u};  // P as the A fragment of one k16 step: a0 = keys 0-7, a2 = keys 8-15; rows + 8 stay zero
#pragma unroll
      for (int t = 0; t < PPS / 8; ++t) {
        const float e0 = exp2f(sc[t][0] - mx), e1 = exp2f(sc[t][1] - mx);  // masked: exp2(-1e30) = 0
        l_run += e0 + e1;
        pa[2 * t] = pack_bf16x2(e0, e1);
      }
#pragma unroll
      for (int n = 0; n < 16; ++n) {
        o[n][0] *= corr;
        o[n][1] *= corr;
      }
      // ---- O += P V: B = V^T fragments via ldmatrix.trans (rows = keys)
      if constexpr (PPS == 16) {
        const uint32_t vaddr = smem_u32(vst) + (uint32_t)((lane & 7) + ((lane >> 3) & 1) * 8) * row_stride + (uint32_t)(lane >> 4) * 16;
#pragma unroll
        for (int n2 = 0; n2 < 8; ++n2) {  // dim tiles 2*n2, 2*n2+1
          uint32_t b0, b1, b2, b3;
          ldmatrix_x4_trans(vaddr + n2 * 32, b0, b1, b2, b3);
          mma_bf16_16816(o[2 * n2], pa, b0, b1);
          mma_bf16_16816(o[2 * n2 + 1], pa, b2, b3);
        }
      } else {  // 8 keys: the k16 step's upper half (keys 8-15) is zero on both operands
        const uint32_t vaddr = smem_u32(vst) + (uint32_t)(lane & 7) * row_stride + (uint32_t)(lane >> 3) * 16;
#pragma unroll
        for (int n4 = 0; n4 < 4; ++n4) {  // dim tiles 4*n4 .. 4*n4+3
          uint32_t b0, b1, b2, b3;
          ldmatrix_x4_trans(vaddr + n4 * 64, b0, b1, b2, b3);
          mma_bf16_16816(o[4 * n4], pa, b0, 0u);
          mma_bf16_16816(o[4 * n4 + 1], pa, b1, 0u);
          mma_bf16_16816(o[4 * n4 + 2], pa, b2, 0u);
          mma_bf16_16816(o[4 * n4 + 3], pa, b3, 0u);
        }
      }
    }
    __syncwarp();
    if (lane == 0) {
      mbar_arrive(&empty[sk]);
      mbar_arrive(&empty[sv]);
    }
  }
  rs.it += 2u * a.n_kvst;
  if (!has_head) return;
  l_run += __shfl_xor_sync(0xffffffffu, l_run, 1);  // the 4 lanes of a row each summed their own columns
  l_run += __shfl_xor_sync(0xffffffffu, l_run, 2);
  if (row >= REP) return;
  // publish this slice's partial for query head g*REP + row; the merge works in the natural-exp domain: m / log2(e)
  m_run *= 0.6931471805599453f;
  const int PSTRIDE = kHeadDim + 2;
  float* mine = p.partial + ((int64_t)blockIdx.x * p.H + g * REP + row) * PSTRIDE;
#pragma unroll
  for (int n = 0; n < 16; ++n) *reinterpret_cast<float2*>(mine + 2 + n * 8 + cq * 2) = make_float2(o[n][0], o[n][1]);
  if (cq == 0) *reinterpret_cast<float2*>(mine) = make_float2(m_run, l_run);
}

// ---- phase 2b: merge the slices.  Unit u = (query head, 32-dim quarter); warp w folds slices w, w+8, ... (all loads issued
// before the first use), the 8 warps are folded through shared memory, lane = dim.
constexpr int MK_CMB_MAX = 20;  // slices per warp held in registers at once
__device__ __forceinline__ void mk_attention_combine(const MkParams& p, int W, int tid, float* scratch) {
  const AttnSlice a = attn_slice(p, W);
  const int lane = tid & 31, warp = tid >> 5;
  const int PSTRIDE = kHeadDim + 2;
  float* sm = scratch;  // [8 warps][34]: m, l, acc[32]
  for (int u = blockIdx.x; u < p.H * 4; u += gridDim.x) {
    const int h = u >> 2, q4 = u & 3;
    float m = kMaskedScore, l = 0.f, acc = 0.f;
    for (int a0 = warp; a0 < a.n_slices; a0 += MK_CONSUMER_WARPS * MK_CMB_MAX) {
      float mt[MK_CMB_MAX], lt[MK_CMB_MAX], at[MK_CMB_MAX];
#pragma unroll
      for (int i = 0; i < MK_CMB_MAX; ++i) {
        const int sl = a0 + i * MK_CONSUMER_WARPS;
        mt[i] = kMaskedScore;
        lt[i] = at[i] = 0.f;
        if (sl < a.n_slices) {
          const float* pp = p.partial + ((int64_t)sl * p.H + h) * PSTRIDE;
          const float2 ml = __ldcg(reinterpret_cast<const float2*>(pp));
          mt[i] = ml.x;
          lt[i] = ml.y;
          at[i] = __ldcg(pp + 2 + q4 * 32 + lane);
        }
      }
      // two passes: the max first, then every slice's weight is independent (no sequential rescale chain)
      float mn = m;
#pragma unroll
      for (int i = 0; i < MK_CMB_MAX; ++i) mn = fmaxf(mn, mt[i]);
      const float c0 = exp2f((m - mn) * kLog2e);
      l *= c0;
      acc *= c0;
#pragma unroll
      for (int i = 0; i < MK_CMB_MAX; ++i) {
        const float c1 = exp2f((mt[i] - mn) * kLog2e);
        l = fmaf(lt[i], c1, l);
        acc = fmaf(at[i], c1, acc);
      }
      m = mn;
    }
    sm[warp * 34 + 2 + lane] = acc;
    if (lane == 0) {
      sm[warp * 34] = m;
      sm[warp * 34 + 1] = l;
    }
    consumer_sync();
    if (warp == 0) {
      float mn = kMaskedScore;
#pragma unroll
      for (int w = 0; w < MK_CONSUMER_WARPS; ++w) mn = fmaxf(mn, sm[w * 34]);
      float lt = 0.f, at = 0.f;
#pragma unroll
      for (int w = 0; w < MK_CONSUMER_WARPS; ++w) {
        const float mw = sm[w * 34];
        const float c = exp2f((mw - mn) * kLog2e);
        lt += sm[w * 34 + 1] * c;
        at += sm[w * 34 + 2 + lane] * c;
      }
      p.abuf[h * kHeadDim + q4 * 32 + lane] = __float2bfloat16_rn(at / lt);
    }
    consumer_sync();
  }
}

// ---- mixture of experts (moe.py:24-32), batch 1 ------------------------------------------------------------------------------

// Router on every CTA (identical, deterministic): logits = bf16(hn . gate^T) (one warp per expert), top-k on the bf16 logits,
// softmax over the k selected in fp32, rounded to bf16 (moe.py:25-27).  Ties: lower expert index first.
__device__ __forceinline__ void moe_route(const MkParams& p, int layer, const uint4* xs, float* red, MoeRoute* route, uint64_t* route_bar, int tid) {
  const int lane = tid & 31, warp = tid >> 5;
  const bf16* gate = p.moe_gate[layer];
  const int kc = p.dim >> 3;
  for (int e = warp; e < p.n_experts; e += MK_CONSUMER_WARPS) {
    const uint4* wrow = reinterpret_cast<const uint4*>(gate + (int64_t)e * p.dim);
    float acc = 0.f;
    for (int i = lane; i < kc; i += 32) {
      const uint4 a = __ldg(wrow + i), x = xs[i];
      const uint32_t aw[4] = {a.x, a.y, a.z, a.w}, xw[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        acc = fmaf(bf16lo(aw[j]), bf16lo(xw[j]), acc);
        acc = fmaf(bf16hi(aw[j]), bf16hi(xw[j]), acc);
      }
    }
    acc = warp_sum(acc);
    if (lane == 0) red[8 + e] = round_bf16(acc);  // red[8..8+E): router logits (E <= 32)
  }
  consumer_sync();
  if (tid == 0) {
    int sel[MK_MAX_TOPK];
    float val[MK_MAX_TOPK];
    unsigned taken = 0;
    for (int j = 0; j < p.top_k; ++j) {
      int best = -1;
      for (int e = 0; e < p.n_experts; ++e)
        if (!((taken >> e) & 1u) && (best < 0 || red[8 + e] > red[8 + best])) best = e;
      taken |= 1u << best;
      sel[j] = best;
      val[j] = red[8 + best];
    }
    float den = 0.f, ex[MK_MAX_TOPK];
    for (int j = 0; j < p.top_k; ++j) {
      ex[j] = expf(val[j] - val[0]);  // val[0] is the maximum
      den += ex[j];
    }
    for (int j = 0; j < p.top_k; ++j) val[j] = round_bf16(ex[j] / den);
    // ascending expert order, weights travelling with their experts
    for (int a = 1; a < p.top_k; ++a)
      for (int b = a; b > 0 && sel[b] < sel[b - 1]; --b) {
        const int ts = sel[b];
        sel[b] = sel[b - 1];
        sel[b - 1] = ts;
        const float tv = val[b];
        val[b] = val[b - 1];
        val[b - 1] = tv;
      }
    for (int j = 0; j < p.top_k; ++j) {
      route->e[j] = sel[j];
      route->w[j] = val[j];
    }
    mbar_arrive(route_bar);  // release: the producers may read `route` and start streaming the selected experts
  }
  consumer_sync();
}

// Expert down projections with the reference's accumulation: for the selected experts in ascending index,
//   y_e = bf16(W2_e g_e);  t_e = bf16(w_e * y_e);  res = (first ? t_e : bf16(res + t_e));   out = bf16(h + res)
// Stage order per group of 8 pairs: expert-major, then chunk-major (mirrored by Producer::moe_down).
template <class Pre, class Epi>
__device__ __forceinline__ void consume_moe_down(const MkParams& p, const MoeRoute& rt, const uint8_t* ring, uint64_t* full, uint64_t* empty,
                                                 int n_stages, RingState& rs, const uint4* xs, int tid, Pre pre, Epi epi) {
  const MatCut c = cut_matrix(p.dim, p.hidden);
  const int lane = tid & 31, warp = tid >> 5;
  const int kc8 = c.kc >> 3;
  const int hid8 = p.hidden >> 3;
  for (int g0 = c.p0; g0 < c.p1; g0 += MK_CONSUMER_WARPS) {
    const int g = min(MK_CONSUMER_WARPS, c.p1 - g0);
    if (warp < g) {
      uint2 prefetched = make_uint2(0u, 0u);
      if (lane == 0) prefetched = pre(2 * (g0 + warp));
      float r0 = 0.f, r1 = 0.f;
      for (int j = 0; j < p.top_k; ++j) {
        float a0 = 0.f, a1 = 0.f;
        for (int ch = 0; ch < c.nch; ++ch)
          consume_pair_stage(ring, full, empty, n_stages, rs.it + (uint32_t)((j * c.nch + ch) * g + warp), xs + j * hid8 + ch * kc8, kc8,
                             lane, a0, a1);
        a0 = warp_sum(a0);
        a1 = warp_sum(a1);
        const float t0 = round_bf16(rt.w[j] * round_bf16(a0)), t1 = round_bf16(rt.w[j] * round_bf16(a1));
        r0 = (j == 0) ? t0 : round_bf16(r0 + t0);  // results starts at zero: bf16(0 + t) == t
        r1 = (j == 0) ? t1 : round_bf16(r1 + t1);
      }
      if (lane == 0) epi(2 * (g0 + warp), r0, r1, prefetched);
    }
    rs.it += (uint32_t)(g * c.nch * p.top_k);
    consumer_sync();
  }
}

// W8: FP8 dense weights (p.layers is an MkLayerFp8 array, no MoE): every layer matrix streams as e4m3, the lm head as bf16.
template <int REP, bool W8 = false>
__global__ void __launch_bounds__(MK_THREADS, 1) decode_megakernel(const MkParams p) {
  extern __shared__ __align__(128) uint8_t smem[];
  // layout: [ring: n_stages x 16 KB][xs: xs_bytes][barriers][reduction scratch]
  uint8_t* ring = smem;
  uint4* xs = reinterpret_cast<uint4*>(smem + (size_t)p.n_stages * MK_STAGE_BYTES);
  uint64_t* full = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(xs) + p.xs_bytes);
  uint64_t* empty = full + MK_MAX_STAGES;
  float* red = reinterpret_cast<float*>(empty + MK_MAX_STAGES);                       // [8]
  MoeRoute* route = reinterpret_cast<MoeRoute*>(red + 48);                            // routing decision of the current MoE layer
  uint64_t* route_bar = reinterpret_cast<uint64_t*>(route + 1);                       // consumers -> producers: "route is valid"

  const int tid = threadIdx.x;
  if (tid == 0) {
    for (int i = 0; i < p.n_stages; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], MK_CONSUMER_WARPS);  // weight stages: the owning warp arrives x8; K/V stages: every warp x1
    }
    mbar_init(route_bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const int q_dim = p.H * kHeadDim, kv_dim = p.KV * kHeadDim;
  RingState rs;
  rs.it = 0;

  if (tid >= MK_CONSUMERS) {
    // ================= producers (one thread per producer warp; weights and old K/V rows never wait for activations) =================
    if ((tid & 31) == 0) producer_main<W8>(p, ring, full, empty, (tid - MK_CONSUMERS) >> 5, route, route_bar);
    return;
  }

  // ================= consumer warps =================
  // barriers completed by previous launches on this workspace.  Nobody writes the word until every CTA of this launch has
  // finished (see the end of the kernel), and launches are stream ordered, so this read cannot race.
  unsigned epoch = ld_acquire_u32(p.bar_epoch);
  const int64_t token = *p.token;
  for (int l = 0; l < p.n_layers; ++l) {
    const MkLayer L = W8 ? reinterpret_cast<const MkLayerFp8*>(p.layers)[l].w : p.layers[l];
    const MkLayerFp8* L8 = W8 ? reinterpret_cast<const MkLayerFp8*>(p.layers) + l : nullptr;
    const int W = p.windows[l];
    const bf16* x_in = (l == 0) ? p.emb + token * p.dim : p.xbuf + (size_t)(l & 1) * p.dim;
    bf16* x_out = p.xbuf + (size_t)((l + 1) & 1) * p.dim;

    // ---- phase 1: RMSNorm + QKV + RoPE + ring scatter ----
    mk_stamp(p, tid, l, 0);
    stage_x(xs, x_in, L.attn_norm, p.dim, p.eps, red, tid);
    mk_stamp(p, tid, l, 1);
    {
      const int slot_row = p.batch_row * W + p.pos % W;
      const float* rope_row = p.rope + (int64_t)p.pos * (kHeadDim / 2) * 2;
      bf16* ck = L.cache_k + (int64_t)slot_row * kv_dim;
      bf16* cv = L.cache_v + (int64_t)slot_row * kv_dim;
      consume_matrix<W8>(q_dim + 2 * kv_dim, p.dim, ring, full, empty, p.n_stages, rs, xs, tid,
                     [&](int n) { return *reinterpret_cast<const uint2*>(rope_row + ((n & (kHeadDim - 1)) >> 1) * 2); },
                     [&](int n, float a0, float a1, uint2 pf) {
        const float y0 = round_bf16(a0), y1 = round_bf16(a1);
        if (n < q_dim + kv_dim) {
          const float2 cs = make_float2(__uint_as_float(pf.x), __uint_as_float(pf.y));
          float re, im;
          ref_cmul(y0, y1, cs.x, cs.y, re, im);
          const uint32_t packed = pack_bf16x2(re, im);
          if (n < q_dim)
            *reinterpret_cast<uint32_t*>(p.qbuf + n) = packed;
          else
            *reinterpret_cast<uint32_t*>(ck + (n - q_dim)) = packed;
        } else {
          *reinterpret_cast<uint32_t*>(cv + (n - q_dim - kv_dim)) = pack_bf16x2(y0, y1);
        }
      }, W8 ? L8->s_qkv : nullptr);
    }
    mk_stamp(p, tid, l, 2);
    grid_barrier(p, tid, epoch, l, 0);
    mk_stamp(p, tid, l, 3);

    // ---- phase 2a: partial attention of my position slice;  2b: merge the slices ----
    if (attn_slice(p, W).pps == 16)
      mk_attention_slice<REP, 16>(p, L, W, ring, full, empty, p.n_stages, rs, tid, l);
    else
      mk_attention_slice<REP, 8>(p, L, W, ring, full, empty, p.n_stages, rs, tid, l);
    mk_stamp(p, tid, l, 12);
    grid_barrier(p, tid, epoch, l, 1);
    mk_stamp(p, tid, l, 13);
    mk_attention_combine(p, W, tid, reinterpret_cast<float*>(xs));
    mk_stamp(p, tid, l, 4);
    grid_barrier(p, tid, epoch, l, 2);
    mk_stamp(p, tid, l, 5);

    // ---- phase 3: wo + residual ----
    stage_x(xs, p.abuf, nullptr, q_dim, 0.f, red, tid);
    consume_matrix<W8>(p.dim, q_dim, ring, full, empty, p.n_stages, rs, xs, tid, [&](int n) { return make_uint2(ldcg_u32(x_in + n), 0u); }, [&](int n, float a0, float a1, uint2 pf) {
      const uint32_t r = pf.x;
      *reinterpret_cast<uint32_t*>(p.hbuf + n) = pack_bf16x2(round_bf16(a0) + bf16lo(r), round_bf16(a1) + bf16hi(r));
    }, W8 ? L8->s_o : nullptr);
    mk_stamp(p, tid, l, 6);
    grid_barrier(p, tid, epoch, l, 3);
    mk_stamp(p, tid, l, 7);

    if (p.n_experts == 0) {
    // ---- phase 4: RMSNorm + gate/up + SiLU*mul ----
      stage_x(xs, p.hbuf, L.ffn_norm, p.dim, p.eps, red, tid);
      consume_matrix<W8>(2 * p.hidden, p.dim, ring, full, empty, p.n_stages, rs, xs, tid, [&](int) { return make_uint2(0u, 0u); }, [&](int n, float a0, float a1, uint2) {
        const float s = round_bf16(ref_silu(round_bf16(a0)));
        p.gbuf[n >> 1] = __float2bfloat16_rn(s * round_bf16(a1));
      }, W8 ? L8->s_13 : nullptr);
      mk_stamp(p, tid, l, 8);
      grid_barrier(p, tid, epoch, l, 4);
      mk_stamp(p, tid, l, 9);

      // ---- phase 5: down + residual ----
      // (Tried: no full barrier here -- stage g chunk by chunk as the barrier words of the CTA range that produced each K-chunk
      //  complete, waiting on those words only.  Correct, but 4 polling rounds + 4 block syncs cost more than the ~5 us gate/up
      //  arrival skew they hide: 345 vs 351 tok/s.)
      stage_x(xs, p.gbuf, nullptr, p.hidden, 0.f, red, tid);
      consume_matrix<W8>(p.dim, p.hidden, ring, full, empty, p.n_stages, rs, xs, tid, [&](int n) { return make_uint2(ldcg_u32(p.hbuf + n), 0u); },
                     [&](int n, float a0, float a1, uint2 pf) {
                       const uint32_t r = pf.x;
                       *reinterpret_cast<uint32_t*>(x_out + n) = pack_bf16x2(round_bf16(a0) + bf16lo(r), round_bf16(a1) + bf16hi(r));
                     }, W8 ? L8->s_2 : nullptr);
    } else if constexpr (!W8) {
      // ---- phase 4 (MoE): RMSNorm + router; gate/up + SiLU*mul of the selected experts (ascending expert index) ----
      stage_x(xs, p.hbuf, L.ffn_norm, p.dim, p.eps, red, tid);
      moe_route(p, l, xs, red, route, route_bar, tid);
      const MoeRoute rt = *route;
      for (int j = 0; j < p.top_k; ++j) {
        bf16* gj = p.gbuf + (size_t)j * p.hidden;
        consume_matrix(2 * p.hidden, p.dim, ring, full, empty, p.n_stages, rs, xs, tid, [&](int) { return make_uint2(0u, 0u); },
                       [&](int n, float a0, float a1, uint2) {
                         const float sv = round_bf16(ref_silu(round_bf16(a0)));
                         gj[n >> 1] = __float2bfloat16_rn(sv * round_bf16(a1));
                       });
      }
      mk_stamp(p, tid, l, 8);
      grid_barrier(p, tid, epoch, l, 4);
      mk_stamp(p, tid, l, 9);
      // ---- phase 5 (MoE): expert down projections, weighted bf16 accumulation in expert order, + residual ----
      stage_x(xs, p.gbuf, nullptr, p.top_k * p.hidden, 0.f, red, tid);
      consume_moe_down(p, rt, ring, full, empty, p.n_stages, rs, xs, tid, [&](int n) { return make_uint2(ldcg_u32(p.hbuf + n), 0u); },
                       [&](int n, float r0, float r1, uint2 pf) {
                         *reinterpret_cast<uint32_t*>(x_out + n) = pack_bf16x2(r0 + bf16lo(pf.x), r1 + bf16hi(pf.x));
                       });
    }
    mk_stamp(p, tid, l, 10);
    grid_barrier(p, tid, epoch, l, 5);
    mk_stamp(p, tid, l, 11);
  }

  // ---- final RMSNorm + lm head (fp32 logits, each a bf16-rounded value) + greedy argmax ----
  stage_x(xs, p.xbuf + (size_t)(p.n_layers & 1) * p.dim, p.final_norm, p.dim, p.eps, red, tid);
  // the maximum argmax_key (common.cuh) over the row is torch.argmax's answer: among equal logits the SMALLEST index
  unsigned long long best = 0ull;
  consume_matrix(p.vocab, p.dim, ring, full, empty, p.n_stages, rs, xs, tid, [&](int) { return make_uint2(0u, 0u); },
                 [&](int n, float a0, float a1, uint2) {
                   const float y0 = round_bf16(a0), y1 = round_bf16(a1);
                   *reinterpret_cast<float2*>(p.logits + n) = make_float2(y0, y1);
                   const unsigned long long k0 = argmax_key(y0, n), k1 = argmax_key(y1, n + 1);
                   best = max(best, max(k0, k1));
                 });
  if (p.next_token != nullptr) {
    // lane 0 of every warp holds its pairs' best; CTA reduce through shared memory, then the last CTA to arrive reduces all
    unsigned long long* sm_best = reinterpret_cast<unsigned long long*>(xs);
    consumer_sync();
    if ((tid & 31) == 0) sm_best[tid >> 5] = best;
    consumer_sync();
    if (tid == 0) {
      unsigned long long b = 0ull;
#pragma unroll
      for (int w = 0; w < MK_CONSUMER_WARPS; ++w) b = max(b, sm_best[w]);
      p.argmax_slots[blockIdx.x] = b;
      __threadfence();
      const int prev = atomicAdd(p.argmax_counter, 1);
      if (prev == (int)gridDim.x - 1) {
        *p.argmax_counter = 0;
        __threadfence();
        unsigned long long g = 0ull;
        for (int c = 0; c < (int)gridDim.x; ++c) g = max(g, __ldcg(p.argmax_slots + c));
        *p.next_token = (long long)(0x7fffffff - (int)(g & 0xffffffffull));
      }
    }
  }
  // publish the barrier epoch for the next launch: the last CTA to get here (all CTAs are past every barrier by then)
  consumer_sync();
  if (tid == 0) {
    __threadfence();
    const int prev = atomicAdd(p.done_counter, 1);
    if (prev == (int)gridDim.x - 1) {
      *p.done_counter = 0;
      st_release_u32(p.bar_epoch, epoch);
    }
  }
}

}  // namespace mb200
