// GQA decode attention over the rotating KV cache for batched decode (B >= 2): TMA-staged K/V tiles, tensor-core scores.
//
// Roofline: HBM.  Algorithmic bytes per (sequence, layer) = 2 (K, V) * kv_len * KV * hd * 2 B.  A kernel that loads K/V rows
// into registers keeps only what its registers can hold in flight (~28 KB per SM at batch 32: 37 % of the HBM rate measured on
// Nemo-12B shapes); here the bytes in flight are decoupled from the math: one producer thread per CTA streams [64 keys x 128 dims]
// K and V tiles of one (sequence, kv head) into a 3-stage shared-memory ring with cp.async.bulk.tensor (two 128B-swizzled
// [64 x 64] boxes per tile; the ring rows are 2 KB apart in the [max_batch * W, KV * hd] cache -- strided rows are the TMA
// engine's job, not 256-byte requests from the SM), 96 KB in flight per CTA, two CTAs per SM.
// CTA = (split s, kv head g, sequence b): it owns ring slots [s*C, (s+1)*C) of that head, C = ceil(kv_len / S), and serves all
// H/KV query heads of the group from the same bytes (no repeat_kv, transformer_layers.py:84).  Softmax over the ring is
// order-free (RoPE was applied with absolute positions before caching), so slots are consumed in slot order like the
// reference's padded-keys mask (cache.py:250-254).  Four consumer warps take 16 keys each of every tile:  S[16 x 16] = Q K^T
// with the REP query heads as MMA rows (mma.sync m16n8k16; the tiles are tiny and softmax lives in the fragments), online
// softmax in fp32, P rounded to bf16, O[16 x 128] += P V.  Warps are merged through shared memory; with S > 1 each split
// publishes its (m, l, acc) partial and the last CTA to arrive per (b, g) merges them.  Slots >= kv_len are uninitialised
// memory in the reference (cache.py:166): their scores are masked by index and their V rows are zeroed in shared memory before
// the PV product.
// REP > 8 (H/KV = 12, Mistral Large 2): query heads 8 .. REP-1 of the group are MMA rows 8 .. REP-1 (the a1 / a3 halves of the Q
// fragment, o[n][2..3], a second running (m, l) per thread).  Their merge arrays (sm_acc, cm, cl: 30 KB at REP = 12) live in the
// K/V ring, which is idle once every tile is consumed, so the CTA keeps the shared-memory size that lets two of them share an SM.
#pragma once
#include "decode_megakernel.cuh"  // mbarrier helpers with the watchdog
#include "gemm_mma.cuh"
#include "gemm_wgmma.cuh"         // tma_load_2d, tensor-map encoder

namespace mb200 {

struct AttnDecodeParams {
  const bf16* q;        // [B, H*hd]
  const bf16* cache_k;  // [max_batch, W, KV, hd]
  const bf16* cache_v;
  const int32_t* kv_len;  // [B]
  bf16* out;              // [B, H*hd]
  float* partial;         // [B, KV, S, REP, hd + 2] (m, l, acc) when S > 1
  int* counters;          // [B, KV] zero-initialised once; self-resetting
  int B, W, H, KV, S;
  float scale;
};

constexpr int ADT_KT = 64;                                 // keys per tile
constexpr int ADT_STAGES = 3;
constexpr int ADT_HALF_BYTES = ADT_KT * 128;               // [64 keys][64 dims] bf16, 128-byte rows
constexpr int ADT_STAGE_BYTES = 4 * ADT_HALF_BYTES;        // K lo | K hi | V lo | V hi = 32 KB
constexpr int ADT_CONSUMER_WARPS = 4;
constexpr int ADT_THREADS = 32 * (ADT_CONSUMER_WARPS + 1);
constexpr int ADT_SMEM = ADT_STAGES * ADT_STAGE_BYTES + 1024 + 64;

// byte offset of 16-byte chunk C (0..15 over the 128 dims) of key row `row` inside a K or V tile (two swizzled halves)
__device__ __forceinline__ uint32_t adt_off(int row, int C) {
  return (uint32_t)((C >> 3) * ADT_HALF_BYTES + row * 128 + (((C & 7) ^ (row & 7)) << 4));
}

// The end of a decode CTA, after every warp has published its (m, l, acc) in sm_m / sm_l / sm_acc and the block has synchronised:
// merge the consumer warps and, with S > 1, the splits (the last CTA of a (b, g) to arrive combines them).  Shared by
// attn_decode_tma_kernel and attn_decode_tma_fp8_kernel (csrc/kv_fp8.cuh).
template <int REP>
__device__ __forceinline__ void adt_merge(const AttnDecodeParams& p, const float (&sm_m)[ADT_CONSUMER_WARPS][REP],
                                          const float (&sm_l)[ADT_CONSUMER_WARPS][REP], const float (&sm_acc)[ADT_CONSUMER_WARPS][REP][kHeadDim],
                                          int& is_last, float* cm, float* cl, int s, int g, int b, int tid, int warp) {
  constexpr float kMasked = -1.0e30f;
  if (warp == ADT_CONSUMER_WARPS) {
    if (p.S == 1) return;  // the producer warp takes no part in the merge
  }

  // ---- merge the warps: thread d (0..127) finishes dim d of every head of the group (log2 domain) ----
  const int d = tid;
  float fm[REP], fl[REP], fa[REP];
  if (warp < ADT_CONSUMER_WARPS) {
#pragma unroll
    for (int r = 0; r < REP; ++r) {
      float mn = kMasked;
#pragma unroll
      for (int w = 0; w < ADT_CONSUMER_WARPS; ++w) mn = fmaxf(mn, sm_m[w][r]);
      float lt = 0.f, at = 0.f;
#pragma unroll
      for (int w = 0; w < ADT_CONSUMER_WARPS; ++w) {
        const float c = exp2f(sm_m[w][r] - mn);  // empty warps: l = acc = 0
        lt += sm_l[w][r] * c;
        at += sm_acc[w][r][d] * c;
      }
      fm[r] = mn;
      fl[r] = lt;
      fa[r] = at;
    }
    if (p.S == 1) {
#pragma unroll
      for (int r = 0; r < REP; ++r) p.out[((int64_t)b * p.H + g * REP + r) * kHeadDim + d] = __float2bfloat16_rn(fa[r] / fl[r]);
      return;
    }
    // ---- publish the partial; the last split of this (b, g) to arrive combines all of them ----
    const int PSTRIDE = kHeadDim + 2;
    float* mine = p.partial + ((((int64_t)b * p.KV + g) * p.S + s) * REP) * PSTRIDE;
#pragma unroll
    for (int r = 0; r < REP; ++r) {
      mine[r * PSTRIDE + 2 + d] = fa[r];
      if (d == 0) {
        mine[r * PSTRIDE + 0] = fm[r];
        mine[r * PSTRIDE + 1] = fl[r];
      }
    }
    __threadfence();
  }
  __syncthreads();
  if (tid == 0) {
    const int prev = atomicAdd(&p.counters[b * p.KV + g], 1);
    is_last = (prev == p.S - 1);
    if (is_last) p.counters[b * p.KV + g] = 0;  // self-reset for the next launch (stream-ordered)
  }
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  const int PSTRIDE = kHeadDim + 2;
  const float* all = p.partial + (((int64_t)b * p.KV + g) * p.S) * REP * PSTRIDE;
  for (int i = tid; i < p.S * REP; i += ADT_THREADS) {
    cm[i] = __ldcg(all + (int64_t)i * PSTRIDE);
    cl[i] = __ldcg(all + (int64_t)i * PSTRIDE + 1);
  }
  __syncthreads();
  if (warp >= ADT_CONSUMER_WARPS) return;
#pragma unroll
  for (int r = 0; r < REP; ++r) {
    float mn = kMasked;
    for (int t = 0; t < p.S; ++t) mn = fmaxf(mn, cm[t * REP + r]);
    float lt = 0.f, at = 0.f;
#pragma unroll 8
    for (int t = 0; t < p.S; ++t) {
      const float c = exp2f(cm[t * REP + r] - mn);
      lt += cl[t * REP + r] * c;
      at += __ldcg(all + ((int64_t)t * REP + r) * PSTRIDE + 2 + d) * c;
    }
    p.out[((int64_t)b * p.H + g * REP + r) * kHeadDim + d] = __float2bfloat16_rn(at / lt);
  }
}

template <int REP>
__global__ void __launch_bounds__(ADT_THREADS, 2)
    attn_decode_tma_kernel(const __grid_constant__ CUtensorMap map_k, const __grid_constant__ CUtensorMap map_v, const AttnDecodeParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + ADT_STAGES * ADT_STAGE_BYTES);
  uint64_t* empty = full + ADT_STAGES;
  constexpr bool HI = REP > 8;  // query heads in MMA rows 8..15 too
  static_assert(REP <= 16, "one m16 MMA tile of query heads");
  __shared__ float sm_m[ADT_CONSUMER_WARPS][REP], sm_l[ADT_CONSUMER_WARPS][REP];
  __shared__ float sm_acc_s[ADT_CONSUMER_WARPS][HI ? 1 : REP][kHeadDim];
  __shared__ int is_last;
  __shared__ float cm_s[64 * (HI ? 1 : REP)], cl_s[64 * (HI ? 1 : REP)];
  typedef float AccArr[ADT_CONSUMER_WARPS][REP][kHeadDim];
  AccArr& sm_acc = HI ? *reinterpret_cast<AccArr*>(smem) : *reinterpret_cast<AccArr*>(&sm_acc_s[0][0][0]);
  float* cm = HI ? reinterpret_cast<float*>(smem + sizeof(AccArr)) : cm_s;
  float* cl = HI ? cm + 64 * REP : cl_s;
  static_assert(!HI || sizeof(AccArr) + 2 * 64 * REP * sizeof(float) <= ADT_STAGES * ADT_STAGE_BYTES, "merge arrays fit the ring");

  const int s = blockIdx.x, g = blockIdx.y, b = blockIdx.z;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  pdl_trigger();
  pdl_wait();  // q, the ring rows of this step and kv_len come from the preceding kernels
  const int len = p.kv_len[b];
  const int C = (len + p.S - 1) / p.S;
  const int k_begin = min(s * C, len), k_end = min(k_begin + C, len);
  const int n_tiles = (k_end - k_begin + ADT_KT - 1) / ADT_KT;

  if (tid == 0) {
    for (int i = 0; i < ADT_STAGES; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], ADT_CONSUMER_WARPS);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_k) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_v) : "memory");
  }
  __syncthreads();

  constexpr float kMasked = -1.0e30f;
  float o[16][4];
  float m_run = kMasked, l_run = 0.f;
  float m_hi = kMasked, l_hi = 0.f;  // HI: MMA row + 8
  const int row = lane >> 2, cq = lane & 3;

  if (warp == ADT_CONSUMER_WARPS) {
    // ================= producer: one thread =================
    if (lane == 0) {
      for (int j = 0; j < n_tiles; ++j) {
        const uint32_t st = j % ADT_STAGES, par = (j / ADT_STAGES) & 1;
        mbar_wait(&empty[st], par ^ 1, 31, j);
        mbar_arrive_expect_tx(&full[st], ADT_STAGE_BYTES);
        uint8_t* base = smem + st * ADT_STAGE_BYTES;
        const int r0 = b * p.W + k_begin + j * ADT_KT, c0 = g * kHeadDim;
        tma_load_2d(base, &map_k, &full[st], c0, r0);
        tma_load_2d(base + ADT_HALF_BYTES, &map_k, &full[st], c0 + 64, r0);
        tma_load_2d(base + 2 * ADT_HALF_BYTES, &map_v, &full[st], c0, r0);
        tma_load_2d(base + 3 * ADT_HALF_BYTES, &map_v, &full[st], c0 + 64, r0);
      }
    }
  } else {
    // ================= consumers: warp w owns keys [16 w, 16 w + 16) of every tile =================
    const float sl2 = p.scale * kLog2e;  // scores are scaled by hd^-0.5 (fp32, like the reference); softmax in the exp2 domain
    uint32_t qa[8][4];
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) {
      qa[ks][0] = qa[ks][1] = qa[ks][2] = qa[ks][3] = 0u;
      if (row < REP) {
        const bf16* qp = p.q + ((int64_t)b * p.H + g * REP + row) * kHeadDim + ks * 16 + cq * 2;
        qa[ks][0] = *reinterpret_cast<const uint32_t*>(qp);
        qa[ks][2] = *reinterpret_cast<const uint32_t*>(qp + 8);
      }
      if (HI && row + 8 < REP) {
        const bf16* qp = p.q + ((int64_t)b * p.H + g * REP + row + 8) * kHeadDim + ks * 16 + cq * 2;
        qa[ks][1] = *reinterpret_cast<const uint32_t*>(qp);
        qa[ks][3] = *reinterpret_cast<const uint32_t*>(qp + 8);
      }
    }
#pragma unroll
    for (int n = 0; n < 16; ++n) o[n][0] = o[n][1] = o[n][2] = o[n][3] = 0.f;

    for (int j = 0; j < n_tiles; ++j) {
      const uint32_t st = j % ADT_STAGES, par = (j / ADT_STAGES) & 1;
      mbar_wait(&full[st], par, 32, j);
      const uint32_t kst = smem_u32(smem + st * ADT_STAGE_BYTES), vst = kst + 2 * ADT_HALF_BYTES;
      const int nk = min(ADT_KT, k_end - (k_begin + j * ADT_KT)) - 16 * warp;  // valid keys among this warp's 16 (may be <= 0)
      if (nk < 16) {
        // V rows of slots past the range hold whatever the ring holds (P = 0 there, but 0 * NaN = NaN): zero them
        for (int i = lane; i < 16 * 16; i += 32) {
          const int r = i >> 4, c = i & 15;
          if (r >= nk) *reinterpret_cast<uint4*>(smem + st * ADT_STAGE_BYTES + 2 * ADT_HALF_BYTES + adt_off(16 * warp + r, c)) = make_uint4(0, 0, 0, 0);
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic writes before the slot is refilled by TMA
        __syncwarp();
      }
      if (nk > 0) {
        float sc[2][4];
#pragma unroll
        for (int t = 0; t < 2; ++t) {
          sc[t][0] = sc[t][1] = sc[t][2] = sc[t][3] = 0.f;
          const int krow = 16 * warp + t * 8 + (lane & 7);
#pragma unroll
          for (int k2 = 0; k2 < 4; ++k2) {
            uint32_t b0, b1, b2, b3;
            ldmatrix_x4(kst + adt_off(krow, k2 * 4 + (lane >> 3)), b0, b1, b2, b3);
            mma_bf16_16816(sc[t], qa[2 * k2], b0, b1);
            mma_bf16_16816(sc[t], qa[2 * k2 + 1], b2, b3);
          }
        }
        float mx = m_run;
#pragma unroll
        for (int t = 0; t < 2; ++t)
#pragma unroll
          for (int c = 0; c < 2; ++c) {
            const int key = t * 8 + cq * 2 + c;
            sc[t][c] = key < nk ? sc[t][c] * sl2 : kMasked;
            mx = fmaxf(mx, sc[t][c]);
          }
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
        const float corr = exp2f(m_run - mx);
        m_run = mx;
        l_run *= corr;
        uint32_t pa[4] = {0u, 0u, 0u, 0u};
#pragma unroll
        for (int t = 0; t < 2; ++t) {
          const float e0 = exp2f(sc[t][0] - mx), e1 = exp2f(sc[t][1] - mx);
          l_run += e0 + e1;
          pa[2 * t] = pack_bf16x2(e0, e1);
        }
#pragma unroll
        for (int n = 0; n < 16; ++n) {
          o[n][0] *= corr;
          o[n][1] *= corr;
        }
        if constexpr (HI) {  // the same online softmax for MMA row + 8 (accumulator elements 2, 3)
          float mx2 = m_hi;
#pragma unroll
          for (int t = 0; t < 2; ++t)
#pragma unroll
            for (int c = 2; c < 4; ++c) {
              const int key = t * 8 + cq * 2 + c - 2;
              sc[t][c] = key < nk ? sc[t][c] * sl2 : kMasked;
              mx2 = fmaxf(mx2, sc[t][c]);
            }
          mx2 = fmaxf(mx2, __shfl_xor_sync(0xffffffffu, mx2, 1));
          mx2 = fmaxf(mx2, __shfl_xor_sync(0xffffffffu, mx2, 2));
          const float corr2 = exp2f(m_hi - mx2);
          m_hi = mx2;
          l_hi *= corr2;
#pragma unroll
          for (int t = 0; t < 2; ++t) {
            const float e2 = exp2f(sc[t][2] - mx2), e3 = exp2f(sc[t][3] - mx2);
            l_hi += e2 + e3;
            pa[2 * t + 1] = pack_bf16x2(e2, e3);
          }
#pragma unroll
          for (int n = 0; n < 16; ++n) {
            o[n][2] *= corr2;
            o[n][3] *= corr2;
          }
        }
        const int vrow = 16 * warp + (lane & 7) + ((lane >> 3) & 1) * 8;
#pragma unroll
        for (int n2 = 0; n2 < 8; ++n2) {
          uint32_t b0, b1, b2, b3;
          ldmatrix_x4_trans(vst + adt_off(vrow, n2 * 2 + (lane >> 4)), b0, b1, b2, b3);
          mma_bf16_16816(o[2 * n2], pa, b0, b1);
          mma_bf16_16816(o[2 * n2 + 1], pa, b2, b3);
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[st]);
    }
    l_run += __shfl_xor_sync(0xffffffffu, l_run, 1);
    l_run += __shfl_xor_sync(0xffffffffu, l_run, 2);
    if constexpr (HI) {
      l_hi += __shfl_xor_sync(0xffffffffu, l_hi, 1);
      l_hi += __shfl_xor_sync(0xffffffffu, l_hi, 2);
    } else if (row < REP) {
#pragma unroll
      for (int n = 0; n < 16; ++n) {
        sm_acc[warp][row][n * 8 + cq * 2] = o[n][0];
        sm_acc[warp][row][n * 8 + cq * 2 + 1] = o[n][1];
      }
      if (cq == 0) {
        sm_m[warp][row] = m_run;
        sm_l[warp][row] = l_run;
      }
    }
  }
  if constexpr (HI) {
    __syncthreads();  // every warp is done with the ring: the merge arrays may overwrite it
    if (warp < ADT_CONSUMER_WARPS) {
#pragma unroll
      for (int n = 0; n < 16; ++n) {
        sm_acc[warp][row][n * 8 + cq * 2] = o[n][0];
        sm_acc[warp][row][n * 8 + cq * 2 + 1] = o[n][1];
      }
      if (cq == 0) {
        sm_m[warp][row] = m_run;
        sm_l[warp][row] = l_run;
      }
      if (row + 8 < REP) {
#pragma unroll
        for (int n = 0; n < 16; ++n) {
          sm_acc[warp][row + 8][n * 8 + cq * 2] = o[n][2];
          sm_acc[warp][row + 8][n * 8 + cq * 2 + 1] = o[n][3];
        }
        if (cq == 0) {
          sm_m[warp][row + 8] = m_hi;
          sm_l[warp][row + 8] = l_hi;
        }
      }
    }
  }
  __syncthreads();
  adt_merge<REP>(p, sm_m, sm_l, sm_acc, is_last, cm, cl, s, g, b, tid, warp);
}

// [rows, cols] bf16 row-major cache seen as a 2-D tensor; box = [64 cols (128 B) x 64 rows], 128-byte swizzle, OOB rows read as zero
inline int make_kv_tensor_map(CUtensorMap* map, const void* base, int64_t rows, int64_t cols) {
  PFN_encodeTiled enc = get_encode_tiled();
  if (enc == nullptr) return fail(MB200_E_CUDA, "cuTensorMapEncodeTiled entry point not available");
  const cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  const cuuint64_t strides[1] = {(cuuint64_t)cols * 2};
  const cuuint32_t box[2] = {64, (cuuint32_t)ADT_KT};
  const cuuint32_t estr[2] = {1, 1};
  const CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                         CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(MB200_E_CUDA, "cuTensorMapEncodeTiled (kv cache) failed (%d) rows=%lld cols=%lld", (int)r, (long long)rows, (long long)cols);
  return MB200_OK;
}

template <int REP>
int launch_attn_decode_tma(const AttnDecodeParams& p, int64_t max_batch_rows, cudaStream_t st) {
  CUtensorMap map_k, map_v;
  int rc = make_kv_tensor_map(&map_k, p.cache_k, max_batch_rows, (int64_t)p.KV * kHeadDim);
  if (rc) return rc;
  rc = make_kv_tensor_map(&map_v, p.cache_v, max_batch_rows, (int64_t)p.KV * kHeadDim);
  if (rc) return rc;
  MB_CHECK_CUDA(cudaFuncSetAttribute(attn_decode_tma_kernel<REP>, cudaFuncAttributeMaxDynamicSharedMemorySize, ADT_SMEM));
  const dim3 grid((unsigned)p.S, (unsigned)p.KV, (unsigned)p.B);
  MB_CHECK_CUDA(launch_pdl(attn_decode_tma_kernel<REP>, grid, dim3(ADT_THREADS), (size_t)ADT_SMEM, st, map_k, map_v, p));
  note_launch("attn_decode_tma_kernel<%d>", REP);
  return MB200_OK;
}

}  // namespace mb200
