// First-prefill attention (varlen, causal, sliding window; every key comes from the new chunk) on wgmma / TMA.
//
// Roofline: tensor pipe / MUFU (one exp2 per score).  CTA = (query head, 128-query tile, sequence); three warpgroups:
//   warpgroup 0     TMA producer (one thread): Q tile once, then K and V tiles of 128 keys into a 3-stage ring (128B-swizzled
//                   [128 x 64] boxes)
//   warpgroups 1-2  64 query rows each: S[64 x 128] = Q K^T with both operands K-major in shared memory; masks (causal + window +
//                   sequence end; edge tiles only) and the online softmax in fp32 on the register fragment (a row is spread over
//                   the four threads of a quad); P -> bf16 stays in registers as the A operand of O[64 x 128] += P V, with V an
//                   MN-major shared-memory operand; final O / l -> bf16 -> global
// The mma.sync kernel (attn_prefill.cuh) remains for chunks that also read the ring (seqpos > 0) and for the cache-less mode.
#pragma once
#include "gemm_wgmma.cuh"

namespace mb200 {

constexpr int FA_BM = 128, FA_BN = 128, FA_THREADS = 384, FA_STAGES = 3;  // warpgroup 0 TMA, warpgroups 1-2 MMA + softmax
constexpr int FA_TILE_BYTES = 128 * kHeadDim * 2;  // one [128 x 128] bf16 tile = two swizzled [128 x 64] boxes = 32 KB
constexpr int FA_SMEM = FA_TILE_BYTES * (1 + 2 * FA_STAGES) + 128 /*barriers*/;  // 229,504 of 232,448 bytes

struct FaParams {
  const int32_t* q_start;  // [B+1]
  bf16* out;               // [T, H*hd]
  int T, B, W, H, KV;
  float scale_log2;
};

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

__global__ void __launch_bounds__(FA_THREADS, 1)
    attn_prefill_wgmma_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k,
                              const __grid_constant__ CUtensorMap map_v, const FaParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];  // SW128 tiles want 1024-byte alignment; there is no room left to pad by hand
  uint8_t* smem = smem_raw;
  if ((smem_u32(smem) & 1023u) != 0) __trap();
  uint8_t* sQ = smem;
  uint8_t* sKV = smem + FA_TILE_BYTES;  // stage s: K at sKV + s*2*TILE, V right after
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + FA_TILE_BYTES * (1 + 2 * FA_STAGES));
  uint64_t* q_full = bars;        // TMA -> consumers
  uint64_t* kv_full = bars + 1;   // [3] TMA -> consumers
  uint64_t* kv_empty = bars + 4;  // [3] consumers (one arrival per warpgroup) -> TMA

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int h = blockIdx.x, b = blockIdx.z, g = h / (p.H / p.KV);
  const int tok0 = p.q_start[b], s_len = p.q_start[b + 1] - tok0;
  // Heads vary fastest and the heavier (later) query tiles are dispatched first: longest-processing-time order for the causal
  // triangle, and the query heads of one KV group read the same K/V tiles at the same time (L2 locality).
  const int qt = (int)gridDim.y - 1 - (int)blockIdx.y;
  const int i0 = qt * FA_BM;
  if (i0 >= s_len) return;
  const int i_end = min(i0 + FA_BM, s_len);
  const int key_lo = max(0, i0 - p.W + 1), key_hi = i_end - 1;  // visible keys of this tile: [key_lo, key_hi]
  const int n_tiles = (key_hi - key_lo + FA_BN) / FA_BN;

  if (threadIdx.x == 0) {
    mbar_init(q_full, 1);
    for (int i = 0; i < FA_STAGES; ++i) {
      mbar_init(&kv_full[i], 1);
      mbar_init(&kv_empty[i], 2);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == 0) {
    // ================= TMA producer =================
    if (lane == 0) {
      mbar_arrive_expect_tx(q_full, FA_TILE_BYTES);
      tma_load_2d(sQ, &map_q, q_full, h * kHeadDim, tok0 + i0);
      tma_load_2d(sQ + FA_TILE_BYTES / 2, &map_q, q_full, h * kHeadDim + 64, tok0 + i0);
      for (int t = 0; t < n_tiles; ++t) {
        const int s = t % FA_STAGES, par = (t / FA_STAGES) & 1;
        mbar_wait_quiet(&kv_empty[s], par ^ 1);
        mbar_arrive_expect_tx(&kv_full[s], 2 * FA_TILE_BYTES);
        uint8_t* sk = sKV + s * 2 * FA_TILE_BYTES;
        const int row = tok0 + key_lo + t * FA_BN;
        tma_load_2d(sk, &map_k, &kv_full[s], g * kHeadDim, row);
        tma_load_2d(sk + FA_TILE_BYTES / 2, &map_k, &kv_full[s], g * kHeadDim + 64, row);
        tma_load_2d(sk + FA_TILE_BYTES, &map_v, &kv_full[s], g * kHeadDim, row);
        tma_load_2d(sk + FA_TILE_BYTES + FA_TILE_BYTES / 2, &map_v, &kv_full[s], g * kHeadDim + 64, row);
      }
    }
  } else if (warp >= 4) {
    // ================= consumer warpgroups: query rows 64 * wg .. + 63 of the tile =================
    const int wg = (warp >> 2) - 1, wt = (int)threadIdx.x & 127;
    const int r = wg * 64 + ((warp & 3) << 4) + (lane >> 2), c0 = 2 * (lane & 3);  // fragment rows r, r + 8; columns c0 + 8j (+1)
    const int ia = i0 + r, ib = ia + 8;  // local query indices; position == index (first prefill: seqpos = 0)
    const bool va = ia < s_len, vb = ib < s_len;
    const uint32_t q_addr = smem_u32(sQ) + wg * 64 * 128;
    float o[64];
    float m_a = -1.0e30f, m_b = -1.0e30f, l_a = 0.f, l_b = 0.f;
    mbar_wait_quiet(q_full, 0);
    for (int t = 0; t < n_tiles; ++t) {
      const int s = t % FA_STAGES, par = (t / FA_STAGES) & 1;
      mbar_wait_quiet(&kv_full[s], par);
      const uint32_t k_addr = smem_u32(sKV + s * 2 * FA_TILE_BYTES);
      // S = Q K^T: 8 k-steps of 16 dims; dims 0..63 / 64..127 in two boxes 16 KB apart
      float sc[64];
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < 8; ++ks) {
        const uint32_t off = (ks >> 2) * (FA_TILE_BYTES / 2) + (ks & 3) * 32;
        wgmma_ss(sc, wgmma_desc_sw128(q_addr + off), wgmma_desc_sw128(k_addr + off), ks ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_acc(sc);
      const int j0 = key_lo + t * FA_BN + c0;
      // Only edge tiles need per-element masks (tile-uniform test): the causal diagonal, the window's lower edge, the ragged
      // end of the sequence.  Interior tiles take the straight-line path.
      const bool edge = (key_lo + t * FA_BN + FA_BN - 1 > i0) || (key_lo + t * FA_BN <= i0 + FA_BM - 1 - p.W) || (i0 + FA_BM > s_len);
      float mra = -3.0e38f, mrb = -3.0e38f;
#pragma unroll
      for (int jb = 0; jb < 16; ++jb) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float& xa = sc[4 * jb + e];
          float& xb = sc[4 * jb + 2 + e];
          if (edge) {
            const int j = j0 + 8 * jb + e;
            const bool oka = va && j <= ia && j > ia - p.W, okb = vb && j <= ib && j > ib - p.W;
            xa = oka ? xa : -INFINITY;  // exp2 gives exactly 0 below
            xb = okb ? xb : -INFINITY;
            mra = fmaxf(mra, oka ? xa : -3.0e38f);
            mrb = fmaxf(mrb, okb ? xb : -3.0e38f);
          } else {
            mra = fmaxf(mra, xa);
            mrb = fmaxf(mrb, xb);
          }
        }
      }
      mra = quad_max(mra);
      mrb = quad_max(mrb);
      const float mxa = fmaxf(m_a, mra > -1.0e38f ? mra * p.scale_log2 : -1.0e30f);
      const float mxb = fmaxf(m_b, mrb > -1.0e38f ? mrb * p.scale_log2 : -1.0e30f);
      if (t > 0) {  // rescale O and the partial row sums to the new maxima (a factor of exactly 1 where a maximum did not grow)
        const float ca = ex2_approx(m_a - mxa), cb = ex2_approx(m_b - mxb);
        l_a *= ca;
        l_b *= cb;
#pragma unroll
        for (int jb = 0; jb < 16; ++jb) {
          o[4 * jb] *= ca, o[4 * jb + 1] *= ca;
          o[4 * jb + 2] *= cb, o[4 * jb + 3] *= cb;
        }
      }
      m_a = mxa;
      m_b = mxb;
      // P = exp2(s * scale - m) as bf16 pairs in the A-operand fragment layout; O += P V, 16 keys per k-step
      uint32_t pk[32];
#pragma unroll
      for (int jb = 0; jb < 16; ++jb) {
        const float ea0 = ex2_approx(fmaf(sc[4 * jb], p.scale_log2, -mxa)), ea1 = ex2_approx(fmaf(sc[4 * jb + 1], p.scale_log2, -mxa));
        const float eb0 = ex2_approx(fmaf(sc[4 * jb + 2], p.scale_log2, -mxb)), eb1 = ex2_approx(fmaf(sc[4 * jb + 3], p.scale_log2, -mxb));
        l_a += ea0 + ea1;
        l_b += eb0 + eb1;
        pk[2 * jb] = pack2_rn(ea0, ea1);
        pk[2 * jb + 1] = pack2_rn(eb0, eb1);
      }
      const uint32_t v_addr = k_addr + FA_TILE_BYTES;
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < 8; ++ks) {  // keys 16 ks .. + 15 = n8 blocks 2 ks, 2 ks + 1 of S; V rows 16 ks (128 B each)
        const uint32_t a[4] = {pk[4 * ks], pk[4 * ks + 1], pk[4 * ks + 2], pk[4 * ks + 3]};
        wgmma_rs_bmn(o, a, wgmma_desc_sw128_mn(v_addr + ks * 2048, FA_TILE_BYTES / 2), (t | ks) ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_acc(o);
      if (wt == 0) mbar_arrive(&kv_empty[s]);  // K/V stage free once S and PV of this tile have read it
    }
    // final: O / l -> bf16 -> global; the row sum is the sum of the quad's partial sums
    l_a = quad_sum(l_a);
    l_b = quad_sum(l_b);
    const float inv_a = va ? 1.f / l_a : 0.f, inv_b = vb ? 1.f / l_b : 0.f;
    bf16* dst_a = p.out + (int64_t)(tok0 + ia) * p.H * kHeadDim + (int64_t)h * kHeadDim + c0;
    bf16* dst_b = dst_a + (int64_t)8 * p.H * kHeadDim;
#pragma unroll
    for (int jb = 0; jb < 16; ++jb) {
      if (va) *reinterpret_cast<uint32_t*>(dst_a + 8 * jb) = pack2_rn(o[4 * jb] * inv_a, o[4 * jb + 1] * inv_a);
      if (vb) *reinterpret_cast<uint32_t*>(dst_b + 8 * jb) = pack2_rn(o[4 * jb + 2] * inv_b, o[4 * jb + 3] * inv_b);
    }
  }
}

// [rows, cols] bf16 row-major, box = [128 rows x 64 cols], 128-byte swizzle
inline int make_tensor_map_rows(CUtensorMap* map, const void* base, int64_t rows, int64_t cols) {
  PFN_encodeTiled enc = get_encode_tiled();
  if (enc == nullptr) return fail(MB200_E_CUDA, "cuTensorMapEncodeTiled entry point not available");
  const cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  const cuuint64_t strides[1] = {(cuuint64_t)cols * 2};
  const cuuint32_t box[2] = {64, 128};
  const cuuint32_t estr[2] = {1, 1};
  const CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                         CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(MB200_E_CUDA, "cuTensorMapEncodeTiled (attention) failed (%d)", (int)r);
  return MB200_OK;
}

// MB200_ATTN=mma forces the mma.sync kernel.  Read at every launch, like the GEMM switches, so the tests can run both kernels on
// the same cases inside one process.
inline bool wgmma_attn_eligible(int64_t T, int64_t max_seqlen) {
  const char* e = getenv("MB200_ATTN");
  const bool forced = e != nullptr && e[0] == 'm';
  return !forced && T >= 128 && max_seqlen >= 128;
}

inline int launch_attn_prefill_wgmma(const void* q, const void* k_new, const void* v_new, const int32_t* q_start, void* out, int64_t T, int64_t B,
                                       int64_t max_seqlen, int64_t W, int64_t H, int64_t KV, cudaStream_t stream) {
  CUtensorMap mq, mk, mv;
  int rc = make_tensor_map_rows(&mq, q, T, H * kHeadDim);
  if (rc) return rc;
  rc = make_tensor_map_rows(&mk, k_new, T, KV * kHeadDim);
  if (rc) return rc;
  rc = make_tensor_map_rows(&mv, v_new, T, KV * kHeadDim);
  if (rc) return rc;
  FaParams p;
  p.q_start = q_start;
  p.out = (bf16*)out;
  p.T = (int)T;
  p.B = (int)B;
  p.W = (int)W;
  p.H = (int)H;
  p.KV = (int)KV;
  p.scale_log2 = 0.08838834764831845f * 1.4426950408889634f;
  MB_CHECK_CUDA(cudaFuncSetAttribute(attn_prefill_wgmma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, FA_SMEM));
  const dim3 grid((unsigned)H, (unsigned)ceil_div(max_seqlen, FA_BM), (unsigned)B);
  attn_prefill_wgmma_kernel<<<grid, FA_THREADS, FA_SMEM, stream>>>(mq, mk, mv, p);
  note_launch("attn_prefill_wgmma_kernel");
  MB_CHECK_LAUNCH("attn_prefill_wgmma_kernel");
  return MB200_OK;
}

}  // namespace mb200
