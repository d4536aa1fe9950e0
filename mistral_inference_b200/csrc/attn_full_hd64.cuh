// Unmasked attention at head_dim 64 on wgmma / TMA: the cache-less mode (causal = 0) of mb200_attn_prefill for the vision
// encoder (vision_encoder.py:99 -> transformer_layers.py:88 with the mask dropped: every query attends to every key of the call).
//
// Roofline: tensor pipe / MUFU (one exp2 per score; at head_dim 64 the exp2 count per FLOP is twice the head_dim-128 kernel's).
// CTA = (query head, 128-query tile); three warpgroups, the structure of attn_prefill_wgmma_kernel:
//   warpgroup 0     TMA producer (one thread): the Q tile once, then K and V tiles of 128 keys into a 4-stage ring (one
//                   128B-swizzled [128 x 64] box each: a row of 64 bf16 is exactly one 128-byte swizzle row)
//   warpgroups 1-2  64 query rows each: S[64 x 128] = Q K^T (4 k-steps), online softmax in fp32 on the register fragment, P -> bf16
//                   in registers as the A operand of O[64 x 64] += P V (V MN-major in shared memory); final O / l -> bf16 -> global
// The only mask is the end of the key sequence, tested on the last tile only.  TMA zero-fills rows >= T (queries and keys), and
// rows >= T are never stored, so any T >= 1 works.
#pragma once
#include "attn_prefill_wgmma.cuh"

namespace mb200 {

constexpr int FH_HD = 64, FH_BM = 128, FH_BN = 128, FH_THREADS = 384, FH_STAGES = 4;
constexpr int FH_TILE_BYTES = 128 * FH_HD * 2;                          // one [128 x 64] bf16 box = 16 KB
constexpr int FH_SMEM = FH_TILE_BYTES * (1 + 2 * FH_STAGES) + 128;      // Q + 4 x (K, V) + barriers = 147,584 bytes

struct FhParams {
  bf16* out;  // [T, H*64]
  int T, H, KV;
  float scale_log2;  // 64^-0.5 * log2(e)
};

__global__ void __launch_bounds__(FH_THREADS, 1)
    attn_full_hd64_wgmma_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k,
                                const __grid_constant__ CUtensorMap map_v, const FhParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw;
  if ((smem_u32(smem) & 1023u) != 0) __trap();
  uint8_t* sQ = smem;
  uint8_t* sKV = smem + FH_TILE_BYTES;  // stage s: K at sKV + s*2*TILE, V right after
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + FH_TILE_BYTES * (1 + 2 * FH_STAGES));
  uint64_t* q_full = bars;
  uint64_t* kv_full = bars + 1;              // [FH_STAGES] TMA -> consumers
  uint64_t* kv_empty = bars + 1 + FH_STAGES;  // [FH_STAGES] consumers (one arrival per warpgroup) -> TMA

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int h = blockIdx.x, g = h / (p.H / p.KV);
  const int i0 = blockIdx.y * FH_BM;
  const int n_tiles = (p.T + FH_BN - 1) / FH_BN;

  if (threadIdx.x == 0) {
    mbar_init(q_full, 1);
    for (int i = 0; i < FH_STAGES; ++i) {
      mbar_init(&kv_full[i], 1);
      mbar_init(&kv_empty[i], 2);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == 0) {
    // ================= TMA producer =================
    if (lane == 0) {
      mbar_arrive_expect_tx(q_full, FH_TILE_BYTES);
      tma_load_2d(sQ, &map_q, q_full, h * FH_HD, i0);
      for (int t = 0; t < n_tiles; ++t) {
        const int s = t % FH_STAGES, par = (t / FH_STAGES) & 1;
        mbar_wait_quiet(&kv_empty[s], par ^ 1);
        mbar_arrive_expect_tx(&kv_full[s], 2 * FH_TILE_BYTES);
        uint8_t* sk = sKV + s * 2 * FH_TILE_BYTES;
        tma_load_2d(sk, &map_k, &kv_full[s], g * FH_HD, t * FH_BN);
        tma_load_2d(sk + FH_TILE_BYTES, &map_v, &kv_full[s], g * FH_HD, t * FH_BN);
      }
    }
  } else if (warp >= 4) {
    // ================= consumer warpgroups: query rows 64 * wg .. + 63 of the tile =================
    const int wg = (warp >> 2) - 1, wt = (int)threadIdx.x & 127;
    const int r = wg * 64 + ((warp & 3) << 4) + (lane >> 2), c0 = 2 * (lane & 3);  // fragment rows r, r + 8; columns c0 + 8j (+1)
    const int ia = i0 + r, ib = ia + 8;
    const uint32_t q_addr = smem_u32(sQ) + wg * 64 * 128;
    float o[32];
    float m_a = -1.0e30f, m_b = -1.0e30f, l_a = 0.f, l_b = 0.f;
    mbar_wait_quiet(q_full, 0);
    for (int t = 0; t < n_tiles; ++t) {
      const int s = t % FH_STAGES, par = (t / FH_STAGES) & 1;
      mbar_wait_quiet(&kv_full[s], par);
      const uint32_t k_addr = smem_u32(sKV + s * 2 * FH_TILE_BYTES);
      float sc[64];
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) wgmma_ss(sc, wgmma_desc_sw128(q_addr + ks * 32), wgmma_desc_sw128(k_addr + ks * 32), ks ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_acc(sc);
      // every tile but the last is full; the last holds at least one key (t * 128 < T)
      const int j0 = t * FH_BN + c0;
      const bool edge = t * FH_BN + FH_BN > p.T;
      float mra = -3.0e38f, mrb = -3.0e38f;
#pragma unroll
      for (int jb = 0; jb < 16; ++jb) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float& xa = sc[4 * jb + e];
          float& xb = sc[4 * jb + 2 + e];
          if (edge && j0 + 8 * jb + e >= p.T) {
            xa = -INFINITY;  // exp2 gives exactly 0 below
            xb = -INFINITY;
          } else {
            mra = fmaxf(mra, xa);
            mrb = fmaxf(mrb, xb);
          }
        }
      }
      mra = quad_max(mra);
      mrb = quad_max(mrb);
      const float mxa = fmaxf(m_a, mra * p.scale_log2), mxb = fmaxf(m_b, mrb * p.scale_log2);
      if (t > 0) {  // rescale O and the partial row sums to the new maxima (a factor of exactly 1 where a maximum did not grow)
        const float ca = ex2_approx(m_a - mxa), cb = ex2_approx(m_b - mxb);
        l_a *= ca;
        l_b *= cb;
#pragma unroll
        for (int jb = 0; jb < 8; ++jb) {
          o[4 * jb] *= ca, o[4 * jb + 1] *= ca;
          o[4 * jb + 2] *= cb, o[4 * jb + 3] *= cb;
        }
      }
      m_a = mxa;
      m_b = mxb;
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
      const uint32_t v_addr = k_addr + FH_TILE_BYTES;
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < 8; ++ks) {  // keys 16 ks .. + 15; V rows 16 ks (128 B each); 64 dims = one swizzle row, no second box
        const uint32_t a[4] = {pk[4 * ks], pk[4 * ks + 1], pk[4 * ks + 2], pk[4 * ks + 3]};
        wgmma_rs_bmn(o, a, wgmma_desc_sw128_mn(v_addr + ks * 2048, FH_TILE_BYTES), (t | ks) ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_acc(o);
      if (wt == 0) mbar_arrive(&kv_empty[s]);
    }
    l_a = quad_sum(l_a);
    l_b = quad_sum(l_b);
    const int64_t ld = (int64_t)p.H * FH_HD;
    bf16* dst_a = p.out + (int64_t)ia * ld + (int64_t)h * FH_HD + c0;
    bf16* dst_b = dst_a + 8 * ld;
    const float inv_a = 1.f / l_a, inv_b = 1.f / l_b;
#pragma unroll
    for (int jb = 0; jb < 8; ++jb) {
      if (ia < p.T) *reinterpret_cast<uint32_t*>(dst_a + 8 * jb) = pack2_rn(o[4 * jb] * inv_a, o[4 * jb + 1] * inv_a);
      if (ib < p.T) *reinterpret_cast<uint32_t*>(dst_b + 8 * jb) = pack2_rn(o[4 * jb + 2] * inv_b, o[4 * jb + 3] * inv_b);
    }
  }
}

inline int launch_attn_full_hd64(const void* q, const void* k, const void* v, void* out, int64_t T, int64_t H, int64_t KV, cudaStream_t stream) {
  CUtensorMap mq, mk, mv;
  int rc = make_tensor_map_rows(&mq, q, T, H * FH_HD);
  if (rc) return rc;
  rc = make_tensor_map_rows(&mk, k, T, KV * FH_HD);
  if (rc) return rc;
  rc = make_tensor_map_rows(&mv, v, T, KV * FH_HD);
  if (rc) return rc;
  FhParams p;
  p.out = (bf16*)out;
  p.T = (int)T;
  p.H = (int)H;
  p.KV = (int)KV;
  p.scale_log2 = 0.125f * 1.4426950408889634f;  // 64^-0.5 (xformers' default scale) * log2(e)
  MB_CHECK_CUDA(cudaFuncSetAttribute(attn_full_hd64_wgmma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, FH_SMEM));
  const dim3 grid((unsigned)H, (unsigned)ceil_div(T, FH_BM));
  attn_full_hd64_wgmma_kernel<<<grid, FH_THREADS, FH_SMEM, stream>>>(mq, mk, mv, p);
  note_launch("attn_full_hd64_wgmma_kernel");
  MB_CHECK_LAUNCH("attn_full_hd64_wgmma_kernel");
  return MB200_OK;
}

}  // namespace mb200
