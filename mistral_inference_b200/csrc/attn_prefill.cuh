// Prefill attention: varlen batch, causal + sliding window, keys = [old ring rows in position order] ++ [new chunk].
//
// Roofline: tensor pipe (4 * hd * visible-keys flops per (query, head)).  Round-1 version: flash-attention
// structure on warp-level mma.sync -- CTA = (64-query tile, query head, sequence), 4 warps x 16 queries, K/V tiles
// of 64 keys double-buffered with cp.async, online softmax in fp32, P rounded to bf16 for the PV product (as any
// tensor-core attention, incl. the reference's xformers/FA2 dispatch, must).  Nothing is materialised: the
// reference's interleave_kv / unrotate / repeat_kv copies (cache.py:94-117, transformer_layers.py:84) become
// address arithmetic -- key at absolute position j of sequence b lives in ring row b*W + j % W if j < seqpos[b]
// (already cached) and in the chunk buffer at token q_start[b] + j - seqpos[b] otherwise.
// Mask (cache.py:240,243-248; SURVEY.md Appendix B): query at absolute position p sees keys in (p - W, p].
#pragma once
#include "gemm_mma.cuh"
#include "kv_fp8.cuh"  // kv_dequant8

namespace mb200 {

constexpr int AP_BQ = 64, AP_BK = 64, AP_THREADS = 128;
constexpr int AP_TILE_BYTES = 64 * kHeadDim * 2;           // one [64][128] bf16 tile = 16 KB
constexpr int AP_SMEM = AP_TILE_BYTES * (1 + 2 * 2);       // Q + 2 stages x (K, V) = 80 KB

struct AttnPrefillParams {
  const bf16* q;      // [T, H*hd]
  const bf16* k_new;  // [T, KV*hd]
  const bf16* v_new;
  const bf16* cache_k;  // [max_batch, W, KV, hd]
  const bf16* cache_v;
  const int32_t* q_start;  // [B+1]
  const int32_t* seqpos;   // [B]
  bf16* out;               // [T, H*hd]
  int T, B, W, H, KV;
  int causal;
  float scale_log2;  // hd^-0.5 * log2(e)
};

// byte offset of 16-byte chunk (0..15) of row (0..63) in a [64][128 bf16] tile; XOR swizzle on the low 3 chunk bits
__device__ __forceinline__ uint32_t ap_swz(int row, int chunk) { return (uint32_t)(row * 256 + (((chunk & 8) | ((chunk ^ row) & 7)) << 4)); }

// Ring rows of an e4m3 cache (csrc/kv_fp8.cuh): cache_k / cache_v of AttnPrefillParams hold the codes, these the exponents.
struct KvFp8Exps {
  const int8_t* k;  // [max_batch * W, KV]
  const int8_t* v;
};

// The kernel body.  FP8: the ring is e4m3, and its rows are rebuilt as bf16 x' with plain loads and shared-memory stores (cp.async
// cannot convert); chunk rows are bf16 k' / v' and take cp.async as in the bf16 kernel, so the two kernels see the same tiles.
template <bool FP8>
__device__ __forceinline__ void attn_prefill_body(const AttnPrefillParams& p, const KvFp8Exps& ex) {
  extern __shared__ __align__(128) uint8_t smem[];
  const uint32_t sQ = (uint32_t)__cvta_generic_to_shared(smem);
  const uint32_t sKV = sQ + AP_TILE_BYTES;  // stage st: K at sKV + st*2*TILE, V right after
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int h = blockIdx.y, b = blockIdx.z;
  const int g = h / (p.H / p.KV);

  int tok0, s_len, pos0, W;
  if (p.causal) {
    tok0 = p.q_start[b];
    s_len = p.q_start[b + 1] - tok0;
    pos0 = p.seqpos[b];
    W = p.W;
  } else {  // cache-less forward: one unmasked block over the whole flattened batch
    tok0 = 0;
    s_len = p.T;
    pos0 = 0;
    W = 0x3fffffff;
  }
  // heavier (later) query tiles first
  const int qt = (int)gridDim.x - 1 - (int)blockIdx.x;
  const int i0 = qt * AP_BQ;
  if (i0 >= s_len) return;
  const int i_end = min(i0 + AP_BQ, s_len);  // exclusive, local query index

  // visible absolute key range of this query tile
  int key_lo, key_hi;  // [key_lo, key_hi]
  if (p.causal) {
    key_lo = max(0, pos0 + i0 - W + 1);
    key_hi = pos0 + i_end - 1;
  } else {
    key_lo = 0;
    key_hi = p.T - 1;
  }
  const int n_tiles = (key_hi - key_lo + AP_BK) / AP_BK;

  const int64_t q_ld = (int64_t)p.H * kHeadDim, kv_ld = (int64_t)p.KV * kHeadDim;

  // ---- async loads ----
  {  // Q tile: 64 rows x 16 chunks
#pragma unroll
    for (int it = 0; it < 8; ++it) {
      const int idx = tid + it * AP_THREADS;
      const int row = idx >> 4, chunk = idx & 15;
      const bool ok = (i0 + row) < s_len;
      const bf16* src = p.q + (int64_t)(tok0 + (ok ? i0 + row : 0)) * q_ld + (int64_t)h * kHeadDim + chunk * 8;
      cp_async16(sQ + ap_swz(row, chunk), src, ok);
    }
  }
  auto load_kv = [&](int stage, int tile) {
    const uint32_t sK = sKV + stage * 2 * AP_TILE_BYTES, sV = sK + AP_TILE_BYTES;
    const int j0 = key_lo + tile * AP_BK;
#pragma unroll
    for (int it = 0; it < 8; ++it) {
      const int idx = tid + it * AP_THREADS;
      const int row = idx >> 4, chunk = idx & 15;
      const int j = j0 + row;
      const bool ok = j <= key_hi;
      if constexpr (FP8) {
        if (ok && j < pos0) {
          const int64_t ring_row = (int64_t)b * p.W + (j % p.W);
          const int64_t off = ring_row * kv_ld + (int64_t)g * kHeadDim + chunk * 8;
          const uint2 kq = *reinterpret_cast<const uint2*>(reinterpret_cast<const uint8_t*>(p.cache_k) + off);
          const uint2 vq = *reinterpret_cast<const uint2*>(reinterpret_cast<const uint8_t*>(p.cache_v) + off);
          const int ek = ex.k[ring_row * p.KV + g], ev = ex.v[ring_row * p.KV + g];
          *reinterpret_cast<uint4*>(smem + (sK - sQ) + ap_swz(row, chunk)) = kv_dequant8(kq, ek);
          *reinterpret_cast<uint4*>(smem + (sV - sQ) + ap_swz(row, chunk)) = kv_dequant8(vq, ev);
          continue;
        }
      }
      const bf16 *ksrc, *vsrc;
      if (ok && j < pos0) {  // already cached: ring slot j % W of sequence b
        const int64_t off = ((int64_t)b * p.W + (j % p.W)) * kv_ld + (int64_t)g * kHeadDim + chunk * 8;
        ksrc = p.cache_k + off;
        vsrc = p.cache_v + off;
      } else {
        const int64_t off = (int64_t)(tok0 + (ok ? j - pos0 : 0)) * kv_ld + (int64_t)g * kHeadDim + chunk * 8;
        ksrc = p.k_new + off;
        vsrc = p.v_new + off;
      }
      cp_async16(sK + ap_swz(row, chunk), ksrc, ok);
      cp_async16(sV + ap_swz(row, chunk), vsrc, ok);
    }
  };
  load_kv(0, 0);
  cp_async_commit();  // group 0 = Q + tile 0

  // ---- per-thread state: rows r0 = lane/4 and r0 + 8 of this warp's 16 queries ----
  float o[16][4];
#pragma unroll
  for (int j = 0; j < 16; ++j)
#pragma unroll
    for (int r = 0; r < 4; ++r) o[j][r] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  uint32_t qf[8][4];
  const int qrow_local[2] = {warp * 16 + (lane >> 2), warp * 16 + (lane >> 2) + 8};
  const int qpos[2] = {pos0 + i0 + qrow_local[0], pos0 + i0 + qrow_local[1]};
  const bool qvalid[2] = {i0 + qrow_local[0] < s_len, i0 + qrow_local[1] < s_len};

  for (int t = 0; t < n_tiles; ++t) {
    if (t + 1 < n_tiles) load_kv((t + 1) & 1, t + 1);
    cp_async_commit();
    cp_async_wait<1>();
    __syncthreads();
    if (t == 0) {
#pragma unroll
      for (int ks = 0; ks < 8; ++ks) {
        const int row = warp * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
        ldmatrix_x4(sQ + ap_swz(row, ks * 2 + (lane >> 4)), qf[ks][0], qf[ks][1], qf[ks][2], qf[ks][3]);
      }
    }
    const uint32_t sK = sKV + (t & 1) * 2 * AP_TILE_BYTES, sV = sK + AP_TILE_BYTES;

    // S = Q K^T  (16 x 64 per warp)
    float sc[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int r = 0; r < 4; ++r) sc[j][r] = 0.f;
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) {
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {  // key n-tiles 2jj, 2jj+1
        uint32_t b0, b1, b2, b3;
        const int row = jj * 16 + (lane & 7) + (lane >> 4) * 8;
        ldmatrix_x4(sK + ap_swz(row, ks * 2 + ((lane >> 3) & 1)), b0, b1, b2, b3);
        mma_bf16_16816(sc[2 * jj], qf[ks], b0, b1);
        mma_bf16_16816(sc[2 * jj + 1], qf[ks], b2, b3);
      }
    }

    // mask + online softmax
    const int j0 = key_lo + t * AP_BK;
    float m_new[2] = {m_run[0], m_run[1]};
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int half = r >> 1;
        const int key = j0 + j * 8 + (lane & 3) * 2 + (r & 1);
        bool ok = qvalid[half] && key <= key_hi;
        if (p.causal) ok = ok && key <= qpos[half] && key > qpos[half] - W;
        sc[j][r] = ok ? sc[j][r] : -INFINITY;
        m_new[half] = fmaxf(m_new[half], sc[j][r]);
      }
    float corr[2], msub[2];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      m_new[hh] = fmaxf(m_new[hh], __shfl_xor_sync(0xffffffffu, m_new[hh], 1));
      m_new[hh] = fmaxf(m_new[hh], __shfl_xor_sync(0xffffffffu, m_new[hh], 2));
      msub[hh] = (m_new[hh] == -INFINITY) ? 0.f : m_new[hh] * p.scale_log2;
      corr[hh] = (m_run[hh] == -INFINITY) ? 0.f : exp2f(m_run[hh] * p.scale_log2 - msub[hh]);
      m_run[hh] = m_new[hh];
    }
    float l_add[2] = {0.f, 0.f};
    uint32_t pf[4][4];  // P as A fragments for 4 k-steps of 16 keys
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float e[4];
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        e[r] = exp2f(sc[j][r] * p.scale_log2 - msub[r >> 1]);  // exp2f(-inf) = 0 for masked keys
        l_add[r >> 1] += e[r];
      }
      pf[j >> 1][(j & 1) * 2 + 0] = pack_bf16x2(e[0], e[1]);
      pf[j >> 1][(j & 1) * 2 + 1] = pack_bf16x2(e[2], e[3]);
    }
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) l_run[hh] = l_run[hh] * corr[hh] + l_add[hh];
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      o[j][0] *= corr[0];
      o[j][1] *= corr[0];
      o[j][2] *= corr[1];
      o[j][3] *= corr[1];
    }
    // O += P V   (A = P from registers, B = V^T via ldmatrix.trans)
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {  // dim n-tiles 2jj, 2jj+1
        uint32_t b0, b1, b2, b3;
        const int row = kk * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
        ldmatrix_x4_trans(sV + ap_swz(row, jj * 2 + (lane >> 4)), b0, b1, b2, b3);
        mma_bf16_16816(o[2 * jj], pf[kk], b0, b1);
        mma_bf16_16816(o[2 * jj + 1], pf[kk], b2, b3);
      }
    }
    __syncthreads();  // everyone is done with stage t&1 before it is refilled
  }
  cp_async_wait<0>();

  // ---- finish: row sums across the 4 lanes of a row, normalise, store ----
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    l_run[hh] += __shfl_xor_sync(0xffffffffu, l_run[hh], 1);
    l_run[hh] += __shfl_xor_sync(0xffffffffu, l_run[hh], 2);
  }
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    if (!qvalid[hh]) continue;
    const float inv = 1.f / l_run[hh];
    bf16* dst = p.out + (int64_t)(tok0 + i0 + qrow_local[hh]) * q_ld + (int64_t)h * kHeadDim + (lane & 3) * 2;
#pragma unroll
    for (int j = 0; j < 16; ++j)
      *reinterpret_cast<uint32_t*>(dst + j * 8) = pack_bf16x2(o[j][hh * 2] * inv, o[j][hh * 2 + 1] * inv);
  }
}

__global__ void __launch_bounds__(AP_THREADS, 2) attn_prefill_kernel(const AttnPrefillParams p) { attn_prefill_body<false>(p, KvFp8Exps{}); }

// Chunked prefill over an e4m3 ring: bit-identical to attn_prefill_kernel on a bf16 ring that holds x'.
__global__ void __launch_bounds__(AP_THREADS, 2) attn_prefill_fp8_kernel(const AttnPrefillParams p, const KvFp8Exps ex) {
  attn_prefill_body<true>(p, ex);
}

}  // namespace mb200
