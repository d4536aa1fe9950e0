// Un-merged LoRA: the low-rank "down" projection  a[T, R] = bf16( x[T, K] * A[R, K]^T )  (lora_A of LoRALinear, lora.py:71-74).
//
// A stacks the lora_A of every output segment of one fused call (q/k/v, w1/w3, wo, w2), R = segments * rank rounded up to 64 with
// zero rows.  The shape is a narrow N (64..512) over a deep K (4096..14336): a [128 x 64] output tile per CTA gives T = 4096,
// R = 64 only 32 CTAs, so K is split across CTAs as well (grid.z), enough to put two CTAs on every SM.  The split is
// deterministic: split s owns k-blocks [s*nk/S, (s+1)*nk/S), writes its fp32 partial tile to its own slot, and a second kernel
// sums the S slots in ascending order and rounds once.  Same inputs and S give the same bits on every run.
// Main loop: mma.sync m16n8k16 fed by a 3-stage cp.async ring, the shared-memory layout and fragment loads of gemm_mma.cuh;
// 8 warps as 4 (rows) x 2 (columns), warp tile 32 x 32.
// The up-projection  L = bf16(a * B^T)  is an ordinary GEMM (run_linear<EPI_STORE>, K = R) and the combine is the EPI_LORA
// stage of epilogue.cuh.
// GROUPED (the experts of a MoE layer, moe.cuh): the rows are the expert-sorted rows of the MoE row plan, and m tile y is the
// plan's tile y -- expert tile_expert[y], rows [tile_row0[y], tile_row0[y] + tile_rows), read on the device, so the launch needs no
// host sync and replays in a graph.  The grid covers the plan's tile capacity; CTAs past plan[0] exit.  A 32- or 64-row plan
// tile leaves the rest of the 128-row CTA tile zero-filled and unstored.
// MASKED (a bank of adapter slots, one slot per row): A stacks n slots of slot_cols rows each, and row t keeps only the columns of
// its own slot, a[t, c] = 0 unless c / slot_cols == row_slot[t] (all of row t when row_slot[t] == -1).  The mask is applied where
// a is written -- the splits == 1 store here, or lora_down_reduce_masked_kernel -- so the split-K partials and the split count
// are those of the unmasked call.  A 64-column tile lies inside one slot (slot_cols is a multiple of 64).
#pragma once
#include <type_traits>

#include "gemm_mma.cuh"
#include "gemm_wgmma.cuh"

namespace mb200 {

constexpr int LD_BM = 128, LD_BN = 64, LD_BK = 64, LD_STAGES = 3, LD_THREADS = 256;
constexpr int LD_STAGE_BYTES = (LD_BM + LD_BN) * LD_BK * 2;
constexpr int LD_SMEM = LD_STAGES * LD_STAGE_BYTES;
constexpr int LD_MAX_SPLITS = 64;

struct LoraDownParams {
  const bf16* x;    // [T, K]
  const bf16* a_w;  // [R, K]
  bf16* out;        // [T, R]        (splits == 1)
  float* partial;   // [S, T, R] fp32 (splits > 1)
  int T, R, K, splits;
};
// GROUPED: T is the plan's row capacity; a_e[e] is expert e's A [R, K] (null for experts of other ranks, never in the plan).  A
// separate type, so that the dense kernel's parameters (and code) stay as they are.
struct LoraDownGroupedParams : LoraDownParams {
  const int32_t* plan;
  int tile_rows;
  const bf16* a_e[MOE_MAX_EXPERTS];
};
// MASKED: row_slot [T] int32, the slot of each row (-1: none); slot_cols, the A rows of one slot.  Also a separate type.
struct LoraDownMaskedParams : LoraDownParams {
  const int32_t* row_slot;
  int slot_cols;
};
template <bool GROUPED, bool MASKED>
using LoraDownArgs = std::conditional_t<GROUPED, LoraDownGroupedParams, std::conditional_t<MASKED, LoraDownMaskedParams, LoraDownParams>>;

template <bool GROUPED, bool MASKED = false>
__global__ void __launch_bounds__(LD_THREADS, 2) lora_down_kernel(const LoraDownArgs<GROUPED, MASKED> p) {
  static_assert(!(GROUPED && MASKED), "lora down: the slot mask is a dense-call mode");
  extern __shared__ __align__(128) uint8_t smem[];
  const uint32_t smem_base = (uint32_t)__cvta_generic_to_shared(smem);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wm = warp >> 1, wn = warp & 1;
  int m0 = blockIdx.y * LD_BM;
  const int n0 = blockIdx.x * LD_BN, split = blockIdx.z;
  const int nk_all = p.K / LD_BK;
  const int kb0 = (int)((int64_t)split * nk_all / p.splits), kb1 = (int)((int64_t)(split + 1) * nk_all / p.splits);
  const int nk = kb1 - kb0;
  pdl_trigger();
  pdl_wait();  // x (and the plan) are the preceding kernels' output, and the partials may reuse memory they read
  int m_end = p.T;
  const bf16* a_w = p.a_w;
  if constexpr (GROUPED) {
    if ((int)blockIdx.y >= p.plan[0]) return;
    const int cap = p.plan[2];
    a_w = p.a_e[p.plan[MOE_PLAN_HEADER + blockIdx.y]];
    m0 = p.plan[MOE_PLAN_HEADER + cap + blockIdx.y];
    m_end = min(m0 + p.tile_rows, p.T);
  }

  auto load_stage = [&](int stage, int kt) {
    const uint32_t sa = smem_base + stage * LD_STAGE_BYTES;
    const uint32_t sb = sa + LD_BM * LD_BK * 2;
    const int k0 = (kb0 + kt) * LD_BK;
#pragma unroll
    for (int i = 0; i < (LD_BM * 8) / LD_THREADS; ++i) {
      const int idx = tid + i * LD_THREADS;
      const int row = idx >> 3, chunk = idx & 7;
      const int gm = m0 + row;
      const bool ok = gm < m_end;
      cp_async16(sa + swz(row, chunk), p.x + (int64_t)(ok ? gm : 0) * p.K + k0 + chunk * 8, ok);
    }
#pragma unroll
    for (int i = 0; i < (LD_BN * 8) / LD_THREADS; ++i) {
      const int idx = tid + i * LD_THREADS;
      const int row = idx >> 3, chunk = idx & 7;
      cp_async16(sb + swz(row, chunk), a_w + (int64_t)(n0 + row) * p.K + k0 + chunk * 8, true);
    }
  };

  float acc[2][4][4];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int r = 0; r < 4; ++r) acc[i][j][r] = 0.f;

#pragma unroll
  for (int s = 0; s < LD_STAGES - 1; ++s) {
    if (s < nk) load_stage(s, s);
    cp_async_commit();
  }
  for (int kt = 0; kt < nk; ++kt) {
    cp_async_wait<LD_STAGES - 2>();
    __syncthreads();
    {
      const int nxt = kt + LD_STAGES - 1;
      if (nxt < nk) load_stage(nxt % LD_STAGES, nxt);
      cp_async_commit();
    }
    const uint32_t sa = smem_base + (kt % LD_STAGES) * LD_STAGE_BYTES;
    const uint32_t sb = sa + LD_BM * LD_BK * 2;
#pragma unroll
    for (int ks = 0; ks < LD_BK / 16; ++ks) {
      uint32_t af[2][4];
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int row = wm * 32 + i * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
        ldmatrix_x4(sa + swz(row, ks * 2 + (lane >> 4)), af[i][0], af[i][1], af[i][2], af[i][3]);
      }
      uint32_t bfr[4][2];
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int row = wn * 32 + j * 16 + (lane & 7) + (lane >> 4) * 8;
        ldmatrix_x4(sb + swz(row, ks * 2 + ((lane >> 3) & 1)), bfr[2 * j][0], bfr[2 * j][1], bfr[2 * j + 1][0], bfr[2 * j + 1][1]);
      }
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) mma_bf16_16816(acc[i][j], af[i], bfr[j][0], bfr[j][1]);
    }
  }
  cp_async_wait<0>();

#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + wn * 32 + j * 8 + (lane & 3) * 2;
      const int r0 = m0 + wm * 32 + i * 16 + (lane >> 2);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = r0 + 8 * h;
        if (r >= m_end) continue;
        if (p.splits == 1) {
          uint32_t v = pack_bf16x2(acc[i][j][2 * h], acc[i][j][2 * h + 1]);
          if constexpr (MASKED) {
            if (p.row_slot[r] != n0 / p.slot_cols) v = 0u;
          }
          *reinterpret_cast<uint32_t*>(p.out + (int64_t)r * p.R + n) = v;
        } else {
          *reinterpret_cast<float2*>(p.partial + ((int64_t)split * p.T + r) * p.R + n) = make_float2(acc[i][j][2 * h], acc[i][j][2 * h + 1]);
        }
      }
    }
}

// out[i] = bf16( ((partial[0][i] + partial[1][i]) + partial[2][i]) + ... ), four columns per thread
__global__ void __launch_bounds__(256) lora_down_reduce_kernel(const float4* __restrict__ partial, uint2* __restrict__ out, int64_t n4, int splits) {
  const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
  pdl_trigger();
  pdl_wait();
  if (i >= n4) return;
  float4 s = partial[i];
  for (int k = 1; k < splits; ++k) {
    const float4 v = partial[(int64_t)k * n4 + i];
    s.x += v.x;
    s.y += v.y;
    s.z += v.z;
    s.w += v.w;
  }
  out[i] = make_uint2(pack_bf16x2(s.x, s.y), pack_bf16x2(s.z, s.w));
}

// The same fixed-order sum for a masked call: r4 = R / 4 float4s per row, slot4 = slot_cols / 4.  A column outside its row's slot
// is written as zero without reading its partials.
__global__ void __launch_bounds__(256) lora_down_reduce_masked_kernel(const float4* __restrict__ partial, uint2* __restrict__ out, int64_t n4,
                                                                      int splits, const int32_t* __restrict__ row_slot, int r4, int slot4) {
  const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
  pdl_trigger();
  pdl_wait();
  if (i >= n4) return;
  if (row_slot[i / r4] != (int)(i % r4) / slot4) {
    out[i] = make_uint2(0u, 0u);
    return;
  }
  float4 s = partial[i];
  for (int k = 1; k < splits; ++k) {
    const float4 v = partial[(int64_t)k * n4 + i];
    s.x += v.x;
    s.y += v.y;
    s.z += v.z;
    s.w += v.w;
  }
  out[i] = make_uint2(pack_bf16x2(s.x, s.y), pack_bf16x2(s.z, s.w));
}

// K splits: enough CTAs for two per SM over `tiles` output tiles, at least 4 k-blocks per split, and partials [S, T, R] that fit
// the caller's scratch.
inline int lora_down_splits(int64_t tiles, int64_t T, int64_t R, int64_t K, size_t scratch_bytes, int sms) {
  int64_t s = (2 * sms + tiles - 1) / tiles;
  const int64_t by_k = (K / LD_BK) / 4, by_scratch = (int64_t)(scratch_bytes / ((size_t)T * R * sizeof(float)));
  if (s > by_k) s = by_k;
  if (s > by_scratch) s = by_scratch;
  if (s > LD_MAX_SPLITS) s = LD_MAX_SPLITS;
  return s < 1 ? 1 : (int)s;
}

// The split partials [S, T, R] -> out [T, R]: the fixed-order sum of lora_down_reduce_kernel (T = the plan's row capacity when grouped:
// rows no plan tile covers sum stale partials into rows nothing reads).
inline int launch_lora_down_reduce(const void* scratch, void* out, int64_t T, int64_t R, int splits, cudaStream_t stream) {
  const int64_t n4 = T * R / 4;
  MB_CHECK_CUDA(launch_pdl(lora_down_reduce_kernel, dim3((unsigned)ceil_div(n4, 256)), dim3(256), 0, stream, (const float4*)scratch, (uint2*)out,
                           n4, splits));
  note_launch("lora_down_reduce_kernel");
  MB_CHECK_LAUNCH("lora_down_reduce_kernel");
  return MB200_OK;
}

inline int launch_lora_down_reduce_masked(const void* scratch, void* out, int64_t T, int64_t R, int splits, const int32_t* row_slot,
                                          int64_t slot_cols, cudaStream_t stream) {
  const int64_t n4 = T * R / 4;
  MB_CHECK_CUDA(launch_pdl(lora_down_reduce_masked_kernel, dim3((unsigned)ceil_div(n4, 256)), dim3(256), 0, stream, (const float4*)scratch,
                           (uint2*)out, n4, splits, row_slot, (int)(R / 4), (int)(slot_cols / 4)));
  note_launch("lora_down_reduce_masked_kernel");
  MB_CHECK_LAUNCH("lora_down_reduce_masked_kernel");
  return MB200_OK;
}

inline int lora_down_sms(int* sms) {
  int dev = 0;
  MB_CHECK_CUDA(cudaGetDevice(&dev));
  MB_CHECK_CUDA(cudaDeviceGetAttribute(sms, cudaDevAttrMultiProcessorCount, dev));
  return MB200_OK;
}

// x [T, K] (already normed), a_w [R, K] -> out [T, R]; `scratch` (scratch_bytes, 16-byte aligned) holds the split partials.
// Both kernels go through launch_pdl: their launch overlaps the predecessor's tail and they wait for it before touching memory.
// row_slot non-null: the MASKED kernels (a bank of slots of slot_cols columns each), with the same grid and split count.
inline int launch_lora_down(const void* x, const void* a_w, void* out, int64_t T, int64_t R, int64_t K, void* scratch, size_t scratch_bytes,
                            cudaStream_t stream, const int32_t* row_slot = nullptr, int64_t slot_cols = 0) {
  MB_CHECK_ARG(K % LD_BK == 0 && R % LD_BN == 0, "lora down: K=%lld and R=%lld must be multiples of 64", (long long)K, (long long)R);
  int sms = 0;
  if (const int rc = lora_down_sms(&sms)) return rc;
  LoraDownParams p;
  p.x = (const bf16*)x;
  p.a_w = (const bf16*)a_w;
  p.out = (bf16*)out;
  p.partial = (float*)scratch;
  p.T = (int)T;
  p.R = (int)R;
  p.K = (int)K;
  p.splits = lora_down_splits((R / LD_BN) * ceil_div(T, LD_BM), T, R, K, scratch_bytes, sms);
  const dim3 grid((unsigned)(R / LD_BN), (unsigned)ceil_div(T, LD_BM), (unsigned)p.splits);
  if (row_slot != nullptr) {
    LoraDownMaskedParams m;
    static_cast<LoraDownParams&>(m) = p;
    m.row_slot = row_slot;
    m.slot_cols = (int)slot_cols;
    MB_CHECK_CUDA(cudaFuncSetAttribute(lora_down_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, LD_SMEM));
    MB_CHECK_CUDA(launch_pdl(lora_down_kernel<false, true>, grid, dim3(LD_THREADS), (size_t)LD_SMEM, stream, m));
    note_launch("lora_down_masked_kernel<%d>", p.splits);
    MB_CHECK_LAUNCH("lora_down_masked_kernel");
    return p.splits > 1 ? launch_lora_down_reduce_masked(scratch, out, T, R, p.splits, row_slot, slot_cols, stream) : MB200_OK;
  }
  MB_CHECK_CUDA(cudaFuncSetAttribute(lora_down_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, LD_SMEM));
  MB_CHECK_CUDA(launch_pdl(lora_down_kernel<false>, grid, dim3(LD_THREADS), (size_t)LD_SMEM, stream, p));
  note_launch("lora_down_kernel<%d>", p.splits);
  MB_CHECK_LAUNCH("lora_down_kernel");
  return p.splits > 1 ? launch_lora_down_reduce(scratch, out, T, R, p.splits, stream) : MB200_OK;
}

// Grouped (MoE experts): xs [rows_cap, K] in the plan's row order, a_host[e] expert e's A [R, K] -> out [rows_cap, R].  The split
// count is sized for `est_mtiles` busy plan tiles (the grouped GEMMs' estimate), so a decode-sized call with one short tile per
// touched expert still puts two CTAs on every SM; it depends on the shape only, so the bits do too.
inline int launch_lora_down_grouped(const void* xs, const void* const* a_host, int E, const int32_t* plan, int tile_rows, int est_mtiles, void* out,
                                    int64_t rows_cap, int64_t R, int64_t K, void* scratch, size_t scratch_bytes, cudaStream_t stream) {
  MB_CHECK_ARG(K % LD_BK == 0 && R % LD_BN == 0, "lora down (grouped): K=%lld and R=%lld must be multiples of 64", (long long)K, (long long)R);
  MB_CHECK_ARG(E >= 1 && E <= MOE_MAX_EXPERTS && rows_cap % tile_rows == 0 && tile_rows <= LD_BM, "lora down (grouped): E=%d rows_cap=%lld tile_rows=%d",
               E, (long long)rows_cap, tile_rows);
  int sms = 0;
  if (const int rc = lora_down_sms(&sms)) return rc;
  LoraDownGroupedParams p = {};
  p.x = (const bf16*)xs;
  p.out = (bf16*)out;
  p.partial = (float*)scratch;
  p.T = (int)rows_cap;
  p.R = (int)R;
  p.K = (int)K;
  p.plan = plan;
  p.tile_rows = tile_rows;
  for (int e = 0; e < E; ++e) p.a_e[e] = (const bf16*)a_host[e];
  p.splits = lora_down_splits((R / LD_BN) * (est_mtiles < 1 ? 1 : est_mtiles), rows_cap, R, K, scratch_bytes, sms);
  MB_CHECK_CUDA(cudaFuncSetAttribute(lora_down_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, LD_SMEM));
  MB_CHECK_CUDA(launch_pdl(lora_down_kernel<true>, dim3((unsigned)(R / LD_BN), (unsigned)(rows_cap / tile_rows), (unsigned)p.splits),
                           dim3(LD_THREADS), (size_t)LD_SMEM, stream, p));
  note_launch("lora_down_grouped_kernel<%d>", p.splits);
  MB_CHECK_LAUNCH("lora_down_grouped_kernel");
  return p.splits > 1 ? launch_lora_down_reduce(scratch, out, rows_cap, R, p.splits, stream) : MB200_OK;
}

}  // namespace mb200
