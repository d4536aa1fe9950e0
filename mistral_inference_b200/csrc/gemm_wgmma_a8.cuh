// FP8 activations times FP8 dense weights on the Hopper FP8 tensor cores (prefill_compute="fp8", include/mistral_b200.h):
// C[T, N] = XQ[T, K] * Q[N, K]^T with both operands e4m3, wgmma.mma_async ... k32.f32.e4m3.e4m3, TMA-fed.
//
// Roofline: FP8 tensor pipe (2*T*N*K flops).  Persistent, warp-specialised kernel, one CTA per SM:
//   warp 0 lane 0   TMA producer: per stage a 128B-swizzled [128 x 128] e4m3 A tile and a [BN x 128] e4m3 W tile.  A 128-element
//                   k-block is 128 bytes per row, so the swizzle atoms and wgmma descriptors are the bf16 kernels'.  There are no
//                   converter warps: warps 1-3 idle.
//   warpgroups 1-2  consumers, 64 tile rows each: per k-block four m64nBNk32 MMAs into `blk` starting from zero, then (promotion)
//                   `acc += blk` on the CUDA cores in IEEE fp32.  The tensor cores never sum more than one k-block of 128 products,
//                   whatever their internal accumulator width; across k-blocks the sum is fp32.  After the last k-block the
//                   epilogue of epilogue.cuh runs on acc with EPI_WSCALE | EPI_ASCALE: bf16(fp32(fp32(s[n] * acc) * 2^e[t])).
// Two accumulator sets cost BN registers per thread: BN = 128 (N % 128 == 0, every real Linear) or 64 (N % 64 == 0 only).
// The tile walk is tile_walk_mn of gemm_wgmma.cuh, single CTA.
//
// The quantisers that write XQ and e (per token, power of two) into the workspace's normed-activation region are at the end.
#pragma once
#include "gemm_wgmma.cuh"

namespace mb200 {

constexpr int A8_BM = 128, A8_BK = 128;  // tile rows; k-block in elements = bytes

template <int BN>
struct A8Cfg {
  static_assert(BN == 64 || BN == 128, "A8 tile width");
  static constexpr int kABytes = A8_BM * A8_BK;
  static constexpr int kBBytes = BN * A8_BK;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kThreads = 384;
  static constexpr int kFit = (227 * 1024 - 1024 - 512) / kStageBytes;
  static constexpr int kStages = kFit > 8 ? 8 : kFit;
  static constexpr int kSmem = kStages * kStageBytes + 1024 /*align*/ + 512 /*barriers*/;
  static_assert(kSmem <= 227 * 1024, "shared memory plan exceeds the 227 KB of an sm_90 block");
};

// One consumer warpgroup's k-block: the 64 tile rows at a_addr against the [BN x 128] W tile, four K = 32 steps of +32 bytes.
template <int BN>
__device__ __forceinline__ void wgmma_kblock_e4m3(float (&blk)[BN / 2], uint32_t a_addr, uint32_t b_addr) {
  const uint64_t adesc = wgmma_desc_sw128(a_addr), bdesc = wgmma_desc_sw128(b_addr);
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < A8_BK / 32; ++k) wgmma_ss_e4m3(blk, adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k), k == 0 ? 0u : 1u);
  wgmma_commit();
}

template <int MODE, int BN>
__global__ void __launch_bounds__(A8Cfg<BN>::kThreads, 1)
    gemm_wgmma_a8_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_w, const TcGemmParams p,
                         const int32_t* __restrict__ a_exp) {
  static_assert((MODE & (EPI_WSCALE | EPI_ASCALE)) == (EPI_WSCALE | EPI_ASCALE), "A8 GEMM: the epilogue applies both scales");
  using Cfg = A8Cfg<BN>;
  constexpr int STAGES = Cfg::kStages, STAGE_BYTES = Cfg::kStageBytes, A_BYTES = Cfg::kABytes;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);  // SW128 wants 1024-B tiles
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES);
  uint64_t* empty = full + STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int cta = (int)blockIdx.x, n_cta = (int)gridDim.x;
  const int num_m = (p.T + A8_BM - 1) / A8_BM, num_n = p.N / BN, num_tiles = num_m * num_n, num_k = p.K / A8_BK;

  if (threadIdx.x == 0) {
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 2);  // one arrival per consumer warpgroup
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_a) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_w) : "memory");
  }
  __syncthreads();

  if (warp == 0) {
    // ================= TMA producer =================
    if (lane == 0) {
      uint32_t it = 0;
      for (int tile = cta; tile < num_tiles; tile += n_cta) {
        int mu, nt;
        tile_walk_mn<12, 12>(tile, num_m, num_n, mu, nt);
        for (int kb = 0; kb < num_k; ++kb, ++it) {
          const uint32_t s = it % STAGES, par = (it / STAGES) & 1;
          mbar_wait_quiet(&empty[s], par ^ 1);
          uint8_t* sa = smem + s * STAGE_BYTES;
          mbar_arrive_expect_tx(&full[s], STAGE_BYTES);
          tma_load_2d(sa, &map_a, &full[s], kb * A8_BK, mu * A8_BM);
          tma_load_2d(sa + A_BYTES, &map_w, &full[s], kb * A8_BK, nt * BN);
        }
      }
    }
  } else if (warp >= 4) {
    // ================= consumer warpgroups: rows 64 * wg .. + 63 of the tile =================
    const int wg = (warp >> 2) - 1, wt = (int)threadIdx.x & 127;
    const int row_in_tile = wg * 64 + ((warp & 3) << 4) + (lane >> 2);  // fragment rows row_in_tile and row_in_tile + 8
    uint32_t it = 0;
    float acc[BN / 2], blk[BN / 2];
    for (int tile = cta; tile < num_tiles; tile += n_cta) {
      int mu, nt;
      tile_walk_mn<12, 12>(tile, num_m, num_n, mu, nt);
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
      for (int kb = 0; kb < num_k; ++kb, ++it) {
        const uint32_t s = it % STAGES, par = (it / STAGES) & 1;
        mbar_wait_quiet(&full[s], par);
        const uint32_t base = smem_u32(smem + s * STAGE_BYTES);
        wgmma_kblock_e4m3<BN>(blk, base + wg * 64 * A8_BK, base + A_BYTES);
        wgmma_wait<0>();
        wgmma_fence_acc(blk);
        if (wt == 0) mbar_arrive(&empty[s]);  // this warpgroup's MMAs have read the stage
        // promotion: the k-block's tensor-core sum joins the fp32 accumulator (one IEEE add per element)
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] += blk[i];
      }
      // epi_fragment with each row's 2^e[t]: rows t0 and t0 + 8 of the fragment
      const int t0 = mu * A8_BM + row_in_tile, nc = nt * BN + 2 * (lane & 3), limit = min(p.T, mu * A8_BM + A8_BM);
      const float s0 = t0 < limit ? exp2_exact(a_exp[t0]) : 0.f, s1 = t0 + 8 < limit ? exp2_exact(a_exp[t0 + 8]) : 0.f;
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        if (t0 < limit) epi_pair<MODE>(p.epi, t0, nc + 8 * j, acc[4 * j], acc[4 * j + 1], s0);
        if (t0 + 8 < limit) epi_pair<MODE>(p.epi, t0 + 8, nc + 8 * j, acc[4 * j + 2], acc[4 * j + 3], s1);
      }
    }
  }
}

// [rows, K] e4m3 (one byte per element), box = [box_rows x 128] bytes, 128-byte swizzle: the K-major wgmma operand layout
inline int make_tensor_map_e4m3_sw128(CUtensorMap* map, const void* base, int64_t rows, int64_t K, int box_rows) {
  PFN_encodeTiled enc = get_encode_tiled();
  if (enc == nullptr) return fail(MB200_E_CUDA, "cuTensorMapEncodeTiled entry point not available");
  const cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)rows};
  const cuuint64_t strides[1] = {(cuuint64_t)K};
  const cuuint32_t box[2] = {(cuuint32_t)A8_BK, (cuuint32_t)box_rows};
  const cuuint32_t estr[2] = {1, 1};
  const CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                         CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(MB200_E_CUDA, "cuTensorMapEncodeTiled (e4m3, sw128) failed (%d) rows=%lld K=%lld", (int)r, (long long)rows, (long long)K);
  return MB200_OK;
}

// Calls the A8 kernel can run: 128-element k-blocks and a tile width that divides N.
inline bool a8_gemm_eligible(int64_t T, int64_t N, int64_t K) { return T >= A8_BM && K % A8_BK == 0 && N % 64 == 0; }

// 128 wherever it divides N; MB200_GEMM_BN=64|128 overrides when it divides N (tests).
inline int a8_bn(int N) {
  const int forced = wgmma_forced_bn();
  if ((forced == 64 || forced == 128) && N % forced == 0) return forced;
  return N % 128 == 0 ? 128 : 64;
}

// g.a: e4m3 [T, K]; g.w: e4m3 [N, K]; g.epi carries w_scale; a_exp: int32 [T].
template <int MODE, int BN>
int launch_gemm_wgmma_a8_bn(const GemmParams& g, const int32_t* a_exp, int sms, cudaStream_t stream) {
  using Cfg = A8Cfg<BN>;
  CUtensorMap map_a, map_w;
  int rc = make_tensor_map_e4m3_sw128(&map_a, g.a, g.T, g.K, A8_BM);
  if (rc) return rc;
  rc = make_tensor_map_e4m3_sw128(&map_w, g.w, g.N, g.K, BN);
  if (rc) return rc;
  TcGemmParams p;
  p.T = g.T;
  p.N = g.N;
  p.K = g.K;
  p.epi = g.epi;
  const int tiles = ceil_div(g.T, A8_BM) * (g.N / BN);
  MB_CHECK_CUDA(cudaFuncSetAttribute(gemm_wgmma_a8_kernel<MODE, BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmem));
  gemm_wgmma_a8_kernel<MODE, BN><<<tiles < sms ? tiles : sms, Cfg::kThreads, Cfg::kSmem, stream>>>(map_a, map_w, p, a_exp);
  note_launch("gemm_wgmma_a8_kernel<%d, %d>", MODE, BN);
  MB_CHECK_LAUNCH("gemm_wgmma_a8_kernel");
  return MB200_OK;
}

template <int MODE>
int launch_gemm_wgmma_a8(const GemmParams& g, const int32_t* a_exp, cudaStream_t stream) {
  int dev = 0, sms = 0;
  MB_CHECK_CUDA(cudaGetDevice(&dev));
  MB_CHECK_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  return a8_bn(g.N) == 128 ? launch_gemm_wgmma_a8_bn<MODE, 128>(g, a_exp, sms, stream) : launch_gemm_wgmma_a8_bn<MODE, 64>(g, a_exp, sms, stream);
}

// ---- per-token e4m3 quantisers ----------------------------------------------------------------------------------------------
// Row t of v (the bf16 input x, or with NORM its RMSNorm output, computed exactly as rmsnorm_kernel computes it):
//   a = max_k |v[t, k]|;  e[t] = 0 if a == 0, else the smallest integer with a <= 448 * 2^e;  xq[t, k] = e4m3_rn(v[t, k] * 2^-e[t])
// A row holding an inf or a NaN gets e[t] = 0 and every code the e4m3 NaN (0x7f), so every output of that token is NaN.
// One CTA per token; the row stays in shared memory between the passes (K * 2 bytes).
constexpr int QA_THREADS = 256;
constexpr uint8_t kE4m3Nan = 0x7f;

// smallest e with a <= 448 * 2^e, for finite a > 0: a = 1.f * 2^E  ->  e = E - 8, plus one when 1.f > 1.75 (448 = 1.75 * 2^8)
__device__ __forceinline__ int act_exponent(float a) {
  int bias = 0;
  if (a < 0x1p-126f) {  // subnormal: scale into the normal range exactly
    a *= 0x1p64f;
    bias = 64;
  }
  const uint32_t b = __float_as_uint(a);
  return (int)(b >> 23) - 127 - 8 + ((b & 0x7fffffu) > 0x600000u ? 1 : 0) - bias;
}

template <bool NORM>
__global__ void __launch_bounds__(QA_THREADS) quantize_act_e4m3_kernel(const uint4* __restrict__ x, const uint4* __restrict__ w,
                                                                      uint8_t* __restrict__ q, int32_t* __restrict__ exps, int dim, float eps) {
  pdl_trigger();
  pdl_wait();  // x is the previous kernel's output
  extern __shared__ uint4 row[];
  __shared__ float red[8];
  __shared__ int bad_any;
  const int kc = dim >> 3;
  const uint4* xr = x + (int64_t)blockIdx.x * kc;
  if (threadIdx.x == 0) bad_any = 0;
  float r = 1.f;
  if constexpr (NORM) {  // rmsnorm_kernel's sum, reduction order and scale
    float ss = 0.f;
    for (int c = threadIdx.x; c < kc; c += QA_THREADS) {
      const uint4 v = xr[c];
      const uint32_t u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float a = bf16lo(u[j]), b = bf16hi(u[j]);
        ss = fmaf(a, a, ss);
        ss = fmaf(b, b, ss);
      }
    }
    ss = warp_sum(ss);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
    __syncthreads();
    float tot = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) tot += red[i];
    r = ref_rsqrt(tot / (float)dim + eps);
    __syncthreads();  // red is reused below
  }
  float amax = 0.f;
  bool bad = false;
  for (int c = threadIdx.x; c < kc; c += QA_THREADS) {
    uint4 v = xr[c];
    if constexpr (NORM) {
      const uint4 g = w[c];
      const uint32_t u[4] = {v.x, v.y, v.z, v.w}, gw[4] = {g.x, g.y, g.z, g.w};
      uint32_t o[4];
#pragma unroll
      for (int j = 0; j < 4; ++j)
        o[j] = pack_bf16x2(round_bf16(bf16lo(u[j]) * r) * bf16lo(gw[j]), round_bf16(bf16hi(u[j]) * r) * bf16hi(gw[j]));
      v = make_uint4(o[0], o[1], o[2], o[3]);
    }
    row[c] = v;
    const uint32_t u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float a = fabsf(bf16lo(u[j])), b = fabsf(bf16hi(u[j]));
      bad |= !(a <= 3.4e38f) || !(b <= 3.4e38f);  // inf or NaN
      amax = fmaxf(amax, fmaxf(a, b));
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = amax;
  if (bad) bad_any = 1;
  __syncthreads();
  float a = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) a = fmaxf(a, red[i]);
  const bool nan_row = bad_any != 0;
  const int e = (nan_row || a == 0.f) ? 0 : act_exponent(a);
  // 2^-e reaches 2^141 (e >= -141): beyond fp32, so the small rows take 2^64 first (exact: their values are below 2^-100)
  const float s1 = e < -100 ? 0x1p64f : 1.f, s2 = exp2_exact(e < -100 ? -e - 64 : -e);
  uint8_t* qr = q + (int64_t)blockIdx.x * dim;
  for (int c = threadIdx.x; c < kc; c += QA_THREADS) {
    const uint4 v = row[c];
    const uint32_t u[4] = {v.x, v.y, v.z, v.w};
    uint32_t o[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const __nv_fp8x2_storage_t lo = __nv_cvt_float2_to_fp8x2(
          make_float2(__fmul_rn(__fmul_rn(bf16lo(u[2 * h]), s1), s2), __fmul_rn(__fmul_rn(bf16hi(u[2 * h]), s1), s2)), __NV_SATFINITE, __NV_E4M3);
      const __nv_fp8x2_storage_t hi = __nv_cvt_float2_to_fp8x2(
          make_float2(__fmul_rn(__fmul_rn(bf16lo(u[2 * h + 1]), s1), s2), __fmul_rn(__fmul_rn(bf16hi(u[2 * h + 1]), s1), s2)), __NV_SATFINITE,
          __NV_E4M3);
      o[h] = (uint32_t)lo | ((uint32_t)hi << 16);
    }
    if (nan_row) o[0] = o[1] = 0x01010101u * kE4m3Nan;
    *reinterpret_cast<uint2*>(qr + 8 * c) = make_uint2(o[0], o[1]);
  }
  if (threadIdx.x == 0) exps[blockIdx.x] = e;
}

inline int launch_quantize_act(const void* x, const void* norm_w, uint8_t* q, int32_t* exps, int64_t T, int64_t dim, float eps,
                               cudaStream_t st) {
  MB_CHECK_ARG(dim % 8 == 0 && dim >= 8 && T >= 0, "quantize_act_e4m3: dim=%lld must be a positive multiple of 8", (long long)dim);
  const size_t smem = (size_t)dim * 2;
  MB_CHECK_ARG(smem <= 200 * 1024, "quantize_act_e4m3: dim=%lld too large for the shared-memory row", (long long)dim);
  if (T == 0) return MB200_OK;
  auto go = [&](auto kernel, const char* name) -> int {
    if (smem > 48 * 1024) MB_CHECK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    MB_CHECK_CUDA(launch_pdl(kernel, dim3((unsigned)T), dim3(QA_THREADS), smem, st, (const uint4*)x, (const uint4*)norm_w, q, exps, (int)dim, eps));
    note_launch("%s", name);
    MB_CHECK_LAUNCH(name);
    return MB200_OK;
  };
  return norm_w ? go(quantize_act_e4m3_kernel<true>, "quantize_act_e4m3_kernel<true>")
                : go(quantize_act_e4m3_kernel<false>, "quantize_act_e4m3_kernel<false>");
}

}  // namespace mb200
