// C[T, N] = A[T, K] * W[N, K]^T  for T > 4 (prefill chunks, batched decode), bf16 in, fp32 accumulate.
//
// Round-1 stepping stone: warp-level mma.sync (HMMA) fed by a 3-stage cp.async pipeline.  It exists so the
// whole path is parity-green end to end; the wgmma/TMA kernel (gemm_wgmma.cuh) takes over the
// tensor-bound shapes.  Tile 128 (tokens) x 128 (out features) x 64, 8 warps as 2 x 4, warp tile 64 x 32.
// Shared-memory rows are 128 B (64 bf16) with the 16-byte chunk index XOR-swizzled by (row & 7), so both
// cp.async stores and ldmatrix loads are bank-conflict free.
#pragma once
#include "epilogue.cuh"

namespace mb200 {

constexpr int GM_BM = 128, GM_BN = 128, GM_BK = 64, GM_STAGES = 3, GM_THREADS = 256;
constexpr int GM_STAGE_BYTES = (GM_BM + GM_BN) * GM_BK * 2;
constexpr int GM_SMEM = GM_STAGES * GM_STAGE_BYTES;

struct GemmParams {
  const void* a;  // [T, K] bf16
  const void* w;  // [N, K] bf16
  int T, N, K;
  EpiParams epi;
};

__device__ __forceinline__ void cp_async16(uint32_t smem_addr, const void* gptr, bool valid) {
  const int sz = valid ? 16 : 0;  // src-size 0 => zero fill
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_addr), "l"(gptr), "r"(sz));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N)); }

__device__ __forceinline__ void ldmatrix_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}
__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}
__device__ __forceinline__ void mma_bf16_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// byte offset of 16-byte chunk `chunk` (0..7) of row `row` inside a [rows][64 bf16] swizzled tile
__device__ __forceinline__ uint32_t swz(int row, int chunk) { return (uint32_t)(row * 128 + ((chunk ^ (row & 7)) << 4)); }

template <int MODE>
__global__ void __launch_bounds__(GM_THREADS, 2) gemm_mma_kernel(const GemmParams p) {
  extern __shared__ __align__(128) uint8_t smem[];
  const uint32_t smem_base = (uint32_t)__cvta_generic_to_shared(smem);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wm = warp >> 2, wn = warp & 3;  // 2 x 4 warps
  const int m0 = blockIdx.y * GM_BM, n0 = blockIdx.x * GM_BN;
  const bf16* A = reinterpret_cast<const bf16*>(p.a);
  const bf16* W = reinterpret_cast<const bf16*>(p.w);
  const int nk = p.K / GM_BK;

  auto load_stage = [&](int stage, int kt) {
    const uint32_t sa = smem_base + stage * GM_STAGE_BYTES;
    const uint32_t sb = sa + GM_BM * GM_BK * 2;
    const int k0 = kt * GM_BK;
#pragma unroll
    for (int i = 0; i < (GM_BM * 8) / GM_THREADS; ++i) {
      const int idx = tid + i * GM_THREADS;
      const int row = idx >> 3, chunk = idx & 7;
      const int gm = m0 + row;
      const bool ok = gm < p.T;
      cp_async16(sa + swz(row, chunk), A + (int64_t)(ok ? gm : 0) * p.K + k0 + chunk * 8, ok);
    }
#pragma unroll
    for (int i = 0; i < (GM_BN * 8) / GM_THREADS; ++i) {
      const int idx = tid + i * GM_THREADS;
      const int row = idx >> 3, chunk = idx & 7;
      const int gn = n0 + row;
      const bool ok = gn < p.N;
      cp_async16(sb + swz(row, chunk), W + (int64_t)(ok ? gn : 0) * p.K + k0 + chunk * 8, ok);
    }
  };

  float acc[4][4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int r = 0; r < 4; ++r) acc[i][j][r] = 0.f;

#pragma unroll
  for (int s = 0; s < GM_STAGES - 1; ++s) {
    if (s < nk) load_stage(s, s);
    cp_async_commit();
  }

  for (int kt = 0; kt < nk; ++kt) {
    cp_async_wait<GM_STAGES - 2>();
    __syncthreads();
    {  // prefetch tile kt + STAGES - 1 into the slot consumed at iteration kt - 1
      const int nxt = kt + GM_STAGES - 1;
      if (nxt < nk) load_stage(nxt % GM_STAGES, nxt);
      cp_async_commit();
    }
    const uint32_t sa = smem_base + (kt % GM_STAGES) * GM_STAGE_BYTES;
    const uint32_t sb = sa + GM_BM * GM_BK * 2;
#pragma unroll
    for (int ks = 0; ks < GM_BK / 16; ++ks) {
      uint32_t af[4][4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int row = wm * 64 + i * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
        const int chunk = ks * 2 + (lane >> 4);
        ldmatrix_x4(sa + swz(row, chunk), af[i][0], af[i][1], af[i][2], af[i][3]);
      }
      uint32_t bfr[4][2];
#pragma unroll
      for (int j = 0; j < 2; ++j) {  // two n8 tiles per ldmatrix.x4
        const int row = wn * 32 + j * 16 + (lane & 7) + (lane >> 4) * 8;
        const int chunk = ks * 2 + ((lane >> 3) & 1);
        ldmatrix_x4(sb + swz(row, chunk), bfr[2 * j][0], bfr[2 * j][1], bfr[2 * j + 1][0], bfr[2 * j + 1][1]);
      }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) mma_bf16_16816(acc[i][j], af[i], bfr[j][0], bfr[j][1]);
    }
  }
  cp_async_wait<0>();

  // epilogue: c0,c1 -> (row = lane/4, cols 2*(lane%4)+{0,1}); c2,c3 -> row + 8
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + wn * 32 + j * 8 + (lane & 3) * 2;
      if (n >= p.N) continue;
      const int r0 = m0 + wm * 64 + i * 16 + (lane >> 2);
      if (r0 < p.T) epi_pair<MODE>(p.epi, r0, n, acc[i][j][0], acc[i][j][1]);
      if (r0 + 8 < p.T) epi_pair<MODE>(p.epi, r0 + 8, n, acc[i][j][2], acc[i][j][3]);
    }
}

template <int MODE>
int launch_gemm_mma(const GemmParams& p, cudaStream_t stream) {
  MB_CHECK_ARG(p.K % GM_BK == 0, "gemm: K=%d must be a multiple of %d", p.K, GM_BK);
  MB_CHECK_ARG(p.N % 2 == 0, "gemm: N=%d must be even", p.N);
  MB_CHECK_CUDA(cudaFuncSetAttribute(gemm_mma_kernel<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, GM_SMEM));
  const dim3 grid(ceil_div(p.N, GM_BN), ceil_div(p.T, GM_BM));
  gemm_mma_kernel<MODE><<<grid, GM_THREADS, GM_SMEM, stream>>>(p);
  note_launch("gemm_mma_kernel<%d>", MODE);
  MB_CHECK_LAUNCH("gemm_mma_kernel");
  return MB200_OK;
}

// Straightforward CUDA-core GEMM used only by tests to cross-check the tensor-core kernels on the GPU.
__global__ void gemm_naive_kernel(const bf16* __restrict__ a, const bf16* __restrict__ w, float* __restrict__ c, int T, int N, int K) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x, t = blockIdx.y;
  if (n >= N || t >= T) return;
  float acc = 0.f;
  for (int k = 0; k < K; ++k) acc = fmaf(__bfloat162float(a[(int64_t)t * K + k]), __bfloat162float(w[(int64_t)n * K + k]), acc);
  c[(int64_t)t * N + n] = acc;
}

}  // namespace mb200
