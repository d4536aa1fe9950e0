// Weight-streaming linear for T <= 4 tokens (decode):  y[t, n] = sum_k x[t, k] * W[n, k]
//
// Roofline: HBM.  Algorithmic bytes = N*K*2 (every weight read exactly once); the activations
// (T*K*2 bytes) are re-read by every CTA from L2.  Each warp owns 2 adjacent weight rows (one RoPE pair /
// one gate-up pair) and streams them with 16-byte no-allocate loads, 4 in flight per row per lane; x lives in
// shared memory (optionally RMS-normalised in place by every CTA -- 8..28 KB, cheaper than a kernel boundary).
#pragma once
#include "epilogue.cuh"
#include "int4.cuh"

namespace mb200 {

constexpr int kSkinnyThreads = 256;
constexpr int kSkinnyWarps = kSkinnyThreads / 32;
constexpr int kSkinnyRowsPerWarp = 2;
constexpr int kSkinnyRowsPerCta = kSkinnyWarps * kSkinnyRowsPerWarp;

struct SkinnyParams {
  const void* x;       // [T, K] bf16
  const void* norm_w;  // [K] bf16 (NORM only)
  const void* w;       // [N, K] bf16
  int N, K;
  float eps;
  EpiParams epi;
  const uint16_t* gscale = nullptr;  // W4: bf16 group scales [N, K/128]
  const int32_t* row_slot = nullptr;  // SKINNY_SLOT_MASK: [T] slot of each token (-1: none)
  int slot_cols = 0;                  // SKINNY_SLOT_MASK: output columns of one slot (a multiple of 64)
};

// Flag OR-ed into EPI_STORE of the bf16 GEMV only: the LoRA down projection of a bank of adapter slots (lora.cuh, MASKED).  Output
// column n of token t is stored as zero unless n / slot_cols == row_slot[t]; the pair n, n + 1 always lies in one slot.
constexpr int SKINNY_SLOT_MASK = 64;

// W8 (FP8 dense weights, launch_skinny_fp8): p.w is e4m3 [N, K] (K % 16 == 0) and MODE carries EPI_WSCALE (the row
// scales in p.epi.w_scale).  Same CTA, x staging and row pairs; a 16-byte load is 16 weights (half the bytes of a bf16 load, still
// 4 in flight per row per lane), each pair converted exactly (e4m3x2_to_float2) and fed to the same fp32 FMAs.
// The staged x plus the kernel's static reduction array red[T][kSkinnyWarps] must fit the block's shared memory: past the default
// 48 KB the launch needs the opt-in attribute (at T * K = 24576 the dynamic part alone is exactly 48 KB, e.g. Mistral Large's
// dim 12288 at two tokens).
inline bool skinny_needs_optin(size_t smem, int T) { return smem + (size_t)T * kSkinnyWarps * sizeof(float) > 48 * 1024; }

// W4 (INT4 dense weights, launch_skinny_int4): p.w is the packed code matrix [N, K/2] (K % 128 == 0), p.gscale its group scales.
// A 16-byte load is 32 weights of one group; the lane converts them to W' (int4x8_to_bf16x2) and feeds the same fp32 FMAs.
template <int T, int MODE, bool NORM, bool W8 = false, bool W4 = false>
__global__ void __launch_bounds__(kSkinnyThreads) skinny_linear_kernel(const SkinnyParams p) {
  static_assert((MODE & SKINNY_SLOT_MASK) == 0 || (MODE == (EPI_STORE | SKINNY_SLOT_MASK) && !W8 && !W4), "slot mask: bf16 EPI_STORE only");
  extern __shared__ __align__(16) uint8_t smem_raw[];
  uint4* xs = reinterpret_cast<uint4*>(smem_raw);  // [T][K/8] 16-byte chunks
  __shared__ float red[T][kSkinnyWarps];

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int kc = p.K >> 3;  // chunks per row

  // ---- stage x (and normalise) ----
  const uint4* xg = reinterpret_cast<const uint4*>(p.x);
  for (int i = tid; i < T * kc; i += kSkinnyThreads) xs[i] = xg[i];
  if constexpr (NORM) {
    __syncthreads();
    float ss[T];
#pragma unroll
    for (int t = 0; t < T; ++t) {
      ss[t] = 0.f;
      for (int c = tid; c < kc; c += kSkinnyThreads) {
        const uint4 v = xs[t * kc + c];
        const uint32_t u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float a = bf16lo(u[j]), b = bf16hi(u[j]);
          ss[t] = fmaf(a, a, ss[t]);
          ss[t] = fmaf(b, b, ss[t]);
        }
      }
      ss[t] = warp_sum(ss[t]);
      if (lane == 0) red[t][warp] = ss[t];
    }
    __syncthreads();
    const uint4* wn = reinterpret_cast<const uint4*>(p.norm_w);
#pragma unroll
    for (int t = 0; t < T; ++t) {
      float tot = 0.f;
#pragma unroll
      for (int w = 0; w < kSkinnyWarps; ++w) tot += red[t][w];
      const float r = ref_rsqrt(tot / (float)p.K + p.eps);
      for (int c = tid; c < kc; c += kSkinnyThreads) {
        const uint4 v = xs[t * kc + c];
        const uint4 g = wn[c];
        const uint32_t u[4] = {v.x, v.y, v.z, v.w};
        const uint32_t gw[4] = {g.x, g.y, g.z, g.w};
        uint32_t o[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          // bf16( bf16(x * r) * w )
          const float a = round_bf16(bf16lo(u[j]) * r) * bf16lo(gw[j]);
          const float b = round_bf16(bf16hi(u[j]) * r) * bf16hi(gw[j]);
          o[j] = pack_bf16x2(a, b);
        }
        xs[t * kc + c] = make_uint4(o[0], o[1], o[2], o[3]);
      }
    }
  }
  __syncthreads();

  // ---- stream the two rows of this warp ----
  const int n0 = (blockIdx.x * kSkinnyWarps + warp) * kSkinnyRowsPerWarp;
  if (n0 >= p.N) return;
  if constexpr (W4) {
    const int kq = p.K >> 5, G = p.K >> 7;  // 16-byte code chunks and scale groups of a row
    const uint4* w0 = reinterpret_cast<const uint4*>(reinterpret_cast<const uint8_t*>(p.w) + (int64_t)n0 * (p.K >> 1));
    const uint4* w1 = w0 + kq;
    const uint16_t* s0 = p.gscale + (int64_t)n0 * G;
    const uint16_t* s1 = s0 + G;
    float acc[2][T];
#pragma unroll
    for (int t = 0; t < T; ++t) acc[0][t] = acc[1][t] = 0.f;

    // 32 weights of each row (k = 32c ..) against x chunks 4c .. 4c + 3
    auto fma32 = [&](const uint4& a, const uint4& b, int c) {
      const uint32_t sa = (uint32_t)__ldg(s0 + (c >> 2)) * 0x10001u, sb = (uint32_t)__ldg(s1 + (c >> 2)) * 0x10001u;
      const uint32_t aq[4] = {a.x, a.y, a.z, a.w}, bq[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int h = 0; h < 4; ++h) {  // weights 8h .. 8h + 7: aw[i] = (W'[i], W'[i + 4])
        uint32_t aw[4], bw[4];
        int4x8_to_bf16x2<false>(aq[h], sa, aw);
        int4x8_to_bf16x2<false>(bq[h], sb, bw);
#pragma unroll
        for (int t = 0; t < T; ++t) {
          const uint4 xv = xs[t * kc + 4 * c + h];
          const uint32_t xw[4] = {xv.x, xv.y, xv.z, xv.w};
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const float xa = (i & 1) ? bf16hi(xw[i >> 1]) : bf16lo(xw[i >> 1]);            // x[i]
            const float xb = (i & 1) ? bf16hi(xw[2 + (i >> 1)]) : bf16lo(xw[2 + (i >> 1)]);  // x[i + 4]
            acc[0][t] = fmaf(bf16lo(aw[i]), xa, acc[0][t]);
            acc[0][t] = fmaf(bf16hi(aw[i]), xb, acc[0][t]);
            acc[1][t] = fmaf(bf16lo(bw[i]), xa, acc[1][t]);
            acc[1][t] = fmaf(bf16hi(bw[i]), xb, acc[1][t]);
          }
        }
      }
    };
    constexpr int U = T == 4 ? 3 : 4;  // 16-byte loads in flight per row per lane, as in W8
    int c = lane;
    for (; c + (U - 1) * 32 < kq; c += U * 32) {
      uint4 a[U], b[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        a[u] = ldg_stream16(w0 + c + u * 32);
        b[u] = ldg_stream16(w1 + c + u * 32);
      }
#pragma unroll
      for (int u = 0; u < U; ++u) fma32(a[u], b[u], c + u * 32);
    }
    for (; c < kq; c += 32) fma32(ldg_stream16(w0 + c), ldg_stream16(w1 + c), c);  // tail
#pragma unroll
    for (int t = 0; t < T; ++t) {
      acc[0][t] = warp_sum(acc[0][t]);
      acc[1][t] = warp_sum(acc[1][t]);
    }
#pragma unroll
    for (int t = 0; t < T; ++t)
      if (lane == t) epi_pair<MODE>(p.epi, t, n0, acc[0][t], acc[1][t]);
    return;
  }
  if constexpr (W8) {
    const int kq = p.K >> 4;  // e4m3 chunks of a weight row
    const uint4* w0 = reinterpret_cast<const uint4*>(reinterpret_cast<const uint8_t*>(p.w) + (int64_t)n0 * p.K);
    const uint4* w1 = w0 + kq;
    float acc[2][T];
#pragma unroll
    for (int t = 0; t < T; ++t) acc[0][t] = acc[1][t] = 0.f;

    // 16 weights of each row against x chunks 2c, 2c + 1
    auto fma16 = [&](const uint4& a, const uint4& b, int c) {
      const uint32_t aq[4] = {a.x, a.y, a.z, a.w}, bq[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int h = 0; h < 2; ++h) {  // weights 8h .. 8h + 7 against x chunk 2c + h
        float2 af[4], bf[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          af[j] = e4m3x2_to_float2(aq[2 * h + (j >> 1)] >> (16 * (j & 1)));
          bf[j] = e4m3x2_to_float2(bq[2 * h + (j >> 1)] >> (16 * (j & 1)));
        }
#pragma unroll
        for (int t = 0; t < T; ++t) {
          const uint4 xv = xs[t * kc + 2 * c + h];
          const uint32_t xw[4] = {xv.x, xv.y, xv.z, xv.w};
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const float xl = bf16lo(xw[j]), xh = bf16hi(xw[j]);
            acc[0][t] = fmaf(af[j].x, xl, acc[0][t]);
            acc[0][t] = fmaf(af[j].y, xh, acc[0][t]);
            acc[1][t] = fmaf(bf[j].x, xl, acc[1][t]);
            acc[1][t] = fmaf(bf[j].y, xh, acc[1][t]);
          }
        }
      }
    };
    constexpr int U = T == 4 ? 3 : 4;  // 16-byte loads in flight per row per lane (3 at T = 4: 4 would spill)
    int c = lane;
    for (; c + (U - 1) * 32 < kq; c += U * 32) {
      uint4 a[U], b[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        a[u] = ldg_stream16(w0 + c + u * 32);
        b[u] = ldg_stream16(w1 + c + u * 32);
      }
#pragma unroll
      for (int u = 0; u < U; ++u) fma16(a[u], b[u], c + u * 32);
    }
    for (; c < kq; c += 32) fma16(ldg_stream16(w0 + c), ldg_stream16(w1 + c), c);  // tail (K/16 not a multiple of 128)
#pragma unroll
    for (int t = 0; t < T; ++t) {
      acc[0][t] = warp_sum(acc[0][t]);
      acc[1][t] = warp_sum(acc[1][t]);
    }
#pragma unroll
    for (int t = 0; t < T; ++t)
      if (lane == t) epi_pair<MODE>(p.epi, t, n0, acc[0][t], acc[1][t]);
    return;
  }
  const uint4* w0 = reinterpret_cast<const uint4*>(p.w) + (int64_t)n0 * kc;
  const uint4* w1 = w0 + kc;

  float acc[2][T];
#pragma unroll
  for (int t = 0; t < T; ++t) acc[0][t] = acc[1][t] = 0.f;

  constexpr int U = 4;  // 16-byte loads in flight per row per lane
  int c = lane;
  for (; c + (U - 1) * 32 < kc; c += U * 32) {
    uint4 a[U], b[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      a[u] = ldg_stream16(w0 + c + u * 32);
      b[u] = ldg_stream16(w1 + c + u * 32);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const uint32_t aw[4] = {a[u].x, a[u].y, a[u].z, a[u].w};
      const uint32_t bw[4] = {b[u].x, b[u].y, b[u].z, b[u].w};
#pragma unroll
      for (int t = 0; t < T; ++t) {
        const uint4 xv = xs[t * kc + c + u * 32];
        const uint32_t xw[4] = {xv.x, xv.y, xv.z, xv.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float xl = bf16lo(xw[j]), xh = bf16hi(xw[j]);
          acc[0][t] = fmaf(bf16lo(aw[j]), xl, acc[0][t]);
          acc[0][t] = fmaf(bf16hi(aw[j]), xh, acc[0][t]);
          acc[1][t] = fmaf(bf16lo(bw[j]), xl, acc[1][t]);
          acc[1][t] = fmaf(bf16hi(bw[j]), xh, acc[1][t]);
        }
      }
    }
  }
  for (; c < kc; c += 32) {  // tail (K/8 not a multiple of 128)
    const uint4 a = ldg_stream16(w0 + c), b = ldg_stream16(w1 + c);
    const uint32_t aw[4] = {a.x, a.y, a.z, a.w};
    const uint32_t bw[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
    for (int t = 0; t < T; ++t) {
      const uint4 xv = xs[t * kc + c];
      const uint32_t xw[4] = {xv.x, xv.y, xv.z, xv.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float xl = bf16lo(xw[j]), xh = bf16hi(xw[j]);
        acc[0][t] = fmaf(bf16lo(aw[j]), xl, acc[0][t]);
        acc[0][t] = fmaf(bf16hi(aw[j]), xh, acc[0][t]);
        acc[1][t] = fmaf(bf16lo(bw[j]), xl, acc[1][t]);
        acc[1][t] = fmaf(bf16hi(bw[j]), xh, acc[1][t]);
      }
    }
  }
#pragma unroll
  for (int t = 0; t < T; ++t) {
    acc[0][t] = warp_sum(acc[0][t]);
    acc[1][t] = warp_sum(acc[1][t]);
  }
#pragma unroll
  for (int t = 0; t < T; ++t)
    if (lane == t) {
      if constexpr ((MODE & SKINNY_SLOT_MASK) != 0) {
        if (p.row_slot[t] != n0 / p.slot_cols) acc[0][t] = acc[1][t] = 0.f;
        epi_pair<EPI_STORE>(p.epi, t, n0, acc[0][t], acc[1][t]);
      } else {
        epi_pair<MODE>(p.epi, t, n0, acc[0][t], acc[1][t]);
      }
    }
}

template <int MODE, bool NORM>
int launch_skinny_fp8(const SkinnyParams& p, int T, cudaStream_t stream) {
  MB_CHECK_ARG(T >= 1 && T <= MB200_SKINNY_MAX_T, "skinny linear (fp8): T=%d out of range", T);
  MB_CHECK_ARG(p.K % 16 == 0 && p.N % kSkinnyRowsPerWarp == 0, "skinny linear (fp8): K=%d must be a multiple of 16, N=%d even", p.K, p.N);
  const size_t smem = (size_t)T * p.K * 2;
  MB_CHECK_ARG(smem <= 200 * 1024, "skinny linear (fp8): T*K too large for shared memory (%zu B)", smem);
  const dim3 grid(ceil_div(p.N, kSkinnyRowsPerCta));
  auto go = [&](auto kernel) -> int {
    if (skinny_needs_optin(smem, T)) MB_CHECK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kernel<<<grid, kSkinnyThreads, smem, stream>>>(p);
    note_launch("skinny_linear_kernel<%d, %d, %s, true>", T, MODE, NORM ? "true" : "false");
    MB_CHECK_LAUNCH("skinny_linear_kernel<fp8>");
    return MB200_OK;
  };
  switch (T) {
    case 1: return go(skinny_linear_kernel<1, MODE, NORM, true>);
    case 2: return go(skinny_linear_kernel<2, MODE, NORM, true>);
    case 3: return go(skinny_linear_kernel<3, MODE, NORM, true>);
    default: return go(skinny_linear_kernel<4, MODE, NORM, true>);
  }
}

// x of up to 4 tokens is staged whole: 224 KB at Mistral Large's w2 (K = 28672), so the bound is the opt-in shared memory of the
// device less the kernel's static reduction array, not the 200 KB of the bf16 and FP8 launchers.
template <int MODE, bool NORM>
int launch_skinny_int4(const SkinnyParams& p, int T, cudaStream_t stream) {
  MB_CHECK_ARG(T >= 1 && T <= MB200_SKINNY_MAX_T, "skinny linear (int4): T=%d out of range", T);
  MB_CHECK_ARG(p.K % kInt4Group == 0 && p.N % kSkinnyRowsPerWarp == 0 && p.gscale != nullptr,
               "skinny linear (int4): K=%d must be a multiple of 128, N=%d even, group scales given", p.K, p.N);
  int dev = 0, optin = 0;
  MB_CHECK_CUDA(cudaGetDevice(&dev));
  MB_CHECK_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  const size_t smem = (size_t)T * p.K * 2;
  MB_CHECK_ARG(smem + (size_t)T * kSkinnyWarps * sizeof(float) <= (size_t)optin, "skinny linear (int4): T*K too large for shared memory (%zu B)", smem);
  const dim3 grid(ceil_div(p.N, kSkinnyRowsPerCta));
  auto go = [&](auto kernel) -> int {
    if (skinny_needs_optin(smem, T)) MB_CHECK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kernel<<<grid, kSkinnyThreads, smem, stream>>>(p);
    note_launch("skinny_linear_kernel<%d, %d, %s, false, true>", T, MODE, NORM ? "true" : "false");
    MB_CHECK_LAUNCH("skinny_linear_kernel<int4>");
    return MB200_OK;
  };
  switch (T) {
    case 1: return go(skinny_linear_kernel<1, MODE, NORM, false, true>);
    case 2: return go(skinny_linear_kernel<2, MODE, NORM, false, true>);
    case 3: return go(skinny_linear_kernel<3, MODE, NORM, false, true>);
    default: return go(skinny_linear_kernel<4, MODE, NORM, false, true>);
  }
}

template <int MODE, bool NORM>
int launch_skinny(const SkinnyParams& p, int T, cudaStream_t stream) {
  MB_CHECK_ARG(T >= 1 && T <= MB200_SKINNY_MAX_T, "skinny linear: T=%d out of range", T);
  MB_CHECK_ARG(p.K % 8 == 0 && p.N % kSkinnyRowsPerWarp == 0, "skinny linear: K=%d must be a multiple of 8, N=%d even", p.K, p.N);
  const size_t smem = (size_t)T * p.K * 2;
  MB_CHECK_ARG(smem <= 200 * 1024, "skinny linear: T*K too large for shared memory (%zu B)", smem);
  const dim3 grid(ceil_div(p.N, kSkinnyRowsPerCta));
  auto go = [&](auto kernel) -> int {
    if (skinny_needs_optin(smem, T)) MB_CHECK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kernel<<<grid, kSkinnyThreads, smem, stream>>>(p);
    note_launch("skinny_linear_kernel<%d, %d, %s>", T, MODE, NORM ? "true" : "false");
    MB_CHECK_LAUNCH("skinny_linear_kernel");
    return MB200_OK;
  };
  switch (T) {
    case 1: return go(skinny_linear_kernel<1, MODE, NORM>);
    case 2: return go(skinny_linear_kernel<2, MODE, NORM>);
    case 3: return go(skinny_linear_kernel<3, MODE, NORM>);
    default: return go(skinny_linear_kernel<4, MODE, NORM>);
  }
}

}  // namespace mb200
