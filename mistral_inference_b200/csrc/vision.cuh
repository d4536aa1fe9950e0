// Data movement of the vision path (vision_encoder.py, transformer.py:122-161): patchify, patch-merge gather, embedding splice.
// All three are memory-bound copies; every FLOP around them runs in the GEMM and attention kernels.
#pragma once
#include "common.cuh"

namespace mb200 {

// Stride-p Conv2d as a GEMM (vision_encoder.py:35-41,85): row (py * gw + px) of `out` holds the p x p patch of every channel in
// the conv weight's flatten order k = c * p^2 + ky * p + kx, zero-padded to k_pad.  Pixels past the last whole patch are never
// read (the convolution floors).  One CTA per patch.
__global__ void patchify_kernel(const bf16* __restrict__ img, bf16* __restrict__ out, int H, int W, int p, int gw, int K, int k_pad) {
  const int row = blockIdx.x, py = row / gw, px = row - py * gw;
  const int pp = p * p;
  for (int k = threadIdx.x; k < k_pad; k += blockDim.x) {
    bf16 v = __float2bfloat16_rn(0.f);
    if (k < K) {
      const int c = k / pp, rem = k - c * pp, ky = rem / p, kx = rem - ky * p;
      v = img[((int64_t)c * H + py * p + ky) * W + px * p + kx];
    }
    out[(int64_t)row * k_pad + k] = v;
  }
}

// PatchMerger.permute (vision_encoder.py:180-228) for one image of h x w patches: output row by * (w/s) + bx, feature
// c * s^2 + ky * s + kx = x[(by*s + ky) * w + bx*s + kx, c] (the unfold order).  One CTA per output row.
__global__ void patch_merge_kernel(const bf16* __restrict__ x, bf16* __restrict__ out, int w, int s, int d) {
  const int row = blockIdx.x, gw = w / s, by = row / gw, bx = row - by * gw;
  const int ss = s * s, D = d * ss;
  for (int f = threadIdx.x; f < D; f += blockDim.x) {
    const int c = f / ss, rem = f - c * ss, ky = rem / s, kx = rem - ky * s;
    out[(int64_t)row * D + f] = x[((int64_t)(by * s + ky) * w + bx * s + kx) * d + c];
  }
}

// Embedding splice (transformer.py:128-160), step 1: ordinal[t] = number of image tokens before t (or -1 for a text token),
// ordinal[T] = number of image tokens.  One CTA scans the ids in blocks of 1024.
constexpr int SPLICE_SCAN_THREADS = 1024;
__global__ void __launch_bounds__(SPLICE_SCAN_THREADS) splice_scan_kernel(const long long* __restrict__ ids, int32_t* __restrict__ ordinal,
                                                                          int T, long long image_token_id) {
  __shared__ int warp_tot[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int base = 0;
  for (int t0 = 0; t0 < T; t0 += SPLICE_SCAN_THREADS) {
    const int t = t0 + (int)threadIdx.x;
    const bool img = t < T && ids[t] == image_token_id;
    const unsigned bal = __ballot_sync(0xffffffffu, img);
    if (lane == 0) warp_tot[warp] = __popc(bal);
    __syncthreads();
    int before = 0, total = 0;
    for (int w = 0; w < SPLICE_SCAN_THREADS / 32; ++w) {
      before += w < warp ? warp_tot[w] : 0;
      total += warp_tot[w];
    }
    if (t < T) ordinal[t] = img ? base + before + __popc(bal & ((1u << lane) - 1u)) : -1;
    base += total;
    __syncthreads();
  }
  if (threadIdx.x == 0) ordinal[T] = base;
}

// step 2: row t = image feature row ordinal[t], or tok_embeddings[ids[t]].  Rows that would read past either table are written
// as zeros (the caller compares ordinal[T] with the feature count and raises).
__global__ void splice_gather_kernel(const long long* __restrict__ ids, const int32_t* __restrict__ ordinal, const uint4* __restrict__ emb,
                                     const uint4* __restrict__ feats, uint4* __restrict__ out, int row_chunks, long long vocab, int n_feats) {
  const int t = blockIdx.x;
  const int o = ordinal[t];
  const uint4* src = nullptr;
  if (o >= 0) {
    if (o < n_feats) src = feats + (int64_t)o * row_chunks;
  } else {
    const long long id = ids[t];
    if (id >= 0 && id < vocab) src = emb + id * row_chunks;
  }
  for (int c = threadIdx.x; c < row_chunks; c += blockDim.x) out[(int64_t)t * row_chunks + c] = src ? src[c] : make_uint4(0, 0, 0, 0);
}

}  // namespace mb200
