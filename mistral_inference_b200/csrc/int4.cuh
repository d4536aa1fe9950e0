// INT4 dense weights (include/mistral_b200.h): symmetric 4-bit codes, one bf16 scale per group of 128 consecutive k of a row.
// This header owns the format on the device: the quantiser, and the conversion of packed codes to the bf16 weights W' that every
// INT4 kernel computes with.  Storage: codes uint8 [N, K/2], byte j of a row = code of k = 2j (low nibble) and 2j + 1 (high
// nibble), each nibble q + 8; scales bf16 [N, K/128].
#pragma once
#include "common.cuh"

namespace mb200 {

constexpr int kInt4Group = 128;

// W' of the eight codes of one 32-bit word (nibble i = the code of k0 + i) under the bf16 scale pair s2 = (s, s), as bf16x2 words.
// Exact in two bf16x2 instructions per pair: (0x4300 | u) is the bf16 128 + u (u = q + 8 <= 15 fits the 7 mantissa bits), so
// sub.rn.bf16x2 by 136 gives q exactly; mul.rn.bf16x2 by s rounds q * s (exact in fp32: 4 + 8 significant bits) once, i.e. it is
// bf16_rn(fp32(q) * fp32(s)).  The masks pick nibbles i and i + 4 into one word, so without NATURAL o[i] = (W'[i], W'[i + 4]) (the
// GEMV pairs them with the matching x itself); with NATURAL a byte permute gives k order, o[j] = (W'[2j], W'[2j + 1]).
template <bool NATURAL>
__device__ __forceinline__ void int4x8_to_bf16x2(uint32_t v, uint32_t s2, uint32_t (&o)[4]) {
  uint32_t t[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) t[i] = ((v >> (4 * i)) & 0x000f000fu) | 0x43004300u;
  if constexpr (NATURAL) {
    const uint32_t a = __byte_perm(t[0], t[1], 0x5410), b = __byte_perm(t[2], t[3], 0x5410);
    const uint32_t c = __byte_perm(t[0], t[1], 0x7632), d = __byte_perm(t[2], t[3], 0x7632);
    t[0] = a, t[1] = b, t[2] = c, t[3] = d;
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    uint32_t q;
    asm("sub.rn.bf16x2 %0, %1, %2;" : "=r"(q) : "r"(t[i]), "r"(0x43084308u));  // - (bf16 136, bf16 136)
    asm("mul.rn.bf16x2 %0, %1, %2;" : "=r"(o[i]) : "r"(q), "r"(s2));
  }
}

// ---- quantiser: one CTA per row, one 16-byte chunk (8 weights) per thread and pass, a group = 16 consecutive lanes --------------
//   a = amax of the group (fp32), s = 1 if a == 0, else bf16_rn(fp32(a / 7)) raised to the smallest positive bf16 if that is 0,
//   q = clamp(rint(fp32(W / s)), -8, 7) (IEEE division: the library is built without fast math; rint rounds half to even).
// Code rows land q_stride bytes apart and scale rows s_stride elements apart, so w1 / w3 fill the interleaved rows of w13 directly.
__global__ void __launch_bounds__(256) quantize_int4_groups_kernel(const uint4* __restrict__ w, int K, uint8_t* __restrict__ q, int64_t q_stride,
                                                                   uint16_t* __restrict__ scale, int64_t s_stride) {
  const int n = blockIdx.x, chunks = K >> 3;
  const uint4* row = w + (int64_t)n * chunks;
  uint32_t* qrow = reinterpret_cast<uint32_t*>(q + (int64_t)n * q_stride);
  uint16_t* srow = scale + (int64_t)n * s_stride;
  for (int c = threadIdx.x; c < chunks; c += 256) {  // chunks % 16 == 0: a half warp is one whole group
    const uint4 v = row[c];
    const uint32_t u[4] = {v.x, v.y, v.z, v.w};
    float amax = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) amax = fmaxf(amax, fmaxf(fabsf(bf16lo(u[j])), fabsf(bf16hi(u[j]))));
    const unsigned half = 0xffffu << (threadIdx.x & 16);  // the other half warp may have left the loop
#pragma unroll
    for (int o = 8; o >= 1; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(half, amax, o));
    uint16_t sb = 0x3f80u;  // 1.0
    if (amax != 0.f) {
      sb = bf16_bits(__fdiv_rn(amax, 7.f));
      if (sb == 0) sb = 1;  // the smallest positive bf16 (a subnormal)
    }
    if ((c & 15) == 0) srow[c >> 4] = sb;
    const float s = bf16_to_float(sb);
    uint32_t out = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float x = (j & 1) ? bf16hi(u[j >> 1]) : bf16lo(u[j >> 1]);
      const float r = fminf(fmaxf(rintf(__fdiv_rn(x, s)), -8.f), 7.f);
      out |= (uint32_t)((int)r + 8) << (4 * j);
    }
    qrow[c] = out;
  }
}

}  // namespace mb200
