// FP8 (e4m3) KV cache: the quantiser / ring writer and the decode attention kernel that reads the e4m3 ring.
//
// Format (include/mistral_b200.h, mb200_kv_quantize).  Per (slot, kv head) row x of hd = 128 bf16 values the ring holds 128 e4m3
// bytes q and one int8 exponent e:
//   e    = max(-124, smallest integer with amax|x| <= 448 * 2^e)   (all-zero row: -124)
//   q[i] = e4m3fn_rn(fp32(x[i]) * 2^-e)                            (exact scaling, one rounding, never above 448)
//   x'   = q * 2^e                                                 (exact in bf16)
// Attention sees x' only, so every kernel that reads the ring rebuilds the bf16 bits of x' exactly (kv_dequant8) and then runs the
// bf16 kernel's arithmetic unchanged: each FP8 variant is bit-identical to its bf16 kernel on a bf16 ring that holds x'.
#pragma once
#include <cuda_fp16.h>
#include <cuda_fp8.h>

#include "attn_decode_tma.cuh"

namespace mb200 {

constexpr int kKvExpMin = -124;  // 2^-9 (smallest e4m3 subnormal) * 2^-124 = 2^-133, the smallest bf16 subnormal

// Two e4m3 codes (low byte first) of a row with exponent e -> the bf16x2 bits of x'.  cvt.rn.f16x2.e4m3x2 is exact (every e4m3
// value, subnormals included, is a normal f16 with the low 7 mantissa bits zero), so for e >= -112 the bf16 bits are the f16
// bits with the exponent rebiased: sign | (E5 + 112 + e) << 7 | M10 >> 3, and zero stays (signed) zero -- integer work only.  Rows
// with e < -112 (amax < 2^-104) can produce bf16 subnormals; they take an exact fp32 product instead.
__device__ __forceinline__ uint32_t kv_dequant2(uint32_t two, int e) {
  const __half2_raw h = __nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)two, __NV_E4M3);
  const uint32_t w = (uint32_t)h.x | ((uint32_t)h.y << 16);
  if (e >= -112) {
    const uint32_t mag = (w >> 3) & 0x0fff0fffu;                       // E5 << 7 | M7 per half
    const uint32_t nz = (mag + 0x7fff7fffu) & 0x80008000u;             // bit 15 of a half: that half is non-zero (no carry out)
    const uint32_t keep = nz - (nz >> 15);                             // 0x7fff per non-zero half
    const uint32_t bias = (uint32_t)(112 + e) << 7;                    // 0 .. 232 << 7: the sum stays inside its half
    return (w & 0x80008000u) | ((mag + (bias | (bias << 16))) & keep);
  }
  const float s = __uint_as_float((uint32_t)(127 + e) << 23);          // 2^e, a normal fp32 for e >= -126
  const float lo = __half2float(__ushort_as_half(h.x)) * s, hi = __half2float(__ushort_as_half(h.y)) * s;  // exact (>= 2^-133)
  return pack_bf16x2(lo, hi);
}

// 8 e4m3 codes (one uint2) -> 8 bf16 of x' (one uint4)
__device__ __forceinline__ uint4 kv_dequant8(uint2 q, int e) {
  return make_uint4(kv_dequant2(q.x & 0xffffu, e), kv_dequant2(q.x >> 16, e), kv_dequant2(q.y & 0xffffu, e), kv_dequant2(q.y >> 16, e));
}

// ---- quantiser / ring writer: one warp per (token, kv head, K|V) row --------------------------------------------------------------
// x' replaces the bf16 row in place when write_back (prefill, before attention), and (q, e) go to ring row cache_rows[t] when
// cache_rows is given and cache_rows[t] >= 0 (only the last W tokens of a chunk are cached, cache.py:226).
struct KvQuantParams {
  bf16* k;  // [T, KV*hd] bf16
  bf16* v;
  uint8_t* cache_k;  // [n_rows, KV*hd] e4m3
  uint8_t* cache_v;
  int8_t* exp_k;  // [n_rows, KV]
  int8_t* exp_v;
  const int32_t* rows;  // [T] or nullptr
  int T, KV, write_back;
};

__global__ void __launch_bounds__(128) kv_quantize_kernel(const KvQuantParams p) {
  pdl_trigger();
  pdl_wait();  // k, v are the QKV GEMM's output
  const int gw = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (gw >= p.T * p.KV * 2) return;
  const int is_v = gw & 1, g = (gw >> 1) % p.KV, t = (gw >> 1) / p.KV;
  bf16* src = (is_v ? p.v : p.k) + ((int64_t)t * p.KV + g) * kHeadDim + lane * 4;
  const uint2 x = *reinterpret_cast<const uint2*>(src);
  const float f[4] = {bf16lo(x.x), bf16hi(x.x), bf16lo(x.y), bf16hi(x.y)};
  const float amax = warp_max(fmaxf(fmaxf(fabsf(f[0]), fabsf(f[1])), fmaxf(fabsf(f[2]), fabsf(f[3]))));
  // smallest e with amax <= 1.75 * 2^(e + 8): amax = m * 2^E, m in [1, 2), needs e >= E - 8 when m <= 1.75, else E - 7
  const uint32_t bits = __float_as_uint(amax);
  const int E = (int)(bits >> 23) - 127;
  const int e = (bits >> 23) == 0 ? kKvExpMin : max(kKvExpMin, E - 8 + ((bits & 0x7fffffu) > 0x600000u ? 1 : 0));
  const float inv = __uint_as_float((uint32_t)(127 - e) << 23);  // 2^-e, normal for e in [-124, 120]
  const uint32_t q01 = __nv_cvt_float2_to_fp8x2(make_float2(f[0] * inv, f[1] * inv), __NV_SATFINITE, __NV_E4M3);
  const uint32_t q23 = __nv_cvt_float2_to_fp8x2(make_float2(f[2] * inv, f[3] * inv), __NV_SATFINITE, __NV_E4M3);
  const uint32_t q = q01 | (q23 << 16);
  if (p.write_back) *reinterpret_cast<uint2*>(src) = make_uint2(kv_dequant2(q01, e), kv_dequant2(q23, e));
  if (p.rows != nullptr) {
    const int row = p.rows[t];
    if (row >= 0) {
      *reinterpret_cast<uint32_t*>((is_v ? p.cache_v : p.cache_k) + ((int64_t)row * p.KV + g) * kHeadDim + lane * 4) = q;
      if (lane == 0) (is_v ? p.exp_v : p.exp_k)[(int64_t)row * p.KV + g] = (int8_t)e;
    }
  }
}

// ---- decode attention over the e4m3 ring -----------------------------------------------------------------------------------------
// attn_decode_tma_kernel with the same CTA, split, softmax and merge; what changes is the tile.  The producer thread TMA-loads one
// [64 keys x 128 B] e4m3 box of K and one of V per tile (16 KB, half the bf16 tile, so the ring has 5 stages instead of 3: 80 KB
// of e4m3 in flight).  Each consumer warp rebuilds x' of its own 16 keys into a private [16 x 128] bf16 tile in the swizzled layout
// the bf16 kernel's ldmatrix reads (K first; once the scores are in registers, V into the same tile) and releases the e4m3 stage as
// soon as both are converted.  The exponents are one byte per key: plain loads, issued one tile ahead.  Slots >= kv_len hold
// arbitrary bytes (NaN codes, extreme exponents): their scores are masked by index and their V rows are written as zero instead of
// converted.
struct AttnDecodeFp8Params {
  AttnDecodeParams a;    // cache_k / cache_v point at the e4m3 rings
  const int8_t* exp_k;   // [max_batch * W, KV]
  const int8_t* exp_v;
};

constexpr int ADF_STAGES = 5;
constexpr int ADF_TILE_BYTES = ADT_KT * kHeadDim;                   // [64 keys][128 dims] e4m3 = 8 KB
constexpr int ADF_STAGE_BYTES = 2 * ADF_TILE_BYTES;                 // K | V
constexpr int ADF_CONV_BYTES = 16 * kHeadDim * 2;                   // one warp's [16 keys][128 dims] bf16 = 4 KB
constexpr int ADF_SMEM = ADF_STAGES * ADF_STAGE_BYTES + ADT_CONSUMER_WARPS * ADF_CONV_BYTES + 1024 + 2 * ADF_STAGES * 8;  // + alignment, full/empty barriers

// byte offset of bf16 16-byte chunk C (0..15) of key r (0..15) in a warp's converted tile: adt_off's layout for 16 rows
__device__ __forceinline__ uint32_t adf_off(int r, int C) { return (uint32_t)((C >> 3) * 2048 + r * 128 + (((C & 7) ^ (r & 7)) << 4)); }

// Converts the e4m3 rows [16 w, 16 w + 16) of a 128B-swizzled [64][128 B] box into the warp's bf16 tile: lane -> key r = lane / 2,
// dims [64 (lane & 1), 64 (lane & 1) + 64).  Rows r >= zero_from are written as zero.
__device__ __forceinline__ void adf_convert(const uint8_t* box, uint8_t* conv, int warp, int lane, int e, int zero_from) {
  const int r = lane >> 1, row = 16 * warp + r;
// Not unrolled: a full unroll spills (168 registers) and measured only 5 % faster.  This loop is what bounds the kernel (DESIGN
// §3.10: with a plain copy in place of kv_dequant8 the kernel runs 3x faster).
#pragma unroll 1
  for (int i = 0; i < 4; ++i) {
    const int c8 = (lane & 1) * 4 + i;  // 16-byte e4m3 chunk: dims [16 c8, 16 c8 + 16)
    uint4 lo = make_uint4(0, 0, 0, 0), hi = lo;
    if (r < zero_from) {
      const uint4 q = *reinterpret_cast<const uint4*>(box + row * 128 + ((c8 ^ (row & 7)) << 4));
      lo = kv_dequant8(make_uint2(q.x, q.y), e);
      hi = kv_dequant8(make_uint2(q.z, q.w), e);
    }
    *reinterpret_cast<uint4*>(conv + adf_off(r, 2 * c8)) = lo;
    *reinterpret_cast<uint4*>(conv + adf_off(r, 2 * c8 + 1)) = hi;
  }
}

template <int REP>
__global__ void __launch_bounds__(ADT_THREADS, 2)
    attn_decode_tma_fp8_kernel(const __grid_constant__ CUtensorMap map_k, const __grid_constant__ CUtensorMap map_v, const AttnDecodeFp8Params fp) {
  const AttnDecodeParams& p = fp.a;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* conv_all = smem + ADF_STAGES * ADF_STAGE_BYTES;
  uint64_t* full = reinterpret_cast<uint64_t*>(conv_all + ADT_CONSUMER_WARPS * ADF_CONV_BYTES);
  uint64_t* empty = full + ADF_STAGES;
  __shared__ float sm_m[ADT_CONSUMER_WARPS][REP], sm_l[ADT_CONSUMER_WARPS][REP];
  __shared__ float sm_acc[ADT_CONSUMER_WARPS][REP][kHeadDim];
  __shared__ int is_last;
  __shared__ float cm[64 * REP], cl[64 * REP];

  const int s = blockIdx.x, g = blockIdx.y, b = blockIdx.z;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  pdl_trigger();
  pdl_wait();  // q, the ring rows of this step and kv_len come from the preceding kernels
  const int len = p.kv_len[b];
  const int C = (len + p.S - 1) / p.S;
  const int k_begin = min(s * C, len), k_end = min(k_begin + C, len);
  const int n_tiles = (k_end - k_begin + ADT_KT - 1) / ADT_KT;

  if (tid == 0) {
    for (int i = 0; i < ADF_STAGES; ++i) {
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
  const int row = lane >> 2, cq = lane & 3;

  if (warp == ADT_CONSUMER_WARPS) {
    // ================= producer: one thread =================
    if (lane == 0) {
      for (int j = 0; j < n_tiles; ++j) {
        const uint32_t st = j % ADF_STAGES, par = (j / ADF_STAGES) & 1;
        mbar_wait(&empty[st], par ^ 1, 31, j);
        mbar_arrive_expect_tx(&full[st], ADF_STAGE_BYTES);
        uint8_t* base = smem + st * ADF_STAGE_BYTES;
        const int r0 = b * p.W + k_begin + j * ADT_KT, c0 = g * kHeadDim;
        tma_load_2d(base, &map_k, &full[st], c0, r0);
        tma_load_2d(base + ADF_TILE_BYTES, &map_v, &full[st], c0, r0);
      }
    }
  } else {
    // ================= consumers: warp w owns keys [16 w, 16 w + 16) of every tile =================
    const float sl2 = p.scale * kLog2e;
    uint8_t* conv = conv_all + warp * ADF_CONV_BYTES;
    const uint32_t cst = smem_u32(conv);
    uint32_t qa[8][4];
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) {
      qa[ks][0] = qa[ks][1] = qa[ks][2] = qa[ks][3] = 0u;
      if (row < REP) {
        const bf16* qp = p.q + ((int64_t)b * p.H + g * REP + row) * kHeadDim + ks * 16 + cq * 2;
        qa[ks][0] = *reinterpret_cast<const uint32_t*>(qp);
        qa[ks][2] = *reinterpret_cast<const uint32_t*>(qp + 8);
      }
    }
#pragma unroll
    for (int n = 0; n < 16; ++n) o[n][0] = o[n][1] = o[n][2] = o[n][3] = 0.f;

    // the exponents of this lane's key (lane / 2) in tile jj, 0 past the range; loaded one tile ahead so that their latency hides
    // behind a tile's work instead of sitting between the stage wait and the conversion
    auto load_exps = [&](int jj, int& ek_, int& ev_) {
      ek_ = ev_ = 0;
      const int key = 16 * warp + (lane >> 1);
      if (jj < n_tiles && key < k_end - (k_begin + jj * ADT_KT)) {
        const int64_t er = ((int64_t)b * p.W + k_begin + jj * ADT_KT + key) * p.KV + g;
        ek_ = fp.exp_k[er];
        ev_ = fp.exp_v[er];
      }
    };
    int ek_next, ev_next;
    load_exps(0, ek_next, ev_next);
    for (int j = 0; j < n_tiles; ++j) {
      const uint32_t st = j % ADF_STAGES, par = (j / ADF_STAGES) & 1;
      const int nk = min(ADT_KT, k_end - (k_begin + j * ADT_KT)) - 16 * warp;  // valid keys among this warp's 16 (may be <= 0)
      const int ek = ek_next, ev = ev_next;
      load_exps(j + 1, ek_next, ev_next);
      mbar_wait(&full[st], par, 32, j);
      const uint8_t* kbox = smem + st * ADF_STAGE_BYTES;
      if (nk > 0) {
        adf_convert(kbox, conv, warp, lane, ek, 16);  // rows past the range: scores are masked by index
        __syncwarp();
        float sc[2][4];
#pragma unroll
        for (int t = 0; t < 2; ++t) {
          sc[t][0] = sc[t][1] = sc[t][2] = sc[t][3] = 0.f;
          const int krow = t * 8 + (lane & 7);
#pragma unroll
          for (int k2 = 0; k2 < 4; ++k2) {
            uint32_t b0, b1, b2, b3;
            ldmatrix_x4(cst + adf_off(krow, k2 * 4 + (lane >> 3)), b0, b1, b2, b3);
            mma_bf16_16816(sc[t], qa[2 * k2], b0, b1);
            mma_bf16_16816(sc[t], qa[2 * k2 + 1], b2, b3);
          }
        }
        __syncwarp();  // K is in registers: the tile takes V next
        adf_convert(kbox + ADF_TILE_BYTES, conv, warp, lane, ev, nk);  // V rows past the range are zero (P = 0 there, 0 * NaN = NaN)
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[st]);
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
        const int vrow = (lane & 7) + ((lane >> 3) & 1) * 8;
#pragma unroll
        for (int n2 = 0; n2 < 8; ++n2) {
          uint32_t b0, b1, b2, b3;
          ldmatrix_x4_trans(cst + adf_off(vrow, n2 * 2 + (lane >> 4)), b0, b1, b2, b3);
          mma_bf16_16816(o[2 * n2], pa, b0, b1);
          mma_bf16_16816(o[2 * n2 + 1], pa, b2, b3);
        }
        __syncwarp();  // the tile is rewritten by the next K
      } else {
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[st]);
      }
    }
    l_run += __shfl_xor_sync(0xffffffffu, l_run, 1);
    l_run += __shfl_xor_sync(0xffffffffu, l_run, 2);
    if (row < REP) {
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
  __syncthreads();
  adt_merge<REP>(p, sm_m, sm_l, sm_acc, is_last, cm, cl, s, g, b, tid, warp);
}

// [rows, cols] e4m3 ring as a 2-D byte tensor; box = [128 cols (128 B) x 64 rows], 128-byte swizzle, OOB rows read as zero
inline int make_kv_fp8_tensor_map(CUtensorMap* map, const void* base, int64_t rows, int64_t cols) {
  PFN_encodeTiled enc = get_encode_tiled();
  if (enc == nullptr) return fail(MB200_E_CUDA, "cuTensorMapEncodeTiled entry point not available");
  const cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  const cuuint64_t strides[1] = {(cuuint64_t)cols};
  const cuuint32_t box[2] = {(cuuint32_t)kHeadDim, (cuuint32_t)ADT_KT};
  const cuuint32_t estr[2] = {1, 1};
  const CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                         CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(MB200_E_CUDA, "cuTensorMapEncodeTiled (e4m3 kv cache) failed (%d) rows=%lld cols=%lld", (int)r, (long long)rows, (long long)cols);
  return MB200_OK;
}

template <int REP>
int launch_attn_decode_tma_fp8(const AttnDecodeFp8Params& fp, int64_t max_batch_rows, cudaStream_t st) {
  const AttnDecodeParams& p = fp.a;
  CUtensorMap map_k, map_v;
  int rc = make_kv_fp8_tensor_map(&map_k, p.cache_k, max_batch_rows, (int64_t)p.KV * kHeadDim);
  if (rc) return rc;
  rc = make_kv_fp8_tensor_map(&map_v, p.cache_v, max_batch_rows, (int64_t)p.KV * kHeadDim);
  if (rc) return rc;
  MB_CHECK_CUDA(cudaFuncSetAttribute(attn_decode_tma_fp8_kernel<REP>, cudaFuncAttributeMaxDynamicSharedMemorySize, ADF_SMEM));
  const dim3 grid((unsigned)p.S, (unsigned)p.KV, (unsigned)p.B);
  MB_CHECK_CUDA(launch_pdl(attn_decode_tma_fp8_kernel<REP>, grid, dim3(ADT_THREADS), (size_t)ADF_SMEM, st, map_k, map_v, fp));
  note_launch("attn_decode_tma_fp8_kernel<%d>", REP);
  return MB200_OK;
}

}  // namespace mb200
