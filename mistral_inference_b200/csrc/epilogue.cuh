// Pair epilogues shared by the weight-streaming GEMV (skinny_linear.cuh) and the tensor-core GEMMs (gemm_mma.cuh, gemm_wgmma.cuh,
// gemm_streamk.cuh).
// Every linear on the hot path hands the epilogue two adjacent fp32 accumulators (columns n, n+1 of
// token t).  That is the natural unit: RoPE rotates the interleaved pair (x[2i], x[2i+1]) (rope.py:18-23)
// and the packed gate/up weight puts w1[i], w3[i] on rows 2i, 2i+1.
#pragma once
#include "common.cuh"

namespace mb200 {

enum EpiMode : int {
  EPI_STORE = 0,     // out[t, n] = bf16(acc)
  EPI_RESIDUAL = 1,  // out[t, n] = bf16( bf16(acc) + residual[t, n] )           (transformer_layers.py:166,168)
  EPI_F32 = 2,       // logits[t, n] = float(bf16(acc))                           (transformer.py:235,240)
  EPI_SWIGLU = 3,    // g[t, n/2] = bf16( bf16(silu(bf16(acc0))) * bf16(acc1) )   (transformer_layers.py:106)
  EPI_QKV_ROPE = 4,  // split into q/k/v, rotate q,k pairs, optional ring scatter  (transformer_layers.py:66-70, cache.py:91-92)
  EPI_MOE_SCALE = 5, // yw[row, n] = bf16( w[row] * bf16(acc) ), stored on every rank of an expert-parallel group  (moe.py:31)
  EPI_BIAS = 6,      // out[t, n] = bf16(acc + bias[n]) (bias may be null: bf16(acc))  nn.Linear(bias=True) (vision_encoder.py:108,114)
  EPI_BIAS_GELU = 7, // out[t, n] = bf16( gelu_erf( bf16(acc + bias[n]) ) )           nn.GELU() after w_in (vision_encoder.py:117)
};
// Flag OR-ed into EPI_STORE / EPI_RESIDUAL / EPI_SWIGLU / EPI_QKV_ROPE / EPI_MOE_SCALE: the un-merged LoRA combine
// (LoRALinear.forward, lora.py:71-74) runs on the Linear's bf16 output before the mode's own work:
//   y = bf16(y + bf16(L[t, n] * scaling))     L = the adapter's up-projection output, bf16 [T, ld_lora]
// (EPI_MOE_SCALE: t is the expert row, so the routing weight and the expert-parallel peer stores take the combined value.)
// Instantiations without the flag compile to the same code as before.
constexpr int EPI_LORA = 16;
// Flag OR-ed into EPI_STORE / EPI_RESIDUAL / EPI_SWIGLU / EPI_QKV_ROPE: FP8 dense weights (include/mistral_b200.h).  The
// accumulator is sum_k x[t, k] * float(q[n, k]); the row scale is applied once, as one fp32 product, before the Linear's rounding:
//   y = bf16(fp32(w_scale[n] * acc))
// Instantiations without the flag compile to the same code as before.
constexpr int EPI_WSCALE = 32;
// Flag OR-ed with EPI_WSCALE: FP8 activations (prefill_compute="fp8", include/mistral_b200.h).  The accumulator is
// sum_k float(xq[t, k]) * float(q[n, k]) over the per-token e4m3 activations xq = e4m3(x * 2^-e[t]); the token's power of two
// (the `ascale` argument of epi_pair, 2^e[t]) comes back after the row scale as one fp32 product:
//   y = bf16(fp32(fp32(w_scale[n] * acc) * 2^e[t]))
// The exponents travel as a kernel argument of their own, so EpiParams and the code of instantiations without the flag are
// unchanged.
constexpr int EPI_ASCALE = 128;  // 64 is SKINNY_SLOT_MASK

constexpr int kMaxPeers = 8;

struct EpiParams {
  void* out = nullptr;             // bf16 [T, ld_out]
  const void* residual = nullptr;  // bf16 [T, ld_out]
  float* out_f32 = nullptr;        // fp32 [T, ld_out]
  int64_t ld_out = 0;
  // EPI_QKV_ROPE
  void* q_out = nullptr;  // [T, q_dim]
  void* k_out = nullptr;  // [T, kv_dim]
  void* v_out = nullptr;  // [T, kv_dim]
  void* cache_k = nullptr;  // [rows, kv_dim]
  void* cache_v = nullptr;
  const int32_t* positions = nullptr;   // [T]
  const int32_t* cache_rows = nullptr;  // [T] or null
  const float* rope = nullptr;          // [n_pos, head_dim / 2, 2]
  int q_dim = 0, kv_dim = 0;
  int head_dim = kHeadDim;              // 64 or 128 (a power of two: the pair index is a mask)
  // EPI_BIAS / EPI_BIAS_GELU
  const void* bias = nullptr;  // bf16 [N] or null
  // EPI_MOE_SCALE: routing weight of each (token, expert) row; the weighted expert output goes to `out` and to the same offset
  // of the mapped buffers of the other ranks (NVLink peer stores; n_peers == 0 when unsharded)
  const void* row_w = nullptr;  // bf16 [rows]
  void* peer_out[kMaxPeers] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  int n_peers = 0;
  // EPI_LORA
  const void* lora_l = nullptr;  // bf16 [T, ld_lora], columns in the weight's row order
  int64_t ld_lora = 0;
  float lora_scaling = 0.f;
  // EPI_WSCALE
  const float* w_scale = nullptr;  // fp32 [N]
};

// 2^e as an fp32 number for e in [-149, 127] (subnormal below -126): exact, so a product with it rounds once
__device__ __forceinline__ float exp2_exact(int e) { return __int_as_float(e >= -126 ? (e + 127) << 23 : 1 << (e + 149)); }

template <int FLAGS>
__device__ __forceinline__ void epi_pair(const EpiParams& p, int t, int n, float acc0, float acc1, float ascale = 1.f) {
  constexpr int MODE = FLAGS & ~(EPI_LORA | EPI_WSCALE | EPI_ASCALE);
  if constexpr ((FLAGS & EPI_WSCALE) != 0) {
    static_assert(MODE == EPI_STORE || MODE == EPI_RESIDUAL || MODE == EPI_SWIGLU || MODE == EPI_QKV_ROPE, "FP8 row scale: unsupported mode");
    const float2 s = *reinterpret_cast<const float2*>(p.w_scale + n);
    acc0 = __fmul_rn(s.x, acc0);
    acc1 = __fmul_rn(s.y, acc1);
  }
  if constexpr ((FLAGS & EPI_ASCALE) != 0) {
    static_assert((FLAGS & (EPI_WSCALE | EPI_LORA)) == EPI_WSCALE, "FP8 activations: FP8 dense weights without LoRA only");
    acc0 = __fmul_rn(acc0, ascale);
    acc1 = __fmul_rn(acc1, ascale);
  }
  // the Linear's own output rounding (bf16 result of nn.Linear)
  float y0 = round_bf16(acc0), y1 = round_bf16(acc1);
  if constexpr ((FLAGS & EPI_LORA) != 0) {
    static_assert(MODE == EPI_STORE || MODE == EPI_RESIDUAL || MODE == EPI_SWIGLU || MODE == EPI_QKV_ROPE || MODE == EPI_MOE_SCALE,
                  "LoRA combine: unsupported mode");
    const uint32_t l = *reinterpret_cast<const uint32_t*>(reinterpret_cast<const uint16_t*>(p.lora_l) + (int64_t)t * p.ld_lora + n);
    y0 = round_bf16(y0 + round_bf16(bf16lo(l) * p.lora_scaling));
    y1 = round_bf16(y1 + round_bf16(bf16hi(l) * p.lora_scaling));
  }
  if constexpr (MODE == EPI_STORE) {
    *reinterpret_cast<uint32_t*>(reinterpret_cast<uint16_t*>(p.out) + (int64_t)t * p.ld_out + n) = pack_bf16x2(y0, y1);
  } else if constexpr (MODE == EPI_RESIDUAL) {
    const uint32_t r = *reinterpret_cast<const uint32_t*>(reinterpret_cast<const uint16_t*>(p.residual) + (int64_t)t * p.ld_out + n);
    *reinterpret_cast<uint32_t*>(reinterpret_cast<uint16_t*>(p.out) + (int64_t)t * p.ld_out + n) =
        pack_bf16x2(y0 + bf16lo(r), y1 + bf16hi(r));
  } else if constexpr (MODE == EPI_F32) {
    *reinterpret_cast<float2*>(p.out_f32 + (int64_t)t * p.ld_out + n) = make_float2(y0, y1);
  } else if constexpr (MODE == EPI_SWIGLU) {
    const float s = round_bf16(ref_silu(y0));
    reinterpret_cast<bf16*>(p.out)[(int64_t)t * p.ld_out + (n >> 1)] = __float2bfloat16_rn(s * y1);
  } else if constexpr (MODE == EPI_MOE_SCALE) {
    const float w = bf16_to_float(reinterpret_cast<const uint16_t*>(p.row_w)[t]);
    const uint32_t packed = pack_bf16x2(w * y0, w * y1);
    const int64_t off = (int64_t)t * p.ld_out + n;
    *reinterpret_cast<uint32_t*>(reinterpret_cast<uint16_t*>(p.out) + off) = packed;
    for (int r = 0; r < p.n_peers; ++r) *reinterpret_cast<uint32_t*>(reinterpret_cast<uint16_t*>(p.peer_out[r]) + off) = packed;
  } else if constexpr (MODE == EPI_BIAS || MODE == EPI_BIAS_GELU) {
    float b0 = y0, b1 = y1;
    if (p.bias != nullptr) {  // addmm: the bias joins the fp32 accumulator before the single rounding
      const uint32_t bb = *reinterpret_cast<const uint32_t*>(reinterpret_cast<const uint16_t*>(p.bias) + n);
      b0 = round_bf16(acc0 + bf16lo(bb));
      b1 = round_bf16(acc1 + bf16hi(bb));
    }
    if constexpr (MODE == EPI_BIAS_GELU) {
      b0 = ref_gelu(b0);
      b1 = ref_gelu(b1);
    }
    *reinterpret_cast<uint32_t*>(reinterpret_cast<uint16_t*>(p.out) + (int64_t)t * p.ld_out + n) = pack_bf16x2(b0, b1);
  } else if constexpr (MODE == EPI_QKV_ROPE) {
    if (n < p.q_dim + p.kv_dim) {  // q or k: rotate
      const int pos = p.positions[t];
      const int i = (n & (p.head_dim - 1)) >> 1;
      const float2 cs = *reinterpret_cast<const float2*>(p.rope + ((int64_t)pos * (p.head_dim >> 1) + i) * 2);
      float re, im;
      ref_cmul(y0, y1, cs.x, cs.y, re, im);
      const uint32_t packed = pack_bf16x2(re, im);
      if (n < p.q_dim) {
        *reinterpret_cast<uint32_t*>(reinterpret_cast<uint16_t*>(p.q_out) + (int64_t)t * p.q_dim + n) = packed;
      } else {
        const int c = n - p.q_dim;
        *reinterpret_cast<uint32_t*>(reinterpret_cast<uint16_t*>(p.k_out) + (int64_t)t * p.kv_dim + c) = packed;
        if (p.cache_rows != nullptr) {
          const int row = p.cache_rows[t];
          if (row >= 0) *reinterpret_cast<uint32_t*>(reinterpret_cast<uint16_t*>(p.cache_k) + (int64_t)row * p.kv_dim + c) = packed;
        }
      }
    } else {  // v: stored as projected
      const int c = n - p.q_dim - p.kv_dim;
      const uint32_t packed = pack_bf16x2(y0, y1);
      *reinterpret_cast<uint32_t*>(reinterpret_cast<uint16_t*>(p.v_out) + (int64_t)t * p.kv_dim + c) = packed;
      if (p.cache_rows != nullptr) {
        const int row = p.cache_rows[t];
        if (row >= 0) *reinterpret_cast<uint32_t*>(reinterpret_cast<uint16_t*>(p.cache_v) + (int64_t)row * p.kv_dim + c) = packed;
      }
    }
  }
}

__device__ __forceinline__ uint32_t pack2_rn(float lo, float hi) {
  const __nv_bfloat162 b = __floats2bfloat162_rn(lo, hi);  // one F2FP: .x (low half) = lo
  return *reinterpret_cast<const uint32_t*>(&b);
}

}  // namespace mb200
