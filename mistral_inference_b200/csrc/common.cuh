// Shared device/host helpers for libmb200 (sm_90a only).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_fp8.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <cstdarg>
#include <cstdio>
#include <cstdlib>

#include "../../include/mistral_b200.h"

namespace mb200 {

// ---- error plumbing (never throw across the C ABI) ------------------------------------------
extern thread_local char g_err[512];
inline int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}
#define MB_CHECK_ARG(cond, ...) \
  do {                          \
    if (!(cond)) return ::mb200::fail(MB200_E_INVALID, __VA_ARGS__); \
  } while (0)
#define MB_CHECK_LAUNCH(what)                                                                        \
  do {                                                                                               \
    cudaError_t e__ = cudaGetLastError();                                                            \
    if (e__ != cudaSuccess) return ::mb200::fail(MB200_E_CUDA, "%s: %s", what, cudaGetErrorString(e__)); \
  } while (0)
#define MB_CHECK_CUDA(expr)                                                                          \
  do {                                                                                               \
    cudaError_t e__ = (expr);                                                                        \
    if (e__ != cudaSuccess) return ::mb200::fail(MB200_E_CUDA, "%s: %s", #expr, cudaGetErrorString(e__)); \
  } while (0)

// ---- launch log (mb200_debug_launch_log): which attention / GEMM / MoE / speculative kernel each call chose --------
// Off unless switched on: one thread-local flag test per launch.  One line per launch, named like the kernel with its template
// arguments ("attn_decode_tma_kernel<8>", "gemm_wgmma_kernel<0, 1, 32, 64>").
constexpr size_t kLaunchLogBytes = 16384;
extern thread_local bool g_launch_log_on;
extern thread_local bool g_launch_log_overflow;
extern thread_local size_t g_launch_log_len;
extern thread_local char g_launch_log[kLaunchLogBytes];
inline void note_launch(const char* fmt, ...) {
  if (!g_launch_log_on) return;
  char line[128];
  va_list ap;
  va_start(ap, fmt);
  const int n = vsnprintf(line, sizeof(line), fmt, ap);
  va_end(ap);
  if (n < 0 || n >= (int)sizeof(line) || g_launch_log_len + n + 2 > kLaunchLogBytes) {
    g_launch_log_overflow = true;
    return;
  }
  snprintf(g_launch_log + g_launch_log_len, kLaunchLogBytes - g_launch_log_len, "%s\n", line);
  g_launch_log_len += n + 1;
}

typedef __nv_bfloat16 bf16;

constexpr int kHeadDim = 128;
constexpr float kLog2e = 1.4426950408889634f;  // softmax runs in the exp2 domain

// ---- bf16 <-> fp32 ---------------------------------------------------------------------------
// A bf16 is the top half of an fp32: widening is a shift, exact.
__device__ __forceinline__ float bf16lo(uint32_t packed) { return __uint_as_float(packed << 16); }
__device__ __forceinline__ float bf16hi(uint32_t packed) { return __uint_as_float(packed & 0xffff0000u); }
// round-to-nearest-even, like every `.to(bfloat16)` rounding point in the reference
__device__ __forceinline__ float round_bf16(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }
__device__ __forceinline__ uint16_t bf16_bits(float x) { return __bfloat16_as_ushort(__float2bfloat16_rn(x)); }
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  return (uint32_t)bf16_bits(lo) | ((uint32_t)bf16_bits(hi) << 16);
}
__device__ __forceinline__ float bf16_to_float(uint16_t b) { return __uint_as_float(((uint32_t)b) << 16); }

// ---- e4m3 -> fp32, exactly ----------------------------------------------------------------------
// Two e4m3 bytes (low byte first) -> their values: cvt.rn.f16x2.e4m3x2 is exact (every e4m3 value is an f16 value) and so is f16 ->
// f32 -- three instructions per pair, no rounding.  Every e4m3 value is also a bf16 value, so a bf16 pack of the result is exact too.
__device__ __forceinline__ float2 e4m3x2_to_float2(uint32_t two) {
  const __half2_raw h = __nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)(two & 0xffffu), __NV_E4M3);
  return __half22float2(*reinterpret_cast<const __half2*>(&h));
}

// ---- memory ----------------------------------------------------------------------------------
// streaming 16-byte load that does not pollute L1 (weights / KV rows are read exactly once per step)
__device__ __forceinline__ uint4 ldg_stream16(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}

// ---- reductions --------------------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Argmax key of logit v at index idx: the maximum over a row's keys is torch.argmax's answer on every fp32 input
// (generate.py:156).  High word: an order-preserving map of the value, with -0.0 equal to +0.0 and every NaN one key above +inf
// (torch treats NaN as the maximum); low word: ~index, so among equal values the smallest index wins.  Shared by the sampling
// kernels and the megakernel's fused lm-head argmax, which must agree.
__device__ __forceinline__ unsigned long long argmax_key(float v, int idx) {
  unsigned u = __float_as_uint(v);
  if (v != v)
    u = 0x7f800001u;
  else if (v == 0.f)
    u = 0u;
  u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
  return ((unsigned long long)u << 32) | (unsigned)(0x7fffffff - idx);
}

// Reference numerics helpers ---------------------------------------------------------------------
// rsqrt as torch's CPU kernel does it: 1 / sqrt(x), both IEEE-rounded (not the 2-ulp rsqrt.approx)
__device__ __forceinline__ float ref_rsqrt(float x) { return __fdiv_rn(1.0f, __fsqrt_rn(x)); }
// silu in fp32: x / (1 + exp(-x))  (transformer_layers.py:106 via nn.functional.silu on bf16 -> fp32 internally)
__device__ __forceinline__ float ref_silu(float x) { return __fdiv_rn(x, 1.0f + expf(-x)); }
// exact-erf GELU in fp32 on a bf16 input, as nn.GELU() computes it: x * 0.5 * (1 + erf(x / sqrt(2)))
__device__ __forceinline__ float ref_gelu(float x) { return __fmul_rn(__fmul_rn(x, 0.5f), __fadd_rn(1.0f, erff(__fmul_rn(x, 0.70710678118654752f)))); }
// complex multiply without FMA contraction, as torch's complex kernel computes it (rope.py:21-22)
__device__ __forceinline__ void ref_cmul(float a, float b, float c, float d, float& re, float& im) {
  re = __fsub_rn(__fmul_rn(a, c), __fmul_rn(b, d));
  im = __fadd_rn(__fmul_rn(a, d), __fmul_rn(b, c));
}

inline int ceil_div(int64_t a, int64_t b) { return (int)((a + b - 1) / b); }

// ---- programmatic dependent launch (PDL) --------------------------------------------------------------------------------------
// The decode step of a batch is ~7 short kernels per layer, each preceded by launch latency and a pipeline fill and followed by
// a drain: measured 10-20 us of fixed cost per weight-streaming GEMM at Nemo-12B shapes, a third of the step.  Kernels launched
// through launch_pdl() may start while their predecessor in the stream is still running: everything up to pdl_wait() -- barrier
// init, tensor-map prefetch and, in the GEMMs, the first ring of WEIGHT tiles, which no kernel ever writes --
// overlaps the predecessor's tail.  pdl_wait() returns once the predecessor grid has completed and its writes are visible (and,
// transitively, everything before it).  A kernel signals with pdl_trigger() that its dependents may be scheduled; the hardware
// launches them only when EVERY CTA of this grid has triggered or exited, i.e. when this grid no longer needs SM resources.
// Both are no-ops in a kernel launched the ordinary way.  MB200_PDL=0 launches everything the ordinary way.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

inline bool pdl_enabled() {
  static int on = -1;
  if (on < 0) {
    const char* e = getenv("MB200_PDL");
    on = (e != nullptr && e[0] == '0') ? 0 : 1;
  }
  return on != 0;
}

template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}

}  // namespace mb200
