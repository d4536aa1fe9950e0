// libmb200.so -- the C ABI declared in include/mistral_b200.h.  Argument checking + kernel dispatch only.
#include <cmath>
#include <cstdlib>
#include <cstring>

#include "attn_decode_tma.cuh"
#include "attn_full_hd64.cuh"
#include "attn_prefill.cuh"
#include "attn_prefill_wgmma.cuh"
#include "decode_megakernel.cuh"
#include "elementwise.cuh"
#include "gemm_mma.cuh"
#include "gemm_streamk.cuh"
#include "gemm_wgmma.cuh"
#include "gemm_wgmma_a8.cuh"
#include "int4.cuh"
#include "kv_fp8.cuh"
#include "lora.cuh"
#include "moe.cuh"
#include "sampling.cuh"
#include "skinny_linear.cuh"
#include "speculative.cuh"
#include "vision.cuh"
#include "workspace.cuh"

namespace mb200 {
thread_local char g_err[512] = "";
thread_local bool g_launch_log_on = false;
thread_local bool g_launch_log_overflow = false;
thread_local size_t g_launch_log_len = 0;
thread_local char g_launch_log[kLaunchLogBytes] = "";
static unsigned long long* g_mk_prof = nullptr;
static unsigned long long* g_mk_prof_bar = nullptr;  // debug: decode megakernel phase timeline buffer (device)

static_assert(MK_BAR_WORDS * 128 <= kWsMkBarFlags.bytes, "one grid-barrier counter per 128-byte line");

// Every shape rule of mb200_decode_step and its shared-memory plan, for a device with `smem_max` bytes of opt-in shared memory
// per block.  mb200_decode_step_supported exposes the same function, so a caller learns before launching whether the step runs.
struct DecodePlan {
  int rep, n_stages;
  size_t xs_bytes, smem;
};
static int decode_plan(int64_t dim, int64_t hidden, int64_t n_heads, int64_t n_kv_heads, int64_t head_dim, int64_t vocab, int64_t n_experts,
                       int64_t top_k, int64_t smem_max, DecodePlan* out, bool w8 = false) {
  MB_CHECK_ARG(head_dim == kHeadDim, "decode_step: head_dim=%lld unsupported (128 only)", (long long)head_dim);
  MB_CHECK_ARG(dim > 0 && hidden > 0 && n_kv_heads >= 1 && n_heads % n_kv_heads == 0, "decode_step: H %% KV != 0");
  const int64_t rep = n_heads / n_kv_heads;
  MB_CHECK_ARG(rep == 1 || rep == 2 || rep == 4 || rep == 6 || rep == 8, "decode_step: H/KV=%lld unsupported (1,2,4,6,8)", (long long)rep);
  MB_CHECK_ARG(n_kv_heads <= MK_CONSUMER_WARPS, "decode_step: n_kv_heads=%lld > %d (one consumer warp per kv head)", (long long)n_kv_heads,
               MK_CONSUMER_WARPS);
  MB_CHECK_ARG(n_kv_heads * kHeadDim * 2 + MK_KV_PAD <= MK_STAGE_BYTES / 8, "decode_step: a ring stage must hold 8 padded K/V position rows");
  const int64_t q_dim = n_heads * head_dim;
  auto cut_ok = [](int64_t K) { const int64_t nch = (K + MK_MAX_KC - 1) / MK_MAX_KC; return K % (nch * 8) == 0; };
  MB_CHECK_ARG(cut_ok(dim) && cut_ok(hidden) && cut_ok(q_dim), "decode_step: dim/hidden/q_dim must split into 16-byte-aligned row chunks");
  // e4m3 layer matrices (cut_matrix with w8): chunks of up to MK_MAX_KC8 bytes, 16-byte aligned
  auto cut8_ok = [](int64_t K) { const int64_t nch = (K + MK_MAX_KC8 - 1) / MK_MAX_KC8; return K % (nch * 16) == 0; };
  MB_CHECK_ARG(!w8 || (cut8_ok(dim) && cut8_ok(hidden) && cut8_ok(q_dim)), "decode_step (fp8): dim/hidden/q_dim must split into 16-byte row chunks");
  MB_CHECK_ARG(!w8 || n_experts == 0, "decode_step (fp8): dense models only");
  MB_CHECK_ARG(vocab > 0 && vocab % 2 == 0, "decode_step: vocab must be even");
  MB_CHECK_ARG(n_experts == 0 || (top_k >= 1 && top_k <= MK_MAX_TOPK && top_k <= n_experts && n_experts <= 32),
               "decode_step: bad MoE arguments (E=%lld, k=%lld)", (long long)n_experts, (long long)top_k);
  // shared memory plan: x buffer (also the attention merge scratch), barriers + reduction scratch, the rest is the ring
  int64_t widest = dim > hidden ? dim : hidden;
  if (q_dim > widest) widest = q_dim;
  size_t xs_bytes = (size_t)widest * 2;
  if (n_experts && xs_bytes < (size_t)top_k * hidden * 2) xs_bytes = (size_t)top_k * hidden * 2;  // g of every selected expert
  if (xs_bytes < 2048) xs_bytes = 2048;  // also the slice-merge scratch of phase 2b
  xs_bytes = (xs_bytes + 127) & ~(size_t)127;
  const size_t tail = 2 * MK_MAX_STAGES * sizeof(uint64_t) + 48 * sizeof(float) + sizeof(MoeRoute) + 8 + 64;
  const int64_t room = smem_max - (int64_t)(xs_bytes + tail);
  int n_stages = room > 0 ? (int)(room / MK_STAGE_BYTES) : 0;
  if (n_stages > MK_MAX_STAGES) n_stages = MK_MAX_STAGES;
  MB_CHECK_ARG(n_stages > MK_CONSUMER_WARPS, "decode_step: not enough shared memory for the weight ring (%d stages, %zu B of activations)",
               n_stages, xs_bytes);
  out->rep = (int)rep;
  out->n_stages = n_stages;
  out->xs_bytes = xs_bytes;
  out->smem = (size_t)n_stages * MK_STAGE_BYTES + xs_bytes + tail;
  return MB200_OK;
}

static int run_rmsnorm(const void* x, const void* w, void* out, int64_t T, int64_t dim, float eps, cudaStream_t st) {
  MB_CHECK_ARG(dim % 8 == 0 && T >= 0, "rmsnorm: dim=%lld must be a multiple of 8", (long long)dim);
  if (T == 0) return MB200_OK;
  MB_CHECK_CUDA(launch_pdl(rmsnorm_kernel, dim3((unsigned)T), dim3(256), 0, st, (const uint4*)x, (const uint4*)w, (uint4*)out, (int)dim, eps));
  return MB200_OK;
}

template <int MODE>
static int run_linear(const void* x, const void* norm_w, const void* w, const EpiParams& epi, int64_t T, int64_t N, int64_t K, float eps,
                      void* workspace, size_t workspace_bytes, cudaStream_t st) {
  MB_CHECK_ARG(T >= 1, "linear: T=%lld", (long long)T);
  if (T <= MB200_SKINNY_MAX_T) {
    SkinnyParams p;
    p.x = x;
    p.norm_w = norm_w;
    p.w = w;
    p.N = (int)N;
    p.K = (int)K;
    p.eps = eps;
    p.epi = epi;
    return norm_w ? launch_skinny<MODE, true>(p, (int)T, st) : launch_skinny<MODE, false>(p, (int)T, st);
  }
  const void* a = x;
  if (norm_w) {
    const WsRegion nr = ws_normed(T, K);
    if (workspace == nullptr || workspace_bytes < nr.end()) return fail(MB200_E_WORKSPACE, "linear: workspace %zu < %zu", workspace_bytes, nr.end());
    void* normed = (uint8_t*)workspace + nr.offset;
    int rc = run_rmsnorm(x, norm_w, normed, T, K, eps, st);
    if (rc) return rc;
    a = normed;
  }
  GemmParams g;
  g.a = a;
  g.w = w;
  g.T = (int)T;
  g.N = (int)N;
  g.K = (int)K;
  g.epi = epi;
  if (streamk_eligible(T, N, K)) return launch_streamk<MODE>(g, workspace, workspace_bytes, st);  // decode-sized batches: HBM-bound
  if (wgmma_gemm_eligible(T, N, K)) return launch_gemm_wgmma<MODE>(g, st);
  return launch_gemm_mma<MODE>(g, st);
}

// Quantised dense weights (include/mistral_b200.h): the bf16 dispatch of run_linear, except that a shape it would give to
// gemm_mma_kernel is refused (that kernel has no quantised variant).  One function for both formats, so the regime choice lives here
// once.  FP8 (INT4 = false): w is e4m3 [N, K], epi.w_scale its fp32 row scales, applied by the epilogue (EPI_WSCALE).  INT4: w is
// the packed code matrix [N, K/2], gscale its bf16 group scales [N, K/128]; the kernels convert to W' and keep the bf16 epilogue.
// A8 (FP8 only): the calls that would run the prefill wgmma kernel (T >= 128, not stream-K) quantise their input per token into the
// workspace and run the e4m3 x e4m3 kernel instead; every other call is the FP8 call unchanged.
template <int MODE, bool INT4, bool A8 = false>
static int run_linear_quant(const void* x, const void* norm_w, const void* w, const uint16_t* gscale, const EpiParams& epi, int64_t T,
                            int64_t N, int64_t K, float eps, void* workspace, size_t workspace_bytes, cudaStream_t st) {
  static_assert(!(A8 && INT4), "FP8 activations: FP8 weights only");
  const char* fmt = INT4 ? "int4" : "fp8";
  constexpr int KMODE = INT4 ? MODE : (MODE | EPI_WSCALE);  // the kernels' epilogue mode
  MB_CHECK_ARG(T >= 1, "linear (%s): T=%lld", fmt, (long long)T);
  if constexpr (INT4) {
    MB_CHECK_ARG(gscale != nullptr && ((uintptr_t)gscale & 1) == 0 && ((uintptr_t)w & 15) == 0, "linear (int4): misaligned or null weights");
    MB_CHECK_ARG(K % kInt4Group == 0, "linear (int4): K=%lld must be a multiple of 128", (long long)K);
  } else {
    MB_CHECK_ARG(epi.w_scale != nullptr && ((uintptr_t)epi.w_scale & 7) == 0, "linear (fp8): w_scale must be an 8-byte aligned fp32 array");
  }
  if (T <= MB200_SKINNY_MAX_T) {
    SkinnyParams p;
    p.x = x;
    p.norm_w = norm_w;
    p.w = w;
    p.N = (int)N;
    p.K = (int)K;
    p.eps = eps;
    p.epi = epi;
    if constexpr (INT4) {
      p.gscale = gscale;
      // attn_qkv always norms its input: no un-normed QKV instantiation (it would spill 8 bytes at T = 4)
      if constexpr (MODE == EPI_QKV_ROPE) return launch_skinny_int4<KMODE, true>(p, (int)T, st);
      else return norm_w ? launch_skinny_int4<KMODE, true>(p, (int)T, st) : launch_skinny_int4<KMODE, false>(p, (int)T, st);
    } else {
      return norm_w ? launch_skinny_fp8<KMODE, true>(p, (int)T, st) : launch_skinny_fp8<KMODE, false>(p, (int)T, st);
    }
  }
  const bool sk = streamk_eligible(T, N, K);
  MB_CHECK_ARG(sk || wgmma_gemm_eligible(T, N, K), "linear (%s): T=%lld N=%lld K=%lld needs the mma.sync GEMM, which has no %s variant", fmt,
               (long long)T, (long long)N, (long long)K, INT4 ? "int4" : "e4m3");
  if constexpr (A8) {
    if (!sk && T >= A8_BM) {
      MB_CHECK_ARG(a8_gemm_eligible(T, N, K), "linear (fp8 activations): N=%lld K=%lld (K must be a multiple of 128 and N of 64)", (long long)N,
                   (long long)K);
      const WsActE4m3 r = ws_act_e4m3(T, K);
      if (workspace == nullptr || workspace_bytes < r.exps.end())
        return fail(MB200_E_WORKSPACE, "linear: workspace %zu < %zu", workspace_bytes, r.exps.end());
      uint8_t* xq = (uint8_t*)workspace + r.q.offset;
      int32_t* exps = (int32_t*)((uint8_t*)workspace + r.exps.offset);
      int rc = launch_quantize_act(x, norm_w, xq, exps, T, K, eps, st);
      if (rc) return rc;
      GemmParams g;
      g.a = xq;
      g.w = w;
      g.T = (int)T;
      g.N = (int)N;
      g.K = (int)K;
      g.epi = epi;
      return launch_gemm_wgmma_a8<KMODE | EPI_ASCALE>(g, exps, st);
    }
  }
  const void* a = x;
  if (norm_w) {
    const WsRegion nr = ws_normed(T, K);
    if (workspace == nullptr || workspace_bytes < nr.end()) return fail(MB200_E_WORKSPACE, "linear: workspace %zu < %zu", workspace_bytes, nr.end());
    void* normed = (uint8_t*)workspace + nr.offset;
    int rc = run_rmsnorm(x, norm_w, normed, T, K, eps, st);
    if (rc) return rc;
    a = normed;
  }
  GemmParams g;
  g.a = a;
  g.w = w;
  g.T = (int)T;
  g.N = (int)N;
  g.K = (int)K;
  g.epi = epi;
  if constexpr (INT4) {
    if (sk) return launch_streamk_int4<KMODE>(g, gscale, workspace, workspace_bytes, st);
    return launch_gemm_wgmma_int4<KMODE>(g, gscale, st);
  } else {
    if (sk) return launch_streamk_fp8<KMODE>(g, workspace, workspace_bytes, st);
    return launch_gemm_wgmma_fp8<KMODE>(g, st);
  }
}

// Un-merged LoRA around one fused Linear (include/mistral_b200.h): down projection -> up projection -> base GEMM whose epilogue
// adds bf16(l * scaling) before the mode's work.  With row_slot (a bank of adapter slots) the down projection masks each row to its
// slot's columns; the up projection and the base GEMM are the same kernels, so the call has the same launches.  For T > MB200_SKINNY_MAX_T the input is normed once into the workspace and both
// the down kernel and the base GEMM read it; for T <= MB200_SKINNY_MAX_T both are weight-streaming GEMVs that norm in-kernel.
template <int MODE>
static int run_linear_lora(const void* x, const void* norm_w, const void* w, EpiParams epi, const mb200_lora* lora, int64_t T, int64_t N,
                           int64_t K, float eps, void* workspace, size_t workspace_bytes, cudaStream_t st) {
  MB_CHECK_ARG(lora && lora->a_w && lora->b_w && lora->a_buf && lora->l_buf, "lora: null pointer");
  const int64_t R = lora->rank_cols;
  MB_CHECK_ARG(R >= 64 && R % 64 == 0 && K % 64 == 0, "lora: rank_cols=%lld and K=%lld must be multiples of 64", (long long)R, (long long)K);
  MB_CHECK_ARG(T >= 1, "lora: T=%lld", (long long)T);
  const int64_t Rc = lora->slot_cols;
  MB_CHECK_ARG(lora->row_slot == nullptr || (Rc >= 64 && Rc % 64 == 0 && R % Rc == 0),
               "lora: slot_cols=%lld must be a multiple of 64 that divides rank_cols=%lld", (long long)Rc, (long long)R);
  MB_CHECK_ARG(((uintptr_t)lora->a_buf & 15) == 0 && ((uintptr_t)lora->l_buf & 15) == 0,
               "lora: a_buf and l_buf must be 16-byte aligned (l_buf doubles as fp32 split-K scratch)");
  const void* xn = x;
  int rc;
  if (T <= MB200_SKINNY_MAX_T) {
    SkinnyParams p;
    p.x = x;
    p.norm_w = norm_w;
    p.w = lora->a_w;
    p.N = (int)R;
    p.K = (int)K;
    p.eps = eps;
    p.epi.out = lora->a_buf;
    p.epi.ld_out = R;
    if (lora->row_slot != nullptr) {
      p.row_slot = lora->row_slot;
      p.slot_cols = (int)Rc;
      constexpr int M = EPI_STORE | SKINNY_SLOT_MASK;
      rc = norm_w ? launch_skinny<M, true>(p, (int)T, st) : launch_skinny<M, false>(p, (int)T, st);
    } else {
      rc = norm_w ? launch_skinny<EPI_STORE, true>(p, (int)T, st) : launch_skinny<EPI_STORE, false>(p, (int)T, st);
    }
  } else {
    if (norm_w) {
      const WsRegion nr = ws_normed(T, K);
      if (workspace == nullptr || workspace_bytes < nr.end()) return fail(MB200_E_WORKSPACE, "linear: workspace %zu < %zu", workspace_bytes, nr.end());
      void* normed = (uint8_t*)workspace + nr.offset;
      rc = run_rmsnorm(x, norm_w, normed, T, K, eps, st);
      if (rc) return rc;
      xn = normed;
      norm_w = nullptr;
    }
    rc = launch_lora_down(xn, lora->a_w, lora->a_buf, T, R, K, lora->l_buf, (size_t)T * N * 2, st, lora->row_slot, Rc);
  }
  if (rc) return rc;
  EpiParams up;
  up.out = lora->l_buf;
  up.ld_out = N;
  rc = run_linear<EPI_STORE>(lora->a_buf, nullptr, lora->b_w, up, T, N, R, 0.f, workspace, workspace_bytes, st);
  if (rc) return rc;
  epi.lora_l = lora->l_buf;
  epi.ld_lora = N;
  epi.lora_scaling = lora->scaling;
  return run_linear<MODE | EPI_LORA>(xn, norm_w, w, epi, T, N, K, eps, workspace, workspace_bytes, st);
}
}  // namespace mb200

using namespace mb200;

extern "C" {

int mb200_abi_version(void) { return MB200_ABI_VERSION; }
const char* mb200_last_error(void) { return g_err; }

int mb200_device_info(int* sm_count, int* max_smem_optin) {
  int dev = 0;
  MB_CHECK_CUDA(cudaGetDevice(&dev));
  if (sm_count) MB_CHECK_CUDA(cudaDeviceGetAttribute(sm_count, cudaDevAttrMultiProcessorCount, dev));
  if (max_smem_optin) MB_CHECK_CUDA(cudaDeviceGetAttribute(max_smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  return MB200_OK;
}

size_t mb200_workspace_bytes(int64_t T, int64_t dim, int64_t n_heads, int64_t n_kv_heads, int64_t head_dim, int64_t hidden, int64_t vocab,
                             int64_t max_batch) {
  (void)vocab;
  (void)head_dim;
  const int64_t widest = dim > hidden ? dim : hidden;
  const int64_t rep = n_kv_heads > 0 ? n_heads / n_kv_heads : 1;
  // stream-K partial slots + normed activations, then room for the split-KV partials (n_splits <= 64) on top
  const size_t s = ws_normed(T, widest).end() + align256(ws_splitkv_partials(max_batch, n_kv_heads, 64, rep).bytes);
  // decode_step scratch for any MoE top-k and up to 256 SMs worth of attention slices
  const size_t mk = decode_scratch(dim, hidden, n_heads, 1, MK_MAX_TOPK, 256).end;
  return s > mk ? s : mk;
}

int mb200_rmsnorm(const void* x, const void* w, void* out, int64_t T, int64_t dim, float eps, void* stream) {
  MB_CHECK_ARG(x && w && out, "rmsnorm: null pointer");
  return run_rmsnorm(x, w, out, T, dim, eps, (cudaStream_t)stream);
}

static int attn_qkv_impl(const void* x, const void* norm_w, const void* wqkv, const float* rope, const int32_t* positions, void* q_out,
                         void* k_out, void* v_out, void* cache_k, void* cache_v, const int32_t* cache_rows, int64_t T, int64_t dim,
                         int64_t n_heads, int64_t n_kv_heads, int64_t head_dim, float eps, void* workspace, size_t workspace_bytes,
                         void* stream, const mb200_lora* lora, const float* w_scale = nullptr, const uint16_t* w_gscale = nullptr,
                         bool a8 = false) {
  MB_CHECK_ARG(x && norm_w && wqkv && rope && positions && q_out && k_out && v_out, "attn_qkv: null pointer");
  MB_CHECK_ARG(head_dim == kHeadDim || head_dim == 64, "attn_qkv: head_dim=%lld unsupported (64 or 128)", (long long)head_dim);
  MB_CHECK_ARG(cache_rows == nullptr || (cache_k && cache_v), "attn_qkv: cache_rows without cache pointers");
  EpiParams e;
  e.q_out = q_out;
  e.k_out = k_out;
  e.v_out = v_out;
  e.cache_k = cache_k;
  e.cache_v = cache_v;
  e.positions = positions;
  e.cache_rows = cache_rows;
  e.rope = rope;
  e.q_dim = (int)(n_heads * head_dim);
  e.kv_dim = (int)(n_kv_heads * head_dim);
  e.head_dim = (int)head_dim;
  const int64_t N = (n_heads + 2 * n_kv_heads) * head_dim;
  if (w_scale) {
    e.w_scale = w_scale;
    if (a8)
      return run_linear_quant<EPI_QKV_ROPE, false, true>(x, norm_w, wqkv, nullptr, e, T, N, dim, eps, workspace, workspace_bytes, (cudaStream_t)stream);
    return run_linear_quant<EPI_QKV_ROPE, false>(x, norm_w, wqkv, nullptr, e, T, N, dim, eps, workspace, workspace_bytes, (cudaStream_t)stream);
  }
  if (w_gscale) return run_linear_quant<EPI_QKV_ROPE, true>(x, norm_w, wqkv, w_gscale, e, T, N, dim, eps, workspace, workspace_bytes,
                                                                 (cudaStream_t)stream);
  if (lora) return run_linear_lora<EPI_QKV_ROPE>(x, norm_w, wqkv, e, lora, T, N, dim, eps, workspace, workspace_bytes, (cudaStream_t)stream);
  return run_linear<EPI_QKV_ROPE>(x, norm_w, wqkv, e, T, N, dim, eps, workspace, workspace_bytes, (cudaStream_t)stream);
}

int mb200_attn_qkv(const void* x, const void* norm_w, const void* wqkv, const float* rope, const int32_t* positions, void* q_out, void* k_out,
                   void* v_out, void* cache_k, void* cache_v, const int32_t* cache_rows, int64_t T, int64_t dim, int64_t n_heads,
                   int64_t n_kv_heads, int64_t head_dim, float eps, void* workspace, size_t workspace_bytes, void* stream) {
  return attn_qkv_impl(x, norm_w, wqkv, rope, positions, q_out, k_out, v_out, cache_k, cache_v, cache_rows, T, dim, n_heads, n_kv_heads,
                       head_dim, eps, workspace, workspace_bytes, stream, nullptr);
}

int mb200_attn_qkv_lora(const void* x, const void* norm_w, const void* wqkv, const float* rope, const int32_t* positions, void* q_out,
                        void* k_out, void* v_out, void* cache_k, void* cache_v, const int32_t* cache_rows, int64_t T, int64_t dim,
                        int64_t n_heads, int64_t n_kv_heads, int64_t head_dim, float eps, void* workspace, size_t workspace_bytes,
                        void* stream, const mb200_lora* lora) {
  MB_CHECK_ARG(lora, "attn_qkv_lora: null adapter");
  return attn_qkv_impl(x, norm_w, wqkv, rope, positions, q_out, k_out, v_out, cache_k, cache_v, cache_rows, T, dim, n_heads, n_kv_heads,
                       head_dim, eps, workspace, workspace_bytes, stream, lora);
}

int mb200_decode_meta(int32_t* seqpos_dev, int32_t* meta_dev, int64_t B, const int32_t* windows_host, int64_t n_windows, void* stream) {
  MB_CHECK_ARG(seqpos_dev && meta_dev && windows_host, "decode_meta: null pointer");
  MB_CHECK_ARG(B >= 1 && n_windows >= 1 && n_windows <= kMaxWindows, "decode_meta: B=%lld, n_windows=%lld (max %d)", (long long)B,
               (long long)n_windows, kMaxWindows);
  DecodeMetaParams p;
  p.seqpos = seqpos_dev;
  p.meta = meta_dev;
  p.B = (int)B;
  p.n_w = (int)n_windows;
  for (int j = 0; j < (int)n_windows; ++j) {
    MB_CHECK_ARG(windows_host[j] >= 1, "decode_meta: window %d", (int)windows_host[j]);
    p.windows[j] = windows_host[j];
  }
  decode_meta_kernel<<<(unsigned)ceil_div(B + 1, 128), 128, 0, (cudaStream_t)stream>>>(p);
  MB_CHECK_LAUNCH("decode_meta_kernel");
  return MB200_OK;
}

int mb200_spec_meta(const int32_t* seqpos_dev, int32_t* meta_dev, int64_t B, int64_t S, const int32_t* windows_host, int64_t n_windows,
                    void* stream) {
  MB_CHECK_ARG(seqpos_dev && meta_dev && windows_host, "spec_meta: null pointer");
  MB_CHECK_ARG(B >= 1 && S >= 1 && B * S <= (1 << 24) && n_windows >= 1 && n_windows <= kMaxWindows,
               "spec_meta: B=%lld, S=%lld, n_windows=%lld (max %d)", (long long)B, (long long)S, (long long)n_windows, kMaxWindows);
  SpecMetaParams p;
  p.seqpos = seqpos_dev;
  p.meta = meta_dev;
  p.B = (int)B;
  p.S = (int)S;
  p.n_w = (int)n_windows;
  for (int j = 0; j < (int)n_windows; ++j) {
    MB_CHECK_ARG(windows_host[j] >= 1, "spec_meta: window %d", (int)windows_host[j]);
    p.windows[j] = windows_host[j];
  }
  const int64_t threads = B * S > B + 1 ? B * S : B + 1;
  spec_meta_kernel<<<(unsigned)ceil_div(threads, 128), 128, 0, (cudaStream_t)stream>>>(p);
  note_launch("spec_meta_kernel");
  MB_CHECK_LAUNCH("spec_meta_kernel");
  return MB200_OK;
}

int mb200_spec_accept_greedy(const float* logits, const int64_t* tokens_dev, int64_t* out_dev, int32_t* n_dev, int32_t* seqpos_dev, int64_t B,
                             int64_t S, int64_t vocab, void* stream) {
  MB_CHECK_ARG(logits && tokens_dev && out_dev && n_dev && seqpos_dev, "spec_accept_greedy: null pointer");
  MB_CHECK_ARG(B >= 1 && S >= 2 && vocab >= 1 && vocab <= 0x7fffffff, "spec_accept_greedy: B=%lld S=%lld vocab=%lld", (long long)B, (long long)S,
               (long long)vocab);
  spec_accept_greedy_kernel<<<(unsigned)B, SP_THREADS, 0, (cudaStream_t)stream>>>(logits, (const long long*)tokens_dev, (long long*)out_dev,
                                                                                 n_dev, seqpos_dev, (int)S, (int)vocab);
  note_launch("spec_accept_greedy_kernel");
  MB_CHECK_LAUNCH("spec_accept_greedy_kernel");
  return MB200_OK;
}

int mb200_spec_accept_sample(const float* logits, const float* draft_logits, const int64_t* tokens_dev, const float* uniform_dev, int64_t* out_dev,
                             int32_t* n_dev, int32_t* seqpos_dev, int64_t B, int64_t S, int64_t vocab, float temperature, float top_p,
                             void* stream) {
  MB_CHECK_ARG(logits && draft_logits && tokens_dev && uniform_dev && out_dev && n_dev && seqpos_dev, "spec_accept_sample: null pointer");
  MB_CHECK_ARG(B >= 1 && S >= 2 && vocab >= 1 && vocab <= 0x7fffffff, "spec_accept_sample: B=%lld S=%lld vocab=%lld", (long long)B, (long long)S,
               (long long)vocab);
  MB_CHECK_ARG(temperature > 0.f && top_p >= 0.f && top_p <= 1.f, "spec_accept_sample: temperature=%g must be > 0 and top_p=%g in [0, 1]",
               (double)temperature, (double)top_p);
  spec_accept_sample_kernel<<<(unsigned)B, SP_THREADS, 0, (cudaStream_t)stream>>>(logits, draft_logits, (const long long*)tokens_dev, uniform_dev,
                                                                                 (long long*)out_dev, n_dev, seqpos_dev, (int)S, (int)vocab,
                                                                                 1.0f / temperature, top_p);
  note_launch("spec_accept_sample_kernel");
  MB_CHECK_LAUNCH("spec_accept_sample_kernel");
  return MB200_OK;
}

int mb200_kv_ring_write(const void* k_new, const void* v_new, void* cache_k, void* cache_v, const int32_t* cache_rows, int64_t T,
                        int64_t n_kv_heads, int64_t head_dim, void* stream) {
  MB_CHECK_ARG(k_new && v_new && cache_k && cache_v && cache_rows, "kv_ring_write: null pointer");
  MB_CHECK_ARG((n_kv_heads * head_dim) % 8 == 0, "kv_ring_write: row not 16-byte aligned");
  if (T == 0) return MB200_OK;
  kv_ring_write_kernel<<<(unsigned)T, 128, 0, (cudaStream_t)stream>>>((const uint4*)k_new, (const uint4*)v_new, (uint4*)cache_k, (uint4*)cache_v,
                                                                      cache_rows, (int)T, (int)(n_kv_heads * head_dim / 8));
  MB_CHECK_LAUNCH("kv_ring_write_kernel");
  return MB200_OK;
}

int mb200_attn_decode(const void* q, const void* cache_k, const void* cache_v, const int32_t* kv_len, void* out, int64_t B, int64_t W,
                      int64_t n_heads, int64_t n_kv_heads, int64_t head_dim, int64_t n_splits, void* workspace, size_t workspace_bytes,
                      void* stream) {
  MB_CHECK_ARG(q && cache_k && cache_v && kv_len && out, "attn_decode: null pointer");
  MB_CHECK_ARG(head_dim == kHeadDim, "attn_decode: head_dim=%lld unsupported (128 only)", (long long)head_dim);
  MB_CHECK_ARG(n_heads % n_kv_heads == 0, "attn_decode: H %% KV != 0");
  const int rep = (int)(n_heads / n_kv_heads);
  MB_CHECK_ARG(n_splits >= 1 && n_splits <= 64, "attn_decode: n_splits=%lld out of [1, 64]", (long long)n_splits);
  MB_CHECK_ARG((size_t)B * n_kv_heads * sizeof(int) <= kWsSplitKvCounters.bytes, "attn_decode: B*KV too large for the counter block");
  AttnDecodeParams p;
  p.q = (const bf16*)q;
  p.cache_k = (const bf16*)cache_k;
  p.cache_v = (const bf16*)cache_v;
  p.kv_len = kv_len;
  p.out = (bf16*)out;
  p.B = (int)B;
  p.W = (int)W;
  p.H = (int)n_heads;
  p.KV = (int)n_kv_heads;
  p.S = (int)n_splits;
  p.scale = 0.08838834764831845f;  // 128^-0.5 (xformers default scale; Attention.scale is unused, SURVEY E-3)
  p.partial = nullptr;
  p.counters = nullptr;
  if (n_splits > 1) {
    const WsRegion pr = ws_splitkv_partials(B, n_kv_heads, n_splits, rep);
    if (workspace == nullptr || workspace_bytes < pr.end()) return fail(MB200_E_WORKSPACE, "attn_decode: workspace %zu < %zu", workspace_bytes, pr.end());
    p.counters = (int*)((uint8_t*)workspace + kWsSplitKvCounters.offset);
    p.partial = (float*)((uint8_t*)workspace + pr.offset);
  }
  cudaStream_t st = (cudaStream_t)stream;
  switch (rep) {
    case 1: return launch_attn_decode_tma<1>(p, B * W, st);
    case 2: return launch_attn_decode_tma<2>(p, B * W, st);
    case 4: return launch_attn_decode_tma<4>(p, B * W, st);
    case 6: return launch_attn_decode_tma<6>(p, B * W, st);
    case 8: return launch_attn_decode_tma<8>(p, B * W, st);
    case 12: return launch_attn_decode_tma<12>(p, B * W, st);
    default: return fail(MB200_E_INVALID, "attn_decode: H/KV=%d unsupported (1,2,4,6,8,12)", rep);
  }
}

int mb200_debug_attn_decode_occupancy(int64_t rep, int* blocks_per_sm) {
  MB_CHECK_ARG(blocks_per_sm, "debug_attn_decode_occupancy: null pointer");
  const void* fn = nullptr;
  switch (rep) {
    case 1: fn = (const void*)attn_decode_tma_kernel<1>; break;
    case 2: fn = (const void*)attn_decode_tma_kernel<2>; break;
    case 4: fn = (const void*)attn_decode_tma_kernel<4>; break;
    case 6: fn = (const void*)attn_decode_tma_kernel<6>; break;
    case 8: fn = (const void*)attn_decode_tma_kernel<8>; break;
    case 12: fn = (const void*)attn_decode_tma_kernel<12>; break;
    default: return fail(MB200_E_INVALID, "debug_attn_decode_occupancy: H/KV=%lld not compiled", (long long)rep);
  }
  MB_CHECK_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, ADT_SMEM));
  MB_CHECK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(blocks_per_sm, fn, ADT_THREADS, ADT_SMEM));
  return MB200_OK;
}

int mb200_attn_prefill(const void* q, const void* k_new, const void* v_new, const void* cache_k, const void* cache_v, const int32_t* q_start,
                       const int32_t* seqpos, void* out, int64_t T, int64_t B, int64_t max_seqlen, int64_t W, int64_t n_heads,
                       int64_t n_kv_heads, int64_t head_dim, int causal, void* stream) {
  MB_CHECK_ARG(q && k_new && v_new && out, "attn_prefill: null pointer");
  MB_CHECK_ARG(!causal || (cache_k && cache_v && q_start && seqpos), "attn_prefill: causal mode needs ring + metadata");
  MB_CHECK_ARG(head_dim == kHeadDim || head_dim == 64, "attn_prefill: head_dim=%lld unsupported (64 or 128)", (long long)head_dim);
  MB_CHECK_ARG(n_heads % n_kv_heads == 0, "attn_prefill: H %% KV != 0");
  if (head_dim == 64) {  // the vision encoder's attention: cache-less and unmasked only
    MB_CHECK_ARG(causal == 0, "attn_prefill: head_dim=64 supports the cache-less mode (causal=0) only, got causal=%d", causal);
    if (T == 0) return MB200_OK;
    return launch_attn_full_hd64(q, k_new, v_new, out, T, n_heads, n_kv_heads, (cudaStream_t)stream);
  }
  if (T == 0) return MB200_OK;
  if (causal == 2 && wgmma_attn_eligible(T, max_seqlen))  // first prefill: every key comes from the chunk -> wgmma / TMA kernel
    return launch_attn_prefill_wgmma(q, k_new, v_new, q_start, out, T, B, max_seqlen, W, n_heads, n_kv_heads, (cudaStream_t)stream);
  AttnPrefillParams p;
  p.q = (const bf16*)q;
  p.k_new = (const bf16*)k_new;
  p.v_new = (const bf16*)v_new;
  p.cache_k = (const bf16*)cache_k;
  p.cache_v = (const bf16*)cache_v;
  p.q_start = q_start;
  p.seqpos = seqpos;
  p.out = (bf16*)out;
  p.T = (int)T;
  p.B = (int)B;
  p.W = (int)W;
  p.H = (int)n_heads;
  p.KV = (int)n_kv_heads;
  p.causal = causal;
  p.scale_log2 = 0.08838834764831845f * 1.4426950408889634f;
  const int64_t span = causal ? max_seqlen : T;
  const dim3 grid((unsigned)ceil_div(span, AP_BQ), (unsigned)n_heads, (unsigned)(causal ? B : 1));
  MB_CHECK_CUDA(cudaFuncSetAttribute(attn_prefill_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, AP_SMEM));
  attn_prefill_kernel<<<grid, AP_THREADS, AP_SMEM, (cudaStream_t)stream>>>(p);
  note_launch("attn_prefill_kernel");
  MB_CHECK_LAUNCH("attn_prefill_kernel");
  return MB200_OK;
}

int mb200_kv_quantize(void* k, void* v, int write_back, void* cache_k, void* cache_v, int8_t* exp_k, int8_t* exp_v, const int32_t* cache_rows,
                      int64_t T, int64_t n_kv_heads, int64_t head_dim, void* stream) {
  MB_CHECK_ARG(k && v, "kv_quantize: null pointer");
  MB_CHECK_ARG(head_dim == kHeadDim, "kv_quantize: head_dim=%lld unsupported (128 only)", (long long)head_dim);
  MB_CHECK_ARG(cache_rows == nullptr || (cache_k && cache_v && exp_k && exp_v), "kv_quantize: cache_rows without ring pointers");
  MB_CHECK_ARG(T >= 0 && n_kv_heads >= 1 && T * n_kv_heads * 2 <= 0x7fffffff, "kv_quantize: T=%lld KV=%lld", (long long)T, (long long)n_kv_heads);
  MB_CHECK_ARG(((uintptr_t)k & 7) == 0 && ((uintptr_t)v & 7) == 0 && ((uintptr_t)cache_k & 3) == 0 && ((uintptr_t)cache_v & 3) == 0,
               "kv_quantize: misaligned pointer");
  if (T == 0 || (!write_back && cache_rows == nullptr)) return MB200_OK;
  KvQuantParams p;
  p.k = (bf16*)k;
  p.v = (bf16*)v;
  p.cache_k = (uint8_t*)cache_k;
  p.cache_v = (uint8_t*)cache_v;
  p.exp_k = exp_k;
  p.exp_v = exp_v;
  p.rows = cache_rows;
  p.T = (int)T;
  p.KV = (int)n_kv_heads;
  p.write_back = write_back ? 1 : 0;
  const int64_t warps = T * n_kv_heads * 2;
  MB_CHECK_CUDA(launch_pdl(kv_quantize_kernel, dim3((unsigned)ceil_div(warps, 4)), dim3(128), 0, (cudaStream_t)stream, p));
  note_launch("kv_quantize_kernel");
  return MB200_OK;
}

int mb200_attn_decode_fp8(const void* q, const void* cache_k, const void* cache_v, const int8_t* exp_k, const int8_t* exp_v, const int32_t* kv_len,
                          void* out, int64_t B, int64_t W, int64_t n_heads, int64_t n_kv_heads, int64_t head_dim, int64_t n_splits,
                          void* workspace, size_t workspace_bytes, void* stream) {
  MB_CHECK_ARG(q && cache_k && cache_v && exp_k && exp_v && kv_len && out, "attn_decode_fp8: null pointer");
  MB_CHECK_ARG(head_dim == kHeadDim, "attn_decode_fp8: head_dim=%lld unsupported (128 only)", (long long)head_dim);
  MB_CHECK_ARG(n_kv_heads >= 1 && n_heads % n_kv_heads == 0, "attn_decode_fp8: H %% KV != 0");
  const int rep = (int)(n_heads / n_kv_heads);
  MB_CHECK_ARG(n_splits >= 1 && n_splits <= 64, "attn_decode_fp8: n_splits=%lld out of [1, 64]", (long long)n_splits);
  MB_CHECK_ARG((size_t)B * n_kv_heads * sizeof(int) <= kWsSplitKvCounters.bytes, "attn_decode_fp8: B*KV too large for the counter block");
  AttnDecodeFp8Params fp;
  AttnDecodeParams& p = fp.a;
  p.q = (const bf16*)q;
  p.cache_k = (const bf16*)cache_k;
  p.cache_v = (const bf16*)cache_v;
  p.kv_len = kv_len;
  p.out = (bf16*)out;
  p.B = (int)B;
  p.W = (int)W;
  p.H = (int)n_heads;
  p.KV = (int)n_kv_heads;
  p.S = (int)n_splits;
  p.scale = 0.08838834764831845f;  // as mb200_attn_decode
  p.partial = nullptr;
  p.counters = nullptr;
  fp.exp_k = exp_k;
  fp.exp_v = exp_v;
  if (n_splits > 1) {
    const WsRegion pr = ws_splitkv_partials(B, n_kv_heads, n_splits, rep);
    if (workspace == nullptr || workspace_bytes < pr.end()) return fail(MB200_E_WORKSPACE, "attn_decode_fp8: workspace %zu < %zu", workspace_bytes, pr.end());
    p.counters = (int*)((uint8_t*)workspace + kWsSplitKvCounters.offset);
    p.partial = (float*)((uint8_t*)workspace + pr.offset);
  }
  cudaStream_t st = (cudaStream_t)stream;
  switch (rep) {
    case 1: return launch_attn_decode_tma_fp8<1>(fp, B * W, st);
    case 2: return launch_attn_decode_tma_fp8<2>(fp, B * W, st);
    case 4: return launch_attn_decode_tma_fp8<4>(fp, B * W, st);
    case 6: return launch_attn_decode_tma_fp8<6>(fp, B * W, st);
    case 8: return launch_attn_decode_tma_fp8<8>(fp, B * W, st);
    default: return fail(MB200_E_INVALID, "attn_decode_fp8: H/KV=%d unsupported (1,2,4,6,8)", rep);
  }
}

int mb200_attn_prefill_fp8(const void* q, const void* k_new, const void* v_new, const void* cache_k, const void* cache_v, const int8_t* exp_k,
                           const int8_t* exp_v, const int32_t* q_start, const int32_t* seqpos, void* out, int64_t T, int64_t B, int64_t max_seqlen,
                           int64_t W, int64_t n_heads, int64_t n_kv_heads, int64_t head_dim, int causal, void* stream) {
  MB_CHECK_ARG(causal == 1 || causal == 2, "attn_prefill_fp8: causal=%d (1 or 2; the cache-less forward has no ring)", causal);
  MB_CHECK_ARG(head_dim == kHeadDim, "attn_prefill_fp8: head_dim=%lld unsupported (128 only)", (long long)head_dim);
  MB_CHECK_ARG(exp_k && exp_v, "attn_prefill_fp8: null pointer");
  // first prefill reads no ring row: the bf16 kernels run it on the chunk's k' / v'
  if (causal == 2) return mb200_attn_prefill(q, k_new, v_new, cache_k, cache_v, q_start, seqpos, out, T, B, max_seqlen, W, n_heads, n_kv_heads, head_dim, 2, stream);
  MB_CHECK_ARG(q && k_new && v_new && out && cache_k && cache_v && q_start && seqpos, "attn_prefill_fp8: null pointer");
  MB_CHECK_ARG(n_kv_heads >= 1 && n_heads % n_kv_heads == 0, "attn_prefill_fp8: H %% KV != 0");
  if (T == 0) return MB200_OK;
  AttnPrefillParams p;
  p.q = (const bf16*)q;
  p.k_new = (const bf16*)k_new;
  p.v_new = (const bf16*)v_new;
  p.cache_k = (const bf16*)cache_k;
  p.cache_v = (const bf16*)cache_v;
  p.q_start = q_start;
  p.seqpos = seqpos;
  p.out = (bf16*)out;
  p.T = (int)T;
  p.B = (int)B;
  p.W = (int)W;
  p.H = (int)n_heads;
  p.KV = (int)n_kv_heads;
  p.causal = 1;
  p.scale_log2 = 0.08838834764831845f * 1.4426950408889634f;
  const KvFp8Exps ex{exp_k, exp_v};
  const dim3 grid((unsigned)ceil_div(max_seqlen, AP_BQ), (unsigned)n_heads, (unsigned)B);
  MB_CHECK_CUDA(cudaFuncSetAttribute(attn_prefill_fp8_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, AP_SMEM));
  attn_prefill_fp8_kernel<<<grid, AP_THREADS, AP_SMEM, (cudaStream_t)stream>>>(p, ex);
  note_launch("attn_prefill_fp8_kernel");
  MB_CHECK_LAUNCH("attn_prefill_fp8_kernel");
  return MB200_OK;
}

int mb200_linear_residual(const void* x, const void* w, const void* residual, void* out, int64_t T, int64_t N, int64_t K, void* workspace,
                          size_t workspace_bytes, void* stream) {
  MB_CHECK_ARG(x && w && out, "linear_residual: null pointer");
  EpiParams e;
  e.out = out;
  e.residual = residual;
  e.ld_out = N;
  if (residual) return run_linear<EPI_RESIDUAL>(x, nullptr, w, e, T, N, K, 0.f, workspace, workspace_bytes, (cudaStream_t)stream);
  return run_linear<EPI_STORE>(x, nullptr, w, e, T, N, K, 0.f, workspace, workspace_bytes, (cudaStream_t)stream);
}

int mb200_attn_qkv_fp8(const void* x, const void* norm_w, const void* w_q, const float* w_scale, const float* rope, const int32_t* positions,
                       void* q_out, void* k_out, void* v_out, void* cache_k, void* cache_v, const int32_t* cache_rows, int64_t T, int64_t dim,
                       int64_t n_heads, int64_t n_kv_heads, int64_t head_dim, float eps, void* workspace, size_t workspace_bytes, void* stream) {
  MB_CHECK_ARG(w_scale, "attn_qkv_fp8: null scale");
  return attn_qkv_impl(x, norm_w, w_q, rope, positions, q_out, k_out, v_out, cache_k, cache_v, cache_rows, T, dim, n_heads, n_kv_heads,
                       head_dim, eps, workspace, workspace_bytes, stream, nullptr, w_scale);
}

int mb200_linear_residual_fp8(const void* x, const void* w_q, const float* w_scale, const void* residual, void* out, int64_t T, int64_t N,
                              int64_t K, void* workspace, size_t workspace_bytes, void* stream) {
  MB_CHECK_ARG(x && w_q && w_scale && out, "linear_residual_fp8: null pointer");
  EpiParams e;
  e.out = out;
  e.residual = residual;
  e.ld_out = N;
  e.w_scale = w_scale;
  if (residual) return run_linear_quant<EPI_RESIDUAL, false>(x, nullptr, w_q, nullptr, e, T, N, K, 0.f, workspace, workspace_bytes, (cudaStream_t)stream);
  return run_linear_quant<EPI_STORE, false>(x, nullptr, w_q, nullptr, e, T, N, K, 0.f, workspace, workspace_bytes, (cudaStream_t)stream);
}

int mb200_ffn_gateup_fp8(const void* x, const void* norm_w, const void* w_q, const float* w_scale, void* g_out, int64_t T, int64_t dim,
                         int64_t hidden, float eps, void* workspace, size_t workspace_bytes, void* stream) {
  MB_CHECK_ARG(x && w_q && w_scale && g_out, "ffn_gateup_fp8: null pointer");
  EpiParams e;
  e.out = g_out;
  e.ld_out = hidden;
  e.w_scale = w_scale;
  return run_linear_quant<EPI_SWIGLU, false>(x, norm_w, w_q, nullptr, e, T, 2 * hidden, dim, eps, workspace, workspace_bytes, (cudaStream_t)stream);
}

int mb200_attn_qkv_fp8a8(const void* x, const void* norm_w, const void* w_q, const float* w_scale, const float* rope, const int32_t* positions,
                         void* q_out, void* k_out, void* v_out, void* cache_k, void* cache_v, const int32_t* cache_rows, int64_t T, int64_t dim,
                         int64_t n_heads, int64_t n_kv_heads, int64_t head_dim, float eps, void* workspace, size_t workspace_bytes, void* stream) {
  MB_CHECK_ARG(w_scale, "attn_qkv_fp8a8: null scale");
  return attn_qkv_impl(x, norm_w, w_q, rope, positions, q_out, k_out, v_out, cache_k, cache_v, cache_rows, T, dim, n_heads, n_kv_heads,
                       head_dim, eps, workspace, workspace_bytes, stream, nullptr, w_scale, nullptr, true);
}

int mb200_linear_residual_fp8a8(const void* x, const void* w_q, const float* w_scale, const void* residual, void* out, int64_t T, int64_t N,
                                int64_t K, void* workspace, size_t workspace_bytes, void* stream) {
  MB_CHECK_ARG(x && w_q && w_scale && out, "linear_residual_fp8a8: null pointer");
  EpiParams e;
  e.out = out;
  e.residual = residual;
  e.ld_out = N;
  e.w_scale = w_scale;
  if (residual)
    return run_linear_quant<EPI_RESIDUAL, false, true>(x, nullptr, w_q, nullptr, e, T, N, K, 0.f, workspace, workspace_bytes, (cudaStream_t)stream);
  return run_linear_quant<EPI_STORE, false, true>(x, nullptr, w_q, nullptr, e, T, N, K, 0.f, workspace, workspace_bytes, (cudaStream_t)stream);
}

int mb200_ffn_gateup_fp8a8(const void* x, const void* norm_w, const void* w_q, const float* w_scale, void* g_out, int64_t T, int64_t dim,
                           int64_t hidden, float eps, void* workspace, size_t workspace_bytes, void* stream) {
  MB_CHECK_ARG(x && w_q && w_scale && g_out, "ffn_gateup_fp8a8: null pointer");
  EpiParams e;
  e.out = g_out;
  e.ld_out = hidden;
  e.w_scale = w_scale;
  return run_linear_quant<EPI_SWIGLU, false, true>(x, norm_w, w_q, nullptr, e, T, 2 * hidden, dim, eps, workspace, workspace_bytes,
                                                   (cudaStream_t)stream);
}

int mb200_quantize_act_e4m3(const void* x, const void* norm_w, void* q, int32_t* exps, int64_t T, int64_t dim, float eps, void* stream) {
  MB_CHECK_ARG(x && q && exps, "quantize_act_e4m3: null pointer");
  MB_CHECK_ARG(((uintptr_t)x & 15) == 0 && ((uintptr_t)norm_w & 15) == 0 && ((uintptr_t)q & 7) == 0 && ((uintptr_t)exps & 3) == 0,
               "quantize_act_e4m3: misaligned pointer");
  return launch_quantize_act(x, norm_w, (uint8_t*)q, exps, T, dim, eps, (cudaStream_t)stream);
}

int mb200_attn_qkv_int4(const void* x, const void* norm_w, const void* w_q, const void* w_gscale, const float* rope, const int32_t* positions,
                        void* q_out, void* k_out, void* v_out, void* cache_k, void* cache_v, const int32_t* cache_rows, int64_t T, int64_t dim,
                        int64_t n_heads, int64_t n_kv_heads, int64_t head_dim, float eps, void* workspace, size_t workspace_bytes, void* stream) {
  MB_CHECK_ARG(w_gscale, "attn_qkv_int4: null group scales");
  return attn_qkv_impl(x, norm_w, w_q, rope, positions, q_out, k_out, v_out, cache_k, cache_v, cache_rows, T, dim, n_heads, n_kv_heads,
                       head_dim, eps, workspace, workspace_bytes, stream, nullptr, nullptr, (const uint16_t*)w_gscale);
}

int mb200_linear_residual_int4(const void* x, const void* w_q, const void* w_gscale, const void* residual, void* out, int64_t T, int64_t N,
                               int64_t K, void* workspace, size_t workspace_bytes, void* stream) {
  MB_CHECK_ARG(x && w_q && w_gscale && out, "linear_residual_int4: null pointer");
  EpiParams e;
  e.out = out;
  e.residual = residual;
  e.ld_out = N;
  const uint16_t* gs = (const uint16_t*)w_gscale;
  if (residual) return run_linear_quant<EPI_RESIDUAL, true>(x, nullptr, w_q, gs, e, T, N, K, 0.f, workspace, workspace_bytes, (cudaStream_t)stream);
  return run_linear_quant<EPI_STORE, true>(x, nullptr, w_q, gs, e, T, N, K, 0.f, workspace, workspace_bytes, (cudaStream_t)stream);
}

int mb200_ffn_gateup_int4(const void* x, const void* norm_w, const void* w_q, const void* w_gscale, void* g_out, int64_t T, int64_t dim,
                          int64_t hidden, float eps, void* workspace, size_t workspace_bytes, void* stream) {
  MB_CHECK_ARG(x && w_q && w_gscale && g_out, "ffn_gateup_int4: null pointer");
  EpiParams e;
  e.out = g_out;
  e.ld_out = hidden;
  return run_linear_quant<EPI_SWIGLU, true>(x, norm_w, w_q, (const uint16_t*)w_gscale, e, T, 2 * hidden, dim, eps, workspace, workspace_bytes,
                                     (cudaStream_t)stream);
}

int mb200_quantize_int4_groups(const void* w, int64_t rows, int64_t K, void* q, int64_t q_row_stride, void* scale, int64_t scale_row_stride,
                               void* stream) {
  MB_CHECK_ARG(w && q && scale, "quantize_int4_groups: null pointer");
  MB_CHECK_ARG(rows >= 1 && rows <= 0x7fffffff && K >= kInt4Group && K % kInt4Group == 0 && K <= (1 << 24),
               "quantize_int4_groups: rows=%lld K=%lld (K a multiple of 128)", (long long)rows, (long long)K);
  MB_CHECK_ARG(q_row_stride >= K / 2 && q_row_stride % 4 == 0 && scale_row_stride >= K / kInt4Group,
               "quantize_int4_groups: q_row_stride=%lld (>= K/2, multiple of 4) scale_row_stride=%lld (>= K/128)", (long long)q_row_stride,
               (long long)scale_row_stride);
  MB_CHECK_ARG(((uintptr_t)w & 15) == 0 && ((uintptr_t)q & 3) == 0 && ((uintptr_t)scale & 1) == 0, "quantize_int4_groups: misaligned pointer");
  quantize_int4_groups_kernel<<<(unsigned)rows, 256, 0, (cudaStream_t)stream>>>((const uint4*)w, (int)K, (uint8_t*)q, q_row_stride,
                                                                                (uint16_t*)scale, scale_row_stride);
  MB_CHECK_LAUNCH("quantize_int4_groups_kernel");
  note_launch("quantize_int4_groups_kernel");
  return MB200_OK;
}

int mb200_linear_residual_lora(const void* x, const void* w, const void* residual, void* out, int64_t T, int64_t N, int64_t K,
                               void* workspace, size_t workspace_bytes, void* stream, const mb200_lora* lora) {
  MB_CHECK_ARG(x && w && out && lora, "linear_residual_lora: null pointer");
  EpiParams e;
  e.out = out;
  e.residual = residual;
  e.ld_out = N;
  cudaStream_t st = (cudaStream_t)stream;
  if (residual) return run_linear_lora<EPI_RESIDUAL>(x, nullptr, w, e, lora, T, N, K, 0.f, workspace, workspace_bytes, st);
  return run_linear_lora<EPI_STORE>(x, nullptr, w, e, lora, T, N, K, 0.f, workspace, workspace_bytes, st);
}

int mb200_linear_bias(const void* x, const void* w, const void* bias, void* out, int64_t T, int64_t N, int64_t K, int gelu, void* workspace,
                      size_t workspace_bytes, void* stream) {
  MB_CHECK_ARG(x && w && out, "linear_bias: null pointer");
  EpiParams e;
  e.out = out;
  e.bias = bias;
  e.ld_out = N;
  if (gelu) return run_linear<EPI_BIAS_GELU>(x, nullptr, w, e, T, N, K, 0.f, workspace, workspace_bytes, (cudaStream_t)stream);
  return run_linear<EPI_BIAS>(x, nullptr, w, e, T, N, K, 0.f, workspace, workspace_bytes, (cudaStream_t)stream);
}

int mb200_vision_patchify(const void* image, void* out, int64_t C, int64_t H, int64_t W, int64_t patch, int64_t k_pad, void* stream) {
  MB_CHECK_ARG(image && out, "vision_patchify: null pointer");
  MB_CHECK_ARG(C >= 1 && patch >= 1 && H >= patch && W >= patch, "vision_patchify: image [%lld, %lld, %lld] has no whole %lld x %lld patch",
               (long long)C, (long long)H, (long long)W, (long long)patch, (long long)patch);
  MB_CHECK_ARG(k_pad >= C * patch * patch && k_pad % 8 == 0, "vision_patchify: k_pad=%lld < C*p*p=%lld or not a multiple of 8", (long long)k_pad,
               (long long)(C * patch * patch));
  const int64_t gh = H / patch, gw = W / patch;
  patchify_kernel<<<(unsigned)(gh * gw), 256, 0, (cudaStream_t)stream>>>((const bf16*)image, (bf16*)out, (int)H, (int)W, (int)patch, (int)gw,
                                                                       (int)(C * patch * patch), (int)k_pad);
  note_launch("patchify_kernel");
  MB_CHECK_LAUNCH("patchify_kernel");
  return MB200_OK;
}

int mb200_patch_merge(const void* x, void* out, int64_t h, int64_t w, int64_t s, int64_t d, void* stream) {
  MB_CHECK_ARG(x && out, "patch_merge: null pointer");
  MB_CHECK_ARG(s >= 1 && h >= 1 && w >= 1 && d >= 1, "patch_merge: h=%lld w=%lld s=%lld d=%lld", (long long)h, (long long)w, (long long)s,
               (long long)d);
  const int64_t rows = (h / s) * (w / s);
  if (rows == 0) return MB200_OK;
  patch_merge_kernel<<<(unsigned)rows, 256, 0, (cudaStream_t)stream>>>((const bf16*)x, (bf16*)out, (int)w, (int)s, (int)d);
  note_launch("patch_merge_kernel");
  MB_CHECK_LAUNCH("patch_merge_kernel");
  return MB200_OK;
}

int mb200_embed_splice(const int64_t* ids, const void* emb, const void* feats, void* out, int32_t* ordinal, int64_t T, int64_t dim, int64_t vocab,
                       int64_t n_feats, int64_t image_token_id, void* stream) {
  MB_CHECK_ARG(ids && emb && out && ordinal && (feats || n_feats == 0), "embed_splice: null pointer");
  MB_CHECK_ARG(dim % 8 == 0 && T >= 0 && n_feats >= 0, "embed_splice: dim=%lld must be a multiple of 8", (long long)dim);
  cudaStream_t st = (cudaStream_t)stream;
  splice_scan_kernel<<<1, SPLICE_SCAN_THREADS, 0, st>>>((const long long*)ids, ordinal, (int)T, (long long)image_token_id);
  note_launch("splice_scan_kernel");
  MB_CHECK_LAUNCH("splice_scan_kernel");
  if (T == 0) return MB200_OK;
  splice_gather_kernel<<<(unsigned)T, 128, 0, st>>>((const long long*)ids, ordinal, (const uint4*)emb, (const uint4*)feats, (uint4*)out,
                                                   (int)(dim / 8), (long long)vocab, (int)n_feats);
  note_launch("splice_gather_kernel");
  MB_CHECK_LAUNCH("splice_gather_kernel");
  return MB200_OK;
}

int mb200_ffn_gateup(const void* x, const void* norm_w, const void* w13, void* g_out, int64_t T, int64_t dim, int64_t hidden, float eps,
                     void* workspace, size_t workspace_bytes, void* stream) {
  MB_CHECK_ARG(x && w13 && g_out, "ffn_gateup: null pointer");
  EpiParams e;
  e.out = g_out;
  e.ld_out = hidden;
  return run_linear<EPI_SWIGLU>(x, norm_w, w13, e, T, 2 * hidden, dim, eps, workspace, workspace_bytes, (cudaStream_t)stream);
}

int mb200_ffn_gateup_lora(const void* x, const void* norm_w, const void* w13, void* g_out, int64_t T, int64_t dim, int64_t hidden, float eps,
                          void* workspace, size_t workspace_bytes, void* stream, const mb200_lora* lora) {
  MB_CHECK_ARG(x && w13 && g_out && lora, "ffn_gateup_lora: null pointer");
  EpiParams e;
  e.out = g_out;
  e.ld_out = hidden;
  return run_linear_lora<EPI_SWIGLU>(x, norm_w, w13, e, lora, T, 2 * hidden, dim, eps, workspace, workspace_bytes, (cudaStream_t)stream);
}

int mb200_lm_head(const void* x, const void* norm_w, const void* w_out, float* logits, int64_t T, int64_t dim, int64_t vocab, float eps,
                  void* workspace, size_t workspace_bytes, void* stream) {
  MB_CHECK_ARG(x && norm_w && w_out && logits, "lm_head: null pointer");
  EpiParams e;
  e.out_f32 = logits;
  e.ld_out = vocab;
  return run_linear<EPI_F32>(x, norm_w, w_out, e, T, vocab, dim, eps, workspace, workspace_bytes, (cudaStream_t)stream);
}

int mb200_argmax_rows(const float* logits, int64_t* out_dev, int64_t T, int64_t vocab, void* stream) {
  MB_CHECK_ARG(logits && out_dev && T >= 0 && vocab >= 1, "argmax_rows: bad arguments");
  if (T == 0) return MB200_OK;
  argmax_rows_kernel<<<(unsigned)T, SP_THREADS, 0, (cudaStream_t)stream>>>(logits, (long long*)out_dev, (int)vocab);
  MB_CHECK_LAUNCH("argmax_rows_kernel");
  return MB200_OK;
}

int mb200_logprob_gather(const float* logits, const int64_t* target_dev, float* out_dev, int64_t T, int64_t vocab, void* stream) {
  MB_CHECK_ARG(logits && target_dev && out_dev && T >= 0 && vocab >= 1, "logprob_gather: bad arguments");
  if (T == 0) return MB200_OK;
  logprob_gather_kernel<<<(unsigned)T, SP_THREADS, 0, (cudaStream_t)stream>>>(logits, (const long long*)target_dev, out_dev, (int)vocab);
  MB_CHECK_LAUNCH("logprob_gather_kernel");
  return MB200_OK;
}

int mb200_sample_top_p(const float* logits, const float* uniform_dev, int64_t* out_dev, int64_t T, int64_t vocab, float temperature,
                       float top_p, void* stream) {
  MB_CHECK_ARG(logits && uniform_dev && out_dev && T >= 0 && vocab >= 1, "sample_top_p: bad arguments");
  MB_CHECK_ARG(temperature > 0.f && top_p >= 0.f && top_p <= 1.f, "sample_top_p: temperature=%g must be > 0 and top_p=%g in [0, 1]",
               (double)temperature, (double)top_p);
  if (T == 0) return MB200_OK;
  sample_top_p_kernel<<<(unsigned)T, SP_THREADS, 0, (cudaStream_t)stream>>>(logits, uniform_dev, (long long*)out_dev, (int)vocab,
                                                                            1.0f / temperature, top_p);
  MB_CHECK_LAUNCH("sample_top_p_kernel");
  return MB200_OK;
}

int mb200_select_tokens(const float* logits, const float* temperature_dev, const float* top_p_dev, const float* presence_dev,
                        const float* frequency_dev, const uint64_t* seeds_dev, const float* uniform_dev, int32_t* step_dev, int32_t* counts_dev,
                        int64_t* out_dev, int64_t B, int64_t vocab, void* stream) {
  MB_CHECK_ARG(logits && temperature_dev && top_p_dev && presence_dev && frequency_dev && step_dev && out_dev && B >= 0 && vocab >= 1 &&
                   vocab <= INT32_MAX,
               "select_tokens: bad arguments");
  MB_CHECK_ARG((seeds_dev == nullptr) != (uniform_dev == nullptr), "select_tokens: exactly one of seeds and uniform");
  if (B == 0) return MB200_OK;
  select_tokens_kernel<<<(unsigned)B, SP_THREADS, 0, (cudaStream_t)stream>>>(logits, temperature_dev, top_p_dev, presence_dev, frequency_dev,
                                                                            (const unsigned long long*)seeds_dev, uniform_dev, step_dev,
                                                                            counts_dev, (long long*)out_dev, (int)vocab);
  MB_CHECK_LAUNCH("select_tokens_kernel");
  note_launch("select_tokens_kernel<%s, %s>", seeds_dev ? "philox" : "uniform", counts_dev ? "counts" : "nocounts");
  return MB200_OK;
}

// ---- mixture of experts (csrc/moe.cuh) ---------------------------------------------------------------------------------------
int mb200_moe_sizes(int64_t T, int64_t n_experts, int64_t top_k, int64_t* tile_rows, int64_t* rows_cap, int64_t* plan_words) {
  MB_CHECK_ARG(T >= 1 && n_experts >= 1 && top_k >= 1, "moe_sizes: bad arguments");
  const int tr = moe_tile_rows(T);
  const int64_t cap = moe_tile_cap(T * top_k, n_experts, tr);
  if (tile_rows) *tile_rows = tr;
  if (rows_cap) *rows_cap = cap * tr;
  if (plan_words) *plan_words = moe_plan_words(T * top_k, n_experts, tr);
  return MB200_OK;
}

int mb200_moe_route(const void* hn, const void* gate_w, int64_t T, int64_t dim, int64_t n_experts, int64_t top_k, int64_t shard_rank,
                    int64_t shard_world, int32_t* sel, void* wts, int32_t* slot, int32_t* plan, void* xs, void* row_w, void* stream) {
  MB_CHECK_ARG(hn && gate_w && sel && wts && slot && plan && xs && row_w, "moe_route: null pointer");
  MB_CHECK_ARG(T >= 1 && dim % 8 == 0, "moe_route: T=%lld dim=%lld", (long long)T, (long long)dim);
  MB_CHECK_ARG(top_k >= 1 && top_k <= MOE_MAX_TOPK && top_k <= n_experts && n_experts <= MOE_MAX_EXPERTS,
               "moe_route: E=%lld (max %d), k=%lld (max %d)", (long long)n_experts, MOE_MAX_EXPERTS, (long long)top_k, MOE_MAX_TOPK);
  MB_CHECK_ARG(shard_world >= 1 && shard_rank >= 0 && shard_rank < shard_world, "moe_route: shard %lld of %lld", (long long)shard_rank,
               (long long)shard_world);
  cudaStream_t st = (cudaStream_t)stream;
  const bool wide = T <= 256;  // decode-sized batches: one CTA per token
  const dim3 blocks(wide ? (unsigned)T : (unsigned)ceil_div(T, 8));
#define MB_ROUTE(EE)                                                                                                                              \
  if (wide)                                                                                                                                       \
    MB_CHECK_CUDA(launch_pdl(moe_route_kernel<EE, true>, blocks, dim3(256), 0, st, (const bf16*)hn, (const bf16*)gate_w, (int)T, (int)dim,      \
                             (int)top_k, sel, (bf16*)wts));                                                                                       \
  else                                                                                                                                            \
    MB_CHECK_CUDA(launch_pdl(moe_route_kernel<EE, false>, blocks, dim3(256), 0, st, (const bf16*)hn, (const bf16*)gate_w, (int)T, (int)dim,     \
                             (int)top_k, sel, (bf16*)wts));
  switch (n_experts) {
    case 2: MB_ROUTE(2) break;
    case 4: MB_ROUTE(4) break;
    case 8: MB_ROUTE(8) break;
    case 16: MB_ROUTE(16) break;
    default: return fail(MB200_E_INVALID, "moe_route: n_experts=%lld unsupported (2, 4, 8, 16)", (long long)n_experts);
  }
#undef MB_ROUTE
  MB_CHECK_LAUNCH("moe_route_kernel");
  note_launch("moe_route_kernel<%d, %s>", (int)n_experts, wide ? "true" : "false");
  const int tile_rows = moe_tile_rows(T);
  const int64_t pairs = T * top_k, cap = moe_tile_cap(pairs, n_experts, tile_rows);
  const size_t plan_smem = ((size_t)n_experts * MP_THREADS + 2 * n_experts + 1) * sizeof(int32_t);
  MB_CHECK_CUDA(cudaFuncSetAttribute(moe_plan_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)plan_smem));
  moe_plan_kernel<<<1, MP_THREADS, plan_smem, st>>>(sel, (int)pairs, (int)n_experts, tile_rows, (int)shard_rank, (int)shard_world, (int)cap, slot, plan);
  MB_CHECK_LAUNCH("moe_plan_kernel");
  note_launch("moe_plan_kernel<%s>", pairs <= 512 ? "short" : "scan");  // the kernel's own switch: a thread per expert, or the 1024-thread scan
  moe_gather_kernel<<<(unsigned)ceil_div(pairs, 8), 256, 0, st>>>((const uint4*)hn, sel, (const bf16*)wts, slot, (int)pairs, (int)top_k, (int)(dim / 8),
                                                                  (int)shard_rank, (int)shard_world, (uint4*)xs, (bf16*)row_w);
  MB_CHECK_LAUNCH("moe_gather_kernel");
  note_launch("moe_gather_kernel");
  return MB200_OK;
}

// The un-merged LoRA stages of one grouped expert Linear [N, K] (include/mistral_b200.h): a = bf16(x A_e^T) over the plan's rows
// (l_buf doubles as the split partials), then L = bf16(a B_e^T) with the bf16 grouped GEMM (K = rank_cols).  The base GEMM's
// EPI_LORA epilogue adds bf16(L * scaling): `epi` gets those fields.
static int moe_lora_stages(const void* x, const mb200_moe_lora* l, const void* const* w_host, int E, int64_t rows_cap, int64_t K, int64_t N,
                           int est, int tile_rows, const int32_t* plan, EpiParams* epi, void* workspace, size_t workspace_bytes, cudaStream_t st) {
  MB_CHECK_ARG(l->a_host && l->b_host && l->a_buf && l->l_buf, "moe lora: null pointer");
  MB_CHECK_ARG(l->rank_cols >= 64 && l->rank_cols % 64 == 0, "moe lora: rank_cols=%lld must be a multiple of 64", (long long)l->rank_cols);
  MB_CHECK_ARG(((uintptr_t)l->a_buf & 15) == 0 && ((uintptr_t)l->l_buf & 15) == 0,
               "moe lora: a_buf and l_buf must be 16-byte aligned (l_buf doubles as fp32 split-K scratch)");
  for (int e = 0; e < E; ++e)
    MB_CHECK_ARG(w_host[e] == nullptr || (l->a_host[e] != nullptr && l->b_host[e] != nullptr), "moe lora: expert %d has weights but no adapter", e);
  int rc = launch_lora_down_grouped(x, l->a_host, E, plan, tile_rows, est, l->a_buf, rows_cap, l->rank_cols, K, l->l_buf, (size_t)rows_cap * N * 2, st);
  if (rc) return rc;
  EpiParams up;
  up.out = l->l_buf;
  up.ld_out = N;
  rc = launch_grouped<EPI_STORE>(l->a_buf, rows_cap, l->rank_cols, N, l->b_host, E, est, tile_rows, plan, up, workspace, workspace_bytes, st,
                                 MoeFmt::BF16, nullptr);
  if (rc) return rc;
  epi->lora_l = l->l_buf;
  epi->ld_lora = N;
  epi->lora_scaling = l->scaling;
  return MB200_OK;
}

// s13 / s2: NULL for bf16 experts; the host arrays of per-row fp32 scale pointers next to e4m3 weights (FP8), or of bf16 group-scale
// pointers next to INT4 codes.  l13 / l2: the un-merged adapters of FP8 experts, or NULL.
static int moe_grouped_ffn(const void* xs, const void* const* w13_host, const void* const* w2_host, MoeFmt fmt, const void* const* s13_host,
                           const void* const* s2_host, const int32_t* plan, const void* row_w, const int32_t* slot, const void* residual, void* g,
                           void* yw, void* out, int64_t T, int64_t dim, int64_t hidden, int64_t n_experts, int64_t top_k, const mb200_moe_comm* comm,
                           void* workspace, size_t workspace_bytes, void* stream, const mb200_moe_lora* l13 = nullptr,
                           const mb200_moe_lora* l2 = nullptr) {
  MB_CHECK_ARG(xs && w13_host && w2_host && plan && row_w && slot && g && yw && out, "moe_grouped_ffn: null pointer");
  MB_CHECK_ARG((l13 == nullptr) == (l2 == nullptr) && (l13 == nullptr || fmt == MoeFmt::FP8), "moe_grouped_ffn: adapters need FP8 experts, both of them");
  MB_CHECK_ARG(T >= 1 && top_k >= 1 && top_k <= MOE_MAX_TOPK && n_experts <= MOE_MAX_EXPERTS && dim % 64 == 0 && hidden % 64 == 0,
               "moe_grouped_ffn: T=%lld k=%lld E=%lld dim=%lld hidden=%lld", (long long)T, (long long)top_k, (long long)n_experts, (long long)dim,
               (long long)hidden);
  MB_CHECK_ARG(fmt != MoeFmt::INT4 || (dim % kInt4Group == 0 && hidden % kInt4Group == 0),
               "moe_grouped_ffn (int4): dim=%lld and hidden=%lld must be multiples of 128", (long long)dim, (long long)hidden);
  const int n_ranks = comm ? comm->n_ranks : 1, my_rank = comm ? comm->my_rank : 0;
  MB_CHECK_ARG(n_ranks >= 1 && n_ranks <= kMaxPeers && my_rank >= 0 && my_rank < n_ranks, "moe_grouped_ffn: rank %d of %d", my_rank, n_ranks);
  cudaStream_t st = (cudaStream_t)stream;
  const int tile_rows = moe_tile_rows(T);
  const int64_t pairs = T * top_k, rows_cap = moe_row_cap(pairs, n_experts, tile_rows);
  int local = 0;
  for (int e = 0; e < (int)n_experts; ++e) local += (w13_host[e] != nullptr);
  MB_CHECK_ARG(local >= 1, "moe_grouped_ffn: this rank owns no expert");
  // expected number of this rank's experts that get at least one row (uniform routing): sizes the decode tile width
  double touched = (double)n_experts * (1.0 - pow(1.0 - (double)top_k / (double)n_experts, (double)T)) * ((double)local / (double)n_experts);
  int est = (int)(touched + 0.5);
  if (est < 1) est = 1;
  if (tile_rows == 128) est = (int)((pairs / n_ranks + tile_rows - 1) / tile_rows) + local;
  EpiParams e1;
  e1.out = g;
  e1.ld_out = hidden;
  int rc;
  if (l13) {
    rc = moe_lora_stages(xs, l13, w13_host, (int)n_experts, rows_cap, dim, 2 * hidden, est, tile_rows, plan, &e1, workspace, workspace_bytes, st);
    if (rc) return rc;
    rc = launch_grouped<EPI_SWIGLU | EPI_LORA>(xs, rows_cap, dim, 2 * hidden, w13_host, (int)n_experts, est, tile_rows, plan, e1, workspace,
                                               workspace_bytes, st, fmt, s13_host);
  } else {
    rc = launch_grouped<EPI_SWIGLU>(xs, rows_cap, dim, 2 * hidden, w13_host, (int)n_experts, est, tile_rows, plan, e1, workspace, workspace_bytes, st,
                                    fmt, s13_host);
  }
  if (rc) return rc;
  EpiParams e2;
  e2.out = yw;
  e2.ld_out = dim;
  e2.row_w = row_w;
  e2.n_peers = n_ranks - 1;
  for (int r = 0; r < n_ranks - 1; ++r) {
    MB_CHECK_ARG(comm->peer_yw[r] != nullptr, "moe_grouped_ffn: peer buffer %d missing", r);
    e2.peer_out[r] = comm->peer_yw[r];
  }
  if (l2) {
    rc = moe_lora_stages(g, l2, w2_host, (int)n_experts, rows_cap, hidden, dim, est, tile_rows, plan, &e2, workspace, workspace_bytes, st);
    if (rc) return rc;
    rc = launch_grouped<EPI_MOE_SCALE | EPI_LORA>(g, rows_cap, hidden, dim, w2_host, (int)n_experts, est, tile_rows, plan, e2, workspace,
                                                  workspace_bytes, st, fmt, s2_host);
  } else {
    rc = launch_grouped<EPI_MOE_SCALE>(g, rows_cap, hidden, dim, w2_host, (int)n_experts, est, tile_rows, plan, e2, workspace, workspace_bytes, st,
                                       fmt, s2_host);
  }
  if (rc) return rc;
  MoeCombineParams c;
  c.yw = (const uint4*)yw;
  c.slot = slot;
  c.residual = (const uint4*)residual;
  c.out = (uint4*)out;
  c.T = (int)T;
  c.k = (int)top_k;
  c.row_chunks = (int)(dim / 8);
  c.n_ranks = n_ranks;
  c.my_rank = my_rank;
  c.my_flags = nullptr;
  c.epoch = nullptr;
  c.done_counter = nullptr;
  for (int r = 0; r < kMaxPeers; ++r) c.peer_flags[r] = nullptr;
  if (n_ranks > 1) {
    MB_CHECK_ARG(comm->my_flags && comm->epoch && comm->done_counter, "moe_grouped_ffn: comm state missing");
    c.my_flags = (unsigned*)comm->my_flags;
    c.epoch = (unsigned*)comm->epoch;
    c.done_counter = (int*)comm->done_counter;
    for (int r = 0; r < n_ranks - 1; ++r) {
      MB_CHECK_ARG(comm->peer_flags[r] != nullptr, "moe_grouped_ffn: peer flags %d missing", r);
      c.peer_flags[r] = (unsigned*)comm->peer_flags[r];
    }
  }
  moe_combine_kernel<<<(unsigned)T, 128, 0, st>>>(c);
  MB_CHECK_LAUNCH("moe_combine_kernel");
  note_launch("moe_combine_kernel");
  return MB200_OK;
}

int mb200_moe_grouped_ffn(const void* xs, const void* const* w13_host, const void* const* w2_host, const int32_t* plan, const void* row_w,
                          const int32_t* slot, const void* residual, void* g, void* yw, void* out, int64_t T, int64_t dim, int64_t hidden,
                          int64_t n_experts, int64_t top_k, const mb200_moe_comm* comm, void* workspace, size_t workspace_bytes, void* stream) {
  return moe_grouped_ffn(xs, w13_host, w2_host, MoeFmt::BF16, nullptr, nullptr, plan, row_w, slot, residual, g, yw, out, T, dim, hidden, n_experts, top_k, comm,
                         workspace, workspace_bytes, stream);
}

int mb200_moe_grouped_ffn_fp8(const void* xs, const void* const* w13_host, const float* const* w13_scale_host, const void* const* w2_host,
                              const float* const* w2_scale_host, const int32_t* plan, const void* row_w, const int32_t* slot, const void* residual,
                              void* g, void* yw, void* out, int64_t T, int64_t dim, int64_t hidden, int64_t n_experts, int64_t top_k,
                              const mb200_moe_comm* comm, void* workspace, size_t workspace_bytes, void* stream) {
  MB_CHECK_ARG(w13_scale_host && w2_scale_host, "moe_grouped_ffn_fp8: null scale table");
  return moe_grouped_ffn(xs, w13_host, w2_host, MoeFmt::FP8, reinterpret_cast<const void* const*>(w13_scale_host),
                         reinterpret_cast<const void* const*>(w2_scale_host), plan, row_w, slot, residual, g, yw, out, T, dim, hidden, n_experts,
                         top_k, comm, workspace, workspace_bytes, stream);
}

int mb200_moe_grouped_ffn_fp8_lora(const void* xs, const void* const* w13_host, const float* const* w13_scale_host, const void* const* w2_host,
                                   const float* const* w2_scale_host, const int32_t* plan, const void* row_w, const int32_t* slot, const void* residual,
                                   void* g, void* yw, void* out, int64_t T, int64_t dim, int64_t hidden, int64_t n_experts, int64_t top_k,
                                   const mb200_moe_comm* comm, void* workspace, size_t workspace_bytes, void* stream, const mb200_moe_lora* lora13,
                                   const mb200_moe_lora* lora2) {
  MB_CHECK_ARG(w13_scale_host && w2_scale_host, "moe_grouped_ffn_fp8_lora: null scale table");
  MB_CHECK_ARG(lora13 && lora2, "moe_grouped_ffn_fp8_lora: null adapter");
  return moe_grouped_ffn(xs, w13_host, w2_host, MoeFmt::FP8, reinterpret_cast<const void* const*>(w13_scale_host),
                         reinterpret_cast<const void* const*>(w2_scale_host), plan, row_w, slot, residual, g, yw, out, T, dim, hidden, n_experts,
                         top_k, comm, workspace, workspace_bytes, stream, lora13, lora2);
}

int mb200_moe_grouped_ffn_int4(const void* xs, const void* const* w13_host, const void* const* w13_gscale_host, const void* const* w2_host,
                               const void* const* w2_gscale_host, const int32_t* plan, const void* row_w, const int32_t* slot, const void* residual,
                               void* g, void* yw, void* out, int64_t T, int64_t dim, int64_t hidden, int64_t n_experts, int64_t top_k,
                               const mb200_moe_comm* comm, void* workspace, size_t workspace_bytes, void* stream) {
  MB_CHECK_ARG(w13_gscale_host && w2_gscale_host, "moe_grouped_ffn_int4: null scale table");
  return moe_grouped_ffn(xs, w13_host, w2_host, MoeFmt::INT4, w13_gscale_host, w2_gscale_host, plan, row_w, slot, residual, g, yw, out, T, dim,
                         hidden, n_experts, top_k, comm, workspace, workspace_bytes, stream);
}

int mb200_quantize_e4m3_rows(const void* w, int64_t rows, int64_t K, void* q, int64_t q_row_stride, float* scale, int64_t scale_stride, void* stream) {
  MB_CHECK_ARG(w && q && scale, "quantize_e4m3_rows: null pointer");
  MB_CHECK_ARG(rows >= 1 && rows <= 0x7fffffff && K >= 8 && K % 8 == 0 && K <= (1 << 24), "quantize_e4m3_rows: rows=%lld K=%lld (K a multiple of 8)",
               (long long)rows, (long long)K);
  MB_CHECK_ARG(q_row_stride >= K && q_row_stride % 8 == 0 && scale_stride >= 1, "quantize_e4m3_rows: q_row_stride=%lld (>= K, multiple of 8) scale_stride=%lld",
               (long long)q_row_stride, (long long)scale_stride);
  MB_CHECK_ARG(((uintptr_t)w & 15) == 0 && ((uintptr_t)q & 7) == 0 && ((uintptr_t)scale & 3) == 0, "quantize_e4m3_rows: misaligned pointer");
  quantize_e4m3_rows_kernel<<<(unsigned)rows, 256, 0, (cudaStream_t)stream>>>((const uint4*)w, (int)K, (uint8_t*)q, q_row_stride, scale, scale_stride);
  MB_CHECK_LAUNCH("quantize_e4m3_rows_kernel");
  note_launch("quantize_e4m3_rows_kernel");
  return MB200_OK;
}

// ---- NVLink peer buffers for the expert-parallel exchange: plain CUDA IPC on cudaMalloc'ed memory ------------------------------
int mb200_comm_alloc(size_t bytes, void** ptr_out) {
  MB_CHECK_ARG(ptr_out && bytes > 0, "comm_alloc: bad arguments");
  MB_CHECK_CUDA(cudaMalloc(ptr_out, bytes));
  MB_CHECK_CUDA(cudaMemset(*ptr_out, 0, bytes));
  MB_CHECK_CUDA(cudaDeviceSynchronize());
  return MB200_OK;
}
int mb200_comm_free(void* ptr) {
  if (ptr) MB_CHECK_CUDA(cudaFree(ptr));
  return MB200_OK;
}
int mb200_comm_export(void* ptr, void* handle_out64) {
  MB_CHECK_ARG(ptr && handle_out64, "comm_export: null pointer");
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
  MB_CHECK_CUDA(cudaIpcGetMemHandle((cudaIpcMemHandle_t*)handle_out64, ptr));
  return MB200_OK;
}
int mb200_comm_open(const void* handle64, void** ptr_out) {
  MB_CHECK_ARG(handle64 && ptr_out, "comm_open: null pointer");
  cudaIpcMemHandle_t h;
  memcpy(&h, handle64, sizeof(h));
  MB_CHECK_CUDA(cudaIpcOpenMemHandle(ptr_out, h, cudaIpcMemLazyEnablePeerAccess));
  return MB200_OK;
}
int mb200_comm_close(void* ptr) {
  if (ptr) MB_CHECK_CUDA(cudaIpcCloseMemHandle(ptr));
  return MB200_OK;
}

}  // extern "C"

// mb200_decode_step and mb200_decode_step_fp8 (w8: layers_dev is an mb200_layer_desc_fp8 array, dense only)
static int decode_step_impl(const void* layers_dev, const int32_t* windows_dev, int64_t n_layers, const void* emb, const void* final_norm,
                            const void* w_out, const float* rope, const int64_t* token_dev, int64_t pos, int64_t batch_row, float* logits,
                            int64_t* next_token_dev, int64_t dim, int64_t hidden, int64_t n_heads, int64_t n_kv_heads, int64_t head_dim,
                            int64_t vocab, float eps, int64_t n_experts, int64_t top_k, const void* const* moe_gate_dev,
                            const void* const* moe_w13_dev, const void* const* moe_w2_dev, void* workspace, size_t workspace_bytes, void* stream,
                            bool w8) {
  static_assert(sizeof(mb200_layer_desc) == sizeof(MkLayer), "layer descriptor layout");
  static_assert(sizeof(mb200_layer_desc_fp8) == sizeof(MkLayerFp8), "FP8 layer descriptor layout");
  MB_CHECK_ARG(layers_dev && windows_dev && emb && final_norm && w_out && rope && token_dev && logits && workspace, "decode_step: null pointer");
  MB_CHECK_ARG(n_experts == 0 || (moe_gate_dev && moe_w13_dev && moe_w2_dev), "decode_step: MoE weight tables missing");
  int dev = 0, sms = 0, smem_max = 0, coop = 0;
  MB_CHECK_CUDA(cudaGetDevice(&dev));
  MB_CHECK_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  MB_CHECK_CUDA(cudaDeviceGetAttribute(&smem_max, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  MB_CHECK_CUDA(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev));
  MB_CHECK_ARG(coop, "decode_step: device does not support cooperative launch");
  DecodePlan plan;
  const int rc = decode_plan(dim, hidden, n_heads, n_kv_heads, head_dim, vocab, n_experts, top_k, smem_max, &plan, w8);
  if (rc) return rc;
  const int rep = plan.rep;

  MkParams p;
  p.layers = reinterpret_cast<const MkLayer*>(layers_dev);
  p.windows = windows_dev;
  p.n_layers = (int)n_layers;
  p.emb = (const bf16*)emb;
  p.final_norm = (const bf16*)final_norm;
  p.w_out = (const bf16*)w_out;
  p.rope = rope;
  p.token = token_dev;
  p.pos = (int)pos;
  p.batch_row = (int)batch_row;
  p.logits = logits;
  p.next_token = (long long*)next_token_dev;
  p.n_experts = (int)n_experts;
  p.top_k = (int)(n_experts ? top_k : 0);
  p.moe_gate = (const bf16* const*)moe_gate_dev;
  p.moe_w13 = (const bf16* const*)moe_w13_dev;
  p.moe_w2 = (const bf16* const*)moe_w2_dev;
  p.dim = (int)dim;
  p.hidden = (int)hidden;
  p.H = (int)n_heads;
  p.KV = (int)n_kv_heads;
  p.vocab = (int)vocab;
  p.eps = eps;
  p.n_stages = plan.n_stages;
  p.xs_bytes = (int)plan.xs_bytes;
  const size_t smem = plan.smem;
  // global scratch: header words + activations + per-slice attention partials
  MB_CHECK_ARG((size_t)sms * sizeof(unsigned long long) <= kWsMkArgmaxSlots.bytes, "decode_step: %d SMs exceed the argmax slots", sms);
  uint8_t* ws = (uint8_t*)workspace;
  p.argmax_counter = (int*)(ws + kWsMkArgmaxCounter.offset);
  p.argmax_slots = (unsigned long long*)(ws + kWsMkArgmaxSlots.offset);
  p.bar_flags = (unsigned*)(ws + kWsMkBarFlags.offset);
  p.bar_epoch = (unsigned*)(ws + kWsMkBarEpoch.offset);
  p.done_counter = (int*)(ws + kWsMkDoneCounter.offset);
  const DecodeScratch sc = decode_scratch(dim, hidden, n_heads, n_experts, top_k, sms);
  p.xbuf = (bf16*)(ws + sc.xbuf);
  p.hbuf = (bf16*)(ws + sc.hbuf);
  p.qbuf = (bf16*)(ws + sc.qbuf);
  p.abuf = (bf16*)(ws + sc.abuf);
  p.gbuf = (bf16*)(ws + sc.gbuf);
  p.partial = (float*)(ws + sc.partial);
  p.prof = g_mk_prof;
  p.prof_bar = g_mk_prof_bar;
  if (workspace_bytes < sc.end) return fail(MB200_E_WORKSPACE, "decode_step: workspace %zu < %zu", workspace_bytes, sc.end);

  void* args[] = {(void*)&p};
  const void* fn = nullptr;
  switch (rep) {
    case 1: fn = w8 ? (const void*)decode_megakernel<1, true> : (const void*)decode_megakernel<1>; break;
    case 2: fn = w8 ? (const void*)decode_megakernel<2, true> : (const void*)decode_megakernel<2>; break;
    case 4: fn = w8 ? (const void*)decode_megakernel<4, true> : (const void*)decode_megakernel<4>; break;
    case 6: fn = w8 ? (const void*)decode_megakernel<6, true> : (const void*)decode_megakernel<6>; break;
    case 8: fn = w8 ? (const void*)decode_megakernel<8, true> : (const void*)decode_megakernel<8>; break;
    default: return fail(MB200_E_INVALID, "decode_step: H/KV=%d unsupported (1,2,4,6,8)", rep);
  }
  if (w8)
    note_launch("decode_megakernel<%d, true>", rep);
  else
    note_launch("decode_megakernel<%d>", rep);
  MB_CHECK_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  MB_CHECK_CUDA(cudaLaunchCooperativeKernel(fn, dim3((unsigned)sms), dim3(MK_THREADS), args, smem, (cudaStream_t)stream));
  return MB200_OK;
}

extern "C" {

int mb200_decode_step(const mb200_layer_desc* layers_dev, const int32_t* windows_dev, int64_t n_layers, const void* emb, const void* final_norm,
                      const void* w_out, const float* rope, const int64_t* token_dev, int64_t pos, int64_t batch_row, float* logits,
                      int64_t* next_token_dev, int64_t dim,
                      int64_t hidden, int64_t n_heads, int64_t n_kv_heads, int64_t head_dim, int64_t vocab, float eps, int64_t n_experts,
                      int64_t top_k, const void* const* moe_gate_dev, const void* const* moe_w13_dev, const void* const* moe_w2_dev,
                      void* workspace, size_t workspace_bytes, void* stream) {
  return decode_step_impl(layers_dev, windows_dev, n_layers, emb, final_norm, w_out, rope, token_dev, pos, batch_row, logits, next_token_dev, dim,
                          hidden, n_heads, n_kv_heads, head_dim, vocab, eps, n_experts, top_k, moe_gate_dev, moe_w13_dev, moe_w2_dev, workspace,
                          workspace_bytes, stream, false);
}

int mb200_decode_step_fp8(const mb200_layer_desc_fp8* layers_dev, const int32_t* windows_dev, int64_t n_layers, const void* emb,
                          const void* final_norm, const void* w_out, const float* rope, const int64_t* token_dev, int64_t pos,
                          int64_t batch_row, float* logits, int64_t* next_token_dev, int64_t dim, int64_t hidden, int64_t n_heads,
                          int64_t n_kv_heads, int64_t head_dim, int64_t vocab, float eps, void* workspace, size_t workspace_bytes, void* stream) {
  return decode_step_impl(layers_dev, windows_dev, n_layers, emb, final_norm, w_out, rope, token_dev, pos, batch_row, logits, next_token_dev, dim,
                          hidden, n_heads, n_kv_heads, head_dim, vocab, eps, 0, 0, nullptr, nullptr, nullptr, workspace, workspace_bytes, stream,
                          true);
}

int mb200_decode_step_fp8_supported(int64_t dim, int64_t hidden, int64_t n_heads, int64_t n_kv_heads, int64_t head_dim, int64_t vocab,
                                    int64_t smem_optin) {
  if (smem_optin <= 0) {
    int dev = 0, smem_max = 0;
    MB_CHECK_CUDA(cudaGetDevice(&dev));
    MB_CHECK_CUDA(cudaDeviceGetAttribute(&smem_max, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    smem_optin = smem_max;
  }
  DecodePlan plan;
  return decode_plan(dim, hidden, n_heads, n_kv_heads, head_dim, vocab, 0, 0, smem_optin, &plan, true);
}

int mb200_debug_decode_scratch(int64_t dim, int64_t hidden, int64_t n_heads, int64_t n_kv_heads, int64_t head_dim, int64_t n_experts,
                               int64_t top_k, size_t* q_offset, size_t* attn_offset) {
  MB_CHECK_ARG(q_offset && attn_offset, "debug_decode_scratch: null pointer");
  size_t off[6];
  const int rc = mb200_debug_decode_buffers(dim, hidden, n_heads, n_kv_heads, head_dim, n_experts, top_k, off);
  if (rc) return rc;
  *q_offset = off[2];
  *attn_offset = off[3];
  return MB200_OK;
}

int mb200_debug_decode_buffers(int64_t dim, int64_t hidden, int64_t n_heads, int64_t n_kv_heads, int64_t head_dim, int64_t n_experts,
                               int64_t top_k, size_t* offsets) {
  MB_CHECK_ARG(offsets, "debug_decode_buffers: null pointer");
  MB_CHECK_ARG(head_dim == kHeadDim && n_kv_heads > 0 && n_heads % n_kv_heads == 0 && dim > 0 && hidden > 0,
               "debug_decode_scratch: bad shape (H=%lld, KV=%lld, hd=%lld)", (long long)n_heads, (long long)n_kv_heads, (long long)head_dim);
  const DecodeScratch sc = decode_scratch(dim, hidden, n_heads, n_experts, top_k, 0);  // the SM count only sizes the last buffer
  offsets[0] = sc.xbuf;
  offsets[1] = sc.hbuf;
  offsets[2] = sc.qbuf;
  offsets[3] = sc.abuf;
  offsets[4] = sc.gbuf;
  offsets[5] = sc.partial;
  return MB200_OK;
}

int mb200_decode_step_supported(int64_t dim, int64_t hidden, int64_t n_heads, int64_t n_kv_heads, int64_t head_dim, int64_t vocab,
                                int64_t n_experts, int64_t top_k, int64_t smem_optin) {
  if (smem_optin <= 0) {
    int dev = 0, smem_max = 0;
    MB_CHECK_CUDA(cudaGetDevice(&dev));
    MB_CHECK_CUDA(cudaDeviceGetAttribute(&smem_max, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    smem_optin = smem_max;
  }
  DecodePlan plan;
  return decode_plan(dim, hidden, n_heads, n_kv_heads, head_dim, vocab, n_experts, top_k, smem_optin, &plan);
}

// Debug: device buffer of [8][n_layers][MK_PROF_WORDS] uint64 that 8 sampled CTAs of the decode megakernel fill with phase
// stamps and producer blocked times (NULL = off; layout next to mk_stamp).
int mb200_debug_set_decode_timeline(void* device_buffer) {
  g_mk_prof = (unsigned long long*)device_buffer;
  return MB200_OK;
}
int mb200_debug_set_barrier_timeline(void* device_buffer) {
  g_mk_prof_bar = (unsigned long long*)device_buffer;
  return MB200_OK;
}

int mb200_debug_launch_log(int enable, char* out, size_t out_bytes) {
  const bool overflow = g_launch_log_overflow;
  const size_t len = g_launch_log_len;
  g_launch_log_on = enable != 0;
  g_launch_log_overflow = false;
  g_launch_log_len = 0;
  if (out != nullptr) {
    if (out_bytes < len + 1) return fail(MB200_E_INVALID, "launch log: %zu bytes recorded, buffer of %zu", len, out_bytes);
    memcpy(out, g_launch_log, len);
    out[len] = '\0';
  }
  if (overflow) return fail(MB200_E_INVALID, "launch log: more than %zu bytes of launches since the last read", kLaunchLogBytes);
  return MB200_OK;
}

// Test-only: CUDA-core fp32-accumulate GEMM (c fp32 [T, N]) used to cross-check the tensor-core kernels on the GPU.
int mb200_test_gemm_naive(const void* a, const void* w, float* c, int64_t T, int64_t N, int64_t K, void* stream) {
  MB_CHECK_ARG(a && w && c, "test_gemm_naive: null pointer");
  const dim3 grid((unsigned)ceil_div(N, 128), (unsigned)T);
  gemm_naive_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>((const bf16*)a, (const bf16*)w, c, (int)T, (int)N, (int)K);
  MB_CHECK_LAUNCH("gemm_naive_kernel");
  return MB200_OK;
}

}  // extern "C"

#ifdef MB200_SK_TRACE
// tracing build only (scripts/trace_streamk.py): copies the stream-K stamp ring to the host and returns the stamp count
extern "C" int mb200_debug_sk_trace(void* host_out, size_t bytes, unsigned* count) {
  using namespace mb200;
  if (bytes < sizeof(sk_trace_buf)) return fail(MB200_E_INVALID, "sk trace: %zu < %zu", bytes, sizeof(sk_trace_buf));
  MB_CHECK_CUDA(cudaDeviceSynchronize());
  MB_CHECK_CUDA(cudaMemcpyFromSymbol(host_out, sk_trace_buf, sizeof(sk_trace_buf)));
  MB_CHECK_CUDA(cudaMemcpyFromSymbol(count, sk_trace_count, sizeof(unsigned)));
  return MB200_OK;
}
#endif
