/*
 * mistral_b200.h -- C ABI of libmb200.so: the sm_90a (H100) implementation of the mistral-inference
 * transformer hot path (Attention block + FeedForward/MoE block + the norm / lm-head either side).
 *
 * The reference (mistralai/mistral-inference @ 2557e12) is pure Python and has NO FFI / plugin
 * boundary (SURVEY.md section 0.3, 8b); its hot path is a sequence of torch / xformers library calls.
 * Each entry point below replaces one group of those call sites and cites them.  The reference-side
 * binding is a ctypes stub (INTEGRATION.md); in this repo the caller is
 * mistral_inference_b200/_abi.py, which mirrors the reference's Python API on top.
 *
 * Conventions (all entry points):
 *   - plain C types only.  Every `*_d` / `const void*` tensor argument is a DEVICE pointer
 *     (torch: tensor.data_ptr()); bf16 tensors are raw 16-bit words, row-major, innermost contiguous.
 *   - `stream` is a cudaStream_t passed as void* (torch.cuda.current_stream().cuda_stream); all work is
 *     enqueued on it; no entry point synchronises, allocates or frees device memory, or touches host
 *     copies of the data.  Scratch comes from the caller-provided `workspace` (device, 256-B aligned).
 *   - returns 0 on success, a negative MB200_E_* code otherwise; mb200_last_error() gives the
 *     thread-local message.  Nothing throws across the boundary.
 *   - integer metadata (positions, rows, lengths) are int32 device arrays.
 *   - head_dim must be 128 (every config in BASELINE.json); mb200_attn_qkv and the cache-less mode of mb200_attn_prefill
 *     also take 64 (the vision encoder).  dims must be multiples of 8 (16-byte rows).
 */
#ifndef MISTRAL_B200_H_
#define MISTRAL_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MB200_ABI_VERSION 5

#define MB200_OK 0
#define MB200_E_INVALID (-1)   /* bad argument / unsupported shape */
#define MB200_E_WORKSPACE (-2) /* workspace too small */
#define MB200_E_CUDA (-3)      /* CUDA runtime / driver error at launch */

int mb200_abi_version(void);
const char* mb200_last_error(void);
/* Number of SMs / max opt-in shared memory of the current device (for the host-side planners). */
int mb200_device_info(int* sm_count, int* max_smem_optin);

/* ---------------------------------------------------------------------------------------------
 * RMSNorm.  out = bf16( bf16( x_f32 * rsqrt(mean(x_f32^2) + eps) ) * w )
 * Replaces RMSNorm.forward (transformer_layers.py:115-120; call sites :165,:167, transformer.py:219).
 * x, out: [T, dim] bf16; w: [dim] bf16.
 */
int mb200_rmsnorm(const void* x, const void* w, void* out, int64_t T, int64_t dim, float eps, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Fused attention input: RMSNorm -> packed QKV projection -> interleaved-pair RoPE (q,k) -> optional
 * scatter of k,v into the rotating KV cache.
 * Replaces attention_norm + wq/wk/wv + apply_rotary_emb + CacheView.update
 * (transformer_layers.py:165,66-70; rope.py:13-23; cache.py:83-92).
 *   x          [T, dim] bf16 (block input, un-normed)
 *   norm_w     [dim] bf16
 *   wqkv       [(H + 2*KV) * hd, dim] bf16: rows = wq ++ wk ++ wv ([out, in] like nn.Linear)
 *   rope       [n_pos, hd/2, 2] fp32 = view_as_real(precompute_freqs_cis(...)) (rope.py:6-10); the vision encoder passes
 *              the 2-D table [side, side, hd/2] flattened to [side^2, hd/2, 2] (rope.py:26-51) and positions row*side + col
 *   head_dim   64 or 128
 *   positions  [T] int32 absolute positions (cache.py:228-230)
 *   q_out      [T, H*hd] bf16; k_out, v_out [T, KV*hd] bf16 (rotated k, raw v)
 *   cache_k/v  [n_rows, KV, hd] bf16 flat ring (cache.py:88-89) and cache_rows [T] int32 = slot + b*W
 *              (cache.py:235) or -1 for tokens that are not cached (to_cache_mask false, cache.py:226).
 *              Pass cache_rows = NULL to skip the scatter (prefill reads the old ring first:
 *              transformer_layers.py:75-76; use mb200_kv_ring_write afterwards).
 * T <= MB200_SKINNY_MAX_T uses the weight-streaming GEMV path (HBM-bound), larger T the tensor-core path.
 * workspace: >= mb200_workspace_bytes(...) for this T.
 */
int mb200_attn_qkv(const void* x, const void* norm_w, const void* wqkv, const float* rope, const int32_t* positions,
                   void* q_out, void* k_out, void* v_out, void* cache_k, void* cache_v, const int32_t* cache_rows,
                   int64_t T, int64_t dim, int64_t n_heads, int64_t n_kv_heads, int64_t head_dim, float eps,
                   void* workspace, size_t workspace_bytes, void* stream);

/* CacheView.update on its own (cache.py:83-92): rows[t] >= 0 ? cache[rows[t]] = src[t]. */
int mb200_kv_ring_write(const void* k_new, const void* v_new, void* cache_k, void* cache_v, const int32_t* cache_rows,
                        int64_t T, int64_t n_kv_heads, int64_t head_dim, void* stream);

/* ---------------------------------------------------------------------------------------------
 * GQA decode attention over the rotating cache (one query token per sequence).
 * Replaces cache.key/value + repeat_kv + memory_efficient_attention with
 * BlockDiagonalCausalWithOffsetPaddedKeysMask (transformer_layers.py:78-88, cache.py:250-254):
 * sequence b attends to ring slots [0, kv_len[b]) of its ring, kv_len = min(pos+1, W); order-free softmax.
 *   q [B, H*hd] bf16; cache_k/v [max_batch, W, KV, hd] bf16; kv_len [B] int32 (device); out [B, H*hd] bf16
 *   n_splits: KV range is cut into this many CTAs per (b, kv head) (flash-decoding), combined in-kernel.
 */
int mb200_attn_decode(const void* q, const void* cache_k, const void* cache_v, const int32_t* kv_len, void* out,
                      int64_t B, int64_t W, int64_t n_heads, int64_t n_kv_heads, int64_t head_dim, int64_t n_splits,
                      void* workspace, size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Prefill attention (varlen, causal, sliding window) reading old keys from the ring and new keys from
 * k_new/v_new.  Replaces interleave_kv + repeat_kv + memory_efficient_attention with
 * BlockDiagonalCausalMask.make_local_attention / BlockDiagonalMask.make_local_attention_from_bottomright
 * (transformer_layers.py:75-76,84-88; cache.py:94-117,240,243-248).
 * Query i of sequence b sits at absolute position p = seqpos[b] + i and attends to absolute positions
 * (p - W, p]; positions < seqpos[b] come from ring slot (pos % W), the rest from the new chunk.
 *   q [T, H*hd]; k_new, v_new [T, KV*hd]; cache_k/v [max_batch, W, KV, hd]; out [T, H*hd] (all bf16)
 *   q_start [B+1] int32 (prefix sums of seqlens), seqpos [B] int32 (tokens already cached) -- device arrays
 *   max_seqlen: max over b of seqlens[b] (grid sizing);  window = W (cache size of this layer)
 *   causal = 2: like 1, and the caller guarantees seqpos[b] == 0 for every sequence (first prefill, cache.py:236-240): no key
 *               comes from the ring, which lets large chunks run on the wgmma / TMA kernel.
 *   causal = 0: the cache-less forward (transformer_layers.py:72-73,88 with mask=None): every query attends
 *               to every new key of the whole flattened batch; ring, q_start, seqpos are ignored.
 * head_dim 64 (the vision encoder, vision_encoder.py:99): causal = 0 only, on its own wgmma / TMA kernel, scale 64^-0.5.
 */
int mb200_attn_prefill(const void* q, const void* k_new, const void* v_new, const void* cache_k, const void* cache_v,
                       const int32_t* q_start, const int32_t* seqpos, void* out, int64_t T, int64_t B, int64_t max_seqlen,
                       int64_t W, int64_t n_heads, int64_t n_kv_heads, int64_t head_dim, int causal, void* stream);

/* ---------------------------------------------------------------------------------------------
 * FP8 (e4m3) KV cache (Python: BufferCache(..., kv_cache="fp8"), Transformer(..., kv_cache="fp8")).  A storage format with an
 * exact definition, not a new numeric path.  Per layer the ring holds, for each (slot, kv head) row x of hd = 128 bf16 values,
 * 128 e4m3 bytes q in cache_k / cache_v [max_batch, W, KV, hd] and one int8 exponent e in exp_k / exp_v [max_batch, W, KV]:
 *   e    = max(-124, smallest integer with amax|x| <= 448 * 2^e)      (all-zero row: -124)
 *   q[i] = e4m3fn_rn(fp32(x[i]) * 2^-e)                               (2^-e scales exactly; one rounding, |q| <= 448)
 *   x'   = q * 2^e                                                    (exact in bf16; -0 stays -0)
 * The FP8-cache model is the bf16 model with k <- k', v <- v' inserted right after RoPE in every forward that has a cache:
 * attention sees only k' and v', from the ring in decode, from the chunk in first prefill, from both in chunked prefill.
 * The -124 clamp makes the smallest e4m3 subnormal (2^-9) times 2^e the smallest bf16 subnormal, so every x' is a bf16 value.
 * Rows with |x| >= 2^127 are outside the format (their amax can round up to 2^128).  Projection: quantising x' again returns x'
 * (the bytes may differ: a largest |q| of exactly 224 re-quantises as e - 1 and 2q), so prefill quantises k / v in place before
 * attention and writes the ring from k' / v' afterwards.  The readers rebuild the bf16 bits of x' exactly, so
 * mb200_attn_decode_fp8 and mb200_attn_prefill_fp8 are bit-identical to mb200_attn_decode / mb200_attn_prefill on a bf16 ring
 * that holds x'.  head_dim 128 only.
 *
 * mb200_kv_quantize: k, v [T, KV*hd] bf16.  write_back != 0: k, v <- k', v' in place.  cache_rows [T] int32 (or NULL): for
 *   cache_rows[t] >= 0, (q, e) of token t go to ring row cache_rows[t] (slot + b*W, as mb200_kv_ring_write).  Decode: ring only;
 *   prefill: in place before attention, then ring only from k' / v' after it.
 * mb200_attn_decode_fp8: mb200_attn_decode reading the e4m3 ring and its exponents.  Workspace: as mb200_attn_decode (the
 *   e4m3 ring needs no scratch of its own, so mb200_workspace_bytes is unchanged).
 * mb200_attn_prefill_fp8: mb200_attn_prefill (causal 1 or 2) reading old keys from the e4m3 ring; k_new / v_new must already
 *   hold k' / v'.  causal = 2 reads no ring row and runs the bf16 kernels.
 */
int mb200_kv_quantize(void* k, void* v, int write_back, void* cache_k, void* cache_v, int8_t* exp_k, int8_t* exp_v,
                      const int32_t* cache_rows, int64_t T, int64_t n_kv_heads, int64_t head_dim, void* stream);
int mb200_attn_decode_fp8(const void* q, const void* cache_k, const void* cache_v, const int8_t* exp_k, const int8_t* exp_v,
                          const int32_t* kv_len, void* out, int64_t B, int64_t W, int64_t n_heads, int64_t n_kv_heads,
                          int64_t head_dim, int64_t n_splits, void* workspace, size_t workspace_bytes, void* stream);
int mb200_attn_prefill_fp8(const void* q, const void* k_new, const void* v_new, const void* cache_k, const void* cache_v,
                           const int8_t* exp_k, const int8_t* exp_v, const int32_t* q_start, const int32_t* seqpos, void* out,
                           int64_t T, int64_t B, int64_t max_seqlen, int64_t W, int64_t n_heads, int64_t n_kv_heads,
                           int64_t head_dim, int causal, void* stream);

/* ---------------------------------------------------------------------------------------------
 * out = residual + bf16( x @ W^T )   (bf16 add, one more rounding).
 * Replaces wo + residual (transformer_layers.py:93,166) and w2 + residual (:106,:168).
 *   x [T, K]; w [N, K]; residual, out [T, N] (out may alias residual).  residual = NULL: plain linear.
 */
int mb200_linear_residual(const void* x, const void* w, const void* residual, void* out, int64_t T, int64_t N, int64_t K,
                          void* workspace, size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * nn.Linear with an optional bias and an optional exact-erf GELU (the vision-language adapter, vision_encoder.py:105-117).
 *   out = bf16(x @ W^T + bias)                       gelu = 0   (bias = NULL: bf16(x @ W^T))
 *   out = bf16(gelu_erf(bf16(x @ W^T + bias)))       gelu != 0
 *   x [T, K]; w [N, K]; bias [N] or NULL; out [T, N]
 */
int mb200_linear_bias(const void* x, const void* w, const void* bias, void* out, int64_t T, int64_t N, int64_t K, int gelu,
                      void* workspace, size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Vision input data movement (vision_encoder.py, transformer.py:122-161).
 * mb200_vision_patchify: one image [C, H, W] bf16 -> the A operand of the stride-p, bias-free patch Conv2d as a GEMM:
 *     out [(H/p) * (W/p), k_pad] bf16, row py * (W/p) + px, column c*p*p + ky*p + kx (the conv weight's flatten order),
 *     columns >= C*p*p zero.  Remainder pixels (H % p, W % p) are dropped, as the convolution floors.
 * mb200_patch_merge: PatchMerger.permute (vision_encoder.py:180-228) of one image of h x w patch features x [h*w, d] ->
 *     out [(h/s) * (w/s), d*s*s], row by * (w/s) + bx, column c*s*s + ky*s + kx = x[(by*s + ky) * w + bx*s + kx, c].
 * mb200_embed_splice: out[t] = feats[number of image tokens before t] where ids[t] == image_token_id, else
 *     emb[ids[t]] (Transformer.embed_vision_language_features).  ids [T] int64; emb [vocab, dim]; feats [n_feats, dim];
 *     out [T, dim]; ordinal [T + 1] int32 scratch (device): on return ordinal[T] holds the number of image tokens -- the
 *     caller compares it with n_feats.  Rows that would read past feats or emb are written as zeros.
 */
int mb200_vision_patchify(const void* image, void* out, int64_t C, int64_t H, int64_t W, int64_t patch, int64_t k_pad, void* stream);
int mb200_patch_merge(const void* x, void* out, int64_t h, int64_t w, int64_t s, int64_t d, void* stream);
int mb200_embed_splice(const int64_t* ids, const void* emb, const void* feats, void* out, int32_t* ordinal, int64_t T, int64_t dim,
                       int64_t vocab, int64_t n_feats, int64_t image_token_id, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Fused FFN input: RMSNorm -> packed gate/up projection -> bf16(silu(a)) * b.
 * Replaces ffn_norm + w1, w3, silu, mul (transformer_layers.py:167,106).
 *   x [T, dim]; norm_w [dim] (NULL = x is already normed, used by MoE experts);
 *   w13 [2*hidden, dim]: row 2i = w1[i] (gate), row 2i+1 = w3[i] (up);  g_out [T, hidden]
 */
int mb200_ffn_gateup(const void* x, const void* norm_w, const void* w13, void* g_out, int64_t T, int64_t dim,
                     int64_t hidden, float eps, void* workspace, size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Un-merged LoRA adapters (params.json `lora` block: every wq/wk/wv/wo/w1/w2/w3 of the text layers is a LoRALinear,
 * lora.py:22-89).  Each *_lora entry point below takes the arguments of its counterpart plus one adapter and computes, for every
 * output column n of the packed weight, following LoRALinear.forward (lora.py:71-74) with xn = the (normed) input:
 *   a   = bf16(xn @ a_w^T)            [T, rank_cols]  lora_A of every segment, fp32 accumulation       -> a_buf
 *   l   = bf16(a  @ b_w^T)            [T, N]          lora_B                                             -> l_buf
 *   y   = bf16(xn @ W^T)                              the base Linear, as in the counterpart
 *   out = bf16(y + bf16(l * scaling))                 `linear(x) + lora * scaling`
 * and then the counterpart's epilogue on `out` unchanged (RoPE + ring scatter / SiLU*mul / residual add).  RMSNorm runs once per
 * call: the down projection and the base GEMM read the same normed rows.  Adapters that are exactly zero give the counterpart's
 * result bit for bit.
 * Packing (done once at load time by the caller), with S segments of rank r (q,k,v: S = 3; w1,w3: S = 2; wo, w2: S = 1):
 *   a_w  [rank_cols, K]: rows s*r .. s*r + r - 1 = lora_A of segment s; rank_cols = S*r rounded up to a multiple of 64, the
 *        padding rows zero.
 *   b_w  [N, rank_cols]: row n = lora_B of n's segment (row n - first row of the segment) in columns s*r .. s*r + r - 1, zeros
 *        elsewhere.  For w13 the rows interleave like w13: row 2i = [B1[i] | 0], row 2i+1 = [0 | B3[i]].
 *   a_buf [T, rank_cols], l_buf [T, N] bf16 device scratch owned by the caller, 16-byte aligned (the workspace contract is
 *        unchanged; MB200_E_INVALID otherwise); the down
 *        projection splits K across CTAs and keeps its fp32 partials in l_buf before the up projection overwrites it.  The split
 *        bounds and the summation order depend on the shape and the device's SM count only, so results are deterministic.
 * A bank of adapter slots, one slot chosen per token (row_slot non-NULL): a_w and b_w stack n adapters of slot_cols columns each,
 * each packed as above (slot j: a_w rows and b_w columns j*slot_cols .. j*slot_cols + slot_cols - 1; rank_cols = n*slot_cols), and
 * the down projection keeps only token t's own slot:
 *   a[t, c] = bf16(xn[t] . a_w[c])  if c / slot_cols == row_slot[t],  0 otherwise (the whole row when row_slot[t] == -1)
 * The up projection and the combine are unchanged (the zero columns add exact zeros), so token t's result depends only on its
 * input, its slot's adapter and the call's shape -- not on the other tokens' slots -- and a token with slot -1 gets the counterpart's
 * result (up to the sign of a zero).  The call has the same launches as with one adapter.  row_slot NULL: one adapter, as above.
 */
typedef struct mb200_lora {
  const void* a_w;          /* [rank_cols, K] bf16 */
  const void* b_w;          /* [N, rank_cols] bf16 */
  int64_t rank_cols;        /* multiple of 64 */
  float scaling;            /* args.lora.scaling */
  void* a_buf;              /* [T, rank_cols] bf16 scratch */
  void* l_buf;              /* [T, N] bf16 scratch */
  const int32_t* row_slot;  /* [T] int32 device: the slot of each token, in [0, rank_cols / slot_cols) or -1; NULL: one adapter */
  int64_t slot_cols;        /* with row_slot: the columns of one slot, a multiple of 64 that divides rank_cols */
} mb200_lora;
int mb200_attn_qkv_lora(const void* x, const void* norm_w, const void* wqkv, const float* rope, const int32_t* positions,
                        void* q_out, void* k_out, void* v_out, void* cache_k, void* cache_v, const int32_t* cache_rows,
                        int64_t T, int64_t dim, int64_t n_heads, int64_t n_kv_heads, int64_t head_dim, float eps,
                        void* workspace, size_t workspace_bytes, void* stream, const mb200_lora* lora);
int mb200_ffn_gateup_lora(const void* x, const void* norm_w, const void* w13, void* g_out, int64_t T, int64_t dim,
                          int64_t hidden, float eps, void* workspace, size_t workspace_bytes, void* stream, const mb200_lora* lora);
int mb200_linear_residual_lora(const void* x, const void* w, const void* residual, void* out, int64_t T, int64_t N, int64_t K,
                               void* workspace, size_t workspace_bytes, void* stream, const mb200_lora* lora);

/* ---------------------------------------------------------------------------------------------
 * Final RMSNorm + lm head, fp32 logits.  Replaces norm + output + .float() (transformer.py:219,235,240).
 *   x [T, dim]; norm_w [dim]; w_out [V, dim]; logits [T, V] fp32 (each value is a bf16-rounded number).
 */
int mb200_lm_head(const void* x, const void* norm_w, const void* w_out, float* logits, int64_t T, int64_t dim,
                  int64_t vocab, float eps, void* workspace, size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Device-side step state of the batched decode loop.  Replaces BufferCache.get_input_metadata for one-token steps
 * (cache.py:197-263: positions, cache_positions, the padded-keys mask's kv_seqlen) and update_seqlens
 * (cache.py:191-192) with one tiny kernel, so a CUDA graph of the decode step replays without host writes.
 *   seqpos_dev [B] int32 (DEVICE, in/out): tokens cached so far per sequence; incremented by one.
 *   meta_dev   [3B + 1 + n_windows * 2B] int32 (DEVICE, out):
 *              positions[B] | q_start[B+1] | seqpos[B] | per distinct window W: cache_rows[B] (= pos %% W + b*W), kv_len[B]
 *   windows_host [n_windows] int32 (HOST array, n_windows <= 8): the distinct cache sizes (cache.py:13-24), ascending.
 */
int mb200_decode_meta(int32_t* seqpos_dev, int32_t* meta_dev, int64_t B, const int32_t* windows_host, int64_t n_windows,
                      void* stream);

/* ---------------------------------------------------------------------------------------------
 * Token selection and log-probabilities on the device (the per-token tail of generate()).
 *   logits [T, vocab] fp32 (the lm head's output), one CTA per row, nothing of size [T, vocab] is written.
 * mb200_argmax_rows:    out[t] = argmax(logits[t]) with the first index on ties -- `sample` with temperature == 0
 *                       (generate.py:154-158).
 * mb200_logprob_gather: out[t] = log_softmax(logits[t])[target[t]] in fp32 (generate.py:101-117,134-135); rows with
 *                       target[t] < 0 are skipped.
 * mb200_sample_top_p:   one draw per row from softmax(logits / temperature) restricted to the nucleus: a token is kept iff
 *                       the probability mass of the tokens ranked before it is <= top_p (generate.py:151-170; the reference
 *                       hard-codes top_p = 0.8, :126).  uniform [T] fp32 in [0, 1) supplies the randomness (torch.rand on the
 *                       device keeps torch.manual_seed semantics); the draw is the inverse CDF over the kept tokens in index
 *                       order -- same distribution as torch.multinomial on the sorted vector, not the same stream.
 *   out / target: int64 device arrays.
 */
int mb200_argmax_rows(const float* logits, int64_t* out_dev, int64_t T, int64_t vocab, void* stream);
int mb200_logprob_gather(const float* logits, const int64_t* target_dev, float* out_dev, int64_t T, int64_t vocab, void* stream);
int mb200_sample_top_p(const float* logits, const float* uniform_dev, int64_t* out_dev, int64_t T, int64_t vocab,
                       float temperature, float top_p, void* stream);

/* ---------------------------------------------------------------------------------------------
 * mb200_select_tokens: one token per row b < B of logits [B, vocab] fp32 with per-row sampling controls (generate()'s
 * temperature / top_p / random_seed / presence_penalty / frequency_penalty).  One CTA per row; nothing of size [B, vocab] is written.
 *   temperature_dev, top_p_dev, presence_dev, frequency_dev [B] fp32: the row's controls.  The caller keeps them in range
 *                  (temperature >= 0 and finite, top_p in [0, 1], penalties finite); the kernel does not check device values.
 *   counts_dev     [B, vocab] int32 or NULL: c[b, v], how often row b's sequence selected v so far.
 *   step_dev       [B] int32: t, the row's step.
 *   seeds_dev [B] uint64 or uniform_dev [B] fp32 in [0, 1): exactly one is non-NULL.
 * Per row b:
 *   1. l'[v] = fp32(l[v] - pen[v]), pen[v] = fp32(fp32(c[v]) * frequency) then + presence (one fp32 add) where c[v] > 0, all
 *      round-to-nearest without FMA.  With counts_dev NULL, or both penalties of the row 0, l' is l bit for bit.
 *   2. temperature == 0: argmax of l' as mb200_argmax_rows (-0 == +0, NaN above +inf, the first index on ties).
 *   3. otherwise the draw of mb200_sample_top_p on l' at (temperature, top_p) with the uniform u:
 *      seeded: u = (x0 >> 8) * 2^-24 with x0 word 0 of Philox4x32-10, key (seed mod 2^32, seed >> 32), counter (t, 0, 0, 0);
 *      else u = uniform_dev[b].
 *   4. out_dev[b] (int64) = the token; then counts_dev[b, token] += 1 (when given) and step_dev[b] += 1, on the device.
 * No argument changes from step to step, so a stream capture of the call replays as a decode loop's selection.
 */
int mb200_select_tokens(const float* logits, const float* temperature_dev, const float* top_p_dev, const float* presence_dev,
                        const float* frequency_dev, const uint64_t* seeds_dev, const float* uniform_dev, int32_t* step_dev,
                        int32_t* counts_dev, int64_t* out_dev, int64_t B, int64_t vocab, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Speculative decoding: a draft model proposes k tokens per sequence, the target scores the S = k + 1 tokens
 * [last, d_1 .. d_k] of every sequence in one forward (the verify step), and an acceptance rule keeps a prefix.
 *
 * mb200_spec_meta: the metadata block BufferCache.build_metadata_host builds for seqlens = [S] * B at the positions
 *   seqpos_dev, for the chunked-prefill layout (T = B * S):
 *     positions[T] | q_start[B+1] | seqpos[B] | per distinct window W: cache_rows[T], kv_len[B]
 *   seqpos_dev [B] int32 (DEVICE, read only); meta_dev [T + 2B + 1 + n_windows * (T + B)] int32 (DEVICE, out);
 *   windows_host as in mb200_decode_meta.  With it a CUDA graph of the verify step replays without host writes.
 *
 * mb200_spec_accept_greedy / mb200_spec_accept_sample, one CTA per sequence b:
 *   logits [B * S, vocab] fp32: the verify step's rows, row b * S + j scores the token after input j;
 *   tokens_dev [B, S] int64: the verify step's input [last, d_1 .. d_k];
 *   out_dev [B, S] int64 (out): d_1 .. d_n, then the target's token, then -1;  n_dev [B] int32 (out): n, the accepted proposals;
 *   seqpos_dev [B] int32 (in/out): advanced by n + 1 (the cached prefix [last, d_1 .. d_n]).
 *   greedy: a_j = argmax of row j with the first index on ties (as mb200_argmax_rows); n = the longest prefix with d_{j+1} == a_j;
 *           the last token is a_n.
 *   sample: standard speculative sampling (Leviathan et al. 2023; Chen et al. 2023) on the nucleus distributions
 *           mb200_sample_top_p draws from at (temperature, top_p): P_j of target row j, Q_j of draft_logits [B * k, vocab]
 *           row b * k + j.  d_{j+1} is accepted iff u[b, j] * Q_j(d) < P_j(d); at the first rejection the last token is drawn
 *           from max(0, P_j - Q_j) renormalised, after k acceptances from P_k, both with u[b, k]; uniform_dev [B, S] fp32 in [0, 1).
 *   The emitted tokens' log-probabilities are mb200_logprob_gather over (logits, out_dev): rows with -1 are skipped.
 */
int mb200_spec_meta(const int32_t* seqpos_dev, int32_t* meta_dev, int64_t B, int64_t S, const int32_t* windows_host, int64_t n_windows,
                    void* stream);
int mb200_spec_accept_greedy(const float* logits, const int64_t* tokens_dev, int64_t* out_dev, int32_t* n_dev, int32_t* seqpos_dev, int64_t B,
                             int64_t S, int64_t vocab, void* stream);
int mb200_spec_accept_sample(const float* logits, const float* draft_logits, const int64_t* tokens_dev, const float* uniform_dev, int64_t* out_dev,
                             int32_t* n_dev, int32_t* seqpos_dev, int64_t B, int64_t S, int64_t vocab, float temperature, float top_p,
                             void* stream);

/* ---------------------------------------------------------------------------------------------
 * Mixture of experts for T > 1 tokens (prefill, batched decode).  Replaces MoeLayer.forward (moe.py:24-32): the gate Linear,
 * torch.topk on the bf16 router logits, the fp32 softmax over the k selected, and the per-expert torch.where / gather /
 * FeedForward / weighted `results[idx] +=` loop (one host sync per expert) -- with no host round trip at all.
 *
 * mb200_moe_sizes:   buffer sizes for T tokens: tile_rows (m-tile height of the grouped GEMMs: 32 / 64 for decode-sized batches,
 *                    128 otherwise), rows_cap (rows of xs / g / yw / row_w: every expert's segment is padded to a multiple of
 *                    tile_rows), plan_words (int32 words of `plan`).
 * mb200_moe_route:   router + routing plan + gather.
 *     hn [T, dim] bf16 = ffn_norm(h); gate_w [E, dim] bf16 (moe.py:20)
 *     sel [T, k] int32, wts [T, k] bf16: the selected experts of each token in ASCENDING expert index with their routing weights
 *     slot [T, k] int32: row of each (token, expert) pair in the expert-sorted buffers (deterministic: token order per expert)
 *     plan [plan_words] int32: device-side description of the grouped GEMMs' m tiles (count, expert and first row of each)
 *     xs [rows_cap, dim] bf16: hn rows gathered by slot; row_w [rows_cap] bf16: routing weight of each row
 *     shard_rank / shard_world: expert parallelism, this rank owns the experts e % shard_world == shard_rank (1 rank: 0 / 1);
 *     slots are numbered over ALL experts on every rank, tiles and gathered rows cover the local experts only.
 * mb200_moe_grouped_ffn: grouped gate/up GEMM (+ SiLU*mul) -> grouped down GEMM whose epilogue rounds the expert output to bf16,
 *     scales by the routing weight, rounds again (moe.py:31) and stores the row locally AND on every peer (comm->peer_yw: NVLink
 *     stores, the expert-parallel exchange is this epilogue) -> combine: out[t] = residual[t] + sum over the token's k rows in
 *     ascending expert index, every step rounded to bf16 like the reference's `+=`.
 *     w13_host / w2_host: HOST arrays of E device pointers (packed gate/up [2*hidden, dim] and down [dim, hidden] of each expert;
 *     NULL for experts of other ranks).  g [rows_cap, hidden], yw [rows_cap, dim] bf16 scratch; out [T, dim]; residual may be NULL.
 *     comm: NULL when unsharded; otherwise the mapped peer buffers and the handshake words (see mb200_comm_* below).  The combine
 *     kernel signals every peer that this rank's rows are written and waits for every peer's signal; `epoch` counts the calls.
 */
typedef struct mb200_moe_comm {
  int32_t n_ranks, my_rank;
  void* peer_yw[8];     /* yw buffer of the other ranks (mapped), n_ranks - 1 entries */
  void* my_flags;       /* uint32 [n_ranks] in this rank's comm buffer: flags[r] written by rank r */
  void* peer_flags[8];  /* the same array on the other ranks (mapped), n_ranks - 1 entries */
  void* epoch;          /* uint32 device word, local: number of completed calls on this buffer */
  void* done_counter;   /* int32 device word, local, zero */
} mb200_moe_comm;
int mb200_moe_sizes(int64_t T, int64_t n_experts, int64_t top_k, int64_t* tile_rows, int64_t* rows_cap, int64_t* plan_words);
int mb200_moe_route(const void* hn, const void* gate_w, int64_t T, int64_t dim, int64_t n_experts, int64_t top_k, int64_t shard_rank,
                    int64_t shard_world, int32_t* sel, void* wts, int32_t* slot, int32_t* plan, void* xs, void* row_w, void* stream);
int mb200_moe_grouped_ffn(const void* xs, const void* const* w13_host, const void* const* w2_host, const int32_t* plan, const void* row_w,
                          const int32_t* slot, const void* residual, void* g, void* yw, void* out, int64_t T, int64_t dim,
                          int64_t hidden, int64_t n_experts, int64_t top_k, const mb200_moe_comm* comm, void* workspace,
                          size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * FP8 (e4m3) expert weights.  A storage format with an exact definition: per row n of an expert matrix W [N, K] (bf16),
 *     s[n] = fp32(amax_k |W[n, k]| / 448)  (IEEE division; s[n] = 1 for an all-zero row)
 *     q[n, k] = e4m3fn_rn(clamp(fp32(W[n, k] / s[n]), -448, 448))  (IEEE division, round to nearest even)
 *     W'[n, k] = bf16_rn(fp32(float(q[n, k]) * s[n]))
 * and the FP8 model computes exactly what the bf16 model computes with expert weights W': every rounding after the weights is the
 * bf16 path's.
 *
 * mb200_quantize_e4m3_rows: q and s of a bf16 matrix w [rows, K] (K a multiple of 8).  Row n of q starts at q + n * q_row_stride
 *     bytes, its scale is scale[n * scale_stride]: with q_row_stride = 2 * K and scale_stride = 2, w1 and w3 (offset by one row
 *     and one scale) fill the interleaved rows of the packed gate/up matrix (row 2i = w1[i], row 2i + 1 = w3[i]).
 * mb200_moe_grouped_ffn_fp8: mb200_moe_grouped_ffn with e4m3 experts: w13_host / w2_host are HOST arrays of E device pointers to
 *     q (packed gate/up [2*hidden, dim] and down [dim, hidden], one byte per element), w13_scale_host / w2_scale_host HOST arrays
 *     of E device pointers to their fp32 row scales ([2*hidden] and [dim]); NULL for experts of other ranks.  The grouped GEMMs
 *     load the e4m3 tiles and convert them to W' in shared memory; tile rows, tile width and the stream-K partition are those of
 *     mb200_moe_grouped_ffn for the same plan, except that 128-row calls never run as 2-CTA clusters.
 */
int mb200_quantize_e4m3_rows(const void* w, int64_t rows, int64_t K, void* q, int64_t q_row_stride, float* scale, int64_t scale_stride,
                             void* stream);
int mb200_moe_grouped_ffn_fp8(const void* xs, const void* const* w13_host, const float* const* w13_scale_host, const void* const* w2_host,
                              const float* const* w2_scale_host, const int32_t* plan, const void* row_w, const int32_t* slot,
                              const void* residual, void* g, void* yw, void* out, int64_t T, int64_t dim, int64_t hidden, int64_t n_experts,
                              int64_t top_k, const mb200_moe_comm* comm, void* workspace, size_t workspace_bytes, void* stream);

/* Un-merged LoRA on FP8 experts (LoRALinear on every expert's w1 / w2 / w3, lora.py:71-74).  Each expert Linear [N, K] computes,
 * on the dequantised W' of the FP8 format above and the rows of the MoE row plan:
 *   a = bf16(x A_e^T)    L = bf16(a B_e^T)    y = bf16( bf16(x W'_e^T) + bf16(L * scaling) )
 * for w1 / w3 before SiLU * mul, and for w2 before the routing weight: yw = bf16(w * y).  The combine is unchanged.
 * mb200_moe_lora: one adapter per expert Linear group, in the packed layout of mb200_lora, whose w13 B rows interleave like w13:
 *   a_host / b_host  HOST arrays of E device pointers to A [rank_cols, K] and B [N, rank_cols] (bf16); NULL for experts of other
 *                    ranks, and non-NULL wherever the expert's weights are
 *   a_buf            [rows_cap, rank_cols] bf16 scratch; l_buf [rows_cap, N] bf16 scratch, 16-byte aligned (it doubles as the fp32
 *                    split-K partials of the down projection); rows_cap from mb200_moe_sizes.  The two adapters of a call may share
 *                    their scratch: the w13 stages are done before the w2 stages start.
 * The down projection a is one launch over the plan's tiles (read on the device: no host sync, graph-replayable), its K split into a
 * fixed number of slices summed in a fixed order, so every run gives the same bits; L is the bf16 grouped GEMM with K = rank_cols. */
typedef struct mb200_moe_lora {
  const void* const* a_host;
  const void* const* b_host;
  int64_t rank_cols; /* multiple of 64 */
  float scaling;     /* args.lora.scaling */
  void* a_buf;
  void* l_buf;
} mb200_moe_lora;
int mb200_moe_grouped_ffn_fp8_lora(const void* xs, const void* const* w13_host, const float* const* w13_scale_host, const void* const* w2_host,
                                   const float* const* w2_scale_host, const int32_t* plan, const void* row_w, const int32_t* slot,
                                   const void* residual, void* g, void* yw, void* out, int64_t T, int64_t dim, int64_t hidden,
                                   int64_t n_experts, int64_t top_k, const mb200_moe_comm* comm, void* workspace, size_t workspace_bytes,
                                   void* stream, const mb200_moe_lora* lora13, const mb200_moe_lora* lora2);

/* INT4 expert weights: the INT4 format of the dense Linears (see mb200_quantize_int4_groups below) applied to every expert matrix;
 * each expert's w1 / w3 fill the interleaved w13 rows (row 2i = w1[i], row 2i + 1 = w3[i]) through the quantiser's row strides.
 * mb200_moe_grouped_ffn_int4: mb200_moe_grouped_ffn with INT4 experts: w13_host / w2_host are HOST arrays of E device pointers to
 *     the codes (uint8 [2*hidden, dim/2] and [dim, hidden/2], 16-byte aligned), w13_gscale_host / w2_gscale_host HOST arrays of E
 *     device pointers to their bf16 group scales ([2*hidden, dim/128] and [dim, hidden/128]); NULL for experts of other ranks.
 *     dim and hidden must be multiples of 128 (else MB200_E_INVALID).  The grouped GEMMs form W' in shared memory; tile rows, tile
 *     width and the stream-K partition are those of mb200_moe_grouped_ffn for the same plan, except that 128-row calls never run as
 *     2-CTA clusters.  Every tile sums the same W' tiles in the same k order as the bf16 call, so the result equals
 *     mb200_moe_grouped_ffn on W' bit for bit at every T. */
int mb200_moe_grouped_ffn_int4(const void* xs, const void* const* w13_host, const void* const* w13_gscale_host, const void* const* w2_host,
                               const void* const* w2_gscale_host, const int32_t* plan, const void* row_w, const int32_t* slot,
                               const void* residual, void* g, void* yw, void* out, int64_t T, int64_t dim, int64_t hidden, int64_t n_experts,
                               int64_t top_k, const mb200_moe_comm* comm, void* workspace, size_t workspace_bytes, void* stream);

/* Buffers that other ranks (one process per GPU) can write: plain cudaMalloc + CUDA IPC.  alloc zero-fills and synchronises;
 * export writes the 64-byte IPC handle to pass to the other processes (e.g. torch.distributed.all_gather_object); open maps a
 * peer's buffer into this process (peer access over NVLink is enabled lazily).  These are the only entry points that allocate. */
int mb200_comm_alloc(size_t bytes, void** ptr_out);
int mb200_comm_free(void* ptr);
int mb200_comm_export(void* ptr, void* handle_out64);
int mb200_comm_open(const void* handle64, void** ptr_out);
int mb200_comm_close(void* ptr);

/* Upper bound of the scratch any entry point above needs for up to T tokens of this geometry. */
size_t mb200_workspace_bytes(int64_t T, int64_t dim, int64_t n_heads, int64_t n_kv_heads, int64_t head_dim,
                             int64_t hidden, int64_t vocab, int64_t max_batch);

/* ---------------------------------------------------------------------------------------------
 * One whole decode step (batch 1) as ONE persistent cooperative kernel: embedding row -> n_layers x
 * [RMSNorm+QKV+RoPE+ring write | GQA attention over the ring | wo+residual | RMSNorm+gate/up+SiLU*mul |
 * down+residual] -> final RMSNorm + lm head.  Replaces one Transformer.forward(next_token, seqlens=[1], cache)
 * call of the decode loop (generate.py:139 -> transformer.py:163-242) including every per-layer library call.
 * Weights stream through a shared-memory ring fed by TMA bulk copies that keep prefetching across the phase
 * (grid) barriers, which is what lets a batch-1 step approach the HBM roofline.
 *   layers_dev   [n_layers] mb200_layer_desc in DEVICE memory (pointers to this layer's packed weights + ring)
 *   windows_dev  [n_layers] int32 ring size W of each layer
 *   token_dev    device int64 scalar (e.g. the previous step's argmax); pos = its absolute position;
 *                batch_row = which row of the [max_batch, W, KV, hd] cache this sequence occupies
 *   logits       [vocab] fp32
 *   next_token_dev  optional device int64: greedy argmax of the logits, first index on ties (torch.argmax, generate.py:156);
 *                NULL to skip.  Feeding it back as token_dev makes the greedy loop one launch per token, nothing on the host.
 *   n_experts/top_k  0/0 for dense FeedForward layers.  Mixture of experts (moe.py:16-32): the layer descriptors' w13/w2 are
 *                ignored; moe_gate_dev [n_layers] (router weight [E, dim]), moe_w13_dev / moe_w2_dev [n_layers * E] are DEVICE arrays
 *                of device pointers.  Router, top-k, softmax over the k and the ascending-expert bf16 accumulation run in-kernel.
 * Requires a device that can co-schedule one CTA per SM (cooperative launch).
 */
typedef struct mb200_layer_desc {
  const void* wqkv;      /* [(H+2KV)*hd, dim] */
  const void* wo;        /* [dim, H*hd] */
  const void* w13;       /* [2*hidden, dim], rows interleaved w1/w3 */
  const void* w2;        /* [dim, hidden] */
  const void* attn_norm; /* [dim] */
  const void* ffn_norm;  /* [dim] */
  void* cache_k;         /* [max_batch, W, KV, hd] */
  void* cache_v;
} mb200_layer_desc;

int mb200_decode_step(const mb200_layer_desc* layers_dev, const int32_t* windows_dev, int64_t n_layers, const void* emb,
                      const void* final_norm, const void* w_out, const float* rope, const int64_t* token_dev, int64_t pos,
                      int64_t batch_row, float* logits, int64_t* next_token_dev, int64_t dim, int64_t hidden, int64_t n_heads, int64_t n_kv_heads,
                      int64_t head_dim, int64_t vocab, float eps, int64_t n_experts, int64_t top_k, const void* const* moe_gate_dev,
                      const void* const* moe_w13_dev, const void* const* moe_w2_dev, void* workspace, size_t workspace_bytes, void* stream);

#define MB200_SKINNY_MAX_T 4

/* Workspace contract: the first 64 KiB of `workspace` hold self-resetting counters (split-KV arrival counts, the decode
 * kernel's grid-barrier words and epoch, stream-K flags); the caller zero-fills the workspace ONCE when allocating it
 * (torch.zeros) and never writes to it afterwards.
 * Concurrency: a workspace carries state BETWEEN and DURING launches, so all calls that share one workspace must be ordered on
 * one stream (or by events); concurrent streams need one workspace each.  The library keeps no other mutable state that affects
 * results: process-wide state is limited to the debug hooks below, environment switches, and the driver entry point
 * for tensor-map encoding.  mb200_last_error() is thread-local. */
#define MB200_WORKSPACE_HEADER_BYTES (64 * 1024)

/* Debug: a device buffer of [8][n_layers][24] uint64 for 8 sampled CTAs (0, 21, ..., 147: every 21st CTA of a grid of up to
 * 168 SMs); NULL switches it off.  Per CTA and layer, words 0..15 are %globaltimer stamps at the phase boundaries and words
 * 16..21 the nanoseconds the weight producers spent blocked (ADDED to the buffer: zero-fill it before the step).  The layout is
 * spelled out next to mk_stamp in csrc/decode_megakernel.cuh.  Used by scripts/mk_timeline.py to see where a decode step spends
 * time. */
int mb200_debug_set_decode_timeline(void* device_buffer);
/* Debug: [n_sm][n_layers][6][2] uint64 arrive/leave stamps of every CTA at every grid barrier (NULL = off). */
int mb200_debug_set_barrier_timeline(void* device_buffer);
/* Debug, per calling thread: the attention, dense GEMM, mixture-of-experts, vision data-movement and speculative-decoding (spec_meta, spec_accept_*)
 * kernels launched since the last call, one line each, named like the
 * kernel with its template arguments (e.g. "attn_decode_tma_kernel<8>", "gemm_wgmma_kernel<0, 1, 32, 64>").  Copies the log
 * into `out` (NUL-terminated; NULL discards it), clears it, and switches recording on (enable != 0) or off.  MB200_E_INVALID
 * when `out` is too small or launches were dropped because the log filled up.  Tests use it to check which kernel a call chose. */
int mb200_debug_launch_log(int enable, char* out, size_t out_bytes);
/* Debug, host only: byte offsets into `workspace` at which mb200_decode_step leaves q of the last layer ([H*hd] bf16, after RoPE)
 * and that layer's attention output ([H*hd] bf16, head-major) for the given geometry.  Both are 256-byte aligned.  Tests use it
 * to check the attention phases of the step on their own.  (offsets[2] and [3] of mb200_debug_decode_buffers.) */
int mb200_debug_decode_scratch(int64_t dim, int64_t hidden, int64_t n_heads, int64_t n_kv_heads, int64_t head_dim, int64_t n_experts,
                               int64_t top_k, size_t* q_offset, size_t* attn_offset);
/* Debug, host only: byte offsets into `workspace` of every buffer mb200_decode_step leaves behind, for the given geometry, in
 * offsets[6]:
 *   [0] x: the residual stream ping-pong, [2][dim] bf16; layer l writes its output to half (l + 1) & 1, the final norm reads
 *       half n_layers & 1
 *   [1] h of the last layer ([dim] bf16, after wo + residual)
 *   [2] q of the last layer ([H*hd] bf16, after RoPE)
 *   [3] the last layer's attention output ([H*hd] bf16, head-major)
 *   [4] g of the last layer ([hidden] bf16 after SiLU * up; for MoE [top_k][hidden], the selected experts in ascending index)
 *   [5] the attention slice partials ([SM count][H][hd + 2] fp32)
 * Each buffer starts on a 256-byte boundary after the workspace header.  Tests use it to check the phases of the step on their own. */
int mb200_debug_decode_buffers(int64_t dim, int64_t hidden, int64_t n_heads, int64_t n_kv_heads, int64_t head_dim, int64_t n_experts,
                               int64_t top_k, size_t* offsets);
/* Host only: MB200_OK when mb200_decode_step accepts these shapes on a device with `smem_optin` bytes of opt-in shared memory
 * per block (<= 0: the current device's), else MB200_E_INVALID with the reason in mb200_last_error().  The same checks run at the
 * start of mb200_decode_step: head_dim, H/KV, KV <= 8, the K chunking of dim / hidden / H*hd, an even vocab, the MoE limits and
 * a ring of at least 9 stages next to the activation buffer (top_k * hidden bf16 for MoE). */
int mb200_decode_step_supported(int64_t dim, int64_t hidden, int64_t n_heads, int64_t n_kv_heads, int64_t head_dim, int64_t vocab,
                                int64_t n_experts, int64_t top_k, int64_t smem_optin);

/* ---------------------------------------------------------------------------------------------
 * FP8 (e4m3) dense weights (Python: Transformer(..., dense_weights="fp8")).  The storage format is that of the FP8 experts: per row
 * n of a Linear's weight W [N, K], s[n] = fp32(amax_k |W[n, k]| / 448) (1 for an all-zero row) and
 * q[n, k] = e4m3fn_rn(clamp(fp32(W[n, k] / s[n]), -448, 448)), written by mb200_quantize_e4m3_rows.  The compute is different
 * from the experts' W' contract: the scale leaves the dot product,
 *     acc[t, n] = fp32 sum over k of x[t, k] * float(q[n, k])      (any order: the operand is q itself, converted exactly)
 *     y[t, n]   = bf16(fp32(s[n] * acc[t, n]))                      (one fp32 product, then the Linear's bf16 rounding)
 * followed by the mode's own epilogue on y exactly as in the bf16 entry points (residual add, SiLU * mul, RoPE + ring scatter).
 * Every e4m3 value is a bf16 value, so the tensor-core kernels feed q to the same bf16 MMAs.  The FP8 dense model is not bit-identical
 * to any bf16 model.
 *
 * mb200_attn_qkv_fp8, mb200_ffn_gateup_fp8, mb200_linear_residual_fp8: the counterpart's arguments with the weight replaced by
 *     w_q (e4m3 [N, K], one byte per element; wqkv rows cat(q, k, v), w13 rows interleaved w1 / w3) and w_scale (fp32 [N]).
 *     Kernel choice is mb200_linear's (T <= 4: weight-streaming GEMV; 5..128 tokens with N % 128 == 0: stream-K; else wgmma, single
 *     CTA at the bf16 tile width); a shape the bf16 path would run on mma.sync (K % 64 != 0, or N not a multiple of 32 below 128
 *     tokens, of 128 or 192 from 128 tokens on) returns MB200_E_INVALID.
 * mb200_decode_step_fp8: mb200_decode_step for a dense model whose layer matrices are e4m3: layers_dev is a DEVICE array of
 *     mb200_layer_desc_fp8.  The norms, the K/V ring, the embedding and the lm head stay bf16.  mb200_decode_step_fp8_supported is
 *     its mb200_decode_step_supported (dense shapes only).
 */
int mb200_attn_qkv_fp8(const void* x, const void* norm_w, const void* w_q, const float* w_scale, const float* rope, const int32_t* positions,
                       void* q_out, void* k_out, void* v_out, void* cache_k, void* cache_v, const int32_t* cache_rows, int64_t T, int64_t dim,
                       int64_t n_heads, int64_t n_kv_heads, int64_t head_dim, float eps, void* workspace, size_t workspace_bytes, void* stream);
int mb200_ffn_gateup_fp8(const void* x, const void* norm_w, const void* w_q, const float* w_scale, void* g_out, int64_t T, int64_t dim,
                         int64_t hidden, float eps, void* workspace, size_t workspace_bytes, void* stream);
int mb200_linear_residual_fp8(const void* x, const void* w_q, const float* w_scale, const void* residual, void* out, int64_t T, int64_t N,
                              int64_t K, void* workspace, size_t workspace_bytes, void* stream);

typedef struct mb200_layer_desc_fp8 {
  mb200_layer_desc layer;  /* wqkv / wo / w13 / w2 point to e4m3 matrices of the shapes above */
  const float* wqkv_scale; /* [(H+2KV)*hd] */
  const float* wo_scale;   /* [dim] */
  const float* w13_scale;  /* [2*hidden] */
  const float* w2_scale;   /* [dim] */
} mb200_layer_desc_fp8;

int mb200_decode_step_fp8(const mb200_layer_desc_fp8* layers_dev, const int32_t* windows_dev, int64_t n_layers, const void* emb,
                          const void* final_norm, const void* w_out, const float* rope, const int64_t* token_dev, int64_t pos,
                          int64_t batch_row, float* logits, int64_t* next_token_dev, int64_t dim, int64_t hidden, int64_t n_heads,
                          int64_t n_kv_heads, int64_t head_dim, int64_t vocab, float eps, void* workspace, size_t workspace_bytes, void* stream);
int mb200_decode_step_fp8_supported(int64_t dim, int64_t hidden, int64_t n_heads, int64_t n_kv_heads, int64_t head_dim, int64_t vocab,
                                    int64_t smem_optin);

/* ---------------------------------------------------------------------------------------------
 * FP8 activations for FP8 dense weights (Python: Transformer(..., dense_weights="fp8", prefill_compute="fp8")).  Opt-in numeric
 * mode of the prefill-sized Linears: both GEMM operands are e4m3 and the product runs on the FP8 tensor cores.
 *
 * Which calls.  Every call of the three _fp8a8 entry points that the _fp8 dispatch above would give to the prefill wgmma kernel
 * (T >= 128 and not stream-K; stream-K takes T <= 128 when N % 128 == 0, so T >= 129 for every Linear of the real shapes).  Every
 * other call (GEMV, stream-K, small-batch wgmma) is the _fp8 entry point's call, kernel and bits.  The rule depends on the call's
 * token count only: chunks of <= 128 tokens compute exactly what the FP8 model computes.
 *
 * Activations.  Row t of the Linear's bf16 input v (wqkv, w13: the RMSNorm output, the same bf16 values mb200_rmsnorm gives; wo, w2:
 * x itself), in fp32:
 *     a[t]      = max_k |v[t, k]|
 *     e[t]      = 0 if a[t] == 0, else the smallest integer with a[t] <= 448 * 2^e[t]     (int32, in [-141, 120] for bf16 inputs)
 *     xq[t, k]  = e4m3fn_rn(v[t, k] * 2^-e[t])       (the power of two scales exactly: the e4m3 rounding is the only one)
 *     A row holding an inf or a NaN gets e[t] = 0 and every xq[t, k] = NaN (0x7f): every output of that token is NaN.
 * Product.  The tensor cores sum each k-block of 128 products float(xq[t, k]) * float(q[n, k]) (k = 128 j .. 128 j + 127) from
 *     zero, and each block sum is added into an IEEE fp32 accumulator on the CUDA cores, blocks in ascending order (promotion
 *     interval: one k-block of 128).  Inside a k-block the sum is the tensor core's, about 14 significant bits wide: on an H100
 *     (tests/test_gpu_fp8_prefill.py) the block sum of 2^16 + 2^j keeps 2^j for j >= 3 and drops it for j <= 2.  It is exact
 *     whenever every product and partial sum of the block is a multiple of a power of two p and below 2^13 * p.
 *         acc[t, n] = fp32 sum over j of block_j[t, n]
 * Output.  y[t, n] = bf16(fp32(fp32(s[n] * acc[t, n]) * 2^e[t])), then the mode's own epilogue exactly as in the _fp8 entry
 *     points (residual add, SiLU * mul, RoPE + ring scatter).
 *
 * mb200_attn_qkv_fp8a8, mb200_ffn_gateup_fp8a8, mb200_linear_residual_fp8a8: the _fp8 signatures.  A call in the FP8-activation
 *     regime needs K % 128 == 0 and N % 64 == 0 (MB200_E_INVALID otherwise) and writes xq and e into the normed-activation scratch
 *     of the workspace (mb200_workspace_bytes is unchanged).
 * mb200_quantize_act_e4m3: xq (e4m3 [T, dim], 8-byte aligned) and e (int32 [T]) of x (bf16 [T, dim], dim % 8 == 0), or of its RMSNorm
 *     output with weight norm_w when norm_w is not NULL.  The quantiser the entry points above run.
 */
int mb200_attn_qkv_fp8a8(const void* x, const void* norm_w, const void* w_q, const float* w_scale, const float* rope, const int32_t* positions,
                         void* q_out, void* k_out, void* v_out, void* cache_k, void* cache_v, const int32_t* cache_rows, int64_t T, int64_t dim,
                         int64_t n_heads, int64_t n_kv_heads, int64_t head_dim, float eps, void* workspace, size_t workspace_bytes, void* stream);
int mb200_ffn_gateup_fp8a8(const void* x, const void* norm_w, const void* w_q, const float* w_scale, void* g_out, int64_t T, int64_t dim,
                           int64_t hidden, float eps, void* workspace, size_t workspace_bytes, void* stream);
int mb200_linear_residual_fp8a8(const void* x, const void* w_q, const float* w_scale, const void* residual, void* out, int64_t T, int64_t N,
                                int64_t K, void* workspace, size_t workspace_bytes, void* stream);
int mb200_quantize_act_e4m3(const void* x, const void* norm_w, void* q, int32_t* exps, int64_t T, int64_t dim, float eps, void* stream);

/* ---------------------------------------------------------------------------------------------
 * INT4 dense weights (Python: Transformer(..., dense_weights="int4")).  Each layer Linear's weight W [N, K] (K % 128 == 0) is
 * stored as symmetric 4-bit codes with one bf16 scale per group g of 128 consecutive k of a row, written by
 * mb200_quantize_int4_groups:
 *     a[n, g]  = max over k in group g of |W[n, k]|                                  (fp32)
 *     s[n, g]  = 1 if a == 0, else bf16_rn(fp32(a / 7)), raised to the smallest positive bf16 (2^-133) if that rounds to 0
 *     q[n, k]  = clamp(rint_even(fp32(W[n, k]) / fp32(s[n, g])), -8, 7)                 (IEEE division)
 *     W'[n, k] = bf16_rn(fp32(q) * fp32(s))                                            (q * s is exact in fp32: one rounding)
 * Storage: codes uint8 [N, K/2], byte j of a row holding q + 8 of k = 2j in its low nibble and of k = 2j + 1 in its high nibble;
 * scales bf16 [N, K/128].  The packing is the bf16 one: wqkv rows cat(q, k, v), w13 rows interleaved w1 / w3.  W' is never
 * materialised in memory: the kernels form it in registers or shared memory with two exact bf16x2 instructions per pair
 * ((0x4300 | (q + 8)) - 136 = q, then one bf16 multiply by s).
 * The INT4 model computes what the bf16 model computes with weights W': every Linear is bf16(x W'^T) with fp32 accumulation,
 * followed by the mode's own epilogue exactly as in the bf16 entry points.  From 128 tokens on the kernels also keep the bf16
 * kernels' tiles and k order, so their results equal the bf16 entry point on W' bit for bit.
 *
 * mb200_quantize_int4_groups: w bf16 [rows, K] contiguous; code row r at q + r * q_row_stride bytes, scale row r at
 *     scale + r * scale_row_stride elements (strided rows: w1 / w3 land in the interleaved w13 rows).
 * mb200_attn_qkv_int4, mb200_ffn_gateup_int4, mb200_linear_residual_int4: the counterpart's arguments with the weight replaced by
 *     w_q (codes [N, K/2]) and w_gscale (bf16 scales [N, K/128]).  Kernel choice is that of the _fp8 trio (T <= 4: weight-streaming
 *     GEMV; 5..128 tokens with N % 128 == 0: stream-K; else wgmma, single CTA at the bf16 tile width); K % 128 != 0, or a shape the
 *     bf16 path would run on mma.sync, returns MB200_E_INVALID.
 */
int mb200_quantize_int4_groups(const void* w, int64_t rows, int64_t K, void* q, int64_t q_row_stride, void* scale, int64_t scale_row_stride,
                               void* stream);
int mb200_attn_qkv_int4(const void* x, const void* norm_w, const void* w_q, const void* w_gscale, const float* rope, const int32_t* positions,
                        void* q_out, void* k_out, void* v_out, void* cache_k, void* cache_v, const int32_t* cache_rows, int64_t T, int64_t dim,
                        int64_t n_heads, int64_t n_kv_heads, int64_t head_dim, float eps, void* workspace, size_t workspace_bytes, void* stream);
int mb200_ffn_gateup_int4(const void* x, const void* norm_w, const void* w_q, const void* w_gscale, void* g_out, int64_t T, int64_t dim,
                          int64_t hidden, float eps, void* workspace, size_t workspace_bytes, void* stream);
int mb200_linear_residual_int4(const void* x, const void* w_q, const void* w_gscale, const void* residual, void* out, int64_t T, int64_t N,
                               int64_t K, void* workspace, size_t workspace_bytes, void* stream);

/* Debug: CTAs of attn_decode_tma_kernel<rep> (rep = H/KV) resident per SM on the current device, from
 * cudaOccupancyMaxActiveBlocksPerMultiprocessor at the kernel's launch configuration. */
int mb200_debug_attn_decode_occupancy(int64_t rep, int* blocks_per_sm);

/* Test-only: CUDA-core fp32 GEMM c[T, N] = a[T, K] w[N, K]^T used to cross-check the tensor-core kernels. */
int mb200_test_gemm_naive(const void* a, const void* w, float* c, int64_t T, int64_t N, int64_t K, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MISTRAL_B200_H_ */
