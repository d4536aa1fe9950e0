// Layout of the workspace every entry point takes (include/mistral_b200.h).  The first MB200_WORKSPACE_HEADER_BYTES are
// persistent: self-resetting counters, zero-filled once by the caller.  After the header lies per-call scratch; the scratch of
// different entry points overlaps, which is safe because calls on one workspace are stream ordered.  Entry points address the
// workspace through the names and functions below only.
#pragma once
#include "common.cuh"

namespace mb200 {

inline size_t align256(size_t v) { return (v + 255) & ~(size_t)255; }

struct WsRegion {
  size_t offset, bytes;
  constexpr size_t end() const { return offset + bytes; }
};

constexpr size_t kWsHeader = MB200_WORKSPACE_HEADER_BYTES;

// Stream-K GEMMs (gemm_streamk.cuh, moe.cuh) launch at most SK_MAX_CTAS CTAs; each has one flag in the header and one
// [128 x 128] fp32 partial slot after it.
constexpr int SK_MAX_CTAS = 160;
constexpr size_t SK_PARTIAL_BYTES = (size_t)SK_MAX_CTAS * 128 * 128 * sizeof(float);

// ---- header regions, in ascending offset order ----
constexpr WsRegion kWsSplitKvCounters = {0, 8192};                  // split-KV decode attention: one int per (sequence, kv head)
constexpr WsRegion kWsMkArgmaxCounter = {12288, sizeof(int)};       // decode megakernel: CTAs that have published their argmax
constexpr WsRegion kWsMkBarFlags = {16384, 8 * 128};                // decode megakernel: grid-barrier counters, one per 128-byte line
constexpr WsRegion kWsMkBarEpoch = {20480, sizeof(unsigned)};       // decode megakernel: barriers completed by earlier launches
constexpr WsRegion kWsMkDoneCounter = {20480 + 128, sizeof(int)};   // decode megakernel: CTAs that have finished this launch
constexpr WsRegion kWsSkFlags = {24576, SK_MAX_CTAS * sizeof(unsigned)};  // stream-K: one flag per CTA
constexpr WsRegion kWsMkArgmaxSlots = {32768, 32768};               // decode megakernel: 8 B per CTA = per SM, so up to 4096 SMs

constexpr WsRegion kWsHeaderRegions[] = {kWsSplitKvCounters, kWsMkArgmaxCounter, kWsMkBarFlags, kWsMkBarEpoch,
                                         kWsMkDoneCounter,   kWsSkFlags,         kWsMkArgmaxSlots};
constexpr bool ws_header_regions_disjoint() {
  const int n = (int)(sizeof(kWsHeaderRegions) / sizeof(kWsHeaderRegions[0]));
  for (int i = 0; i + 1 < n; ++i)
    if (kWsHeaderRegions[i].end() > kWsHeaderRegions[i + 1].offset) return false;
  return kWsHeaderRegions[n - 1].end() <= kWsHeader;
}
static_assert(ws_header_regions_disjoint(), "workspace header regions overlap or end past MB200_WORKSPACE_HEADER_BYTES");

// ---- scratch after the header ----
// Stream-K partial slots: SK_PARTIAL_BYTES from the end of the header.
constexpr WsRegion kWsSkPartials = {kWsHeader, SK_PARTIAL_BYTES};
// Activations normed once for a tensor-core GEMM ([T, K] bf16): after the stream-K slots, which that GEMM may use.
inline WsRegion ws_normed(int64_t T, int64_t K) { return {kWsSkPartials.end(), align256((size_t)T * K * 2)}; }
// FP8 activations (prefill_compute="fp8") in the same region: e4m3 codes [T, K], then the int32 exponents [T] on a 256-byte
// boundary.  T*K rounded up to 256 plus 4T bytes fit in the 2*T*K bytes of ws_normed for every K >= 128.
struct WsActE4m3 {
  WsRegion q, exps;
};
inline WsActE4m3 ws_act_e4m3(int64_t T, int64_t K) {
  const WsRegion nr = ws_normed(T, K);
  const WsRegion q = {nr.offset, align256((size_t)T * K)};
  return {q, {q.end(), (size_t)T * sizeof(int32_t)}};
}
// Split-KV decode attention partials: [B, KV, S, rep, hd + 2] fp32 (m, l, acc).
inline WsRegion ws_splitkv_partials(int64_t B, int64_t KV, int64_t S, int64_t rep) {
  return {kWsHeader, (size_t)B * KV * S * rep * (kHeadDim + 2) * sizeof(float)};
}

// Global scratch of mb200_decode_step, as byte offsets: each buffer starts on a 256-byte boundary.
// mb200_debug_decode_buffers (and mb200_debug_decode_scratch) report the offsets from the same function, so tests read what the kernel wrote.
struct DecodeScratch {
  size_t xbuf, hbuf, qbuf, abuf, gbuf, partial, end;
};
inline DecodeScratch decode_scratch(int64_t dim, int64_t hidden, int64_t n_heads, int64_t n_experts, int64_t top_k, int sms) {
  const size_t q_dim = (size_t)n_heads * kHeadDim;
  DecodeScratch s;
  size_t off = kWsHeader;
  auto take = [&](size_t bytes) { const size_t r = off; off += align256(bytes); return r; };
  s.xbuf = take((size_t)2 * dim * 2);
  s.hbuf = take((size_t)dim * 2);
  s.qbuf = take(q_dim * 2);
  s.abuf = take(q_dim * 2);
  s.gbuf = take((size_t)(n_experts ? top_k : 1) * hidden * 2);
  s.partial = take((size_t)sms * n_heads * (kHeadDim + 2) * sizeof(float));  // [slice = CTA][H][m, l, acc[128]]
  s.end = off;
  return s;
}

}  // namespace mb200
