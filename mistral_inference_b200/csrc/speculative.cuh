// Speculative decoding on the device: the verify step's metadata and the acceptance of the draft's proposals.
//
//   spec_meta_kernel           the metadata block of a verify forward (S = k + 1 tokens per sequence) at device-side positions
//   spec_accept_greedy_kernel  longest prefix of proposals equal to the target's argmax, then the target's argmax
//   spec_accept_sample_kernel  speculative sampling (Leviathan et al. 2023; Chen et al. 2023) on the nucleus distributions
//
// A round verifies the S tokens [last, d1 .. dk] of every sequence in one forward; row j of its logits is the target's
// distribution for the token after input j, i.e. for proposal d_{j+1} (j < k) or for the bonus token (j = k).  Both acceptance
// kernels write, per sequence b: out[b, 0 .. n_b] (d_1 .. d_{n_b}, then the target's own token), out[b, j] = -1 for j > n_b,
// n_out[b] = n_b, and advance seqpos[b] by n_b + 1 -- the cached prefix [last, d_1 .. d_{n_b}] -- so the next round's verify
// step reads its positions from the device.  One CTA per sequence; the row passes are those of sampling.cuh.
#pragma once
#include "elementwise.cuh"
#include "sampling.cuh"

namespace mb200 {

// The block BufferCache.build_metadata_host builds for seqlens = [S] * B at positions seqpos (cache.py:197-263), for the chunked
// prefill layout: positions[T] | q_start[B + 1] | seqpos[B] | per distinct window W: cache_rows[T], kv_len[B]  (T = B * S).
// seqpos is read, not advanced: the acceptance kernel advances it by what the round keeps.
struct SpecMetaParams {
  const int32_t* seqpos;  // [B]
  int32_t* meta;          // [T + 2B + 1 + n_w * (T + B)]
  int B, S, n_w;
  int windows[kMaxWindows];
};
__global__ void spec_meta_kernel(const SpecMetaParams p) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int T = p.B * p.S;
  int32_t* q_start = p.meta + T;
  int32_t* seqpos_out = q_start + p.B + 1;
  int32_t* per_w = seqpos_out + p.B;
  if (i < T) {  // one token
    const int b = i / p.S, local = i - b * p.S;
    const int pos = p.seqpos[b] + local;
    p.meta[i] = pos;
    int32_t* o = per_w;
    for (int j = 0; j < p.n_w; ++j) {
      const int W = p.windows[j];
      o[i] = local >= p.S - W ? pos % W + b * W : -1;  // only the last W tokens of the chunk are cached (cache.py:226)
      o += T + p.B;
    }
  }
  if (i <= p.B) {  // one sequence, and q_start's end
    q_start[i] = i * p.S;
    if (i == p.B) return;
    const int sp = p.seqpos[i];
    seqpos_out[i] = sp;
    int32_t* o = per_w + T;
    for (int j = 0; j < p.n_w; ++j) {
      const int W = p.windows[j];
      o[i] = min(sp + min(p.S, W), W);
      o += T + p.B;
    }
  }
}

// Greedy: a_j = argmax(row j) with the first index on ties (mb200_argmax_rows); n = the longest prefix with d_{j+1} == a_j.
__global__ void __launch_bounds__(SP_THREADS) spec_accept_greedy_kernel(const float* __restrict__ logits, const long long* __restrict__ tokens,
                                                                        long long* __restrict__ out, int* __restrict__ n_out,
                                                                        int* __restrict__ seqpos, int S, int V) {
  const int b = blockIdx.x;
  const long long* tk = tokens + (int64_t)b * S;
  long long* o = out + (int64_t)b * S;
  __shared__ int best_sm;
  int n = S - 1;
  for (int j = 0; j < S; ++j) {
    const int a = block_argmax(logits + ((int64_t)b * S + j) * V, V);
    if (threadIdx.x == 0) best_sm = a;
    __syncthreads();
    const int best = best_sm;  // the next call's first barrier orders this read before thread 0's next write
    if (j == S - 1 || (long long)best != tk[j + 1]) {
      n = j;
      if (threadIdx.x == 0) o[j] = best;
      break;
    }
    if (threadIdx.x == 0) o[j] = tk[j + 1];
  }
  if (threadIdx.x == 0) {
    for (int j = n + 1; j < S; ++j) o[j] = -1;
    n_out[b] = n;
    seqpos[b] += n + 1;
  }
}

// The nucleus distribution of one row as speculative sampling needs it: P(i) = prob(i) / Z_kept for prob(i) >= tau, else 0 --
// exactly the distribution mb200_sample_top_p draws from.
struct NucleusDist {
  NucleusRow r;
  float tau, inv_kept;
  __device__ __forceinline__ float kept(int i) const {  // prob(i) on the kept set (the unnormalised weights of sample_top_p)
    const float p = r.prob(i);
    return p >= tau ? p : 0.f;
  }
  __device__ __forceinline__ float at(int i) const { return kept(i) * inv_kept; }
};

__device__ __forceinline__ NucleusDist nucleus_dist(const float* __restrict__ row, int V, float inv_temperature, float top_p, float* scratch) {
  NucleusDist d;
  d.r = nucleus_row(row, V, inv_temperature, scratch);
  d.tau = nucleus_tau(d.r, V, top_p, scratch);
  float s = 0.f;
  for (int i = threadIdx.x; i < V; i += SP_THREADS) s += d.kept(i);
  d.inv_kept = 1.0f / block_sum(s, scratch);
  return d;
}

// Sampled: for j < k accept d_{j+1} iff u[b, j] < P_j(d) / Q_j(d) (as u * Q < P); at the first rejection draw from
// max(0, P_j - Q_j) renormalised; after k acceptances draw the bonus token from P_k.  P_j: target row j, Q_j: draft row j
// (draft_logits [B * k, V], row b * k + j), both through the nucleus of sampling.cuh at the same temperature and top_p.  The
// final draw uses u[b, k].  A residual that rounds to nothing everywhere (P_j == Q_j up to rounding, where a rejection has
// probability 0) draws from P_j instead.
__global__ void __launch_bounds__(SP_THREADS) spec_accept_sample_kernel(const float* __restrict__ logits, const float* __restrict__ draft_logits,
                                                                        const long long* __restrict__ tokens, const float* __restrict__ uniform,
                                                                        long long* __restrict__ out, int* __restrict__ n_out,
                                                                        int* __restrict__ seqpos, int S, int V, float inv_temperature,
                                                                        float top_p) {
  const int b = blockIdx.x, k = S - 1;
  const long long* tk = tokens + (int64_t)b * S;
  const float* u = uniform + (int64_t)b * S;
  long long* o = out + (int64_t)b * S;
  __shared__ float scratch[SP_WARPS];
  int n = k, last = -1;
  for (int j = 0; j < k; ++j) {
    const NucleusDist p = nucleus_dist(logits + ((int64_t)b * S + j) * V, V, inv_temperature, top_p, scratch);
    const NucleusDist q = nucleus_dist(draft_logits + ((int64_t)b * k + j) * V, V, inv_temperature, top_p, scratch);
    const int d = (int)tk[j + 1];
    if (u[j] * q.at(d) < p.at(d)) {
      if (threadIdx.x == 0) o[j] = d;
      continue;
    }
    n = j;
    // __fsub_rn: the difference of the two ROUNDED probabilities the acceptance test compared.  A contracted
    // fma(kept_p, inv_kept_p, -q) leaves the product's rounding error where P == Q, a residual of pure noise.
    last = block_draw([&](int i) { return fmaxf(__fsub_rn(p.at(i), q.at(i)), 0.f); }, V, u[k]);
    if (last < 0) last = block_draw([&](int i) { return p.kept(i); }, V, u[k]);
    break;
  }
  if (n == k) {
    const NucleusDist p = nucleus_dist(logits + ((int64_t)b * S + k) * V, V, inv_temperature, top_p, scratch);
    last = block_draw([&](int i) { return p.kept(i); }, V, u[k]);
  }
  if (threadIdx.x == 0) {
    o[n] = last;
    for (int j = n + 1; j < S; ++j) o[j] = -1;
    n_out[b] = n;
    seqpos[b] += n + 1;
  }
}

}  // namespace mb200
