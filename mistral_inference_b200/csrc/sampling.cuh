// Device-side token selection and log-probabilities (SURVEY.md N1): the per-token tail of generate().
//
//   argmax_rows_kernel      greedy pick: torch.argmax(logits, -1) (generate.py:156), first index on ties
//   logprob_gather_kernel   log_softmax(logits, -1)[t, target[t]] (generate.py:101-117,134-135) without materialising [T, V]
//   sample_top_p_kernel     softmax(logits / temperature) -> nucleus (top-p) filter -> one draw (generate.py:151-170)
//   select_tokens_kernel    per-row sampling controls: presence / frequency penalties applied on load, then greedy or nucleus
//                           with the row's own temperature, top_p and (seeded Philox or caller) uniform
// The row argmax, the nucleus and the draw are device functions that the speculative acceptance kernels share.  They read a row
// through a loader (RawRow: the logits as they are; PenalisedRow: the penalised logits), so no penalised copy is ever written.
//
// All three are one CTA per row over fp32 logits [T, V] (the lm head's output).  Roofline: HBM/L2 -- V * 4 bytes per row and
// pass; argmax and logprob are single-pass (online log-sum-exp), top-p re-reads its row (L2 resident) during the threshold
// search.  Reductions are fixed-order (warp shuffles, then warp 0 over the per-warp partials): results are deterministic.
#pragma once
#include "common.cuh"

namespace mb200 {

constexpr int SP_THREADS = 1024;
constexpr int SP_WARPS = SP_THREADS / 32;

// block-wide reductions over SP_THREADS threads; `scratch` holds SP_WARPS values; result broadcast to every thread
__device__ __forceinline__ float block_sum(float v, float* scratch) {
  v = warp_sum(v);
  __syncthreads();  // scratch reuse
  if ((threadIdx.x & 31) == 0) scratch[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = scratch[threadIdx.x & 31];  // SP_WARPS == 32: every lane reads one partial
  t = warp_sum(t);
  return t;
}
__device__ __forceinline__ float block_max(float v, float* scratch) {
  v = warp_max(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) scratch[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = scratch[threadIdx.x & 31];
  t = warp_max(t);
  return t;
}

// A row of fp32 logits as the selection reads it: row(i) is element i.
struct RawRow {
  const float* p;
  __device__ __forceinline__ float operator()(int i) const { return p[i]; }
};

// argmax of one row with the first index on ties; the result is valid in thread 0 (the shared partials may be reused once
// every thread has passed a __syncthreads after the call)
template <typename Row>
__device__ __forceinline__ int block_argmax(const Row& row, int V) {
  unsigned long long best = 0ull;
  for (int i = threadIdx.x; i < V; i += SP_THREADS) best = max(best, argmax_key(row(i), i));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) best = max(best, __shfl_xor_sync(0xffffffffu, best, o));
  __shared__ unsigned long long sm[SP_WARPS];
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = best;
  __syncthreads();
  if (threadIdx.x < 32) {
    best = sm[threadIdx.x];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) best = max(best, __shfl_xor_sync(0xffffffffu, best, o));
  }
  return 0x7fffffff - (int)(best & 0xffffffffull);
}
__device__ __forceinline__ int block_argmax(const float* __restrict__ row, int V) { return block_argmax(RawRow{row}, V); }

__global__ void __launch_bounds__(SP_THREADS) argmax_rows_kernel(const float* __restrict__ logits, long long* __restrict__ out, int V) {
  const int best = block_argmax(logits + (int64_t)blockIdx.x * V, V);
  if (threadIdx.x == 0) out[blockIdx.x] = (long long)best;
}

// out[t] = logits[t, target[t]] - max - log(sum(exp(logits[t, :] - max)))   (fp32, like torch.log_softmax on fp32 logits)
// rows with target[t] < 0 are skipped (out untouched).
__global__ void __launch_bounds__(SP_THREADS) logprob_gather_kernel(const float* __restrict__ logits, const long long* __restrict__ target,
                                                                    float* __restrict__ out, int V) {
  const long long tgt = target[blockIdx.x];
  if (tgt < 0) return;
  const float* row = logits + (int64_t)blockIdx.x * V;
  __shared__ float scratch[SP_WARPS];
  float m = -INFINITY;
  for (int i = threadIdx.x; i < V; i += SP_THREADS) m = fmaxf(m, row[i]);
  m = block_max(m, scratch);
  float s = 0.f;
  for (int i = threadIdx.x; i < V; i += SP_THREADS) s += expf(row[i] - m);
  s = block_sum(s, scratch);
  if (threadIdx.x == 0) out[blockIdx.x] = (row[tgt] - m) - logf(s);
}

// Nucleus sampling, one draw per row.  The reference (generate.py:151-170):
//   probs = softmax(logits / temperature); sort descending; keep token j iff (mass of the tokens ranked before j) <= p;
//   renormalise; torch.multinomial(1).
// Without a sort: token i is kept iff S(p_i) <= top_p with S(q) = sum of probabilities strictly greater than q, i.e. the kept
// set is {i : p_i >= tau} for the smallest probability tau with S(tau) <= top_p; tau is found by bisection on the fp32 bit
// pattern (exact after 32 steps; probabilities are positive, so the patterns are ordered like the values).  The draw is the
// inverse CDF over the kept tokens in index order with the caller's uniform u[row] in [0, 1) -- the same distribution as
// multinomial over the sorted, renormalised vector (order is irrelevant).  Tokens with EQUAL probability at the cut are kept or
// dropped together, where the reference's unstable sort keeps an arbitrary subset of them.
//
// The pieces are shared with the speculative-sampling acceptance (speculative.cuh), which needs the same nucleus of two rows:
//   NucleusRow   softmax(row / temperature): the row maximum m and 1/Z, prob(i) = exp(row[i] / T - m) / Z
//   nucleus_tau  the threshold tau of the kept set {i : prob(i) >= tau}
//   block_draw   inverse-CDF draw over nonnegative weights w(i) in index order
template <typename Row>
struct NucleusRowOf {
  Row row;
  float inv_temperature, m, inv_z;
  __device__ __forceinline__ float prob(int i) const { return expf(row(i) * inv_temperature - m) * inv_z; }
};
using NucleusRow = NucleusRowOf<RawRow>;

template <typename Row>
__device__ __forceinline__ NucleusRowOf<Row> nucleus_row(const Row& row, int V, float inv_temperature, float* scratch) {
  float m = -INFINITY;
  for (int i = threadIdx.x; i < V; i += SP_THREADS) m = fmaxf(m, row(i) * inv_temperature);
  m = block_max(m, scratch);
  float z = 0.f;
  for (int i = threadIdx.x; i < V; i += SP_THREADS) z += expf(row(i) * inv_temperature - m);
  z = block_sum(z, scratch);
  return NucleusRowOf<Row>{row, inv_temperature, m, 1.0f / z};
}
__device__ __forceinline__ NucleusRow nucleus_row(const float* __restrict__ row, int V, float inv_temperature, float* scratch) {
  return nucleus_row(RawRow{row}, V, inv_temperature, scratch);
}

template <typename Row>
__device__ __forceinline__ float nucleus_tau(const NucleusRowOf<Row>& r, int V, float top_p, float* scratch) {
  // bisection on the bit pattern of tau in (0, 1]: invariant S(hi) <= top_p (S(1.0) = 0), S(lo) > top_p or lo = 0
  unsigned lo = 0u, hi = __float_as_uint(1.0f);
  while (hi - lo > 1u) {
    const unsigned mid = lo + (hi - lo) / 2u;
    const float q = __uint_as_float(mid);
    float s = 0.f;
    for (int i = threadIdx.x; i < V; i += SP_THREADS) {
      const float p = r.prob(i);
      s += p > q ? p : 0.f;
    }
    s = block_sum(s, scratch);
    if (s <= top_p)
      hi = mid;
    else
      lo = mid;
  }
  // kept set: p_i >= tau where tau = the smallest ACTUAL probability > lo's value ... any p in (value(lo), value(hi)] equals
  // value(hi) (adjacent floats), so "p >= value(hi)" is exact.  If even the largest probability alone exceeds top_p the first
  // token is still kept (its preceding mass is 0 <= p), which S(p_max) = 0 <= top_p guarantees here too.
  return __uint_as_float(hi);
}

// One draw from the weights w(i) >= 0, i < V: the token where u * sum(w) falls in the prefix sums over index order (u in
// [0, 1)).  Every thread returns the token.  -1 only when every weight is 0.
template <typename Weight>
__device__ __forceinline__ int block_draw(const Weight& weight, int V, float u) {
  __shared__ float warp_mass[SP_WARPS];
  // mass of the weights, then the draw: thread-contiguous chunks so that a prefix over threads is a prefix over indices
  const int per = (V + SP_THREADS - 1) / SP_THREADS;
  const int i0 = threadIdx.x * per, i1 = min(V, i0 + per);
  float mine = 0.f;
  for (int i = i0; i < i1; ++i) mine += weight(i);
  // inclusive scan over threads: within the warp, then over the warps
  float incl = mine;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float t = __shfl_up_sync(0xffffffffu, incl, o);
    if ((threadIdx.x & 31) >= o) incl += t;
  }
  __syncthreads();
  if ((threadIdx.x & 31) == 31) warp_mass[threadIdx.x >> 5] = incl;
  __syncthreads();
  float before = 0.f, total = 0.f;
  for (int w = 0; w < SP_WARPS; ++w) {
    const float wm = warp_mass[w];
    if (w < (int)(threadIdx.x >> 5)) before += wm;
    total += wm;
  }
  // the winner is the LOWEST weighted thread with target < upper(t).  Each lane's scan associates its fp32 additions
  // differently, so a zero-mass thread's upper(t) can exceed its weighted predecessor's by an ulp; a rule that also required
  // target >= upper(t-1) would leave that interval to nobody.  With this rule every target below the last weighted upper(t) has
  // exactly one claimant, and the claimant's walk starts at upper(t-1): a target below it takes the thread's first weighted
  // token, the inverse CDF's neighbour across the ulp.  Only a target past every weighted upper(t) falls through below.
  __shared__ float upper_sm[SP_THREADS];
  __shared__ int winner_tid, winner;
  const float upper = before + incl;
  upper_sm[threadIdx.x] = upper;
  if (threadIdx.x == 0) {
    winner_tid = SP_THREADS;
    winner = -1;
  }
  __syncthreads();
  const float lower = threadIdx.x ? upper_sm[threadIdx.x - 1] : 0.f;
  total = upper_sm[SP_THREADS - 1];
  const float target = u * total;
  if (mine > 0.f && target < upper) atomicMin(&winner_tid, (int)threadIdx.x);
  __syncthreads();
  if ((int)threadIdx.x == winner_tid) {
    float run = lower;
    int pick = -1;
    for (int i = i0; i < i1; ++i) {
      const float w = weight(i);
      if (w > 0.f) {
        pick = i;  // last weighted token so far: the fallback when rounding pushes the target past the chunk's sum
        run += w;
        if (target < run) break;
      }
    }
    winner = pick;
  }
  __syncthreads();
  if (threadIdx.x == 0 && winner < 0) {  // target == total after rounding: the last weighted token overall
    for (int i = V - 1; i >= 0; --i)
      if (weight(i) > 0.f) {
        winner = i;
        break;
      }
  }
  __syncthreads();
  const int out = winner;
  __syncthreads();  // winner may be reused by the caller's next draw
  return out;
}

__global__ void __launch_bounds__(SP_THREADS) sample_top_p_kernel(const float* __restrict__ logits, const float* __restrict__ uniform,
                                                                  long long* __restrict__ out, int V, float inv_temperature, float top_p) {
  __shared__ float scratch[SP_WARPS];
  const NucleusRow r = nucleus_row(logits + (int64_t)blockIdx.x * V, V, inv_temperature, scratch);
  const float tau = nucleus_tau(r, V, top_p, scratch);
  const int winner = block_draw([&](int i) { const float p = r.prob(i); return p >= tau ? p : 0.f; }, V, uniform[blockIdx.x]);
  if (threadIdx.x == 0) out[blockIdx.x] = winner;
}

// ---- per-row sampling controls (generate(temperature=[...], top_p=..., random_seed=..., presence_penalty=..., ...)) -------------
// Penalised logits as the selection loads them: l'[v] = fp32(l[v] - pen[v]) with pen[v] = fp32(c[v] * frequency), plus presence
// (one fp32 add) where c[v] > 0; c[v] counts the times the sequence generated v.  Round-to-nearest, no FMA contraction.  A NULL
// count row (no count table, or both penalties of the row 0) reads the logits unchanged.
struct PenalisedRow {
  const float* p;
  const int* count;
  float presence, frequency;
  __device__ __forceinline__ float operator()(int i) const {
    const float x = p[i];
    if (count == nullptr) return x;
    const int c = count[i];
    float pen = __fmul_rn((float)c, frequency);
    if (c > 0) pen = __fadd_rn(pen, presence);
    return __fsub_rn(x, pen);
  }
};

// Philox4x32-10 (Salmon et al., SC'11), the Random123 constants.
__device__ __forceinline__ uint4 philox4x32_10(uint4 ctr, uint2 key) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r) {
      key.x += 0x9E3779B9u;
      key.y += 0xBB67AE85u;
    }
    const unsigned lo0 = 0xD2511F53u * ctr.x, hi0 = __umulhi(0xD2511F53u, ctr.x);
    const unsigned lo1 = 0xCD9E8D57u * ctr.z, hi1 = __umulhi(0xCD9E8D57u, ctr.z);
    ctr = make_uint4(hi1 ^ ctr.y ^ key.x, lo1, hi0 ^ ctr.w ^ key.y, lo0);
  }
  return ctr;
}

// The uniform of a seeded sequence at its step t: the top 24 bits of word 0 of Philox4x32-10 with key (seed mod 2^32, seed >> 32)
// and counter (t, 0, 0, 0), times 2^-24 -- exactly representable, in [0, 1).
__device__ __forceinline__ float philox_uniform(unsigned long long seed, unsigned step) {
  const uint4 x = philox4x32_10(make_uint4(step, 0u, 0u, 0u), make_uint2((unsigned)seed, (unsigned)(seed >> 32)));
  return (float)(x.x >> 8) * 0x1p-24f;
}

// One CTA per row b: temperature[b] == 0 is greedy (block_argmax), otherwise the nucleus draw of sample_top_p_kernel at
// (temperature[b], top_p[b]) with u = philox_uniform(seeds[b], step[b]) when seeds is given, else uniform[b].  Then thread 0 adds 1
// to counts[b, token] (when a table is given) and to step[b]: the barrier before it orders every thread's reads of the row's counts
// and step before the increment.  Nothing the host changes between steps is an argument, so a captured launch replays as is.
__global__ void __launch_bounds__(SP_THREADS) select_tokens_kernel(const float* __restrict__ logits, const float* __restrict__ temperature,
                                                                   const float* __restrict__ top_p, const float* __restrict__ presence,
                                                                   const float* __restrict__ frequency, const unsigned long long* __restrict__ seeds,
                                                                   const float* __restrict__ uniform, int* step, int* counts,
                                                                   long long* __restrict__ out, int V) {
  const int b = blockIdx.x;
  const float pres = presence[b], freq = frequency[b];
  int* cnt = counts != nullptr ? counts + (int64_t)b * V : nullptr;
  const PenalisedRow row{logits + (int64_t)b * V, (cnt != nullptr && (pres != 0.f || freq != 0.f)) ? cnt : nullptr, pres, freq};
  const float t = temperature[b];
  int token;
  if (t == 0.f) {
    token = block_argmax(row, V);  // valid in thread 0, the only reader
  } else {
    __shared__ float scratch[SP_WARPS];
    const auto r = nucleus_row(row, V, __fdiv_rn(1.0f, t), scratch);
    const float tau = nucleus_tau(r, V, top_p[b], scratch);
    const float u = seeds != nullptr ? philox_uniform(seeds[b], (unsigned)step[b]) : uniform[b];
    token = block_draw([&](int i) { const float p = r.prob(i); return p >= tau ? p : 0.f; }, V, u);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    out[b] = token;
    if (cnt != nullptr && token >= 0) cnt[token] += 1;
    step[b] += 1;
  }
}

}  // namespace mb200
