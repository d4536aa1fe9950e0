"""Speculative decoding: `generate(..., draft=...)` (Leviathan et al. 2023; Chen et al. 2023).

A small draft model that shares the target's vocabulary proposes k = draft_tokens tokens per sequence; the target scores the
k + 1 tokens [last, d_1 .. d_k] of every sequence in ONE forward (the verify step: `Transformer.verify_static`, a CUDA-graph
replay of the chunked-prefill path at T = B * (k + 1)); an acceptance kernel keeps a prefix of the proposals and appends one token
of the target's own.  Greedy output is the target's argmax choices; sampled output keeps the target's nucleus distribution exactly
(csrc/speculative.cuh).  Per round and sequence b at target position p_b (tokens cached):

  1. draft: k steps on the draft's own cache (decode megakernel at B = 1, the CUDA-graph step at B > 1), each picked with `pick`
     (greedy, or mb200_sample_top_p at the same temperature and top-p); with sampling the k fp32 logit rows are kept (q).
     Catch-up: when the previous round accepted all k proposals, the draft never cached d_k, so its first step takes two tokens
     (d_k, then the new last) through the ragged `last_token_logits` forward.
  2. verify: target logits [B * (k + 1), V].
  3. accept: mb200_spec_accept_greedy / _sample write the emitted tokens and n_b, and advance the verify step's device positions by
     n_b + 1; mb200_logprob_gather over the same logits gives the emitted tokens' log-probabilities (untempered, as without a draft).
  4. readback: ONE device-to-host copy per round -- n (and, with eos_id, each sequence's first eos index): 4 B (8 B) bytes.  The
     host advances both caches' lengths (the draft is rewound to the accepted prefix: rejected ring rows are simply overwritten
     later) and decides whether to stop.  The sync is the simple choice because the draft's batch-1 megakernel takes its position
     from the host, and the next round's shape (catch-up or not) depends on n; it costs one round trip per k + 1 tokens at best.

Tokens and log-probabilities stay on the device until the end.  A sequence that has emitted max_tokens keeps running (a round
computes every sequence) but is held at the position where it crossed max_tokens and its tokens are dropped, so no position ever
passes max(prompt) + max_tokens + k.  Rejected proposals overwrite ring slots past the accepted prefix, so a layer whose ring would
wrap within that length could not roll back: such caches are refused.
"""
from typing import List, Optional, Tuple

import torch

from . import _abi
from .cache import BufferCache, get_cache_sizes
from .generate import TOP_P, _PromptPlan, pick
from .transformer import Transformer

_NO_EOS = 2 ** 30


def check_draft(model: Transformer, draft: Transformer, images, prompts: List[List[int]], max_tokens: int, draft_tokens: int) -> None:
    """The refusals of generate(..., draft=...), raised before anything is allocated."""
    if draft_tokens < 1:
        raise ValueError(f"draft_tokens={draft_tokens}: a draft proposes at least one token per round")
    if draft.args.vocab_size != model.args.vocab_size:
        raise ValueError(f"the draft's vocabulary ({draft.args.vocab_size} tokens) differs from the model's ({model.args.vocab_size}): "
                         "speculative decoding needs a draft that shares the tokenizer")
    for name, m in (("model", model), ("draft", draft)):
        if m.num_pipeline_ranks != 1 or m.expert_parallel[1] != 1:
            raise ValueError(f"speculative decoding runs single-device models: the {name} has pipeline ranks or expert parallelism")
        if len(prompts) > m.args.max_batch_size:
            raise ValueError(f"{len(prompts)} prompts exceed the {name}'s max_batch_size={m.args.max_batch_size}")
    if images:
        raise ValueError("speculative decoding takes text prompts only: images with a draft are not supported")
    need = max(len(p) for p in prompts) + max_tokens + draft_tokens
    for name, m in (("model", model), ("draft", draft)):
        short = [w for w in get_cache_sizes(m.n_local_layers, need, m.args.sliding_window) if w < need]
        if short:
            raise ValueError(f"the {name}'s sliding window of {min(short)} tokens would wrap its KV ring within max(prompt) + max_tokens + "
                             f"draft_tokens = {need} tokens: a rejected proposal overwrites a ring slot that a windowed layer still needs, "
                             "so such a cache cannot roll back (generate without a draft, or keep the generation inside the window)")


def check_draft_controls(controls, top_p) -> None:
    """Per-sequence sampling controls are not built for speculative decoding: the acceptance kernels take one temperature and
    top_p for the batch, and penalties would need the counts rolled back when proposals are rejected.  `controls` is
    generate.sampling_controls' result (None: every control a scalar, no seed, no penalty)."""
    if controls is not None or top_p != TOP_P:
        raise ValueError(f"speculative decoding (draft=...) takes one scalar temperature and top_p={TOP_P}: per-sequence "
                         "temperatures, another top_p, random_seed and presence / frequency penalties with a draft model are not built")


def _prefill(m: Transformer, plan: _PromptPlan, cache: BufferCache, want_logprobs: bool):
    """The prompt, chunk by chunk: (prompt log-probabilities per chunk, logits [B, V] of each sequence's last token)."""
    dev = m.device
    prompt_lp: List[torch.Tensor] = []
    last_logits: Optional[torch.Tensor] = None
    for flat, seqlens, targets, _ in plan.chunks:
        ids = torch.tensor(flat, dtype=torch.long, device=dev)
        if want_logprobs:
            lp, last_logits = m.forward_logprobs(ids, seqlens, cache, torch.tensor(targets, dtype=torch.long, device=dev))
            prompt_lp.append(lp)
        else:
            last_logits = m.last_token_logits(ids, seqlens, cache)
    return prompt_lp, last_logits


@torch.inference_mode()
def generate_speculative(prompts: List[List[int]], model: Transformer, draft: Transformer, images, *, max_tokens: int, temperature: float,
                         chunk_size: Optional[int], eos_id: Optional[int], draft_tokens: int) -> Tuple[List[List[int]], List[List[float]]]:
    check_draft(model, draft, images, prompts, max_tokens, draft_tokens)
    model, draft = model.eval(), draft.eval()
    dev = model.device
    plan = _PromptPlan(prompts, chunk_size)
    B, V, k = plan.B, model.args.vocab_size, draft_tokens
    S = k + 1
    ring = max(plan.lens) + max_tokens + k
    caches = []
    for m in (model, draft):
        c = BufferCache(m.n_local_layers, m.args.max_batch_size, ring, m.args.n_kv_heads, m.args.head_dim, m.args.sliding_window,
                        kv_cache=m.kv_cache)
        c.to(device=dev, dtype=m.dtype)
        c.reset()
        caches.append(c)
    tcache, dcache = caches

    prompt_lp, last_logits = _prefill(model, plan, tcache, True)
    _prefill(draft, plan, dcache, False)
    assert last_logits is not None and last_logits.shape == (B, V)

    cap = max_tokens + S  # room for a round's overshoot, then one column where masked-out tokens land
    gen_tok = torch.zeros(B, cap, dtype=torch.long, device=dev)
    gen_lp = torch.zeros(B, cap, dtype=torch.float32, device=dev)
    last = torch.zeros(B, dtype=torch.long, device=dev)
    eos_pos = torch.full((B,), _NO_EOS, dtype=torch.int32, device=dev)  # first eos index per sequence
    if max_tokens > 0:
        pick(last_logits, temperature, TOP_P, out=last)
        gen_lp[:, 0] = _abi.logprob_gather(last_logits, last)
        gen_tok[:, 0] = last
        if eos_id is not None:
            eos_pos.masked_fill_(last == eos_id, 0)

    emitted = [min(max_tokens, 1)] * B          # tokens in each sequence's stream (host mirror of emitted_dev)
    emitted_dev = torch.tensor(emitted, dtype=torch.long, device=dev)
    first_eos = [_NO_EOS] * B
    catch = [False] * B                          # the draft lacks d_k of the previous round
    props = torch.zeros(k, B, dtype=torch.long, device=dev)       # props[j]: proposal d_{j+1} of every sequence
    vtoks = torch.zeros(B, S, dtype=torch.long, device=dev)       # the verify step's input [last, d_1 .. d_k]
    out_tok = torch.zeros(B, S, dtype=torch.long, device=dev)
    n_dev = torch.zeros(B, dtype=torch.int32, device=dev)
    lp_round = torch.zeros(B, S, dtype=torch.float32, device=dev)
    q_rows = torch.empty(B, k, V, dtype=torch.float32, device=dev) if temperature > 0 else None
    ar = torch.arange(S, device=dev)
    readback = torch.empty(2 * B if eos_id is not None else B, dtype=torch.int32).pin_memory()

    def stop_at() -> int:
        if eos_id is not None and max(first_eos) < max_tokens:
            return max(first_eos)  # every sequence has finished: the step where the last one did is excluded
        return max_tokens

    while min(emitted) < stop_at():
        t0, d0 = list(tcache._kv_seqlens_host), list(dcache._kv_seqlens_host)
        # ---- 1. draft: k proposals per sequence
        if any(catch):
            pieces = []
            for b in range(B):
                pieces += ([props[k - 1, b:b + 1]] if catch[b] else []) + [last[b:b + 1]]
            logits = draft.last_token_logits(torch.cat(pieces), [2 if c else 1 for c in catch], dcache)
        else:
            logits = draft.next_token_logits(last, dcache)
        for j in range(k):
            if j > 0:
                logits = draft.next_token_logits(props[j - 1], dcache)
            if q_rows is not None:
                q_rows[:, j].copy_(logits)
            pick(logits, temperature, TOP_P, out=props[j],
                 fused_argmax=draft.last_argmax if draft.last_argmax_valid_for(logits) else None)
        # ---- 2. verify
        vtoks[:, 0] = last
        vtoks[:, 1:] = props.t()
        vlogits, seqpos = model.verify_static(vtoks, tcache)
        # ---- 3. accept (advances seqpos by n + 1), log-probabilities of the emitted tokens
        if q_rows is None:
            _abi.spec_accept_greedy(vlogits, vtoks, out_tok, n_dev, seqpos)
        else:
            u = torch.rand(B, S, dtype=torch.float32, device=dev)
            _abi.spec_accept_sample(vlogits, q_rows.view(B * k, V), vtoks, u, out_tok, n_dev, seqpos, temperature, TOP_P)
        _abi.logprob_gather(vlogits, out_tok.view(-1), out=lp_round.view(-1))
        n64 = n_dev.long()
        live = emitted_dev < max_tokens
        keep = (ar[None, :] <= n64[:, None]) & live[:, None]
        at = torch.where(keep, emitted_dev[:, None] + ar[None, :], cap - 1)
        gen_tok.scatter_(1, at, out_tok)
        gen_lp.scatter_(1, at, lp_round)
        if eos_id is not None:
            hit = torch.where(keep & (out_tok == eos_id), at, _NO_EOS).amin(1).to(torch.int32)
            torch.minimum(eos_pos, hit, out=eos_pos)
        emitted_dev += torch.where(live, n64 + 1, 0)
        last.copy_(out_tok.gather(1, n64[:, None]).squeeze(1))
        # ---- 4. the round's one device-to-host copy
        if eos_id is not None:
            readback.copy_(torch.cat([n_dev, eos_pos]))
        else:
            readback.copy_(n_dev)
        rb = readback.tolist()
        n = rb[:B]
        if eos_id is not None:
            first_eos = rb[B:]
        model.verify_accepted(tcache, S, [p + a + 1 for p, a in zip(t0, n)])
        tl, dl = [], []
        for b in range(B):
            if emitted[b] >= max_tokens:     # held: it stays where it crossed max_tokens
                tl.append(t0[b])
                dl.append(d0[b])
                continue
            emitted[b] += n[b] + 1
            if emitted[b] >= max_tokens:     # crossed now: hold it at this round's start (its draft cache covers that prefix)
                tl.append(t0[b])
                dl.append(t0[b])
                catch[b] = False
                continue
            tl.append(t0[b] + n[b] + 1)
            catch[b] = n[b] == k
            dl.append(tl[b] - 1 if catch[b] else tl[b])
        tcache._kv_seqlens_host = tl
        dcache._kv_seqlens_host = dl

    if eos_id is not None:
        first_eos = eos_pos.tolist()  # also covers a first token that no round has read back
    stop = stop_at() if max_tokens > 0 else 0
    tokens: List[List[int]] = gen_tok[:, :stop].tolist() if stop > 0 else []
    gen_lp_host = gen_lp[:, :stop].tolist() if stop > 0 else [[] for _ in range(B)]
    logprobs: List[List[float]] = [[] for _ in range(B)]
    for (_, _, targets, where), lp in zip(plan.chunks, prompt_lp):
        for (b, _), t, v in zip(where, targets, lp.tolist()):
            if t >= 0:
                logprobs[b].append(v)
    for b in range(B):
        logprobs[b].extend(gen_lp_host[b])
    return tokens, logprobs
