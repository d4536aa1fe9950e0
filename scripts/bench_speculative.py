"""Speculative decoding on one H100: what a round costs, part by part, and the speed-up it gives as a function of the acceptance rate.

With random weights a draft almost never agrees with its target, so the acceptance rate of a real pair cannot be measured here.
This script measures the parts of a round and derives the rest:
  * t_decode  the target's plain decode step (the path generate() takes without a draft),
  * t_draft   one draft decode step (megakernel at B = 1 where the draft has one, else the per-layer CUDA graph),
  * t_verify  one replay of the target's verify graph at k + 1 tokens per sequence (Transformer.verify_static),
  * t_accept  the greedy and the sampled acceptance kernels on the verify logits.
  T_round(k) = k * t_draft + t_verify(k) + t_accept(k).  With i.i.d. acceptance rate a per proposal a round emits
  E(a, k) = (1 - a^(k+1)) / (1 - a) tokens per sequence, so speculation pays iff E > T_round / t_decode (the break-even length).
  The tokens/s at a = 0.5 / 0.7 / 0.9 are DERIVED from the measured component times, not measured end to end.
One end-to-end generate(..., draft=...) per pair (greedy, k = 4, batch 1) checks the round-time model against a real loop: its
decode time (generate with N tokens minus generate with 1) against rounds * T_round(4) + the per-round overheads it leaves out.

Pairs: the Mistral Large 2 shape (88 layers, INT4) with a Mistral-7B-shaped INT4 draft (vocabulary 32768), and the Nemo-12B shape
(40 layers, FP8) with a 7B-shaped FP8 draft (vocabulary 131072); batch 1 at a 4k context, plus one batched point.  Weights are
seeded (N(0, 0.02)); the card's name, power limit and maximum SM clock are read in the same run.
Run: python scripts/bench_speculative.py [--quick] [--only large2,nemo]
"""
import argparse
import json
import sys
import time
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
sys.path.insert(0, str(Path(__file__).resolve().parent))
import bench_fp8_dense as B8  # noqa: E402
import bench_int4_dense as B4  # noqa: E402
import mistral_inference_b200 as mi  # noqa: E402
import synth  # noqa: E402
from mistral_inference_b200 import _abi  # noqa: E402

TEMP, TOP_P = 0.7, 0.8
RATES = (0.5, 0.7, 0.9)
# name: (target shape, layers, format), (draft shape, layers, format, vocabulary), [(batch, context)]
PAIRS = {
    "large2": (("mistral-large-2", 88, "int4"), ("mistral-7b", 32, "int4", 32768), [(1, 4096), (4, 1024)]),
    "nemo": (("mistral-nemo-12b", 40, "fp8"), ("mistral-7b", 32, "fp8", 131072), [(1, 4096), (8, 4096)]),
}


def seeded(name: str, n_layers: int, max_batch: int, fmt: str, seed: int, **over):
    """bench_int4_dense.seeded_model with shape overrides (the drafts take their target's vocabulary and, like Mistral-7B v0.3,
    no sliding window)."""
    saved = synth.SHAPES[name]
    synth.SHAPES[name] = dict(saved, **over)
    try:
        return B4.seeded_model(name, n_layers, max_batch, fmt, seed)
    finally:
        synth.SHAPES[name] = saved


def expected_tokens(a: float, k: int) -> float:
    return float(k + 1) if a >= 1 else (1 - a ** (k + 1)) / (1 - a)


def components(m, d, B: int, ctx: int, reps: int) -> dict:
    V = m.args.vocab_size
    tc = B8.filled_cache(m, B, ctx, reps * 4 + 64)
    dc = B8.filled_cache(d, B, ctx, reps * 4 + 64)
    tok = torch.zeros(B, dtype=torch.long, device="cuda")
    for _ in range(3):  # eager warm-up, capture, replay
        m.decode_static(tok, tc)
        d.decode_static(tok, dc)
    t_decode = min(B8.timed(lambda: m.decode_static(tok, tc), reps) for _ in range(3))
    t_draft = min(B8.timed(lambda: d.decode_static(tok, dc), reps) for _ in range(3))
    tc._kv_seqlens_host = [ctx] * B
    out = {"batch": B, "context": ctx, "t_decode_ms": round(t_decode, 3), "t_draft_ms": round(t_draft, 3),
           "target_path": B4.path_of(m, B), "draft_path": B4.path_of(d, B), "k": {}}
    for k in range(1, 5):
        S = k + 1
        vt = torch.randint(0, V, (B, S), device="cuda")
        for _ in range(3):
            m.verify_static(vt, tc)
        m.verify_accepted(tc, S, tc._kv_seqlens_host)  # the device positions equal the host's: replays upload nothing
        t_verify = min(B8.timed(lambda: m.verify_static(vt, tc), reps) for _ in range(3))
        logits, _ = m.verify_static(vt, tc)
        q = torch.randn(B * k, V, device="cuda")
        u = torch.rand(B, S, device="cuda")
        o = torch.empty(B, S, dtype=torch.long, device="cuda")
        n = torch.empty(B, dtype=torch.int32, device="cuda")
        sp = torch.zeros(B, dtype=torch.int32, device="cuda")
        t_greedy = min(B8.timed(lambda: _abi.spec_accept_greedy(logits, vt, o, n, sp), reps) for _ in range(3))
        t_sample = min(B8.timed(lambda: _abi.spec_accept_sample(logits, q, vt, u, o, n, sp, TEMP, TOP_P), reps) for _ in range(3))
        t_round = k * t_draft + t_verify + t_greedy
        t_round_s = k * t_draft + t_verify + t_sample
        row = {"t_verify_ms": round(t_verify, 3), "verify_over_decode": round(t_verify / t_decode, 2),
               "t_accept_greedy_ms": round(t_greedy, 4), "t_accept_sample_ms": round(t_sample, 4),
               "t_round_greedy_ms": round(t_round, 3), "break_even_tokens_per_round": round(t_round / t_decode, 2),
               "derived_tok_s": {"plain": round(B * 1000 / t_decode, 1),
                                 **{f"a={a}": round(B * 1000 * expected_tokens(a, k) / t_round, 1) for a in RATES},
                                 **{f"a={a} sampled": round(B * 1000 * expected_tokens(a, k) / t_round_s, 1) for a in RATES}}}
        out["k"][k] = row
        print(f"  B={B} ctx={ctx} k={k}", json.dumps(row), flush=True)
    del tc, dc
    torch.cuda.empty_cache()
    return out


def end_to_end(m, d, ctx: int, N: int) -> dict:
    """Greedy generate with k = 4 at batch 1 from a ctx-token prompt; rounds and accepted proposals counted at the accept kernel."""
    k = 4
    prompt = [synth.synth_prompt(ctx, m.args.vocab_size, 3)]
    seen = []
    orig = _abi.spec_accept_greedy

    def record(logits, tokens, out, n, seqpos):
        orig(logits, tokens, out, n, seqpos)
        seen.append(n.clone())

    def run(max_tokens: int) -> float:
        seen.clear()
        torch.cuda.synchronize()
        t = time.perf_counter()
        mi.generate(prompt, m, max_tokens=max_tokens, temperature=0.0, draft=d, draft_tokens=k)
        torch.cuda.synchronize()
        return (time.perf_counter() - t) * 1000

    _abi.spec_accept_greedy = record
    try:
        run(N)  # warm-up: loads modules, captures nothing that survives (each generate builds its caches)
        t1 = run(1)
        tN = run(N)
        accepted = int(sum(int(x[0]) for x in seen))
        rounds = len(seen)
    finally:
        _abi.spec_accept_greedy = orig
    return {"prompt": ctx, "max_tokens": N, "k": k, "rounds": rounds, "accepted_proposals": accepted,
            "decode_ms": round(tN - t1, 1), "ms_per_round": round((tN - t1) / max(rounds, 1), 3)}


def pair(name: str, quick: bool, out: dict) -> None:
    (ts, tl, tf), (ds, dl, df, dv), points = PAIRS[name]
    if quick:
        tl, dl, points = 4, 4, [(1, 1024), (points[1][0], 512)]
    maxb = max(b for b, _ in points)
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    m = seeded(ts, tl, maxb, tf, 7)
    d = seeded(ds, dl, maxb, df, 8, vocab_size=dv, sliding_window=None)
    res = {"target": f"{ts} x{tl} {tf}", "draft": f"{ds} x{dl} {df} (vocab {dv})",
           "target_gb": round(B8.nbytes(m) / 1e9, 2), "draft_gb": round(B8.nbytes(d) / 1e9, 2), "points": []}
    print(name, json.dumps({k: v for k, v in res.items() if k != "points"}), flush=True)
    for B, ctx in points:
        res["points"].append(components(m, d, B, ctx, 5 if quick else 20))
    torch.cuda.reset_peak_memory_stats()
    res["end_to_end"] = e2e = end_to_end(m, d, points[0][1], 16 if quick else 128)
    c = res["points"][0]
    e2e["model_ms_per_round"] = c["k"][4]["t_round_greedy_ms"]
    e2e["peak_gb_models_and_both_caches"] = round(torch.cuda.max_memory_allocated() / 1e9, 2)
    print(name, "end_to_end", json.dumps(e2e), flush=True)
    out[name] = res
    del m, d
    torch.cuda.empty_cache()


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--only", default="large2,nemo")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_speculative needs a GPU: no timing exists without one")
    out = {"card": B8.card()}
    print("card", out["card"], flush=True)
    for name in a.only.split(","):
        pair(name, a.quick, out)
    out["card_after"] = B8.card()
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
