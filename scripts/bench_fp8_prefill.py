"""FP8 activations for FP8 dense weights (prefill_compute="fp8") on one H100: prefill time against bf16 and FP8 A16.

Reports, with the card's name, power limit and maximum SM clock read in the same run (bf16, FP8 A16 and FP8 A8 alternated in one
process):
  1. the Linear kernels alone (STORE epilogue) at T = 512, 1024 and 4096 for the 7B and Nemo-12B wqkv, wo, w13 and w2 shapes: time
     in the three configurations, A8's share of the 1,979 TFLOP/s FP8 data-sheet rate, and the time of its per-token quantiser;
  2. whole-model first prefill, layers + final norm (forward_partial: no lm head): the 7B shape with 4096 tokens (32 layers) and
     the Nemo-12B shape with 32 sequences of 1024 tokens (40 layers);
  3. with --profile (a run of its own): a torch.profiler breakdown of the A8 7B prefill by kernel family;
  4. drift on seeded synthetic weights (4-layer 7B shape, vocab 32768, 4 prompts of 64-700 tokens, 64 greedy tokens of the bf16
     model teacher-forced into each model): the largest logit difference and the top-1 agreement of A8 against bf16 and against
     FP8 A16.
Weights of the timing runs are random (the FP8 models hold the e4m3 rows of the bf16 model's weights), not a checkpoint.
Run: python scripts/bench_fp8_prefill.py [--quick] [--only linears,prefill,drift] [--profile]
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import mistral_inference_b200 as mi  # noqa: E402
import synth  # noqa: E402
from mistral_inference_b200 import _abi  # noqa: E402
from mistral_inference_b200.cache import BufferCache  # noqa: E402
from mistral_inference_b200.transformer import Transformer  # noqa: E402
from oracle import fp8 as F8  # noqa: E402

FP8_PEAK = 1979e12  # H100 SXM data sheet, dense FP8
BF16_PEAK = 989e12
HD = 128
CONFIGS = ("bf16", "fp8", "fp8a8")


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e!r})"


def timed(fn, reps: int) -> float:
    """Mean ms of fn() over reps calls, CUDA events around the whole loop."""
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def alternate(fns: dict, reps: int, rounds: int = 3) -> dict:
    """Best-of-rounds mean ms of each fn, the fns alternated round by round (after one warm-up call each)."""
    for f in fns.values():
        f()
    torch.cuda.synchronize()
    res = {k: [] for k in fns}
    for _ in range(rounds):
        for k, f in fns.items():
            res[k].append(timed(f, reps))
    return {k: min(v) for k, v in res.items()}


# ----------------------------------------------------------------------------- 1. the Linears
def linears(out: dict, quick: bool) -> None:
    rows = []
    for name in ("mistral-7b", "mistral-nemo-12b"):
        p = synth.shape(name)
        dim, hidden, H, KV = p["dim"], p["hidden_dim"], p["n_heads"], p["n_kv_heads"]
        shapes = (("wqkv", (H + 2 * KV) * HD, dim), ("wo", dim, H * HD), ("w13", 2 * hidden, dim), ("w2", dim, hidden))
        for T in ((512, 4096) if quick else (512, 1024, 4096)):
            for lin, N, K in shapes:
                g = torch.Generator(device="cuda").manual_seed(T + N)
                x = torch.randn(T, K, generator=g, device="cuda").to(torch.bfloat16)
                w = (torch.randn(N, K, generator=g, device="cuda") * 0.02).to(torch.bfloat16)
                q, s = F8.quantize_rows(w)
                o = torch.empty(T, N, dtype=torch.bfloat16, device="cuda")
                xq = torch.empty(T, K, dtype=torch.uint8, device="cuda")
                xe = torch.empty(T, dtype=torch.int32, device="cuda")
                ws = _abi.Workspace(_abi.workspace_bytes(T, max(N, K), 32, 8, HD, max(N, K), 0, 64), torch.device("cuda"))
                fns = {"bf16": lambda: _abi.linear_residual(x, w, None, o, ws),
                       "fp8": lambda: _abi.linear_residual_fp8(x, q, s, None, o, ws),
                       "fp8a8": lambda: _abi.linear_residual_fp8(x, q, s, None, o, ws, a8=True),
                       "quantiser": lambda: _abi.lib().mb200_quantize_act_e4m3(x.data_ptr(), None, xq.data_ptr(), xe.data_ptr(), T, K, 0.0,
                                                                               _abi._stream())}
                ms = alternate(fns, 5 if quick else 20)
                flop = 2.0 * T * N * K
                row = {"shape": name, "linear": lin, "T": T, "N": N, "K": K, **{f"{k}_us": round(v * 1e3, 1) for k, v in ms.items()},
                       "a8_tflops": round(flop / (ms["fp8a8"] * 1e-3) / 1e12, 1),
                       "a8_share_of_fp8_peak": round(flop / (ms["fp8a8"] * 1e-3) / FP8_PEAK, 3),
                       "a8_gemm_share_of_fp8_peak": round(flop / ((ms["fp8a8"] - ms["quantiser"]) * 1e-3) / FP8_PEAK, 3),
                       "bf16_share_of_bf16_peak": round(flop / (ms["bf16"] * 1e-3) / BF16_PEAK, 3)}
                print("linear", json.dumps(row), flush=True)
                rows.append(row)
                del x, w, q, s, o, ws, xq, xe
        torch.cuda.empty_cache()
    out["linears"] = rows


# ----------------------------------------------------------------------------- 2. whole-model prefill
def models(name: str, n_layers: int, max_batch: int) -> dict:
    """A bf16 model with random weights, the FP8 model holding the e4m3 rows of the same weights, and the same FP8 model with
    prefill_compute="fp8" (its parameters copied from the FP8 model)."""
    p = synth.shape(name, n_layers=n_layers)
    args = mi.TransformerArgs.from_dict(dict(p))
    args.max_batch_size = max_batch
    bf = Transformer.empty(args, "cuda", torch.bfloat16).eval()
    with torch.no_grad():
        for prm in bf.parameters():
            prm.normal_(0.0, 0.02)
        for blk in bf.layers.values():
            blk.attention_norm.weight.fill_(1.0)
            blk.ffn_norm.weight.fill_(1.0)
    ms = {"bf16": bf}
    for cfg, pc in (("fp8", "bf16"), ("fp8a8", "fp8")):
        m = Transformer.empty(args, "cuda", torch.bfloat16, dense_weights="fp8", prefill_compute=pc).eval()
        with torch.no_grad():
            if cfg == "fp8":
                m.tok_embeddings.weight.copy_(bf.tok_embeddings.weight)
                m.norm.weight.copy_(bf.norm.weight)
                m.output_weight.copy_(bf.output_weight)
                for k in bf.layers:
                    b8, bb = m.layers[k], bf.layers[k]
                    b8.attention_norm.weight.copy_(bb.attention_norm.weight)
                    b8.ffn_norm.weight.copy_(bb.ffn_norm.weight)
                    for n in ("wq", "wk", "wv", "wo"):
                        b8.attention.quantize_(n, getattr(bb.attention, n).weight)
                    for n in ("w1", "w2", "w3"):
                        b8.feed_forward.quantize_(n, getattr(bb.feed_forward, n).weight)
            else:
                for (ka, a), (kb, b) in zip(m.named_parameters(), ms["fp8"].named_parameters()):
                    assert ka == kb
                    a.copy_(b)
        ms[cfg] = m
    return ms


def prefill_run(ms: dict, lens: list, reps: int):
    args = ms["bf16"].args
    ids = torch.randint(0, args.vocab_size, (sum(lens),), device="cuda")
    caches = {f: BufferCache(m.n_local_layers, len(lens), max(lens), args.n_kv_heads, HD, None).to("cuda", torch.bfloat16)
              for f, m in ms.items()}

    def go(f):
        def run():
            caches[f].reset()
            ms[f].forward_partial(ids, lens, caches[f])
        return run

    return alternate({f: go(f) for f in ms}, reps), go


def prefill(out: dict, quick: bool) -> None:
    rows = []
    for name, n_layers, lens in (("mistral-7b", 32, [4096]), ("mistral-nemo-12b", 40, [1024] * 32)):
        if quick:
            n_layers = 4
        ms = models(name, n_layers, len(lens))
        t = prefill_run(ms, lens, 2 if quick else 5)[0]  # keeps no reference to the models or their caches
        row = {"shape": name, "layers": n_layers, "tokens": f"{len(lens)} x {lens[0]}", **{f"{k}_ms": round(v, 2) for k, v in t.items()},
               "a8_over_fp8": round(t["fp8a8"] / t["fp8"], 3), "a8_over_bf16": round(t["fp8a8"] / t["bf16"], 3)}
        print("prefill", json.dumps(row), flush=True)
        rows.append(row)
        del ms
        torch.cuda.empty_cache()
    out["prefill"] = rows


def profile(out: dict, quick: bool) -> None:
    ms = models("mistral-7b", 4 if quick else 32, 1)
    ms = {"fp8": ms["fp8"], "fp8a8": ms["fp8a8"]}
    for f in list(ms):
        _, go = prefill_run({"bf16": ms[f]}, [4096], 1)
        run = go("bf16")
        run()
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            run()
            torch.cuda.synchronize()
        fam = {}
        for ev in prof.key_averages():
            key = ev.key.split("<")[0].split("(")[0]
            t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
            fam[key] = fam.get(key, 0.0) + t / 1e3
        top = dict(sorted(((k, round(v, 2)) for k, v in fam.items() if v > 0.05), key=lambda kv: -kv[1]))
        print(f"profile {f}", json.dumps(top), flush=True)
        out[f"profile_{f}_ms"] = top
    del ms
    torch.cuda.empty_cache()


# ----------------------------------------------------------------------------- 4. drift
def drift(out: dict, quick: bool) -> None:
    p = synth.shape("mistral-7b", n_layers=4, vocab_size=32768)
    sd = synth.synth_state_dict(p, 3, torch.bfloat16, "cuda")
    ms = {}
    for cfg in CONFIGS:
        args = mi.TransformerArgs.from_dict(dict(p))
        args.max_batch_size = 4
        kw = {} if cfg == "bf16" else {"dense_weights": "fp8", "prefill_compute": "fp8" if cfg == "fp8a8" else "bf16"}
        m = Transformer.empty(args, "cuda", torch.bfloat16, **kw)
        m.load_state_dict(sd)
        ms[cfg] = m.eval()
    del sd
    prompts = [synth.synth_prompt(n, p["vocab_size"], 7 + i) for i, n in enumerate((512, 300, 700, 64))]
    n_new = 16 if quick else 64
    toks, _ = mi.generate(prompts, ms["bf16"], max_tokens=n_new, temperature=0.0)
    caches = {f: BufferCache(4, 4, max(len(x) for x in prompts) + n_new + 1, p["n_kv_heads"], HD, p.get("sliding_window")).to("cuda", torch.bfloat16)
              for f in ms}
    logits = {}
    for f, m in ms.items():
        ids = torch.tensor(sum(prompts, []), device="cuda")
        logits[f] = [m.forward(ids, [len(x) for x in prompts], caches[f])[torch.tensor([len(x) for x in prompts]).cumsum(0) - 1]]
        for s in range(n_new - 1):
            nxt = torch.tensor([t[s] for t in toks], device="cuda")
            logits[f].append(m.forward(nxt, [1] * 4, caches[f]).clone())

    def compare(a: str, b: str):
        worst, agree, total, worst_first = 0.0, 0, 0, 0.0
        for i, (la, lb) in enumerate(zip(logits[a], logits[b])):
            d = (la - lb).abs().max().item()
            worst = max(worst, d)
            if i == 0:
                worst_first = d
            agree += int((la.argmax(-1) == lb.argmax(-1)).sum())
            total += la.shape[0]
        return {"max_abs_logit_diff": round(worst, 4), "max_abs_logit_diff_after_prefill": round(worst_first, 4),
                "top1_agreement": round(agree / total, 4), "picks": total}

    row = {"shape": "mistral-7b x4 layers, vocab 32768, synthetic", "prompts": [len(x) for x in prompts], "new_tokens": n_new,
           "a8_vs_bf16": compare("fp8a8", "bf16"), "a8_vs_fp8": compare("fp8a8", "fp8"), "fp8_vs_bf16": compare("fp8", "bf16"),
           "logit_absmax": round(max(x.abs().max().item() for x in logits["bf16"]), 2)}
    print("drift", json.dumps(row), flush=True)
    out["drift"] = row
    del ms
    torch.cuda.empty_cache()


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true", help="few layers and steps (a check that the script runs)")
    ap.add_argument("--only", default="", help="comma-separated sections: linears,prefill,drift")
    ap.add_argument("--profile", action="store_true", help="only the torch.profiler breakdown of the 7B 4096-token prefill")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_fp8_prefill: no CUDA device")
    torch.manual_seed(0)
    out = {"card": card(), "sm_count": torch.cuda.get_device_properties(0).multi_processor_count}
    print("card:", out["card"], flush=True)
    if a.profile:
        profile(out, a.quick)
    else:
        only = set(filter(None, a.only.split(",")))
        for key, fn in (("linears", linears), ("prefill", prefill), ("drift", drift)):
            if not only or key in only:
                fn(out, a.quick)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
