"""INT4 dense weights on one H100: Mistral Large 2 on one card, and what the format buys and costs on the smaller models.

Reports, with the card's name, power limit and maximum SM clock read in the same run:
  1. Mistral Large 2 shape, 88 layers, INT4, its weights seeded and quantised on the device one bf16 tensor at a time: model bytes
     and the build's peak; a 4096-token prefill; batch-1 decode tok/s at a 4k context with its share of 3.35 TB/s from the step's
     own bytes (codes, scales, the bf16 lm head, one embedding row, the norms, the K/V ring); a batch-8 decode step at a 4k context
     (or the largest batch that fits) with its peak memory;
  2. Mistral-7B (32 layers) and Nemo-12B (40 layers) shapes, batch 1 at a 4k context in bf16 / FP8 / INT4, alternated in one
     process, naming the path each ran (decode megakernel or per-layer CUDA graph); the Nemo batch-32 step at a 1k context;
  3. the Linears alone at T = 1, 4, 32, 128, 4096 for the 7B wqkv, w13 and w2 shapes in the three formats, with each format's
     share of 3.35 TB/s from its own weight bytes (INT4: N * K / 2 codes + N * K / 64 scale bytes);
  4. drift on seeded synthetic weights (a 4-layer 7B shape): the largest logit difference and the top-1 agreement between the INT4
     and the bf16 model, teacher-forced on the bf16 model's greedy tokens.
Quality on a real checkpoint is not measured here: no checkpoint is used, the weights are random.
Run: python scripts/bench_int4_dense.py [--quick] [--only large,small,linears,drift]
"""
import argparse
import json
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
sys.path.insert(0, str(Path(__file__).resolve().parent))
import bench_fp8_dense as B8  # noqa: E402
import mistral_inference_b200 as mi  # noqa: E402
import synth  # noqa: E402
from mistral_inference_b200 import _abi  # noqa: E402
from mistral_inference_b200.cache import BufferCache  # noqa: E402
from mistral_inference_b200.transformer import Transformer  # noqa: E402

HBM_BPS = B8.HBM_BPS
HD = 128
FORMATS = ("bf16", "fp8", "int4")


def seeded_model(name: str, n_layers: int, max_batch: int, fmt: str, seed: int = 0) -> Transformer:
    """A model whose bf16 weights are N(0, 0.02) from a per-tensor seed, built on the device one tensor at a time: quantised
    formats never hold more than the model plus one bf16 tensor."""
    p = synth.shape(name, n_layers=n_layers)
    args = mi.TransformerArgs.from_dict(dict(p))
    args.max_batch_size = max_batch
    m = Transformer.empty(args, "cuda", torch.bfloat16, dense_weights=fmt).eval()
    g = torch.Generator(device="cuda")

    def rnd(shape, i):
        g.manual_seed(seed * 1000003 + i)
        return torch.randn(shape, generator=g, device="cuda", dtype=torch.bfloat16) * 0.02

    with torch.no_grad():
        m.tok_embeddings.weight.copy_(rnd(m.tok_embeddings.weight.shape, 1))
        m.output_weight.copy_(rnd(m.output_weight.shape, 2))
        m.norm.weight.fill_(1.0)
        i = 10
        for blk in m.layers.values():
            blk.attention_norm.weight.fill_(1.0)
            blk.ffn_norm.weight.fill_(1.0)
            att, ff = blk.attention, blk.feed_forward
            shapes = {"wq": (att.q_dim, args.dim), "wk": (att.kv_dim, args.dim), "wv": (att.kv_dim, args.dim), "wo": (args.dim, att.q_dim),
                      "w1": (args.hidden_dim, args.dim), "w3": (args.hidden_dim, args.dim), "w2": (args.dim, args.hidden_dim)}
            for n, shp in shapes.items():
                w = rnd(shp, i)
                i += 1
                mod = att if n in ("wq", "wk", "wv", "wo") else ff
                if fmt == "int4":
                    mod.quantize_int4_(n, w)
                elif fmt == "fp8":
                    mod.quantize_(n, w)
                else:
                    getattr(mod, n).weight.copy_(w)
                del w
    return m


def path_of(m: Transformer, B: int) -> str:
    return "megakernel" if m._megakernel_ok(B) else "graph"


def step_bytes(m: Transformer, ctx: int, B: int = 1) -> int:
    a = m.args
    layer = sum(t.numel() * t.element_size() for n, t in m.named_parameters() if n.startswith("layers."))
    return layer + m.output_weight.numel() * 2 + B * a.dim * 2 + a.dim * 2 + B * 2 * ctx * a.n_kv_heads * HD * 2 * m.n_local_layers


def decode_rate(m: Transformer, B: int, ctx: int, steps: int, rounds: int):
    cache = B8.filled_cache(m, B, ctx, rounds * steps + 16)
    tok = torch.zeros(B, dtype=torch.long, device="cuda")
    for _ in range(3):  # eager warm-up, capture, replay
        m.decode_static(tok, cache)
    res = [B8.timed(lambda: m.decode_static(tok, cache), steps) for _ in range(rounds)]
    return res, cache


def large(out: dict, quick: bool) -> None:
    n_layers = 4 if quick else 88
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    m = seeded_model("mistral-large-2", n_layers, 8, "int4", seed=7)
    torch.cuda.synchronize()
    row = {"shape": f"mistral-large-2 x{n_layers} layers, int4", "model_gb": round(B8.nbytes(m) / 1e9, 2),
           "build_peak_gb": round((torch.cuda.max_memory_allocated() - base) / 1e9, 2)}
    print("large_build", json.dumps(row), flush=True)
    out["large_build"] = row
    a = m.args
    # 4096-token prefill
    T = 4096
    ids = torch.randint(0, a.vocab_size, (T,), device="cuda")
    pf = BufferCache(m.n_local_layers, 1, T, a.n_kv_heads, HD, None).to("cuda", torch.bfloat16)

    def prefill():
        pf.reset()
        m.forward(ids, [T], pf)

    prefill()
    res = [B8.timed(prefill, 1 if quick else 2) for _ in range(2 if quick else 3)]
    row = {"tokens": T, "layers": n_layers, "prefill_ms": round(min(res), 1), "all_ms": [round(x, 1) for x in res]}
    print("large_prefill", json.dumps(row), flush=True)
    out["large_prefill"] = row
    del pf
    torch.cuda.empty_cache()
    # batch-1 decode at a 4k context
    ctx = 4096
    res, cache = decode_rate(m, 1, ctx, 10 if quick else 50, 3)
    ms_step = min(res)
    b = step_bytes(m, ctx)
    row = {"B": 1, "context": ctx, "path": path_of(m, 1), "step_ms": round(ms_step, 3), "tok_s": round(1e3 / ms_step, 1),
           "all_tok_s": [round(1e3 / t, 1) for t in res], "step_bytes_gb": round(b / 1e9, 2), "hbm_share": round(b / (ms_step * 1e-3) / HBM_BPS, 3)}
    print("large_decode_b1", json.dumps(row), flush=True)
    out["large_decode_b1"] = row
    del cache
    torch.cuda.empty_cache()
    # the largest batch (of 8, 4, 2) whose 4k step fits, with its peak memory
    for B in (8, 4, 2):
        try:
            torch.cuda.reset_peak_memory_stats()
            res, cache = decode_rate(m, B, ctx, 5 if quick else 20, 3)
        except torch.cuda.OutOfMemoryError:
            torch.cuda.empty_cache()
            continue
        ms_step = min(res)
        b = step_bytes(m, ctx, B)
        row = {"B": B, "context": ctx, "path": path_of(m, B), "step_ms": round(ms_step, 3), "tok_s": round(B * 1e3 / ms_step, 1),
               "step_bytes_gb": round(b / 1e9, 2), "hbm_share": round(b / (ms_step * 1e-3) / HBM_BPS, 3),
               "peak_gb": round(torch.cuda.max_memory_allocated() / 1e9, 2),
               "device_gb": round(torch.cuda.get_device_properties(0).total_memory / 1e9, 2)}
        print("large_decode_batch", json.dumps(row), flush=True)
        out["large_decode_batch"] = row
        del cache
        break
    del m
    torch.cuda.empty_cache()


def small(out: dict, quick: bool) -> None:
    for name, L in (("mistral-7b", 32), ("mistral-nemo-12b", 40)):
        ms = {f: seeded_model(name, 4 if quick else L, 1, f, seed=3) for f in FORMATS}
        ctx, steps = 4096, 30 if quick else 200
        caches, res = {}, {f: [] for f in FORMATS}
        for f, m in ms.items():
            caches[f] = B8.filled_cache(m, 1, ctx, 6 * steps + 16)
            for _ in range(3):
                m.decode_static(torch.zeros(1, dtype=torch.long, device="cuda"), caches[f])
        tok = torch.zeros(1, dtype=torch.long, device="cuda")
        for _ in range(3 if quick else 5):
            for f, m in ms.items():
                res[f].append(B8.timed(lambda: m.decode_static(tok, caches[f]), steps))
        for f, m in ms.items():
            t = min(res[f])
            b = step_bytes(m, ctx)
            row = {"shape": name, "format": f, "path": path_of(m, 1), "layers": m.n_local_layers, "step_ms": round(t, 3),
                   "tok_s": round(1e3 / t, 1), "all_tok_s": [round(1e3 / x, 1) for x in res[f]], "step_bytes_gb": round(b / 1e9, 3),
                   "hbm_share": round(b / (t * 1e-3) / HBM_BPS, 3)}
            print("decode_b1", json.dumps(row), flush=True)
            out.setdefault("decode_b1", []).append(row)
        del ms, caches
        torch.cuda.empty_cache()
    # Nemo batch 32 at a 1k context
    B, ctx = 32, 1024
    ms = {f: seeded_model("mistral-nemo-12b", 4 if quick else 40, B, f, seed=3) for f in FORMATS}
    steps = 5 if quick else 20
    caches = {f: B8.filled_cache(m, B, ctx, 4 * steps + 16) for f, m in ms.items()}
    tok = torch.zeros(B, dtype=torch.long, device="cuda")
    for f, m in ms.items():
        for _ in range(3):
            m.next_token_logits(tok, caches[f])
    res = {f: [] for f in FORMATS}
    for _ in range(3):
        for f, m in ms.items():
            res[f].append(B8.timed(lambda: m.next_token_logits(tok, caches[f]), steps))
    for f, m in ms.items():
        row = {"format": f, "B": B, "context": ctx, "layers": m.n_local_layers, "step_ms": round(min(res[f]), 3),
               "weights_gb": round(B8.nbytes(m) / 1e9, 2)}
        print("decode_nemo_b32", json.dumps(row), flush=True)
        out.setdefault("decode_nemo_b32", []).append(row)
    del ms, caches
    torch.cuda.empty_cache()


def linears(out: dict, quick: bool) -> None:
    dim, hidden, q_dim, kv_dim = 4096, 14336, 4096, 1024
    shapes = {"wqkv": (q_dim + 2 * kv_dim, dim), "w13": (2 * hidden, dim), "w2": (dim, hidden)}
    for name, (N, K) in shapes.items():
        w = (torch.randn(N, K, device="cuda") * 0.02).to(torch.bfloat16)
        q8 = torch.empty(N, K, dtype=torch.uint8, device="cuda")
        s8 = torch.empty(N, dtype=torch.float32, device="cuda")
        _abi.quantize_e4m3_rows(w, q8, s8)
        q4 = torch.empty(N, K // 2, dtype=torch.uint8, device="cuda")
        s4 = torch.empty(N, K // 128, dtype=torch.bfloat16, device="cuda")
        _abi.quantize_int4_groups(w, q4, s4)
        wbytes = {"bf16": 2 * N * K, "fp8": N * K + 4 * N, "int4": N * K // 2 + 2 * N * K // 128}
        for T in (1, 4, 32, 128, 4096):
            ws = _abi.Workspace(_abi.workspace_bytes(T, max(K, dim), 32, 8, 128, max(K, hidden), 0, 1), torch.device("cuda"))
            x = torch.randn(T, K, device="cuda").to(torch.bfloat16)
            o = torch.empty(T, N, dtype=torch.bfloat16, device="cuda")
            calls = {"bf16": lambda: _abi.linear_residual(x, w, None, o, ws), "fp8": lambda: _abi.linear_residual_fp8(x, q8, s8, None, o, ws),
                     "int4": lambda: _abi.linear_residual_int4(x, q4, s4, None, o, ws)}
            names = {f: ",".join(sorted({n.split("<")[0] for n in B8.launched(c)})) for f, c in calls.items()}
            reps = 5 if T == 4096 else (20 if quick else 200)
            res = {f: [] for f in calls}
            for _ in range(3):
                for f, c in calls.items():
                    res[f].append(B8.timed(c, reps))
            row = {"linear": name, "N": N, "K": K, "T": T, "kernels": names}
            for f in calls:
                t = min(res[f])
                row[f"{f}_us"] = round(t * 1e3, 1)
                row[f"{f}_hbm_share"] = round(wbytes[f] / (t * 1e-3) / HBM_BPS, 3)
                row[f"{f}_tflops"] = round(2 * T * N * K / (t * 1e-3) / 1e12, 1)
            print("linear", json.dumps(row), flush=True)
            out.setdefault("linears", []).append(row)
        del w, q8, s8, q4, s4
        torch.cuda.empty_cache()


def drift(out: dict, quick: bool) -> None:
    p = synth.shape("mistral-7b", n_layers=4, vocab_size=32768)
    sd = synth.synth_state_dict(p, 3, torch.bfloat16, "cuda")
    ms = {}
    for fmt in ("bf16", "int4"):
        args = mi.TransformerArgs.from_dict(dict(p))
        args.max_batch_size = 4
        m = Transformer.empty(args, "cuda", torch.bfloat16, dense_weights=fmt)
        m.load_state_dict(sd)
        ms[fmt] = m.eval()
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
    worst, agree, total = 0.0, 0, 0
    for lb, l4 in zip(logits["bf16"], logits["int4"]):
        worst = max(worst, (lb - l4).abs().max().item())
        agree += int((lb.argmax(-1) == l4.argmax(-1)).sum())
        total += lb.shape[0]
    row = {"shape": "mistral-7b x4 layers, synthetic", "prompts": [len(x) for x in prompts], "new_tokens": n_new,
           "max_abs_logit_diff": round(worst, 4), "top1_agreement": round(agree / total, 4), "picks": total,
           "logit_absmax": round(max(x.abs().max().item() for x in logits["bf16"]), 2)}
    print("drift", json.dumps(row), flush=True)
    out["drift"] = row
    del ms
    torch.cuda.empty_cache()


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true", help="few layers and steps (a check that the script runs)")
    ap.add_argument("--only", default="", help="comma-separated sections: large,small,linears,drift")
    a = ap.parse_args()
    torch.manual_seed(0)
    out = {"card": B8.card(), "sm_count": torch.cuda.get_device_properties(0).multi_processor_count}
    print("card:", out["card"], flush=True)
    only = set(filter(None, a.only.split(",")))
    for key, fn in (("large", large), ("small", small), ("linears", linears), ("drift", drift)):
        if not only or key in only:
            fn(out, a.quick)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
