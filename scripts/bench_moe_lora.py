"""Un-merged LoRA adapters on Mixtral-8x7B with FP8 experts, on one GPU: what the adapters cost.

Builds the full model (32 layers, `expert_weights="fp8"`, bf16 attention) from seeded synthetic weights (synth.py), each expert
matrix generated in bf16 on the device and quantised into place, once without adapters and once each with r = 16 and r = 64
adapters on every Linear (the attention's wq/wk/wv/wo and every expert's w1/w2/w3; seeded values, loaded in place).  The three
models do not fit together, so the model-level numbers are taken one model after another in the same process; the grouped expert
FFN of one layer is timed with the three configurations alternated.  Reports, per configuration:
  * model bytes, adapter bytes and the peak device memory of the build;
  * a 4096-token prefill, batch-1 decode ms/token at a 4k context and one batch-32 decode step at a 512 context (graph replays),
    with the peak memory of the run;
  * the grouped expert FFN (router + gate/up + down + combine, with the adapters' down and up projections) of one layer at
    T = 1, 8, 32 and 4096.
`--profile` adds a torch.profiler run of each adapted model (16 batch-1 decode steps, one 4096-token prefill) that sums device time
per kernel family (`--trace-dir DIR` also writes the Chrome traces).  Prints the card's name and power limit with the numbers, then one
JSON line.
Run: python scripts/bench_moe_lora.py [--layers N] [--profile]
"""
import argparse
import ctypes
import json
import subprocess
import sys
import time
from collections import defaultdict
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import mistral_inference_b200 as mi  # noqa: E402
import synth  # noqa: E402
from mistral_inference_b200 import _abi  # noqa: E402
from mistral_inference_b200.args import LoraArgs  # noqa: E402
from mistral_inference_b200.cache import BufferCache  # noqa: E402
from mistral_inference_b200.moe import Fp8Expert, MoeBuffers  # noqa: E402
from mistral_inference_b200.transformer import Transformer  # noqa: E402
from mistral_inference_b200.transformer_layers import LoraAdapter  # noqa: E402

RANKS = (0, 16, 64)  # 0: no adapters (args.lora unset)
ADAPTER_SCALE = 0.02


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e!r})"


def build(p, seed: int, rank: int, max_batch: int) -> Transformer:
    d = dict(p, lora=dict(rank=rank, scaling=2.0)) if rank else dict(p)
    args = mi.TransformerArgs.from_dict(d)
    args.max_batch_size = max_batch
    m = Transformer.empty(args, "cuda", torch.bfloat16, expert_weights="fp8")
    with torch.no_grad():
        for k, shape in synth.state_dict_shapes(p):
            assert m._assign(k, synth.synth_tensor(k, shape, seed, torch.bfloat16, "cuda")), k
        if rank:  # adapter tensors one at a time, straight into the packed adapters
            for k, v in m.state_dict().items():
                if "lora_" in k:
                    assert m._assign(k, (synth.synth_tensor(k, tuple(v.shape), seed + 1, torch.float32, "cuda") * ADAPTER_SCALE).to(torch.bfloat16))
    return m.eval()


def timed(fn, reps: int) -> float:
    """Mean ms of fn() over reps calls, CUDA events around the whole loop."""
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def model_numbers(m: Transformer, p) -> dict:
    V = p["vocab_size"]
    out = {}
    toks = torch.tensor(synth.synth_prompt(4096, V, 1), device="cuda")

    def prefill():
        cache = BufferCache(m.n_local_layers, 1, 4096 + 256, p["n_kv_heads"], p["head_dim"], None).to(m.device, m.dtype)
        m.forward(toks, [4096], cache)
        return cache

    torch.cuda.reset_peak_memory_stats()
    prefill()  # warm-up
    retries = torch.cuda.memory_stats().get("num_alloc_retries", 0)
    ms = []
    for _ in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        cache = prefill()
        torch.cuda.synchronize()
        ms.append((time.perf_counter() - t0) * 1e3)
        if len(ms) < 3:
            del cache
    out["prefill_4096_ms"] = min(ms)
    out["prefill_4096_all_ms"] = [round(x, 1) for x in ms]
    # allocations the caching allocator could only serve after freeing its cache (a device-wide synchronisation each)
    out["prefill_alloc_retries"] = torch.cuda.memory_stats().get("num_alloc_retries", 0) - retries
    nxt = torch.tensor([3], device="cuda")
    for _ in range(8):  # eager step, capture, replays
        nxt = m.next_token_logits(nxt, cache).argmax(-1)
    ms = [timed(lambda: m.next_token_logits(m.last_argmax, cache), 64) for _ in range(3)]
    out["decode_b1_ctx4k_ms"] = min(ms)
    out["decode_b1_ctx4k_all_ms"] = [round(x, 3) for x in ms]
    out["decode_b1_finite"] = bool(torch.isfinite(m.next_token_logits(m.last_argmax, cache)).all())
    del cache
    torch.cuda.empty_cache()
    B, L = 32, 512
    cache = BufferCache(m.n_local_layers, B, L + 128, p["n_kv_heads"], p["head_dim"], None).to(m.device, m.dtype)
    toks = torch.tensor(synth.synth_prompt(B * L, V, 2), device="cuda").view(B, L)
    for c0 in range(0, L, 512):
        m.forward(toks[:, c0:c0 + 512].reshape(-1), [min(512, L - c0)] * B, cache)
    nxt = torch.arange(B, device="cuda")
    for _ in range(4):
        nxt = m.next_token_logits(nxt, cache).argmax(-1)
    ms = [timed(lambda: m.next_token_logits(m.last_argmax, cache), 16) for _ in range(3)]
    out["decode_b32_ctx512_step_ms"] = min(ms)
    out["decode_b32_finite"] = bool(torch.isfinite(m.next_token_logits(m.last_argmax, cache)).all())
    out["run_peak_gb"] = torch.cuda.max_memory_allocated() / 1e9
    del cache
    torch.cuda.empty_cache()
    return out


def family(name: str) -> str:
    for f in ("lora_down_reduce", "lora_down", "gemm_streamk_grouped_fp8", "gemm_wgmma_grouped_fp8", "gemm_streamk_grouped",
              "gemm_wgmma_grouped", "skinny_linear", "gemm_streamk", "gemm_wgmma", "moe_route", "moe_plan", "moe_gather", "moe_combine",
              "attn", "rmsnorm", "lm_head", "elementwise", "fill", "copy"):
        if f in name:
            return f
    return "other"


def profile(m: Transformer, p, out_dir) -> dict:
    from torch.profiler import ProfilerActivity, profile as tprofile

    V = p["vocab_size"]
    cache = BufferCache(m.n_local_layers, 1, 1024 + 64, p["n_kv_heads"], p["head_dim"], None).to(m.device, m.dtype)
    m.forward(torch.tensor(synth.synth_prompt(1024, V, 3), device="cuda"), [1024], cache)
    nxt = torch.tensor([3], device="cuda")
    for _ in range(4):
        nxt = m.next_token_logits(nxt, cache).argmax(-1)
    torch.cuda.synchronize()
    res = {}
    pcache = BufferCache(m.n_local_layers, 1, 4096 + 64, p["n_kv_heads"], p["head_dim"], None).to(m.device, m.dtype)
    ptoks = torch.tensor(synth.synth_prompt(4096, V, 4), device="cuda")
    for what, fn in (("decode_b1_x16", lambda: [m.next_token_logits(m.last_argmax, cache) for _ in range(16)]),
                     ("prefill_4096", lambda: m.forward(ptoks, [4096], pcache))):
        with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        fam = defaultdict(float)
        for ev in prof.key_averages():
            t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
            if t:
                fam[family(ev.key)] += t / 1e3
        res[what] = {k: round(v, 3) for k, v in sorted(fam.items(), key=lambda kv: -kv[1])}
        if out_dir is not None:
            prof.export_chrome_trace(str(Path(out_dir) / f"moe_lora_{what}.json"))
    return res


def ffn_numbers(p, seed: int) -> list:
    """One layer's grouped expert FFN: no adapters, r = 16 and r = 64, over the same routing, alternated."""
    dim, hidden = p["dim"], p["hidden_dim"]
    E, k = p["moe"]["num_experts"], p["moe"]["num_experts_per_tok"]
    gate = synth.synth_tensor("layers.0.feed_forward.gate.weight", (E, dim), seed, torch.bfloat16, "cuda")
    lora = {r: LoraArgs.from_dict(dict(rank=r, scaling=2.0)) if r else None for r in RANKS}
    experts = {r: [] for r in RANKS}
    for e in range(E):
        ws = {n: synth.synth_tensor(f"layers.0.feed_forward.experts.{e}.{n}.weight", shp, seed, torch.bfloat16, "cuda")
              for n, shp in (("w1", (hidden, dim)), ("w3", (hidden, dim)), ("w2", (dim, hidden)))}
        for r in RANKS:
            x = Fp8Expert(dim, hidden, lora[r]).to("cuda", torch.bfloat16)  # (the e4m3 and scale tensors are integers: kept)
            for n, t in ws.items():
                x.quantize_(n, t)
            for mod in x.modules():
                if isinstance(mod, LoraAdapter):
                    g = torch.Generator(device="cuda").manual_seed(seed * 7 + e)
                    mod.a.copy_(torch.randn(mod.a.shape, generator=g, device="cuda") * ADAPTER_SCALE)
                    mod.b.copy_(torch.randn(mod.b.shape, generator=g, device="cuda") * ADAPTER_SCALE)
            experts[r].append(x)
    tab = lambda ts: (ctypes.c_void_p * E)(*[t.data_ptr() for t in ts])  # noqa: E731
    rows = []
    for T in (1, 8, 32, 4096):
        g = torch.Generator(device="cuda").manual_seed(T)
        hn = torch.randn(T, dim, generator=g, device="cuda").to(torch.bfloat16)
        res = torch.zeros_like(hn)
        wsp = _abi.Workspace(_abi.workspace_bytes(T, dim, 1, 1, 128, hidden, 0, 1), torch.device("cuda"))
        runs = {}
        for r in RANKS:
            xs = experts[r]
            R13 = xs[0].w13_lora.rank_cols if r else 0
            b = MoeBuffers(T, dim, hidden, E, k, torch.device("cuda"), torch.bfloat16, lora_cols=R13)
            _abi.moe_route(hn, gate, E, k, 0, 1, b)
            out = torch.empty_like(hn)
            t8 = (tab([x.w13_q for x in xs]), tab([x.w13_scale_bits for x in xs]), tab([x.w2_q for x in xs]), tab([x.w2_scale_bits for x in xs]))
            if r:
                R2 = xs[0].w2_lora.rank_cols
                l13 = _abi.moe_lora_struct(tab([x.w13_lora.a for x in xs]), tab([x.w13_lora.b for x in xs]), R13, 2.0, b.lora_a, b.lora_l)
                l2 = _abi.moe_lora_struct(tab([x.w2_lora.a for x in xs]), tab([x.w2_lora.b for x in xs]), R2, 2.0,
                                          b.lora_a.view(-1)[: b.rows_cap * R2].view(b.rows_cap, R2), b.lora_l)
                runs[r] = (lambda b=b, t8=t8, out=out, l13=l13, l2=l2:
                           _abi.moe_grouped_ffn_fp8_lora(b, *t8, res, out, T, dim, hidden, E, k, None, wsp, l13, l2))
            else:
                runs[r] = lambda b=b, t8=t8, out=out: _abi.moe_grouped_ffn_fp8(b, *t8, res, out, T, dim, hidden, E, k, None, wsp)
        reps = 10 if T == 4096 else 100
        for f in runs.values():
            f()
        torch.cuda.synchronize()
        ms = {r: [] for r in runs}
        for _ in range(5):  # alternated
            for r, f in runs.items():
                ms[r].append(timed(f, reps))
        row = dict(T=T)
        for r, v in ms.items():
            row[f"r{r}_ms" if r else "plain_ms"] = round(sorted(v)[2], 4)
        rows.append(row)
        print("  " + json.dumps(row), flush=True)
    return rows


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=None, help="default: the model's own 32")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--trace-dir", default=None, help="with --profile: write the Chrome traces here")
    ap.add_argument("--ranks", default="0,16,64", help="model-level configurations, 0 = no adapters")
    ap.add_argument("--no-ffn", action="store_true", help="skip the one-layer grouped FFN comparison")
    a = ap.parse_args()
    ranks = [int(x) for x in a.ranks.split(",")]
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    p = synth.shape("mixtral-8x7b", **({"n_layers": a.layers} if a.layers else {}))
    res = {"card": card(), "model": "mixtral-8x7b", "experts": "fp8", "layers": p["n_layers"], "configs": {}}
    print(f"card: {res['card']}", flush=True)
    for r in ranks:
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        t0 = time.perf_counter()
        m = build(p, a.seed, r, 32)
        torch.cuda.synchronize()
        c = {"build_s": round(time.perf_counter() - t0, 1),
             "model_gb": round(sum(t.numel() * t.element_size() for t in m.parameters()) / 1e9, 3),
             "adapter_gb": round(sum(t.numel() * t.element_size() for mod in m.modules() if isinstance(mod, LoraAdapter)
                                     for t in mod.parameters()) / 1e9, 3),
             "build_peak_gb": round(torch.cuda.max_memory_allocated() / 1e9, 2)}
        c.update({k: (round(v, 3) if isinstance(v, float) else v) for k, v in model_numbers(m, p).items()})
        if a.profile and r:
            c["profile_device_ms"] = profile(m, p, a.trace_dir)
        res["configs"][f"r{r}" if r else "plain"] = c
        print(f"{'r' + str(r) if r else 'plain'}: {json.dumps(c)}", flush=True)
        del m
    torch.cuda.empty_cache()
    if not a.no_ffn:
        res["grouped_ffn"] = ffn_numbers(p, a.seed)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
