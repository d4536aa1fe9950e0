"""Pixtral-12B vision encoder on one GPU: ms per encoder forward (+ projection to the text dim), algorithmic TFLOPS, and the
head_dim-64 attention kernel alone against torch's scaled_dot_product_attention on the same q/k/v.  Prints one JSON line.

Synthetic seeded weights of the `pixtral-12b` shape (24 layers, hidden 1024, 16 heads of 64, intermediate 4096, adapter to 5120);
1 image and 4 images of 1024 x 1024 (4096 / 16384 patches: every patch attends to every patch of the call).
FLOPs are computed from shapes: 2*T*N*K per linear (conv as a GEMM with K = 3*16*16, QKV, wo, w1/w3, w2, adapter w_in / w_out) and
4*T^2*hd*H per layer for the unmasked attention; the share of peak is over the H100 SXM data-sheet dense BF16 figure.

    python scripts/bench_vision.py [--images 1 4] [--reps 10] [--out results/bench_vision.json]
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

REPO = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(REPO))

import torch  # noqa: E402

import mistral_inference_b200 as mi  # noqa: E402
import synth  # noqa: E402
from mistral_inference_b200 import _abi  # noqa: E402
from mistral_inference_b200.transformer import Transformer  # noqa: E402

PEAK_BF16_TFLOPS = 989.0  # H100 SXM data sheet, dense BF16


def encoder_flops(p: dict, T: int) -> dict:
    ve = p["vision_encoder"]
    d, inter, L, H = ve["hidden_size"], ve["intermediate_size"], ve["num_hidden_layers"], ve["num_attention_heads"]
    hd = d // H
    k_conv = ve["num_channels"] * ve["patch_size"] ** 2
    gemm = 2 * T * d * k_conv + L * (2 * T * 3 * d * d + 2 * T * d * d + 2 * T * 2 * inter * d + 2 * T * d * inter)
    adapter = 2 * T * p["dim"] * d + 2 * T * p["dim"] * p["dim"]
    attn = L * 4 * T * T * hd * H
    return {"gemm": gemm + adapter, "attention": attn, "total": gemm + adapter + attn}


def gpu_info() -> dict:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in q.split(",")]
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:  # noqa: BLE001
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": f"unavailable ({e})", "max_sm_clock": "unavailable"}


def time_ms(fn, reps: int, warmup: int = 2) -> float:
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(reps):
        fn()
    stop.record()
    torch.cuda.synchronize()
    return start.elapsed_time(stop) / reps


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, nargs="+", default=[1, 4])
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_vision needs a GPU"
    dev = torch.device("cuda", 0)
    p = synth.shape("pixtral-12b")
    args = mi.TransformerArgs.from_dict(dict(p))
    args.max_batch_size = 1
    # only the vision modules and the embedding are needed: a one-layer text model keeps the allocation small
    args.n_layers = 1
    model = Transformer.empty(args, dev, torch.bfloat16)
    keys = dict(synth.state_dict_shapes(dict(p, n_layers=1)))
    with torch.no_grad():
        for k, shp in keys.items():
            model._assign(k, synth.synth_tensor(k, shp, 1, device=dev))
    ve = model.vision_encoder
    H, hd = p["vision_encoder"]["num_attention_heads"], ve.head_dim
    result = {"model": "pixtral-12b vision encoder + adapter (synthetic weights)", "peak_tflops_datasheet_bf16": PEAK_BF16_TFLOPS, "runs": []}
    for n_img in a.images:
        imgs = [synth.synth_image(3, 1024, 1024, i).to(dev) for i in range(n_img)]
        T = 4096 * n_img

        def encode():
            f = ve(imgs)
            return model.vision_language_adapter(f, ve.workspace(f.shape[0]))

        with torch.inference_mode():
            ms = time_ms(encode, a.reps)
            g = torch.Generator(device=dev).manual_seed(0)
            q, k, v = (torch.randn(T, H * hd, device=dev, generator=g).to(torch.bfloat16) for _ in range(3))
            out = torch.empty_like(q)
            attn_ms = time_ms(lambda: _abi.attn_prefill(q, k, v, None, None, None, None, out, 1, T, 0, H, H, hd, causal=False), a.reps * 2)
            try:
                qs, ks, vs = (x.view(T, H, hd).transpose(0, 1)[None] for x in (q, k, v))
                sdpa_ms = time_ms(lambda: torch.nn.functional.scaled_dot_product_attention(qs, ks, vs), a.reps * 2)
                sdpa = {"ms": round(sdpa_ms, 4)}
            except Exception as e:  # noqa: BLE001
                sdpa = {"error": str(e)[:200]}
        fl = encoder_flops(p, T)
        run = {"images": n_img, "patches": T, "encoder_ms": round(ms, 3), "algorithmic_tflop": round(fl["total"] / 1e12, 3),
               "tflops": round(fl["total"] / ms / 1e9, 1), "fraction_of_datasheet_peak": round(fl["total"] / ms / 1e9 / PEAK_BF16_TFLOPS, 3),
               "attention_tflop_per_layer": round(fl["attention"] / p["vision_encoder"]["num_hidden_layers"] / 1e12, 3),
               "attn_kernel_ms_per_layer": round(attn_ms, 4),
               "attn_kernel_tflops": round(fl["attention"] / p["vision_encoder"]["num_hidden_layers"] / attn_ms / 1e9, 1),
               "torch_sdpa_same_qkv": sdpa}
        result["runs"].append(run)
    result.update(gpu_info())
    line = json.dumps(result)
    print(line)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
