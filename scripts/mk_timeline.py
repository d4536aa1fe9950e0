"""Debug: per-phase timeline of the decode megakernel, Mistral-7B shape at kv_len 4096, and how much HBM time each bubble costs.
usage (on the GPU): python scripts/mk_timeline.py [n_layers]      (MB200_LIB_PATH selects the library, as everywhere)

Ideal times come from the shape's bytes (bench.decode_bytes_per_step) over bench.measured_peaks(); the ring's coverage is the
time one SM's share of that bandwidth takes to fill the ring, i.e. how long a consumer stall can last before the SM's
producers block on a full ring and its share of HBM goes idle."""
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import bench  # noqa: E402
import synth  # noqa: E402
from mistral_inference_b200 import _abi  # noqa: E402
from mistral_inference_b200.cache import BufferCache  # noqa: E402

STAMPS, WORDS = 16, 24  # timeline words per sampled CTA and layer (decode_megakernel.cuh, next to mk_stamp)
STAGE_BYTES, MAX_STAGES = 16 * 1024 + 16 * 16, 12  # MK_STAGE_BYTES, MK_MAX_STAGES
KV_LEN = 4096

L = int(sys.argv[1]) if len(sys.argv) > 1 else 8
p = synth.shape("mistral-7b", n_layers=L)
model = bench.build_gpu_model(p, 1)
cache = BufferCache(L, 1, KV_LEN + 64, p["n_kv_heads"], p["head_dim"], p["sliding_window"]).to(model.device, model.dtype)
for i in cache.cache_k:
    cache.cache_k[i].normal_()
    cache.cache_v[i].normal_()
cache._kv_seqlens_host = [5000]  # past the 4096-slot window: every layer attends over KV_LEN rows
tok = torch.tensor([17], device="cuda")
for _ in range(3):
    model.decode_static(tok, cache)
sm_count, smem_optin = _abi.device_info()
buf = torch.zeros(8 * L * WORDS, dtype=torch.int64, device="cuda")  # zeroed: the producers' blocked times are added to it
_abi.set_decode_timeline(buf)
bbuf = torch.zeros(sm_count * L * 6 * 2, dtype=torch.int64, device="cuda")
_abi.set_barrier_timeline(bbuf)
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
model.decode_static(tok, cache)
e1.record()
torch.cuda.synchronize()
_abi.set_decode_timeline(None)
_abi.set_barrier_timeline(None)

peaks = bench.measured_peaks()
layer_bytes = (bench.decode_bytes_per_step(p, KV_LEN) - bench.decode_bytes_per_step(dict(p, n_layers=0), KV_LEN)) / L
ideal_layer_us = layer_bytes / (peaks["hbm_gbs"] * 1e3)
# the ring: what decode_plan (abi.cu) leaves of the opt-in shared memory next to the activation buffer and the barrier tail
widest = max(p["dim"], p["hidden_dim"], p["n_heads"] * p["head_dim"])
xs_bytes = (max(2 * widest, 2048) + 127) // 128 * 128
n_stages = min(MAX_STAGES, (smem_optin - xs_bytes - (2 * MAX_STAGES * 8 + 48 * 4 + 32 + 8 + 64)) // STAGE_BYTES)
sm_share_gbs = peaks["hbm_gbs"] / sm_count
ring_us = n_stages * STAGE_BYTES / (sm_share_gbs * 1e3)
print(f"{torch.cuda.get_device_name()}, {sm_count} SMs; HBM {peaks['hbm_gbs']:.0f} GB/s ({peaks['source']}) = {sm_share_gbs:.1f} GB/s per SM; "
      f"ring {n_stages} x {STAGE_BYTES} B covers {ring_us:.2f} us of one SM's share")
print(f"kernel total {e0.elapsed_time(e1) * 1000:.1f} us for {L} layers + lm head; ideal per layer {ideal_layer_us:.1f} us "
      f"({layer_bytes / 1e6:.1f} MB at {peaks['hbm_gbs']:.0f} GB/s)")

t = buf.cpu().view(8, L, WORDS).double() / 1000.0  # us; sampled CTAs 0, 21, 42, ... (7 of them on 132 SMs)
active = [s for s in range(8) if 21 * s < sm_count]
t = t[active]
# (name, from stamp, to stamp, is a bubble: the consumers do not take stages from the ring)
phases = [("stage_x + RMSNorm", 0, 1, True), ("QKV gemv", 1, 2, False), ("barrier after QKV", 2, 3, True),
          ("attention slice", 3, 12, False), ("barrier after slice", 12, 13, True), ("slice merge", 13, 4, True),
          ("barrier after merge", 4, 5, True), ("stage_x + WO gemv", 5, 6, False), ("barrier after WO", 6, 7, True),
          ("stage_x + RMSNorm + GATEUP", 7, 8, False), ("barrier after GATEUP", 8, 9, True), ("stage_x + DOWN", 9, 10, False),
          ("barrier after DOWN", 10, 11, True)]
print(f"phase durations (us), median over layers 1.. per sampled CTA: min / CTA 0 / max   [bubbles: ring covers {ring_us:.2f} us]")
for name, a, b, bubble in phases:
    med = (t[:, 1:, b] - t[:, 1:, a]).median(1).values
    note = f"   bubble, {max(0.0, med.max().item() - ring_us):5.2f} us past the ring at the max" if bubble else ""
    print(f"  {name:28s} min {med.min():7.2f}   cta0 {med[0]:7.2f}   max {med.max():7.2f}{note}")
sub = torch.stack([t[:, 1:, 14] - t[:, 1:, 3], t[:, 1:, 15] - t[:, 1:, 3]], -1).median(1).values
print("  inside attention, since the phase start (us; first K/V stage ready | last K/V stage ready) per sampled CTA:",
      [[round(x, 2) for x in row] for row in sub.tolist()])
print(f"  layer total (cta0) {(t[0, 1:, 11] - t[0, 1:, 0]).median().item():8.2f} us   (ideal {ideal_layer_us:.1f} us)")

# producers' blocked time per layer (mean of the two producers), median over layers 1.. (the last layer also carries the lm head)
blk = t[:, :, STAMPS:STAMPS + 6].view(len(active), L, 3, 2).mean(-1)  # [cta, layer, kind]
mid = blk[:, 1:L - 1] if L > 2 else blk
print("producer blocked time per layer (us; median over layers 1..L-2, per sampled CTA min / median / max):")
for k, name in enumerate(["ring full (waiting for a free slot)", "in-flight cap", "ring full for 1 us or more (idle HBM share)"]):
    med = mid[:, :, k].median(1).values
    print(f"  {name:44s} min {med.min():7.2f}   median {med.median():7.2f}   max {med.max():7.2f}")

bt = bbuf.cpu().view(sm_count, L, 6, 2).double() / 1000.0
arr, lea = bt[:, 1:, :, 0], bt[:, 1:, :, 1]
print("ALL CTAs, per barrier (median over layers 1..): arrival skew (last - first arrive) | latency (first leave - last arrive) | leave spread")
for b, nm in enumerate(["after QKV", "after slice partial", "after slice merge", "after WO", "after GATEUP", "after DOWN"]):
    skew = (arr[:, :, b].max(0).values - arr[:, :, b].min(0).values).median().item()
    lat = (lea[:, :, b].min(0).values - arr[:, :, b].max(0).values).median().item()
    spread = (lea[:, :, b].max(0).values - lea[:, :, b].min(0).values).median().item()
    slow = arr[:, :, b].argmax(0).mode().values.item()
    print(f"  {nm:20s} skew {skew:6.2f}   latency {lat:6.2f}   leave spread {spread:6.2f}   (most often last: CTA {slow})")
