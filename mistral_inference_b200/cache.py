"""Rotating KV cache (API mirror of mistral_inference/cache.py:140-263).

Same storage contract as the reference -- per layer `cache_k[i]`, `cache_v[i]` of shape
[max_batch, W_i, n_kv_heads, head_dim], token at absolute position p of sequence b in slot p % W_i
(cache.py:235), `kv_seqlens[b]` = tokens seen -- but the per-forward metadata is different in kind:
the reference builds xformers mask objects and bool/index tensors per LAYER with Python list
comprehensions and `.tolist()` syncs (cache.py:197-263); here one small int32 block is built on the host
with numpy (sequence lengths are host-known), uploaded with ONE copy per forward and shared by all
layers with the same window.  The kernels derive masks from (positions, seqpos, W) arithmetically.
"""
from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple, Union

import numpy as np
import torch

SlidingWindow = Union[None, int, List[Optional[int]]]
KV_CACHE_FORMATS = ("bf16", "fp8")


def get_cache_sizes(n_layers: int, max_seq_len: int, sliding_window: SlidingWindow) -> List[int]:
    """cache.py:13-24."""
    if sliding_window is None:
        return n_layers * [max_seq_len]
    elif isinstance(sliding_window, int):
        return n_layers * [sliding_window]
    else:
        assert isinstance(sliding_window, list), f"Expected list, got {type(sliding_window)}"
        assert n_layers % len(sliding_window) == 0, f"Expected n_layers % len(sliding_window) == 0, got {n_layers} % {len(sliding_window)}"
        num_repeats = n_layers // len(sliding_window)
        return num_repeats * [w if w is not None else max_seq_len for w in sliding_window]


@dataclass
class CacheInputMetadata:
    """What one layer's kernels need for this forward (device int32 tensors are views into one upload)."""
    positions: torch.Tensor   # [T] absolute positions (rope + masks)
    cache_rows: torch.Tensor  # [T] flat ring row slot + b*W, or -1 when the token is not cached (cache.py:226,235)
    kv_len: torch.Tensor      # [B] decode only: valid ring slots once this token is written = min(seqpos+1, W)
    q_start: torch.Tensor     # [B+1] prefix sums of seqlens
    seqpos: torch.Tensor      # [B] tokens already cached before this forward
    prefill: bool             # first or subsequent prefill (cache.py:236-237); False = one-token decode
    first_prefill: bool       # nothing cached yet for any sequence (cache.py:236,239)
    seqlens: List[int]
    max_seqlen: int
    window: int               # W of this layer


class CacheView:
    """cache.py:70-137: one layer's ring plus the metadata of this forward."""

    def __init__(self, cache_k: torch.Tensor, cache_v: torch.Tensor, metadata: CacheInputMetadata, kv_seqlens_host: List[int],
                 cache_k_exp: Optional[torch.Tensor] = None, cache_v_exp: Optional[torch.Tensor] = None):
        self.cache_k = cache_k
        self.cache_v = cache_v
        self.cache_k_exp = cache_k_exp  # FP8 cache: int8 exponents [max_batch, W, KV] of the e4m3 rows (None for bf16)
        self.cache_v_exp = cache_v_exp
        self.metadata = metadata
        self.kv_seqlens_host = kv_seqlens_host

    @property
    def max_seq_len(self) -> int:
        return self.cache_k.shape[1]

    @property
    def key(self) -> torch.Tensor:
        return self.cache_k[: len(self.kv_seqlens_host)]

    @property
    def value(self) -> torch.Tensor:
        return self.cache_v[: len(self.kv_seqlens_host)]

    @property
    def prefill(self) -> bool:
        return self.metadata.prefill

    @property
    def fp8(self) -> bool:
        return self.cache_k_exp is not None


class BufferCache:
    """Rectangular rotating cache; constructor and methods as cache.py:140-195.

    kv_cache="fp8" stores every row as e4m3 codes with one int8 power-of-two exponent per (slot, kv head): `cache_k[i]` /
    `cache_v[i]` are torch.float8_e4m3fn [max_batch, W, KV, hd] and `cache_k_exp[i]` / `cache_v_exp[i]` int8 [max_batch, W, KV]
    (format: include/mistral_b200.h, mb200_kv_quantize).  Half the bytes of the bf16 cache plus 1/128 for the exponents."""

    def __init__(self, n_layers: int, max_batch_size: int, max_seq_len: int, n_kv_heads: int, head_dim: int,
                 sliding_window: SlidingWindow = None, kv_cache: str = "bf16"):
        if kv_cache not in KV_CACHE_FORMATS:
            raise ValueError(f"kv_cache={kv_cache!r}: expected one of {KV_CACHE_FORMATS}")
        if kv_cache == "fp8" and head_dim != 128:
            raise ValueError(f"kv_cache='fp8' needs head_dim 128 (got {head_dim})")
        self.kv_cache = kv_cache
        self.max_seq_len = max_seq_len
        self.n_kv_heads = n_kv_heads
        self.head_dim = head_dim
        self.n_layers = n_layers
        self.max_batch_size = max_batch_size
        self.cache_sizes: List[int] = get_cache_sizes(n_layers, max_seq_len, sliding_window)
        assert len(self.cache_sizes) == n_layers, f"Expected {n_layers} cache sizes, got {len(self.cache_sizes)}"
        self.cache_k: Dict[int, torch.Tensor] = {}
        self.cache_v: Dict[int, torch.Tensor] = {}
        self.cache_k_exp: Dict[int, torch.Tensor] = {}
        self.cache_v_exp: Dict[int, torch.Tensor] = {}
        for i, cache_size in enumerate(self.cache_sizes):
            if kv_cache == "fp8":
                self.cache_k[i] = torch.empty((max_batch_size, cache_size, n_kv_heads, head_dim), dtype=torch.float8_e4m3fn)
                self.cache_v[i] = torch.empty((max_batch_size, cache_size, n_kv_heads, head_dim), dtype=torch.float8_e4m3fn)
                self.cache_k_exp[i] = torch.empty((max_batch_size, cache_size, n_kv_heads), dtype=torch.int8)
                self.cache_v_exp[i] = torch.empty((max_batch_size, cache_size, n_kv_heads), dtype=torch.int8)
            else:
                self.cache_k[i] = torch.empty((max_batch_size, cache_size, n_kv_heads, head_dim))
                self.cache_v[i] = torch.empty((max_batch_size, cache_size, n_kv_heads, head_dim))
        # host copy of the valid length per batch element (the reference keeps it on the device and syncs, cache.py:217)
        self._kv_seqlens_host: Optional[List[int]] = None

    # -- reference API --------------------------------------------------------------------------
    def get_view(self, layer_id: int, metadata: CacheInputMetadata) -> CacheView:
        assert self._kv_seqlens_host is not None
        return CacheView(self.cache_k[layer_id], self.cache_v[layer_id], metadata, self._kv_seqlens_host,
                         self.cache_k_exp.get(layer_id), self.cache_v_exp.get(layer_id))

    def reset(self) -> None:
        self._kv_seqlens_host = None

    def init_kvseqlens(self, batch_size: int) -> None:
        self._kv_seqlens_host = [0] * batch_size

    @property
    def kv_seqlens(self) -> Optional[torch.Tensor]:
        if self._kv_seqlens_host is None:
            return None
        return torch.tensor(self._kv_seqlens_host, device=self.device, dtype=torch.long)

    @property
    def device(self) -> torch.device:
        return self.cache_k[0].device

    def to(self, device: torch.device, dtype: torch.dtype) -> "BufferCache":
        """Moves the cache; a bf16 cache takes `dtype`, an FP8 cache keeps its element format (e4m3 codes, int8 exponents)."""
        for i in range(self.n_layers):
            if self.kv_cache == "fp8":
                self.cache_k[i] = self.cache_k[i].to(device=device)
                self.cache_v[i] = self.cache_v[i].to(device=device)
                self.cache_k_exp[i] = self.cache_k_exp[i].to(device=device)
                self.cache_v_exp[i] = self.cache_v_exp[i].to(device=device)
            else:
                self.cache_k[i] = self.cache_k[i].to(device=device, dtype=dtype)
                self.cache_v[i] = self.cache_v[i].to(device=device, dtype=dtype)
        return self

    @property
    def nbytes(self) -> int:
        """Bytes of every ring (and, for an FP8 cache, its exponents)."""
        tensors = list(self.cache_k.values()) + list(self.cache_v.values()) + list(self.cache_k_exp.values()) + list(self.cache_v_exp.values())
        return sum(t.numel() * t.element_size() for t in tensors)

    def update_seqlens(self, seqlens: List[int]) -> None:
        assert self._kv_seqlens_host is not None
        self._kv_seqlens_host = [a + b for a, b in zip(self._kv_seqlens_host, seqlens)]

    # -- metadata ---------------------------------------------------------------------------------
    def get_input_metadata(self, seqlens: List[int]) -> List[CacheInputMetadata]:
        """One CacheInputMetadata per layer (shared objects for layers with equal W)."""
        host, layout = self.build_metadata_host(seqlens)
        dev = torch.from_numpy(host).to(self.device, non_blocking=False)
        return self.metadata_from_block(dev, layout, seqlens)

    def build_metadata_host(self, seqlens: List[int]) -> Tuple[np.ndarray, dict]:
        """Packs [positions | q_start | seqpos | (cache_rows, kv_len) per distinct W] into one int32 array."""
        if self._kv_seqlens_host is None:
            self.init_kvseqlens(len(seqlens))
        assert self._kv_seqlens_host is not None
        assert len(seqlens) == len(self._kv_seqlens_host), (
            f"Batch size is {len(self._kv_seqlens_host)}, got {len(seqlens)}, did you forget to reset cache?")
        assert len(seqlens) > 0, seqlens
        seqpos = np.asarray(self._kv_seqlens_host, dtype=np.int64)
        sl = np.asarray(seqlens, dtype=np.int64)
        B, T = len(seqlens), int(sl.sum())
        first_prefill = bool(seqpos[0] == 0)
        subsequent_prefill = bool((sl > 1).any())
        if first_prefill:
            assert (seqpos == 0).all(), seqpos.tolist()  # cache.py:239
        q_start = np.zeros(B + 1, dtype=np.int64)
        np.cumsum(sl, out=q_start[1:])
        batch_idx = np.repeat(np.arange(B, dtype=np.int64), sl)
        local = np.arange(T, dtype=np.int64) - q_start[batch_idx]
        positions = seqpos[batch_idx] + local
        distinct = sorted(set(self.cache_sizes))
        total = T + (B + 1) + B + len(distinct) * (T + B)
        host = np.empty(total, dtype=np.int32)
        layout = {"T": T, "B": B, "prefill": first_prefill or subsequent_prefill, "first_prefill": first_prefill, "max_seqlen": int(sl.max()), "windows": distinct}
        o = 0
        host[o:o + T] = positions; o += T
        host[o:o + B + 1] = q_start; o += B + 1
        host[o:o + B] = seqpos; o += B
        for W in distinct:
            cached = local >= (sl[batch_idx] - W)  # only the last W tokens of each chunk (cache.py:226)
            rows = np.where(cached, positions % W + batch_idx * W, -1)
            host[o:o + T] = rows; o += T
            host[o:o + B] = np.minimum(seqpos + np.minimum(sl, W), W); o += B
        return host, layout

    def metadata_from_block(self, dev: torch.Tensor, layout: dict, seqlens: List[int]) -> List[CacheInputMetadata]:
        T, B = layout["T"], layout["B"]
        o = 0
        positions = dev[o:o + T]; o += T
        q_start = dev[o:o + B + 1]; o += B + 1
        seqpos = dev[o:o + B]; o += B
        per_w: Dict[int, CacheInputMetadata] = {}
        for W in layout["windows"]:
            rows = dev[o:o + T]; o += T
            kv_len = dev[o:o + B]; o += B
            per_w[W] = CacheInputMetadata(positions=positions, cache_rows=rows, kv_len=kv_len, q_start=q_start, seqpos=seqpos,
                                          prefill=layout["prefill"], first_prefill=layout["first_prefill"], seqlens=list(seqlens), max_seqlen=layout["max_seqlen"], window=W)
        return [per_w[W] for W in self.cache_sizes]
