"""ctypes binding of libmb200.so (C ABI: include/mistral_b200.h).

This is the only place Python touches the native library.  There is NO fallback: if the library is
missing or a call fails, an exception is raised (the product path never routes through PyTorch
reference math or the CPU oracle).
"""
import ctypes
import os
from ctypes import c_char_p, c_float, c_int, c_int64, c_size_t, c_void_p
from pathlib import Path
from typing import NamedTuple, Optional

import torch

_LIB_PATH = Path(os.environ.get("MB200_LIB_PATH") or Path(__file__).resolve().parent / "libmb200.so")  # override: A/B builds of experiments
_lib: Optional[ctypes.CDLL] = None

ABI_VERSION = 5
SKINNY_MAX_T = 4
WORKSPACE_HEADER_BYTES = 64 * 1024

# name -> (restype, argtypes); mirrors include/mistral_b200.h declaration by declaration
_SIGNATURES = {
    "mb200_abi_version": (c_int, []),
    "mb200_last_error": (c_char_p, []),
    "mb200_device_info": (c_int, [ctypes.POINTER(c_int), ctypes.POINTER(c_int)]),
    "mb200_rmsnorm": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_float, c_void_p]),
    "mb200_attn_qkv": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                               c_void_p, c_int64, c_int64, c_int64, c_int64, c_int64, c_float, c_void_p, c_size_t, c_void_p]),
    "mb200_kv_ring_write": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int64, c_void_p]),
    "mb200_attn_decode": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int64, c_int64,
                                  c_int64, c_void_p, c_size_t, c_void_p]),
    "mb200_attn_prefill": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int64,
                                   c_int64, c_int64, c_int64, c_int64, c_int64, c_int, c_void_p]),
    "mb200_kv_quantize": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int64, c_void_p]),
    "mb200_attn_decode_fp8": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int64,
                                      c_int64, c_int64, c_void_p, c_size_t, c_void_p]),
    "mb200_attn_prefill_fp8": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                       c_int64, c_int64, c_int64, c_int64, c_int64, c_int64, c_int64, c_int, c_void_p]),
    "mb200_linear_residual": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int64, c_void_p, c_size_t, c_void_p]),
    "mb200_linear_bias": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int, c_void_p, c_size_t, c_void_p]),
    "mb200_vision_patchify": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int64, c_int64, c_void_p]),
    "mb200_patch_merge": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int64, c_void_p]),
    "mb200_embed_splice": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int64, c_int64, c_void_p]),
    "mb200_ffn_gateup": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int64, c_float, c_void_p, c_size_t,
                                 c_void_p]),
    "mb200_attn_qkv_lora": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                    c_void_p, c_int64, c_int64, c_int64, c_int64, c_int64, c_float, c_void_p, c_size_t, c_void_p, c_void_p]),
    "mb200_ffn_gateup_lora": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int64, c_float, c_void_p, c_size_t,
                                      c_void_p, c_void_p]),
    "mb200_linear_residual_lora": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int64, c_void_p, c_size_t, c_void_p,
                                           c_void_p]),
    "mb200_lm_head": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int64, c_float, c_void_p, c_size_t,
                              c_void_p]),
    "mb200_decode_meta": (c_int, [c_void_p, c_void_p, c_int64, c_void_p, c_int64, c_void_p]),
    "mb200_argmax_rows": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_void_p]),
    "mb200_logprob_gather": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_void_p]),
    "mb200_sample_top_p": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_float, c_float, c_void_p]),
    "mb200_select_tokens": (c_int, [c_void_p] * 10 + [c_int64, c_int64, c_void_p]),
    "mb200_spec_meta": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_void_p, c_int64, c_void_p]),
    "mb200_spec_accept_greedy": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int64, c_void_p]),
    "mb200_spec_accept_sample": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int64,
                                         c_float, c_float, c_void_p]),
    "mb200_moe_sizes": (c_int, [c_int64, c_int64, c_int64, ctypes.POINTER(c_int64), ctypes.POINTER(c_int64), ctypes.POINTER(c_int64)]),
    "mb200_moe_route": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int64, c_int64, c_int64, c_void_p, c_void_p, c_void_p, c_void_p,
                                c_void_p, c_void_p, c_void_p]),
    "mb200_moe_grouped_ffn": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64,
                                      c_int64, c_int64, c_int64, c_int64, c_void_p, c_void_p, c_size_t, c_void_p]),
    "mb200_quantize_e4m3_rows": (c_int, [c_void_p, c_int64, c_int64, c_void_p, c_int64, c_void_p, c_int64, c_void_p]),
    "mb200_moe_grouped_ffn_fp8": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                          c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int64, c_int64, c_void_p, c_void_p, c_size_t, c_void_p]),
    "mb200_moe_grouped_ffn_fp8_lora": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                               c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int64, c_int64, c_void_p, c_void_p,
                                               c_size_t, c_void_p, c_void_p, c_void_p]),
    "mb200_moe_grouped_ffn_int4": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                           c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int64, c_int64, c_void_p, c_void_p, c_size_t, c_void_p]),
    "mb200_comm_alloc": (c_int, [c_size_t, ctypes.POINTER(c_void_p)]),
    "mb200_comm_free": (c_int, [c_void_p]),
    "mb200_comm_export": (c_int, [c_void_p, c_void_p]),
    "mb200_comm_open": (c_int, [c_void_p, ctypes.POINTER(c_void_p)]),
    "mb200_comm_close": (c_int, [c_void_p]),
    "mb200_workspace_bytes": (c_size_t, [c_int64] * 8),
    "mb200_decode_step": (c_int, [c_void_p, c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int64,
                                  c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int64, c_int64, c_int64, c_float, c_int64, c_int64, c_void_p,
                                  c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "mb200_debug_set_decode_timeline": (c_int, [c_void_p]),
    "mb200_debug_set_barrier_timeline": (c_int, [c_void_p]),
    "mb200_debug_launch_log": (c_int, [c_int, c_void_p, c_size_t]),
    "mb200_debug_decode_scratch": (c_int, [c_int64] * 7 + [ctypes.POINTER(c_size_t), ctypes.POINTER(c_size_t)]),
    "mb200_debug_decode_buffers": (c_int, [c_int64] * 7 + [ctypes.POINTER(c_size_t)]),
    "mb200_decode_step_supported": (c_int, [c_int64] * 9),
    "mb200_attn_qkv_fp8": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                   c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int64, c_int64, c_float, c_void_p, c_size_t, c_void_p]),
    "mb200_ffn_gateup_fp8": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int64, c_float, c_void_p,
                                     c_size_t, c_void_p]),
    "mb200_linear_residual_fp8": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int64, c_void_p,
                                          c_size_t, c_void_p]),
    "mb200_attn_qkv_fp8a8": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                     c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int64, c_int64, c_float, c_void_p, c_size_t, c_void_p]),
    "mb200_ffn_gateup_fp8a8": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int64, c_float, c_void_p,
                                       c_size_t, c_void_p]),
    "mb200_linear_residual_fp8a8": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int64, c_void_p,
                                            c_size_t, c_void_p]),
    "mb200_quantize_act_e4m3": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_float, c_void_p]),
    "mb200_decode_step_fp8": (c_int, [c_void_p, c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int64,
                                      c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int64, c_int64, c_int64, c_float, c_void_p, c_size_t,
                                      c_void_p]),
    "mb200_decode_step_fp8_supported": (c_int, [c_int64] * 7),
    "mb200_quantize_int4_groups": (c_int, [c_void_p, c_int64, c_int64, c_void_p, c_int64, c_void_p, c_int64, c_void_p]),
    "mb200_attn_qkv_int4": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                    c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int64, c_int64, c_float, c_void_p, c_size_t, c_void_p]),
    "mb200_ffn_gateup_int4": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int64, c_float, c_void_p,
                                      c_size_t, c_void_p]),
    "mb200_linear_residual_int4": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int64, c_void_p,
                                           c_size_t, c_void_p]),
    "mb200_debug_attn_decode_occupancy": (c_int, [c_int64, ctypes.POINTER(c_int)]),
    "mb200_test_gemm_naive": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int64, c_void_p]),
}


class Mb200Error(RuntimeError):
    pass


def library_path() -> Path:
    return _LIB_PATH


def lib() -> ctypes.CDLL:
    """Loads libmb200.so once.  Raises (never falls back) when it is missing or has the wrong ABI."""
    global _lib
    if _lib is not None:
        return _lib
    if not _LIB_PATH.exists():
        raise Mb200Error(
            f"{_LIB_PATH} not found: build it with `python -m mistral_inference_b200.build` "
            "(there is no PyTorch/CPU fallback for the hot path)")
    handle = ctypes.CDLL(str(_LIB_PATH), mode=os.RTLD_LOCAL if hasattr(os, "RTLD_LOCAL") else 0)
    for name, (restype, argtypes) in _SIGNATURES.items():
        fn = getattr(handle, name)  # AttributeError if a declared symbol is not exported
        fn.restype = restype
        fn.argtypes = argtypes
    if handle.mb200_abi_version() != ABI_VERSION:
        raise Mb200Error(f"libmb200 ABI {handle.mb200_abi_version()} != expected {ABI_VERSION}")
    _lib = handle
    return handle


def _check(rc: int, what: str) -> None:
    if rc != 0:
        msg = lib().mb200_last_error()
        raise Mb200Error(f"{what} failed ({rc}): {msg.decode() if msg else '?'}")


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    if t is None:
        return None
    assert t.is_cuda and t.is_contiguous(), "libmb200 takes contiguous CUDA tensors"
    return t.data_ptr()


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


class Workspace:
    """Caller-owned scratch handed to every entry point (zero-filled once: the first 64 KiB hold self-resetting
    counters, see MB200_WORKSPACE_HEADER_BYTES).  Also owns the model-wide mixture-of-experts row buffers and, for an
    expert-parallel model, the NVLink peer memory of the group (mistral_inference_b200/moe.py)."""

    def __init__(self, nbytes: int, device: torch.device):
        self.buf = torch.zeros(max(int(nbytes), WORKSPACE_HEADER_BYTES + 256), dtype=torch.uint8, device=device)
        self._moe: dict = {}
        self._comm = None

    def moe_buffers(self, T: int, dim: int, hidden: int, E: int, k: int, dtype: torch.dtype, comm=None, parity: int = 0, lora_cols: int = 0):
        from .moe import MoeBuffers

        key = (T, dim, hidden, E, k, parity if comm is not None else 0, id(comm), lora_cols)
        b = self._moe.get(key)
        if b is None:
            if len(self._moe) >= 8:  # prompt chunks of many different lengths: keep the pool small
                self._moe.clear()
            yw_ptr = comm.yw_ptr(parity) if comm is not None else None
            b = self._moe[key] = MoeBuffers(T, dim, hidden, E, k, self.buf.device, dtype, yw_ptr=yw_ptr, lora_cols=lora_cols)
        return b

    def expert_comm(self, layer, T: int, dim: int):
        """The group's peer memory, (re)created collectively when a call needs more rows than it holds."""
        from .moe import ExpertComm

        _, rows_cap, _ = moe_sizes(T, layer.args.num_experts, layer.args.num_experts_per_tok)
        if self._comm is None or self._comm.rows_cap < rows_cap or self._comm.dim != dim:
            if self._comm is not None:
                torch.cuda.synchronize()
                self._comm.close()
                self._moe.clear()
            g, G = layer.expert_shard
            self._comm = ExpertComm(g, G, layer.expert_group, rows_cap, dim, self.buf.device)
        return self._comm

    @property
    def ptr(self) -> int:
        return self.buf.data_ptr()

    @property
    def nbytes(self) -> int:
        return self.buf.numel()


def workspace_bytes(T: int, dim: int, n_heads: int, n_kv_heads: int, head_dim: int, hidden: int, vocab: int, max_batch: int) -> int:
    return int(lib().mb200_workspace_bytes(T, dim, n_heads, n_kv_heads, head_dim, hidden, vocab, max_batch))


def device_info():
    sm, smem = c_int(0), c_int(0)
    _check(lib().mb200_device_info(ctypes.byref(sm), ctypes.byref(smem)), "mb200_device_info")
    return sm.value, smem.value


# ----------------------------------------------------------------------------- thin typed wrappers
def rmsnorm(x: torch.Tensor, w: torch.Tensor, eps: float, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    T, dim = x.shape
    out = torch.empty_like(x) if out is None else out
    _check(lib().mb200_rmsnorm(_ptr(x), _ptr(w), _ptr(out), T, dim, eps, _stream()), "mb200_rmsnorm")
    return out


def attn_qkv(x, norm_w, wqkv, rope, positions, q_out, k_out, v_out, cache_k, cache_v, cache_rows, n_heads, n_kv_heads, head_dim, eps,
             ws: Workspace) -> None:
    T, dim = x.shape
    _check(lib().mb200_attn_qkv(_ptr(x), _ptr(norm_w), _ptr(wqkv), _ptr(rope), _ptr(positions), _ptr(q_out), _ptr(k_out), _ptr(v_out),
                                _ptr(cache_k), _ptr(cache_v), _ptr(cache_rows), T, dim, n_heads, n_kv_heads, head_dim, eps, ws.ptr,
                                ws.nbytes, _stream()), "mb200_attn_qkv")


def kv_ring_write(k_new, v_new, cache_k, cache_v, cache_rows, n_kv_heads, head_dim) -> None:
    _check(lib().mb200_kv_ring_write(_ptr(k_new), _ptr(v_new), _ptr(cache_k), _ptr(cache_v), _ptr(cache_rows), k_new.shape[0],
                                     n_kv_heads, head_dim, _stream()), "mb200_kv_ring_write")


def attn_decode(q, cache_k, cache_v, kv_len, out, n_heads, n_kv_heads, head_dim, n_splits, ws: Workspace) -> None:
    B = q.shape[0]
    W = cache_k.shape[1]
    _check(lib().mb200_attn_decode(_ptr(q), _ptr(cache_k), _ptr(cache_v), _ptr(kv_len), _ptr(out), B, W, n_heads, n_kv_heads, head_dim,
                                   n_splits, ws.ptr, ws.nbytes, _stream()), "mb200_attn_decode")


def attn_prefill(q, k_new, v_new, cache_k, cache_v, q_start, seqpos, out, B, max_seqlen, W, n_heads, n_kv_heads, head_dim,
                 causal: bool, first_prefill: bool = False) -> None:
    _check(lib().mb200_attn_prefill(_ptr(q), _ptr(k_new), _ptr(v_new), _ptr(cache_k), _ptr(cache_v), _ptr(q_start), _ptr(seqpos),
                                    _ptr(out), q.shape[0], B, max_seqlen, W, n_heads, n_kv_heads, head_dim, (2 if first_prefill else 1) if causal else 0,
                                    _stream()), "mb200_attn_prefill")


def kv_quantize(k, v, write_back: bool, cache_k=None, cache_v=None, exp_k=None, exp_v=None, cache_rows=None) -> None:
    """FP8 KV cache (include/mistral_b200.h): k, v [T, KV*hd] bf16 <- k', v' when `write_back`; (q, e) of each token t with
    cache_rows[t] >= 0 into the e4m3 ring cache_k / cache_v [.., KV, hd] and its int8 exponents exp_k / exp_v [.., KV]."""
    KV = exp_k.shape[-1] if exp_k is not None else k.shape[1] // 128
    _check(lib().mb200_kv_quantize(_ptr(k), _ptr(v), int(write_back), _ptr(cache_k), _ptr(cache_v), _ptr(exp_k), _ptr(exp_v), _ptr(cache_rows),
                                   k.shape[0], KV, k.shape[1] // KV, _stream()), "mb200_kv_quantize")


def attn_decode_fp8(q, cache_k, cache_v, exp_k, exp_v, kv_len, out, n_heads, n_kv_heads, head_dim, n_splits, ws: Workspace) -> None:
    B = q.shape[0]
    W = cache_k.shape[1]
    _check(lib().mb200_attn_decode_fp8(_ptr(q), _ptr(cache_k), _ptr(cache_v), _ptr(exp_k), _ptr(exp_v), _ptr(kv_len), _ptr(out), B, W, n_heads,
                                       n_kv_heads, head_dim, n_splits, ws.ptr, ws.nbytes, _stream()), "mb200_attn_decode_fp8")


def attn_prefill_fp8(q, k_new, v_new, cache_k, cache_v, exp_k, exp_v, q_start, seqpos, out, B, max_seqlen, W, n_heads, n_kv_heads, head_dim,
                     first_prefill: bool = False) -> None:
    _check(lib().mb200_attn_prefill_fp8(_ptr(q), _ptr(k_new), _ptr(v_new), _ptr(cache_k), _ptr(cache_v), _ptr(exp_k), _ptr(exp_v), _ptr(q_start),
                                        _ptr(seqpos), _ptr(out), q.shape[0], B, max_seqlen, W, n_heads, n_kv_heads, head_dim,
                                        2 if first_prefill else 1, _stream()), "mb200_attn_prefill_fp8")


def linear_residual(x, w, residual, out, ws: Workspace) -> None:
    T, K = x.shape
    N = w.shape[0]
    _check(lib().mb200_linear_residual(_ptr(x), _ptr(w), _ptr(residual), _ptr(out), T, N, K, ws.ptr, ws.nbytes, _stream()),
           "mb200_linear_residual")


def linear_bias(x, w, bias, out, gelu: bool, ws: Workspace) -> None:
    """out = bf16(x @ w^T + bias), optionally followed by the exact-erf GELU (bias may be None)."""
    T, K = x.shape
    _check(lib().mb200_linear_bias(_ptr(x), _ptr(w), _ptr(bias), _ptr(out), T, w.shape[0], K, int(gelu), ws.ptr, ws.nbytes, _stream()),
           "mb200_linear_bias")


def vision_patchify(image: torch.Tensor, out: torch.Tensor, patch: int) -> None:
    """image [C, H, W] bf16 -> out [(H//p) * (W//p), k_pad] (the patch Conv2d's GEMM operand, zero-padded columns)."""
    C, H, W = image.shape
    _check(lib().mb200_vision_patchify(_ptr(image), _ptr(out), C, H, W, patch, out.shape[1], _stream()), "mb200_vision_patchify")


def patch_merge(x: torch.Tensor, out: torch.Tensor, h: int, w: int, s: int) -> None:
    """PatchMerger.permute of one image of h x w patch features x [h*w, d] -> out [(h//s) * (w//s), d*s*s]."""
    _check(lib().mb200_patch_merge(_ptr(x), _ptr(out), h, w, s, x.shape[1], _stream()), "mb200_patch_merge")


def embed_splice(ids: torch.Tensor, emb: torch.Tensor, feats: torch.Tensor, out: torch.Tensor, image_token_id: int) -> int:
    """Text embedding rows with image feature rows at the image-token positions; returns the number of image tokens in `ids`
    (one 4-byte device-to-host read)."""
    T, V, dim = ids.shape[0], emb.shape[0], emb.shape[1]
    assert ids.dtype == torch.long
    ordinal = torch.empty(T + 1, dtype=torch.int32, device=ids.device)
    _check(lib().mb200_embed_splice(_ptr(ids), _ptr(emb), _ptr(feats), _ptr(out), _ptr(ordinal), T, dim, V, feats.shape[0], image_token_id,
                                    _stream()), "mb200_embed_splice")
    return int(ordinal[T].item())


def ffn_gateup(x, norm_w, w13, g_out, eps, ws: Workspace) -> None:
    T, dim = x.shape
    hidden = w13.shape[0] // 2
    _check(lib().mb200_ffn_gateup(_ptr(x), _ptr(norm_w), _ptr(w13), _ptr(g_out), T, dim, hidden, eps, ws.ptr, ws.nbytes, _stream()),
           "mb200_ffn_gateup")


# ---- FP8 dense weights (include/mistral_b200.h): w_q is the e4m3 matrix as uint8 [N, K], w_scale its fp32 row scales [N] ----
def _check_fp8(w_q: torch.Tensor, w_scale: torch.Tensor) -> None:
    assert w_q.dtype == torch.uint8 and w_scale.dtype == torch.float32 and w_scale.shape == (w_q.shape[0],), (w_q.dtype, w_scale.dtype)


def attn_qkv_fp8(x, norm_w, w_q, w_scale, rope, positions, q_out, k_out, v_out, cache_k, cache_v, cache_rows, n_heads, n_kv_heads, head_dim,
                 eps, ws: Workspace, *, a8: bool = False) -> None:
    """a8: the prefill-sized calls take FP8 activations (mb200_attn_qkv_fp8a8); every other call is the same as without."""
    _check_fp8(w_q, w_scale)
    T, dim = x.shape
    fn, name = (lib().mb200_attn_qkv_fp8a8, "mb200_attn_qkv_fp8a8") if a8 else (lib().mb200_attn_qkv_fp8, "mb200_attn_qkv_fp8")
    _check(fn(_ptr(x), _ptr(norm_w), _ptr(w_q), _ptr(w_scale), _ptr(rope), _ptr(positions), _ptr(q_out), _ptr(k_out), _ptr(v_out), _ptr(cache_k),
              _ptr(cache_v), _ptr(cache_rows), T, dim, n_heads, n_kv_heads, head_dim, eps, ws.ptr, ws.nbytes, _stream()), name)


def ffn_gateup_fp8(x, norm_w, w_q, w_scale, g_out, eps, ws: Workspace, *, a8: bool = False) -> None:
    _check_fp8(w_q, w_scale)
    T, dim = x.shape
    hidden = w_q.shape[0] // 2
    fn, name = (lib().mb200_ffn_gateup_fp8a8, "mb200_ffn_gateup_fp8a8") if a8 else (lib().mb200_ffn_gateup_fp8, "mb200_ffn_gateup_fp8")
    _check(fn(_ptr(x), _ptr(norm_w), _ptr(w_q), _ptr(w_scale), _ptr(g_out), T, dim, hidden, eps, ws.ptr, ws.nbytes, _stream()), name)


def linear_residual_fp8(x, w_q, w_scale, residual, out, ws: Workspace, *, a8: bool = False) -> None:
    _check_fp8(w_q, w_scale)
    T, K = x.shape
    N = w_q.shape[0]
    fn, name = ((lib().mb200_linear_residual_fp8a8, "mb200_linear_residual_fp8a8") if a8
                else (lib().mb200_linear_residual_fp8, "mb200_linear_residual_fp8"))
    _check(fn(_ptr(x), _ptr(w_q), _ptr(w_scale), _ptr(residual), _ptr(out), T, N, K, ws.ptr, ws.nbytes, _stream()), name)


def quantize_act_e4m3(x: torch.Tensor, norm_w: Optional[torch.Tensor] = None, eps: float = 0.0):
    """(xq uint8 [T, dim], e int32 [T]): the per-token e4m3 activations of x, or of its RMSNorm output with norm_w (include/mistral_b200.h)."""
    assert x.dtype == torch.bfloat16 and x.dim() == 2 and x.is_contiguous(), (x.dtype, x.shape)
    T, dim = x.shape
    q = torch.empty(T, dim, dtype=torch.uint8, device=x.device)
    e = torch.empty(T, dtype=torch.int32, device=x.device)
    _check(lib().mb200_quantize_act_e4m3(_ptr(x), _ptr(norm_w), _ptr(q), _ptr(e), T, dim, eps, _stream()), "mb200_quantize_act_e4m3")
    return q, e


# ---- INT4 dense weights (include/mistral_b200.h): w_q the packed codes uint8 [N, K/2], w_gscale the bf16 group scales [N, K/128] ----
def _check_int4(w_q: torch.Tensor, w_gscale: torch.Tensor) -> None:
    assert w_q.dtype == torch.uint8 and w_gscale.dtype == torch.bfloat16, (w_q.dtype, w_gscale.dtype)
    assert w_q.is_contiguous() and w_gscale.is_contiguous() and w_gscale.shape == (w_q.shape[0], w_q.shape[1] // 64), \
        (tuple(w_q.shape), tuple(w_gscale.shape))


def attn_qkv_int4(x, norm_w, w_q, w_gscale, rope, positions, q_out, k_out, v_out, cache_k, cache_v, cache_rows, n_heads, n_kv_heads,
                  head_dim, eps, ws: Workspace) -> None:
    _check_int4(w_q, w_gscale)
    T, dim = x.shape
    _check(lib().mb200_attn_qkv_int4(_ptr(x), _ptr(norm_w), _ptr(w_q), _ptr(w_gscale), _ptr(rope), _ptr(positions), _ptr(q_out),
                                     _ptr(k_out), _ptr(v_out), _ptr(cache_k), _ptr(cache_v), _ptr(cache_rows), T, dim, n_heads, n_kv_heads,
                                     head_dim, eps, ws.ptr, ws.nbytes, _stream()), "mb200_attn_qkv_int4")


def ffn_gateup_int4(x, norm_w, w_q, w_gscale, g_out, eps, ws: Workspace) -> None:
    _check_int4(w_q, w_gscale)
    T, dim = x.shape
    hidden = w_q.shape[0] // 2
    _check(lib().mb200_ffn_gateup_int4(_ptr(x), _ptr(norm_w), _ptr(w_q), _ptr(w_gscale), _ptr(g_out), T, dim, hidden, eps, ws.ptr,
                                       ws.nbytes, _stream()), "mb200_ffn_gateup_int4")


def linear_residual_int4(x, w_q, w_gscale, residual, out, ws: Workspace) -> None:
    _check_int4(w_q, w_gscale)
    T, K = x.shape
    N = w_q.shape[0]
    _check(lib().mb200_linear_residual_int4(_ptr(x), _ptr(w_q), _ptr(w_gscale), _ptr(residual), _ptr(out), T, N, K, ws.ptr, ws.nbytes,
                                            _stream()), "mb200_linear_residual_int4")


def attn_decode_occupancy(rep: int) -> int:
    """CTAs of attn_decode_tma_kernel<rep> resident per SM on the current device."""
    n = c_int(0)
    _check(lib().mb200_debug_attn_decode_occupancy(rep, ctypes.byref(n)), "mb200_debug_attn_decode_occupancy")
    return int(n.value)


def quantize_int4_groups(w: torch.Tensor, q: torch.Tensor, gscale: torch.Tensor) -> None:
    """q (uint8 [rows, K/2]) and gscale (bf16 [rows, K/128]) of the bf16 matrix w [rows, K]; both may be row-strided views."""
    rows, K = w.shape
    assert w.dtype == torch.bfloat16 and w.is_contiguous() and q.dtype == torch.uint8 and gscale.dtype == torch.bfloat16, \
        (w.dtype, q.dtype, gscale.dtype)
    assert q.shape == (rows, K // 2) and q.stride(1) == 1 and gscale.shape == (rows, K // 128) and gscale.stride(1) == 1, \
        (tuple(q.shape), tuple(gscale.shape))
    assert q.is_cuda and gscale.is_cuda and w.device == q.device == gscale.device
    _check(lib().mb200_quantize_int4_groups(_ptr(w), rows, K, q.data_ptr(), q.stride(0), gscale.data_ptr(), gscale.stride(0), _stream()),
           "mb200_quantize_int4_groups")


class LoraStruct(ctypes.Structure):
    """mb200_lora (include/mistral_b200.h)."""
    _fields_ = [("a_w", c_void_p), ("b_w", c_void_p), ("rank_cols", c_int64), ("scaling", c_float), ("a_buf", c_void_p), ("l_buf", c_void_p),
                ("row_slot", c_void_p), ("slot_cols", c_int64)]


def lora_struct(a_w: torch.Tensor, b_w: torch.Tensor, scaling: float, a_buf: torch.Tensor, l_buf: torch.Tensor,
                row_slot: Optional[torch.Tensor] = None, slot_cols: int = 0) -> LoraStruct:
    """One adapter of a fused Linear: packed a_w [R, K], b_w [N, R], scratch a_buf [>= T, R] and l_buf [>= T, N] (bf16).  With
    `row_slot` (int32 [T] on the device) a_w / b_w are a bank of slots of `slot_cols` columns each and token t uses slot
    row_slot[t] (-1: none)."""
    R = a_w.shape[0]
    assert b_w.shape[1] == R and a_buf.shape[-1] == R and l_buf.shape[-1] == b_w.shape[0]
    if row_slot is not None:
        assert row_slot.dtype == torch.int32 and row_slot.is_cuda and row_slot.is_contiguous() and row_slot.shape[0] >= a_buf.shape[0], \
            (row_slot.dtype, tuple(row_slot.shape))
        assert slot_cols > 0 and R % slot_cols == 0, (R, slot_cols)
    return LoraStruct(_ptr(a_w), _ptr(b_w), R, scaling, _ptr(a_buf), _ptr(l_buf), _ptr(row_slot), slot_cols if row_slot is not None else 0)


def _lora_ref(lora: LoraStruct):
    return ctypes.cast(ctypes.pointer(lora), c_void_p)


def attn_qkv_lora(x, norm_w, wqkv, rope, positions, q_out, k_out, v_out, cache_k, cache_v, cache_rows, n_heads, n_kv_heads, head_dim, eps,
                  ws: Workspace, lora: LoraStruct) -> None:
    T, dim = x.shape
    _check(lib().mb200_attn_qkv_lora(_ptr(x), _ptr(norm_w), _ptr(wqkv), _ptr(rope), _ptr(positions), _ptr(q_out), _ptr(k_out), _ptr(v_out),
                                     _ptr(cache_k), _ptr(cache_v), _ptr(cache_rows), T, dim, n_heads, n_kv_heads, head_dim, eps, ws.ptr,
                                     ws.nbytes, _stream(), _lora_ref(lora)), "mb200_attn_qkv_lora")


def ffn_gateup_lora(x, norm_w, w13, g_out, eps, ws: Workspace, lora: LoraStruct) -> None:
    T, dim = x.shape
    hidden = w13.shape[0] // 2
    _check(lib().mb200_ffn_gateup_lora(_ptr(x), _ptr(norm_w), _ptr(w13), _ptr(g_out), T, dim, hidden, eps, ws.ptr, ws.nbytes, _stream(),
                                       _lora_ref(lora)), "mb200_ffn_gateup_lora")


def linear_residual_lora(x, w, residual, out, ws: Workspace, lora: LoraStruct) -> None:
    T, K = x.shape
    N = w.shape[0]
    _check(lib().mb200_linear_residual_lora(_ptr(x), _ptr(w), _ptr(residual), _ptr(out), T, N, K, ws.ptr, ws.nbytes, _stream(),
                                            _lora_ref(lora)), "mb200_linear_residual_lora")


def lm_head(x, norm_w, w_out, logits, eps, ws: Workspace) -> None:
    T, dim = x.shape
    _check(lib().mb200_lm_head(_ptr(x), _ptr(norm_w), _ptr(w_out), _ptr(logits), T, dim, w_out.shape[0], eps, ws.ptr, ws.nbytes,
                               _stream()), "mb200_lm_head")


def argmax_rows(logits: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    T, V = logits.shape
    assert logits.dtype == torch.float32
    out = torch.empty(T, dtype=torch.long, device=logits.device) if out is None else out
    _check(lib().mb200_argmax_rows(_ptr(logits), _ptr(out), T, V, _stream()), "mb200_argmax_rows")
    return out


def logprob_gather(logits: torch.Tensor, target: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """log_softmax(logits, -1)[t, target[t]] (rows with target < 0 are left untouched)."""
    T, V = logits.shape
    assert logits.dtype == torch.float32 and target.dtype == torch.long and target.shape == (T,)
    out = torch.zeros(T, dtype=torch.float32, device=logits.device) if out is None else out
    _check(lib().mb200_logprob_gather(_ptr(logits), _ptr(target), _ptr(out), T, V, _stream()), "mb200_logprob_gather")
    return out


def sample_top_p(logits: torch.Tensor, uniform: torch.Tensor, temperature: float, top_p: float, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    T, V = logits.shape
    assert logits.dtype == torch.float32 and uniform.dtype == torch.float32 and uniform.shape == (T,)
    out = torch.empty(T, dtype=torch.long, device=logits.device) if out is None else out
    _check(lib().mb200_sample_top_p(_ptr(logits), _ptr(uniform), _ptr(out), T, V, temperature, top_p, _stream()), "mb200_sample_top_p")
    return out


def select_tokens(logits: torch.Tensor, temperature: torch.Tensor, top_p: torch.Tensor, presence: torch.Tensor, frequency: torch.Tensor,
                  step: torch.Tensor, out: torch.Tensor, *, seeds: Optional[torch.Tensor] = None, uniform: Optional[torch.Tensor] = None,
                  counts: Optional[torch.Tensor] = None) -> torch.Tensor:
    """One token per row with per-row controls (mb200_select_tokens): the four controls [B] fp32, `step` [B] int32 and `counts`
    [B, V] int32 (or None) are advanced in place; `seeds` [B] int64 holding the uint64 bit patterns, or `uniform` [B] fp32."""
    T, V = logits.shape
    assert logits.dtype == torch.float32 and (seeds is None) != (uniform is None)
    for t in (temperature, top_p, presence, frequency):
        assert t.dtype == torch.float32 and t.shape == (T,)
    assert step.dtype == torch.int32 and step.shape == (T,) and out.dtype == torch.long and out.shape == (T,)
    assert seeds is None or (seeds.dtype in (torch.int64, torch.uint64) and seeds.shape == (T,))
    assert uniform is None or (uniform.dtype == torch.float32 and uniform.shape == (T,))
    assert counts is None or (counts.dtype == torch.int32 and counts.shape == (T, V))
    _check(lib().mb200_select_tokens(_ptr(logits), _ptr(temperature), _ptr(top_p), _ptr(presence), _ptr(frequency), _ptr(seeds), _ptr(uniform),
                                     _ptr(step), _ptr(counts), _ptr(out), T, V, _stream()), "mb200_select_tokens")
    return out


# ---- speculative decoding (include/mistral_b200.h): the verify step's metadata and the acceptance kernels ----
def spec_meta_words(B: int, S: int, n_windows: int) -> int:
    """int32 words of the metadata block of a verify step of S tokens per sequence."""
    return B * S + 2 * B + 1 + n_windows * (B * S + B)


def spec_meta(seqpos_dev: torch.Tensor, meta_dev: torch.Tensor, S: int, windows) -> None:
    """Device-side metadata of a verify step of S tokens per sequence at the positions `seqpos_dev` (read, not advanced)."""
    B = seqpos_dev.shape[0]
    arr = (ctypes.c_int32 * len(windows))(*[int(w) for w in windows])
    assert seqpos_dev.dtype == torch.int32 and meta_dev.dtype == torch.int32 and meta_dev.numel() >= spec_meta_words(B, S, len(windows))
    _check(lib().mb200_spec_meta(_ptr(seqpos_dev), _ptr(meta_dev), B, S, ctypes.cast(arr, c_void_p), len(windows), _stream()), "mb200_spec_meta")


def _check_accept(logits: torch.Tensor, tokens: torch.Tensor, out: torch.Tensor, n: torch.Tensor, seqpos: torch.Tensor):
    B, S = tokens.shape
    assert logits.dtype == torch.float32 and logits.shape[0] == B * S and tokens.dtype == torch.long
    assert out.dtype == torch.long and out.shape == (B, S) and n.dtype == torch.int32 and n.shape == (B,)
    assert seqpos.dtype == torch.int32 and seqpos.shape == (B,)
    return B, S, logits.shape[1]


def spec_accept_greedy(logits: torch.Tensor, tokens: torch.Tensor, out: torch.Tensor, n: torch.Tensor, seqpos: torch.Tensor) -> None:
    """Greedy acceptance of the proposals tokens[:, 1:] against the verify logits [B * S, V]; advances `seqpos` by n + 1."""
    B, S, V = _check_accept(logits, tokens, out, n, seqpos)
    _check(lib().mb200_spec_accept_greedy(_ptr(logits), _ptr(tokens), _ptr(out), _ptr(n), _ptr(seqpos), B, S, V, _stream()),
           "mb200_spec_accept_greedy")


def spec_accept_sample(logits: torch.Tensor, draft_logits: torch.Tensor, tokens: torch.Tensor, uniform: torch.Tensor, out: torch.Tensor,
                       n: torch.Tensor, seqpos: torch.Tensor, temperature: float, top_p: float) -> None:
    """Speculative sampling on the nucleus distributions: draft_logits [B * (S - 1), V] are the rows the proposals were drawn from,
    uniform [B, S] fp32; advances `seqpos` by n + 1."""
    B, S, V = _check_accept(logits, tokens, out, n, seqpos)
    assert draft_logits.dtype == torch.float32 and draft_logits.shape == (B * (S - 1), V)
    assert uniform.dtype == torch.float32 and uniform.shape == (B, S)
    _check(lib().mb200_spec_accept_sample(_ptr(logits), _ptr(draft_logits), _ptr(tokens), _ptr(uniform), _ptr(out), _ptr(n), _ptr(seqpos), B, S,
                                          V, temperature, top_p, _stream()), "mb200_spec_accept_sample")


class MoeCommStruct(ctypes.Structure):
    """mb200_moe_comm (include/mistral_b200.h)."""
    _fields_ = [("n_ranks", ctypes.c_int32), ("my_rank", ctypes.c_int32), ("peer_yw", c_void_p * 8), ("my_flags", c_void_p),
                ("peer_flags", c_void_p * 8), ("epoch", c_void_p), ("done_counter", c_void_p)]


def moe_sizes(T: int, E: int, k: int):
    tr, rc, pw = c_int64(0), c_int64(0), c_int64(0)
    _check(lib().mb200_moe_sizes(T, E, k, ctypes.byref(tr), ctypes.byref(rc), ctypes.byref(pw)), "mb200_moe_sizes")
    return tr.value, rc.value, pw.value


def moe_route(hn: torch.Tensor, gate_w: torch.Tensor, E: int, k: int, shard_rank: int, shard_world: int, b) -> None:
    """Router + row plan + gather into the buffers `b` (moe.MoeBuffers)."""
    T, dim = hn.shape
    _check(lib().mb200_moe_route(_ptr(hn), _ptr(gate_w), T, dim, E, k, shard_rank, shard_world, _ptr(b.sel), _ptr(b.wts), _ptr(b.slot), _ptr(b.plan),
                                 _ptr(b.xs), _ptr(b.row_w), _stream()), "mb200_moe_route")


def moe_grouped_ffn(b, w13_host, w2_host, residual: Optional[torch.Tensor], out: torch.Tensor, T: int, dim: int, hidden: int, E: int, k: int,
                    comm: Optional[MoeCommStruct], ws: "Workspace") -> None:
    _check(lib().mb200_moe_grouped_ffn(_ptr(b.xs), ctypes.cast(w13_host, c_void_p), ctypes.cast(w2_host, c_void_p), _ptr(b.plan), _ptr(b.row_w),
                                       _ptr(b.slot), _ptr(residual), _ptr(b.g), b.yw_ptr, _ptr(out), T, dim, hidden, E, k,
                                       ctypes.cast(ctypes.pointer(comm), c_void_p) if comm is not None else None, ws.ptr, ws.nbytes, _stream()),
           "mb200_moe_grouped_ffn")


def moe_grouped_ffn_fp8(b, w13_host, s13_host, w2_host, s2_host, residual: Optional[torch.Tensor], out: torch.Tensor, T: int, dim: int,
                        hidden: int, E: int, k: int, comm: Optional[MoeCommStruct], ws: "Workspace") -> None:
    """moe_grouped_ffn with e4m3 experts: host arrays of E device pointers to the weights and to their fp32 row scales."""
    _check(lib().mb200_moe_grouped_ffn_fp8(_ptr(b.xs), ctypes.cast(w13_host, c_void_p), ctypes.cast(s13_host, c_void_p),
                                           ctypes.cast(w2_host, c_void_p), ctypes.cast(s2_host, c_void_p), _ptr(b.plan), _ptr(b.row_w),
                                           _ptr(b.slot), _ptr(residual), _ptr(b.g), b.yw_ptr, _ptr(out), T, dim, hidden, E, k,
                                           ctypes.cast(ctypes.pointer(comm), c_void_p) if comm is not None else None, ws.ptr, ws.nbytes,
                                           _stream()), "mb200_moe_grouped_ffn_fp8")


class MoeLoraStruct(ctypes.Structure):
    """mb200_moe_lora (include/mistral_b200.h)."""
    _fields_ = [("a_host", c_void_p), ("b_host", c_void_p), ("rank_cols", c_int64), ("scaling", c_float), ("a_buf", c_void_p), ("l_buf", c_void_p)]


def moe_lora_struct(a_host, b_host, rank_cols: int, scaling: float, a_buf: torch.Tensor, l_buf: torch.Tensor) -> MoeLoraStruct:
    """The adapters of one grouped expert Linear: host arrays of E device pointers to A [R, K] and B [N, R], and the MoE scratch
    a_buf [>= rows_cap, R], l_buf [>= rows_cap, N] (bf16)."""
    assert a_buf.shape[-1] == rank_cols and rank_cols % 64 == 0
    return MoeLoraStruct(ctypes.cast(a_host, c_void_p), ctypes.cast(b_host, c_void_p), rank_cols, scaling, _ptr(a_buf), _ptr(l_buf))


def moe_grouped_ffn_fp8_lora(b, w13_host, s13_host, w2_host, s2_host, residual: Optional[torch.Tensor], out: torch.Tensor, T: int, dim: int,
                             hidden: int, E: int, k: int, comm: Optional[MoeCommStruct], ws: "Workspace", lora13: MoeLoraStruct,
                             lora2: MoeLoraStruct) -> None:
    """moe_grouped_ffn_fp8 with the un-merged adapters of every expert's w1 / w3 (`lora13`) and w2 (`lora2`)."""
    _check(lib().mb200_moe_grouped_ffn_fp8_lora(_ptr(b.xs), ctypes.cast(w13_host, c_void_p), ctypes.cast(s13_host, c_void_p),
                                                ctypes.cast(w2_host, c_void_p), ctypes.cast(s2_host, c_void_p), _ptr(b.plan), _ptr(b.row_w),
                                                _ptr(b.slot), _ptr(residual), _ptr(b.g), b.yw_ptr, _ptr(out), T, dim, hidden, E, k,
                                                ctypes.cast(ctypes.pointer(comm), c_void_p) if comm is not None else None, ws.ptr, ws.nbytes,
                                                _stream(), ctypes.cast(ctypes.pointer(lora13), c_void_p),
                                                ctypes.cast(ctypes.pointer(lora2), c_void_p)), "mb200_moe_grouped_ffn_fp8_lora")


def moe_grouped_ffn_int4(b, w13_host, s13_host, w2_host, s2_host, residual: Optional[torch.Tensor], out: torch.Tensor, T: int, dim: int,
                         hidden: int, E: int, k: int, comm: Optional[MoeCommStruct], ws: "Workspace") -> None:
    """moe_grouped_ffn with INT4 experts: host arrays of E device pointers to the packed codes and to their bf16 group scales."""
    _check(lib().mb200_moe_grouped_ffn_int4(_ptr(b.xs), ctypes.cast(w13_host, c_void_p), ctypes.cast(s13_host, c_void_p),
                                            ctypes.cast(w2_host, c_void_p), ctypes.cast(s2_host, c_void_p), _ptr(b.plan), _ptr(b.row_w),
                                            _ptr(b.slot), _ptr(residual), _ptr(b.g), b.yw_ptr, _ptr(out), T, dim, hidden, E, k,
                                            ctypes.cast(ctypes.pointer(comm), c_void_p) if comm is not None else None, ws.ptr, ws.nbytes,
                                            _stream()), "mb200_moe_grouped_ffn_int4")


def quantize_e4m3_rows(w: torch.Tensor, q: torch.Tensor, scale: torch.Tensor) -> None:
    """q (uint8 [rows, K], rows may be strided) and scale (fp32 [rows], may be strided) of the bf16 matrix w [rows, K]."""
    rows, K = w.shape
    assert w.dtype == torch.bfloat16 and q.dtype == torch.uint8 and scale.dtype == torch.float32, (w.dtype, q.dtype, scale.dtype)
    assert q.shape == (rows, K) and q.stride(1) == 1 and scale.shape == (rows,), (tuple(q.shape), tuple(scale.shape))
    assert q.is_cuda and scale.is_cuda and w.device == q.device == scale.device
    _check(lib().mb200_quantize_e4m3_rows(_ptr(w), rows, K, q.data_ptr(), q.stride(0), scale.data_ptr(), scale.stride(0), _stream()),
           "mb200_quantize_e4m3_rows")


def comm_alloc(nbytes: int) -> int:
    p = c_void_p(0)
    _check(lib().mb200_comm_alloc(nbytes, ctypes.byref(p)), "mb200_comm_alloc")
    return int(p.value)


def comm_free(ptr: int) -> None:
    _check(lib().mb200_comm_free(ptr), "mb200_comm_free")


def comm_export(ptr: int) -> bytes:
    h = ctypes.create_string_buffer(64)
    _check(lib().mb200_comm_export(ptr, ctypes.cast(h, c_void_p)), "mb200_comm_export")
    return h.raw


def comm_open(handle: bytes) -> int:
    h = ctypes.create_string_buffer(handle, 64)
    p = c_void_p(0)
    _check(lib().mb200_comm_open(ctypes.cast(h, c_void_p), ctypes.byref(p)), "mb200_comm_open")
    return int(p.value)


def comm_close(ptr: int) -> None:
    _check(lib().mb200_comm_close(ptr), "mb200_comm_close")


def decode_meta(seqpos_dev: torch.Tensor, meta_dev: torch.Tensor, windows) -> None:
    """Device-side metadata of a one-token step for every sequence; advances `seqpos_dev` (include/mistral_b200.h)."""
    B = seqpos_dev.shape[0]
    arr = (ctypes.c_int32 * len(windows))(*[int(w) for w in windows])
    assert seqpos_dev.dtype == torch.int32 and meta_dev.dtype == torch.int32 and meta_dev.numel() >= 3 * B + 1 + 2 * B * len(windows)
    _check(lib().mb200_decode_meta(_ptr(seqpos_dev), _ptr(meta_dev), B, ctypes.cast(arr, c_void_p), len(windows), _stream()), "mb200_decode_meta")


def decode_step(layers_dev, windows_dev, n_layers, emb, final_norm, w_out, rope, token_dev, pos, batch_row, logits, next_token, dim, hidden,
                n_heads, n_kv_heads, head_dim, vocab, eps, ws: Workspace, n_experts: int = 0, top_k: int = 0, moe_gate=None, moe_w13=None,
                moe_w2=None) -> None:
    _check(lib().mb200_decode_step(_ptr(layers_dev), _ptr(windows_dev), n_layers, _ptr(emb), _ptr(final_norm), _ptr(w_out), _ptr(rope),
                                   _ptr(token_dev), pos, batch_row, _ptr(logits), _ptr(next_token), dim, hidden, n_heads, n_kv_heads, head_dim,
                                   vocab, eps, n_experts, top_k, _ptr(moe_gate), _ptr(moe_w13), _ptr(moe_w2), ws.ptr, ws.nbytes, _stream()),
           "mb200_decode_step")


def decode_step_fp8(layers_dev, windows_dev, n_layers, emb, final_norm, w_out, rope, token_dev, pos, batch_row, logits, next_token, dim,
                    hidden, n_heads, n_kv_heads, head_dim, vocab, eps, ws: Workspace) -> None:
    """decode_step for a dense FP8 model: layers_dev holds one mb200_layer_desc_fp8 (12 pointers) per layer."""
    _check(lib().mb200_decode_step_fp8(_ptr(layers_dev), _ptr(windows_dev), n_layers, _ptr(emb), _ptr(final_norm), _ptr(w_out), _ptr(rope),
                                       _ptr(token_dev), pos, batch_row, _ptr(logits), _ptr(next_token), dim, hidden, n_heads, n_kv_heads,
                                       head_dim, vocab, eps, ws.ptr, ws.nbytes, _stream()), "mb200_decode_step_fp8")


def decode_step_fp8_unsupported(dim, hidden, n_heads, n_kv_heads, head_dim, vocab, smem_optin: int = 0) -> Optional[str]:
    """decode_step_unsupported for decode_step_fp8 (dense shapes)."""
    if lib().mb200_decode_step_fp8_supported(dim, hidden, n_heads, n_kv_heads, head_dim, vocab, smem_optin) == 0:
        return None
    msg = lib().mb200_last_error()
    return msg.decode() if msg else "?"


def set_decode_timeline(buf: Optional[torch.Tensor]) -> None:
    _check(lib().mb200_debug_set_decode_timeline(_ptr(buf)), "mb200_debug_set_decode_timeline")


def set_barrier_timeline(buf: Optional[torch.Tensor]) -> None:
    _check(lib().mb200_debug_set_barrier_timeline(_ptr(buf)), "mb200_debug_set_barrier_timeline")


def launch_log(enable: bool) -> list:
    """Names of the attention / GEMM / MoE / speculative-decoding kernels launched from this thread since the last call (empty while recording is off);
    clears the log and switches recording on or off (include/mistral_b200.h)."""
    buf = ctypes.create_string_buffer(32768)
    _check(lib().mb200_debug_launch_log(int(enable), ctypes.cast(buf, c_void_p), len(buf)), "mb200_debug_launch_log")
    return buf.value.decode().splitlines()


def decode_scratch(dim, hidden, n_heads, n_kv_heads, head_dim, n_experts: int = 0, top_k: int = 0):
    """(q offset, attention-output offset) in bytes of the workspace that decode_step writes (include/mistral_b200.h)."""
    q, a = c_size_t(0), c_size_t(0)
    _check(lib().mb200_debug_decode_scratch(dim, hidden, n_heads, n_kv_heads, head_dim, n_experts, top_k, ctypes.byref(q), ctypes.byref(a)),
           "mb200_debug_decode_scratch")
    return q.value, a.value


class DecodeBuffers(NamedTuple):
    """Byte offsets into the workspace of every buffer decode_step leaves behind (include/mistral_b200.h)."""
    x: int        # [2][dim] bf16 residual ping-pong: layer l writes half (l + 1) & 1
    h: int        # [dim] bf16
    q: int        # [H * 128] bf16
    attn: int     # [H * 128] bf16
    g: int        # [hidden] bf16, or [top_k][hidden] for MoE
    partial: int  # [SM count][H][130] fp32


def decode_buffers(dim, hidden, n_heads, n_kv_heads, head_dim, n_experts: int = 0, top_k: int = 0) -> DecodeBuffers:
    off = (c_size_t * 6)()
    _check(lib().mb200_debug_decode_buffers(dim, hidden, n_heads, n_kv_heads, head_dim, n_experts, top_k, off), "mb200_debug_decode_buffers")
    return DecodeBuffers(*[int(v) for v in off])


def decode_step_unsupported(dim, hidden, n_heads, n_kv_heads, head_dim, vocab, n_experts: int = 0, top_k: int = 0,
                            smem_optin: int = 0) -> Optional[str]:
    """None when decode_step accepts these shapes on a device with `smem_optin` bytes of opt-in shared memory per block (0: the
    current device), else the reason it would refuse them."""
    if lib().mb200_decode_step_supported(dim, hidden, n_heads, n_kv_heads, head_dim, vocab, n_experts, top_k, smem_optin) == 0:
        return None
    msg = lib().mb200_last_error()
    return msg.decode() if msg else "?"


def test_gemm_naive(a, w) -> torch.Tensor:
    T, K = a.shape
    c = torch.empty(T, w.shape[0], dtype=torch.float32, device=a.device)
    _check(lib().mb200_test_gemm_naive(_ptr(a), _ptr(w), _ptr(c), T, w.shape[0], K, _stream()), "mb200_test_gemm_naive")
    return c
