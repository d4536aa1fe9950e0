"""CPU-side checks of the boundary: the C-ABI library loads and exports every symbol include/mistral_b200.h
declares (no compute without a GPU), and the host-side mirror of the reference API behaves like the reference."""
import ctypes
import re
from pathlib import Path

import numpy as np
import pytest
import torch

import mistral_inference_b200 as mi
import synth
from mistral_inference_b200 import _abi
from mistral_inference_b200.build import build_library
from mistral_inference_b200.cache import BufferCache
from mistral_inference_b200.transformer import Transformer

REPO = Path(__file__).resolve().parents[1]


@pytest.fixture(scope="module")
def built():
    return build_library()


def test_header_symbols_exported(built):
    header = (REPO / "include" / "mistral_b200.h").read_text()
    declared = set(re.findall(r"\b(mb200_[a-z0-9_]+)\s*\(", header))
    assert len(declared) >= 12
    handle = ctypes.CDLL(str(built))
    for name in declared:
        assert hasattr(handle, name), f"{name} declared in mistral_b200.h but not exported by libmb200.so"
    # and the ctypes table covers exactly the header
    assert declared == set(_abi._SIGNATURES), declared ^ set(_abi._SIGNATURES)


def test_workspace_header_size_matches_the_header():
    header = (REPO / "include" / "mistral_b200.h").read_text()
    m = re.search(r"#define MB200_WORKSPACE_HEADER_BYTES \((\d+) \* (\d+)\)", header)
    assert m, "MB200_WORKSPACE_HEADER_BYTES not found in the form (a * b)"
    assert _abi.WORKSPACE_HEADER_BYTES == int(m.group(1)) * int(m.group(2))


def test_library_loads_and_reports_version(built):
    assert _abi.lib().mb200_abi_version() == _abi.ABI_VERSION
    assert _abi.workspace_bytes(16, 4096, 32, 8, 128, 14336, 32000, 1) > _abi.WORKSPACE_HEADER_BYTES


def test_argument_errors_do_not_need_a_gpu(built):
    rc = _abi.lib().mb200_attn_decode(None, None, None, None, None, 1, 1, 4, 2, 128, 1, None, 0, None)
    assert rc == -1 and b"null pointer" in _abi.lib().mb200_last_error()
    rc = _abi.lib().mb200_rmsnorm(1, 1, 1, 1, 4095, 1e-5, None)
    assert rc == -1 and b"multiple of 8" in _abi.lib().mb200_last_error()


def test_launch_log_records_nothing_for_rejected_calls(built):
    _abi.launch_log(True)
    assert _abi.lib().mb200_attn_decode(None, None, None, None, None, 1, 1, 4, 2, 128, 1, None, 0, None) == -1
    assert _abi.launch_log(False) == []
    assert _abi.launch_log(False) == []  # recording off: still empty


@pytest.mark.parametrize("dim,hidden,H,KV,E,k", [(256, 256, 4, 2, 0, 0), (4096, 14336, 32, 8, 0, 0), (5120, 14336, 32, 8, 0, 0),
                                                (6144, 16384, 48, 8, 8, 2), (256, 256, 40, 5, 0, 0), (4096, 14336, 32, 8, 8, 4),
                                                (4112, 4112, 8, 1, 16, 4)])
def test_decode_scratch_offsets(built, dim, hidden, H, KV, E, k):
    """Where decode_step leaves q and the attention output: 256-byte aligned, after the header, apart, inside the workspace.
    The same for every buffer mb200_debug_decode_buffers reports (both residual halves, h, q, the attention output, g of every
    selected expert, the slice partials of up to 256 SMs): aligned, after the header, disjoint, inside the workspace, and q /
    attention where mb200_debug_decode_scratch puts them."""
    q, a = _abi.decode_scratch(dim, hidden, H, KV, 128, E, k)
    nb = H * 128 * 2
    total = _abi.workspace_bytes(1, dim, H, KV, 128, hidden, 32000, 1)
    assert q % 256 == 0 and a % 256 == 0
    assert _abi.WORKSPACE_HEADER_BYTES <= q and _abi.WORKSPACE_HEADER_BYTES <= a
    assert q + nb <= a or a + nb <= q
    assert max(q, a) + nb <= total
    assert _abi.lib().mb200_debug_decode_scratch(dim, hidden, H, KV, 64, E, k, None, None) == -1

    b = _abi.decode_buffers(dim, hidden, H, KV, 128, E, k)
    assert (b.q, b.attn) == (q, a)
    sizes = {"x": 2 * dim * 2, "h": dim * 2, "q": nb, "attn": nb, "g": (k if E else 1) * hidden * 2, "partial": 256 * H * 130 * 4}
    spans = sorted((getattr(b, name), getattr(b, name) + n, name) for name, n in sizes.items())
    for lo, hi, name in spans:
        assert lo % 256 == 0, name
        assert lo >= _abi.WORKSPACE_HEADER_BYTES, name
        assert hi <= total, f"{name} ends at {hi} > workspace {total}"
    for (_, hi, x), (lo, _, y) in zip(spans, spans[1:]):
        assert hi <= lo, f"{x} overlaps {y}"
    assert _abi.lib().mb200_debug_decode_buffers(dim, hidden, H, KV, 64, E, k, None) == -1
    assert _abi.lib().mb200_debug_decode_buffers(dim, hidden, H, KV, 128, E, k, None) == -1


H100_SMEM = 227 * 1024  # opt-in shared memory per block of an H100


@pytest.mark.parametrize("name,shape,E,k,ok", [
    ("mistral-7b", (4096, 14336, 32, 8, 32000), 0, 0, True),
    ("nemo-12b", (5120, 14336, 32, 8, 131072), 0, 0, True),
    ("mixtral-8x7b", (4096, 14336, 32, 8, 32000), 8, 2, True),
    ("mixtral-8x7b-k3", (4096, 14336, 32, 8, 32000), 8, 3, False),
    ("mixtral-8x7b-k4", (4096, 14336, 32, 8, 32000), 8, 4, False),
    ("mixtral-8x22b", (6144, 16384, 48, 8, 32768), 8, 2, True),
    ("mixtral-8x22b-k3", (6144, 16384, 48, 8, 32768), 8, 3, False),
    ("k4-widest", (4096, 10272, 32, 8, 32000), 8, 4, True),
    ("k4-one-step-wider", (4096, 10296, 32, 8, 32000), 8, 4, False),
    ("k5", (4096, 4096, 32, 8, 32000), 8, 5, False),
    ("kv16", (4096, 4096, 32, 16, 32000), 0, 0, False),
    ("rep3", (4096, 4096, 24, 8, 32000), 0, 0, False),
    ("odd-vocab", (4096, 4096, 32, 8, 32001), 0, 0, False),
    ("hidden-4100", (4096, 4100, 32, 8, 32000), 0, 0, False),
    ("hidden-4112", (4096, 4112, 32, 8, 32000), 0, 0, True),
])
def test_decode_step_supported_on_h100(built, name, shape, E, k, ok):
    """The megakernel's shape rules at an H100's 227 KB of opt-in shared memory, without a GPU: the real dense and k = 2 MoE
    shapes run; k = 3 on Mixtral-8x7B / 8x22B and k = 4 on Mixtral-8x7B leave fewer than 9 ring stages and are refused, like the
    K chunking that is not 16-byte aligned (4100 = 2 x 2050), an odd vocab, KV > 8 and uncompiled head ratios."""
    dim, hidden, H, KV, V = shape
    why = _abi.decode_step_unsupported(dim, hidden, H, KV, 128, V, E, k, smem_optin=H100_SMEM)
    assert (why is None) == ok, why


def test_no_cpu_fallback():
    p = synth.shape("tiny")
    args = mi.TransformerArgs.from_dict(p)
    args.max_batch_size = 1
    m = Transformer(args).to(torch.bfloat16)
    with pytest.raises(_abi.Mb200Error):
        m.forward(torch.tensor([1, 2, 3]), [3])


def test_product_does_not_import_oracle():
    for f in (REPO / "mistral_inference_b200").glob("*.py"):
        src = f.read_text()
        assert "import oracle" not in src and "from oracle" not in src, f"{f} imports the oracle"


@pytest.mark.parametrize("name", ["tiny", "tiny-moe"])
def test_state_dict_roundtrip_reference_keys(name):
    p = synth.shape(name)
    args = mi.TransformerArgs.from_dict(p)
    m = Transformer(args).to(torch.bfloat16)
    sd = synth.synth_state_dict(p, 5)
    m.load_state_dict(sd)
    out = m.state_dict()
    assert list(out) and set(out) == set(sd)
    for k in sd:
        assert torch.equal(out[k], sd[k]), k
    with pytest.raises(ValueError):
        m.load_state_dict({"bogus.weight": torch.zeros(1)})


def test_from_folder_and_pipeline_key_filtering(tmp_path):
    p = synth.shape("tiny", n_layers=4)
    synth.write_model_folder(tmp_path, p, 2)
    m = Transformer.from_folder(tmp_path, max_batch_size=3, device="cpu")
    assert m.args.max_batch_size == 3 and m.n_local_layers == 4 and m.dtype == torch.bfloat16
    sd = synth.synth_state_dict(p, 2)
    # rank 1 of 2 owns layers 2,3 + norm + output, no embeddings (transformer.py:56-79,94-98)
    args = mi.TransformerArgs.from_dict(p)
    r1 = Transformer(args, pipeline_rank=1, num_pipeline_ranks=2).to(torch.bfloat16)
    r1.load_state_dict(sd)
    assert list(r1.layers.keys()) == ["2", "3"] and r1.tok_embeddings is None and r1.norm is not None
    assert torch.equal(r1.state_dict()["layers.3.feed_forward.w3.weight"], sd["layers.3.feed_forward.w3.weight"])


def test_cache_metadata_matches_reference_docstring():
    """cache.py:199-206 example: seqlens [5,7,2], W=3 -> to_cache_mask / cache_positions."""
    c = BufferCache(1, 3, 20, 2, 128, 3)
    c._kv_seqlens_host = [4, 1, 3]
    host, layout = c.build_metadata_host([5, 7, 2])
    T = 14
    rows = host[T + 4 + 3: T + 4 + 3 + T]
    assert rows.tolist() == [-1, -1, 0, 1, 2, -1, -1, -1, -1, 5, 3, 4, 6, 7]
    assert host[:T].tolist() == [4, 5, 6, 7, 8, 1, 2, 3, 4, 5, 6, 7, 3, 4]
    assert layout["prefill"] is True


def test_cache_metadata_against_oracle_ring():
    """Rows/kv_len agree with the oracle's ring bookkeeping through prefill chunks and decode steps."""
    rng = np.random.default_rng(0)
    for W in (4, 7, 64):
        c = BufferCache(1, 2, 64, 2, 128, W)
        seen = [0, 0]
        for step in range(12):
            sl = [int(rng.integers(1, 9)), int(rng.integers(1, 9))] if step < 4 else [1, 1]
            host, layout = c.build_metadata_host(sl)
            T = sum(sl)
            rows = host[T + 3 + 2: T + 3 + 2 + T]
            kv_len = host[T + 3 + 2 + T:]
            o = 0
            for b, s in enumerate(sl):
                for t in range(s):
                    want = (seen[b] + t) % W + b * W if t >= s - W else -1
                    assert rows[o + t] == want
                o += s
                assert kv_len[b] == min(seen[b] + min(s, W), W)
            c.update_seqlens(sl)
            seen = [a + b for a, b in zip(seen, sl)]


def test_load_lora_merges_like_the_reference():
    """Merged LoRA (lora.py:92-139): weight + (B @ A) * scaling lands in the packed buffers under the reference's key names."""
    import torch

    import mistral_inference_b200 as mi
    import synth
    from mistral_inference_b200.transformer import Transformer

    p = synth.shape("tiny-moe", n_layers=1)
    args = mi.TransformerArgs.from_dict(dict(p))
    m = Transformer(args).to(torch.bfloat16)
    sd = synth.synth_state_dict(p, 4)
    m.load_state_dict(sd)
    g = torch.Generator().manual_seed(0)
    rank = 4
    lora = {}
    for name in ("layers.0.attention.wq", "layers.0.attention.wv", "layers.0.attention.wo", "layers.0.feed_forward.experts.3.w1",
                 "layers.0.feed_forward.experts.3.w2", "layers.0.feed_forward.experts.5.w3"):
        out_f, in_f = sd[name + ".weight"].shape
        lora[name + ".lora_A.weight"] = (torch.randn(rank, in_f, generator=g) * 0.1).to(torch.bfloat16)
        lora[name + ".lora_B.weight"] = (torch.randn(out_f, rank, generator=g) * 0.1).to(torch.bfloat16)
    m._load_lora_state_dict(lora, scaling=2.0)
    got = m.state_dict()
    for key, w in sd.items():
        name = key[: -len(".weight")]
        want = w + (lora[name + ".lora_B.weight"] @ lora[name + ".lora_A.weight"]) * 2.0 if (name + ".lora_B.weight") in lora else w
        assert torch.equal(got[key], want), key
