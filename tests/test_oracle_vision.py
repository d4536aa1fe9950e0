"""CPU checks of the vision path: params.json parsing, the reference's vision state-dict keys (round trip, padding, pipeline-rank
filtering, from_folder), the 2-D RoPE table, and the oracle restatement (oracle/vision.py) pinned against the reference's own
modules (tests/golden/reference/vision_pins.safetensors, made by oracle/make_vision_pins.py).  Bit-exact where the torch build,
CPU ISA level and thread count match the fixture's; elsewhere fp32-accumulation-order noise through the bf16 roundings is
allowed."""
import hashlib

import numpy as np
import pytest
import torch

import mistral_inference_b200 as mi
import synth
from mistral_inference_b200.args import VisionEncoderArgs
from mistral_inference_b200.rope import precompute_freqs_cis_2d
from mistral_inference_b200.transformer import Transformer
from oracle import restatement as R
from oracle import vision as V
from oracle.make_vision_pins import PIN_ROPE2D, PIN_ROPE2D_ROWS, VISION_CASES, VISION_PINS_FILE, case_images, case_params

from .util import LOGPROB_TOL, oracle_args, same_machine_as_golden


@pytest.fixture(scope="module")
def pins():
    import safetensors
    import safetensors.torch

    with safetensors.safe_open(str(VISION_PINS_FILE), "pt") as f:
        meta = f.metadata()
    return safetensors.torch.load_file(str(VISION_PINS_FILE)), meta


def test_vision_args_reference_defaults():
    a = mi.TransformerArgs.from_dict(synth.shape("pixtral-12b"))
    ve = a.vision_encoder
    assert isinstance(ve, VisionEncoderArgs)
    assert (ve.hidden_size, ve.num_attention_heads, ve.hidden_size // ve.num_attention_heads) == (1024, 16, 64)
    minimal = dict(hidden_size=128, num_channels=3, image_size=4, patch_size=2, intermediate_size=256, num_hidden_layers=1,
                   num_attention_heads=2)
    ve = mi.TransformerArgs.from_dict(dict(synth.shape("tiny"), vision_encoder=minimal)).vision_encoder
    # args.py:21-26
    assert (ve.rope_theta, ve.image_token_id, ve.adapter_bias, ve.spatial_merge_size, ve.add_pre_mm_projector_layer_norm,
            ve.mm_projector_id) == (1e4, 10, True, 1, False, "")
    assert mi.TransformerArgs.from_dict(synth.shape("tiny")).vision_encoder is None


def test_rope_2d_table_matches_reference_bits(pins):
    gold, meta = pins
    d, side, theta = PIN_ROPE2D["dim"], PIN_ROPE2D["side"], PIN_ROPE2D["theta"]
    ours = torch.view_as_real(precompute_freqs_cis_2d(d, side, side, theta)).contiguous()
    oracle = torch.view_as_real(V.rope_table_2d(d, side, side, theta)).contiguous()
    assert torch.equal(ours, oracle)
    rows = torch.stack([ours[r, c] for r, c in PIN_ROPE2D_ROWS])
    if same_machine_as_golden(meta):
        assert torch.equal(rows, gold["rope2d_rows"])
        assert hashlib.sha256(ours.numpy().tobytes()).hexdigest() == meta["rope2d_sha256"]
    else:
        torch.testing.assert_close(rows, gold["rope2d_rows"], rtol=1e-6, atol=1e-6)


def _close(got, want, what):
    torch.testing.assert_close(got.float(), want.float(), rtol=2 ** -6, atol=2e-2 * float(want.abs().max()), msg=what)


@pytest.mark.parametrize("name", list(VISION_CASES))
def test_oracle_vision_vs_reference(pins, name):
    gold, meta = pins
    p = case_params(name)
    w = synth.synth_state_dict(p, 3, torch.bfloat16)
    prompts = VISION_CASES[name][2]
    imgs = [torch.tensor(im, dtype=torch.bfloat16) for ims in case_images(name) for im in ims]
    with torch.inference_mode():
        enc = V.encoder_forward(imgs, w, p["vision_encoder"])
        emb = V.embed(torch.tensor(sum(prompts, [])), imgs, w, p["vision_encoder"])
    exact = same_machine_as_golden(meta)
    if exact:
        assert torch.equal(enc, gold[f"{name}/encoder"])
        assert torch.equal(emb, gold[f"{name}/embed"])
    else:
        _close(enc, gold[f"{name}/encoder"], "encoder")
        _close(emb, gold[f"{name}/embed"], "embed")
    om = V.MultimodalOracle(R.OracleTransformer(oracle_args(p, len(prompts)), w), p["vision_encoder"], imgs)
    toks, lps = R.generate(prompts, om, max_tokens=7)
    t_ref = gold[f"{name}/tokens"].tolist()
    lp_ref = torch.split(gold[f"{name}/logprobs"], gold[f"{name}/lengths"].tolist())
    if exact:
        assert toks == t_ref
        assert [x.tolist() for x in lp_ref] == lps
    else:
        for tr, to, lr, lo in zip(t_ref, toks, lp_ref, lps):
            n = next((i for i, (a, b) in enumerate(zip(tr, to)) if a != b), len(tr))
            m = len(lo) - len(to) + n
            torch.testing.assert_close(torch.tensor(lo[:m], dtype=torch.float64), lr[:m], rtol=0, atol=LOGPROB_TOL)


@pytest.mark.parametrize("shape", ["pixtral-ref-test", "pixtral-ref-test-merge", "tiny-pixtral"])
def test_vision_state_dict_roundtrip_reference_keys(shape):
    p = synth.shape(shape)
    m = Transformer(mi.TransformerArgs.from_dict(p)).to(torch.bfloat16)
    sd = synth.synth_state_dict(p, 5)
    m.load_state_dict(sd)
    out = m.state_dict()
    assert set(out) == set(sd)
    for k in sd:
        assert out[k].shape == sd[k].shape and torch.equal(out[k], sd[k]), k
    ve = m.vision_encoder
    assert ve.k_pad % 64 == 0 and ve.k_pad >= ve.k_conv
    assert torch.count_nonzero(ve.patch_conv_weight[:, ve.k_conv:]) == 0
    with pytest.raises(ValueError):
        m.load_state_dict({"vision_encoder.transformer.layers.99.attention.wq.weight": torch.zeros(1)})
    text_only = Transformer(mi.TransformerArgs.from_dict(synth.shape("tiny"))).to(torch.bfloat16)
    with pytest.raises(ValueError):
        text_only.load_state_dict({"vision_encoder.ln_pre.weight": torch.zeros(1)})


def test_patch_conv_padding_for_patch_14():
    p = synth.shape("pixtral-ref-test")
    p["vision_encoder"] = dict(p["vision_encoder"], patch_size=14, image_size=56)
    m = Transformer(mi.TransformerArgs.from_dict(p)).to(torch.bfloat16)
    assert (m.vision_encoder.k_conv, m.vision_encoder.k_pad) == (588, 640)
    sd = synth.synth_state_dict(p, 1)
    m.vision_encoder.patch_conv_weight.fill_(7)  # stale memory must not survive a load
    m.load_state_dict(sd)
    assert torch.equal(m.state_dict()["vision_encoder.patch_conv.weight"], sd["vision_encoder.patch_conv.weight"])
    assert torch.count_nonzero(m.vision_encoder.patch_conv_weight[:, 588:]) == 0


def test_vision_keys_only_on_pipeline_rank_0():
    p = synth.shape("pixtral-ref-test-merge", n_layers=2)
    sd = synth.synth_state_dict(p, 2)
    args = mi.TransformerArgs.from_dict(p)
    r0 = Transformer(args, pipeline_rank=0, num_pipeline_ranks=2).to(torch.bfloat16)
    r1 = Transformer(args, pipeline_rank=1, num_pipeline_ranks=2).to(torch.bfloat16)
    r0.load_state_dict(sd)
    r1.load_state_dict(sd)
    vision = [k for k in sd if k.startswith(("vision_encoder.", "vision_language_adapter.", "patch_merger.", "pre_mm_projector_norm."))]
    assert vision and all(r0._owns_key(k) and not r1._owns_key(k) for k in vision)
    assert r1.vision_encoder is None and not any(k in r1.state_dict() for k in vision)
    assert all(torch.equal(r0.state_dict()[k], sd[k]) for k in vision)


def test_from_folder_streams_a_pixtral_folder(tmp_path):
    p = synth.shape("pixtral-ref-test-merge")
    synth.write_model_folder(tmp_path, p, 4)
    m = Transformer.from_folder(tmp_path, max_batch_size=2, device="cpu")
    assert m.vision_encoder is not None and m.patch_merger is not None and m.pre_mm_projector_norm is not None
    assert m.vision_language_adapter.w_in.bias is None  # adapter_bias = False
    sd = synth.synth_state_dict(p, 4)
    got = m.state_dict()
    assert set(got) == set(sd) and all(torch.equal(got[k], sd[k]) for k in sd)


def test_image_input_checks():
    p = synth.shape("pixtral-ref-test")
    m = Transformer(mi.TransformerArgs.from_dict(p)).to(torch.bfloat16)
    ve = m.vision_encoder
    assert ve.patch_grid([torch.zeros(3, 5, 4)]) == [(2, 2)]  # the convolution floors
    with pytest.raises(IndexError):  # more patches per side than the 2-D table (image_size // patch_size = 2)
        ve.patch_grid([torch.zeros(3, 6, 4)])
    with pytest.raises(RuntimeError):
        ve.patch_grid([torch.zeros(3, 1, 4)])
    with pytest.raises(RuntimeError):
        ve.patch_grid([torch.zeros(1, 4, 4)])
    with pytest.raises(AssertionError):  # generate.py:56: no chunked prefill with images
        mi.generate([[1, 2]], m, images=[[torch.zeros(3, 4, 4).numpy()]], max_tokens=1, temperature=0.0, chunk_size=1)


def test_text_shapes_unchanged_by_vision_support():
    """bench.py's synthetic checkpoints: no vision key appears for a shape without a vision_encoder block."""
    for name in ("mistral-7b", "mistral-nemo-12b", "mixtral-8x7b", "tiny", "tiny-moe", "ref-test"):
        assert not any(k.startswith("vision") for k, _ in synth.state_dict_shapes(synth.shape(name)))


# ----------------------------------------------------------------------------- the head_dim-64 attention test's comparator
# (tests/test_gpu_vision.py, whose docstring gives the exactness argument): q = 0 and V[j, h*64 + d] = 1 iff d < 63 and
# (j + h) % 63 == d, or d == 63 and j >= 63, so head h of every query row is c_hd / n with c_hd the number of visible keys with a
# 1 in column d.
VIS_T = [1, 63, 64, 65, 127, 128, 129, 255, 256, 257, 1000, 4096, 4097]
H_VIS = 16


def visible_expected(T: int, H: int = H_VIS, extra=None, drop=None) -> np.ndarray:
    """[H, 64] float64 c_hd / n, optionally with one key added (index `extra`, past the end) or dropped."""
    keys = np.arange(T)
    if drop is not None:
        keys = keys[keys != drop]
    if extra is not None:
        keys = np.append(keys, extra)
    out = np.zeros((H, 64))
    for h in range(H):
        np.add.at(out[h], (keys + h) % 63, 1.0)
        out[h, 63] = np.count_nonzero(keys >= 63)
    return out / len(keys)


def visible_matches(got: np.ndarray, want: np.ndarray) -> bool:
    """Every element within 1 bf16 ulp of `want` (2^(floor(log2 |want|) - 7)) and exactly 0 where `want` is."""
    zero = want == 0
    nz = want[~zero]
    ulp = 2.0 ** (np.floor(np.log2(np.abs(nz))) - 7)
    return bool(np.all(got[zero] == 0) and np.all(np.abs(got[~zero] - nz) <= ulp))


def test_visible_set_comparator_rejects_single_key_changes():
    for T in VIS_T:
        base = visible_expected(T)
        bf = torch.tensor(base).to(torch.bfloat16).double().numpy()
        assert visible_matches(bf, base), T
        # every added key (each residue, before and past the flag column's edge) and every dropped key changes a count by one
        for r in range(127):
            assert not visible_matches(bf, visible_expected(T, extra=T + r)), (T, "add", r)
        for j in sorted(set(list(range(min(T, 127))) + list(range(max(0, T - 127), T)))):
            if T > 1:
                assert not visible_matches(bf, visible_expected(T, drop=j)), (T, "drop", j)
        shifted = np.roll(base, 1, axis=0)  # head h reads head h-1's values
        if not np.array_equal(shifted, base):
            assert not visible_matches(bf, shifted), (T, "head")


