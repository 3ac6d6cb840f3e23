"""CPU (-m "not gpu"): the CLIP score's host side — the oracle's Pillow resample against PIL itself, the library's tap
tables, the golden's digests, the weight loader, truncation and pooling, and the argument checks that fail before any
CUDA call."""
import ctypes as C
import json
from pathlib import Path

import numpy as np
import pytest
import torch
from PIL import Image

from oracle import clip_score as oc

GOLD = np.load(Path(__file__).parent / "golden" / "clip_score.npz")
SIZES = [(512, 1024), (1024, 512), (512, 512), (299, 299), (300, 517), (225, 225), (224, 224), (17, 9)]


@pytest.mark.parametrize("hw", SIZES)
def test_oracle_resize_bit_equal_to_pillow(hw):
    img = np.random.default_rng(hw[0] * 7 + hw[1]).integers(0, 256, (*hw, 3), dtype=np.uint8)
    hr, wr = oc.resized_size(*hw)
    assert min(hr, wr) == 224
    pil = np.asarray(Image.fromarray(img).resize((wr, hr), resample=Image.BICUBIC))
    assert np.array_equal(oc.resize_u8(img, hr, wr), pil)


@pytest.mark.parametrize("hw", SIZES + [(223, 100), (224, 300), (4000, 3000)])
def test_library_tap_tables_equal_the_oracle(hw):
    from panfusion_b200 import _lib
    l = _lib.lib()
    n = l.pf_clip_prep_taps_ints(*hw)
    buf = (C.c_int * n)()
    assert l.pf_clip_prep_taps(*hw, buf) == 0
    assert np.array_equal(np.frombuffer(buf, np.int32), oc.tap_table(*hw))


def test_resized_size_follows_the_processor():
    assert oc.resized_size(512, 1024) == (224, 448)
    assert oc.resized_size(1024, 512) == (448, 224)
    assert oc.resized_size(224, 300) == (224, 300)  # short side already 224: no resample
    assert oc.resized_size(17, 9) == (423, 224)


def test_golden_digests_regenerate_from_the_seed():
    seed = int(GOLD["seed"])
    assert oc.state_sha256(oc.seeded_state(seed)) == str(GOLD["weights_sha256"])
    assert oc.image_digest(oc.golden_images(seed)) == str(GOLD["images_sha256"])
    ids, _ = oc.pad_ids(oc.golden_prompts(seed))
    assert np.array_equal(ids.numpy(), GOLD["input_ids"])
    assert GOLD["lengths"].max() > 77 and (GOLD["input_ids"][:, :77] == oc.EOS).any(1).sum() == len(ids) - 1
    s = GOLD["scores"]
    assert s.max() > 20 and s.min() < -20  # the shared projection component spreads the scores over both signs
    assert float(GOLD["compute_pos"]) > 20 and float(GOLD["mean_neg"]) < -5 and float(GOLD["compute_neg"]) == 0


def _tiny_config():
    from transformers import CLIPConfig
    cfg = CLIPConfig(text_config=dict(vocab_size=49408, hidden_size=128, intermediate_size=256, num_hidden_layers=2,
                                      num_attention_heads=2, max_position_embeddings=77, hidden_act="quick_gelu",
                                      eos_token_id=2),
                     vision_config=dict(hidden_size=128, intermediate_size=256, num_hidden_layers=2,
                                        num_attention_heads=2, image_size=224, patch_size=16, hidden_act="quick_gelu"),
                     projection_dim=64)
    cfg._attn_implementation = "eager"
    cfg.text_config._attn_implementation = "eager"
    cfg.vision_config._attn_implementation = "eager"
    return cfg


@pytest.fixture(scope="module")
def tiny():
    from transformers import CLIPModel
    torch.manual_seed(0)
    return CLIPModel(_tiny_config()).double().eval()


def test_loader_accepts_the_three_sources(tiny, tmp_path):
    from panfusion_b200.clip_score import CLIPEncoder, expected_shapes
    a = CLIPEncoder(tiny)
    b = CLIPEncoder(tiny.state_dict(), tiny.config)
    tiny.float().save_pretrained(tmp_path)  # config.json + model.safetensors, as an HF snapshot holds them
    tiny.double()
    assert (tmp_path / "config.json").is_file() and (tmp_path / "model.safetensors").is_file()
    c = CLIPEncoder(str(tmp_path))
    assert c.path == tmp_path and a.path is None
    want = expected_shapes(a.cfg)
    assert len(want) == 13 + 2 * 16 * 2
    for k in want:
        assert torch.equal(a._sd[k], b._sd[k]) and torch.equal(a._sd[k], c._sd[k])
    d = tmp_path / "bin"
    d.mkdir()
    torch.save(tiny.float().state_dict(), d / "pytorch_model.bin")
    tiny.double()
    (d / "config.json").write_text((tmp_path / "config.json").read_text())
    assert torch.equal(CLIPEncoder(str(d))._sd["visual_projection.weight"], a._sd["visual_projection.weight"])


def test_loader_rejects_bad_sources(tiny, tmp_path):
    from panfusion_b200.clip_score import CLIPEncoder
    with pytest.raises(ValueError, match="not a local directory"):
        CLIPEncoder("openai/clip-vit-base-patch16")
    sd = dict(tiny.state_dict())
    del sd["vision_model.encoder.layers.1.mlp.fc2.bias"]
    with pytest.raises(ValueError, match="missing key 'vision_model.encoder.layers.1.mlp.fc2.bias'"):
        CLIPEncoder(sd, tiny.config)
    sd = dict(tiny.state_dict())
    sd["text_projection.weight"] = sd["text_projection.weight"][:, :-1]
    with pytest.raises(ValueError, match="'text_projection.weight' has shape"):
        CLIPEncoder(sd, tiny.config)
    with pytest.raises(ValueError, match="needs its config"):
        CLIPEncoder(tiny.state_dict())
    cfg = json.loads(tiny.config.to_json_string())
    cfg["vision_config"]["num_attention_heads"] = 4
    with pytest.raises(ValueError, match="head dim 32"):
        CLIPEncoder(tiny.state_dict(), cfg)
    (tmp_path / "config.json").write_text(json.dumps(cfg))
    with pytest.raises(ValueError, match="model.safetensors or pytorch_model.bin"):
        CLIPEncoder(str(tmp_path))


def test_truncation_and_argmax_pooling(tiny):
    """A prompt longer than 77 tokens loses its EOS; the text tower pools at input_ids.argmax(-1), as transformers
    4.26.1 does (the installed transformers does the same for eos_token_id == 2)."""
    from panfusion_b200.clip_score import CLIPEncoder, CLIPScore, eos_rows
    rows = oc.golden_prompts(int(GOLD["seed"]))
    tok = lambda text, padding=True, return_tensors="pt": {"input_ids": oc.pad_ids([rows[int(t[1:])] for t in text])[0]}
    m = CLIPScore(clip=CLIPEncoder(tiny), tokenizer=tok)
    with pytest.warns(UserWarning, match="longer than max_position_embeddings=77"):
        ids = m.token_ids(["p0", "p8"])
    assert ids.shape == (2, 77) and ids[1, -1] != oc.EOS and (ids[1] != oc.EOS).all()
    pool = eos_rows(ids)
    assert pool[0] == len(rows[0]) - 1 and pool[1] == int(torch.tensor(rows[8][:77]).argmax())
    with torch.no_grad():
        out = tiny.text_model(input_ids=ids, attention_mask=torch.ones_like(ids))
    assert torch.equal(out.pooler_output, out.last_hidden_state[torch.arange(2), pool])
    short = m.token_ids(["p0", "p1"])
    assert short.shape[1] == max(len(rows[0]), len(rows[1]))


def test_argument_checks_fail_before_cuda(tiny):
    from panfusion_b200 import _lib
    from panfusion_b200.clip_score import CLIPEncoder, CLIPScore
    l = _lib.lib()
    V = C.c_void_p
    assert l.pf_clip_prep(None, 1, 1, 8, 8, V(0x1000), V(0x2000), _lib.PF_F16, None) == -1
    assert b"null pointer" in l.pf_last_error()
    assert l.pf_clip_prep(V(0x1000), 1, 1, 8, 8, V(0x1000), V(0x2000), _lib.PF_BF16, None) == -1
    assert l.pf_clip_prep(V(0x1000), 0, 1, 8, 8, V(0x1002), V(0x2000), _lib.PF_F16, None) == -1
    assert b"misaligned" in l.pf_last_error()
    args = [V(0x1000)] * 5 + [C.c_float(1e-5), 2, 768, V(0x2000), _lib.PF_F16]
    assert l.pf_clip_embed(*args, V(0x3008), None) == -1 and b"16-byte" in l.pf_last_error()
    assert l.pf_clip_embed(*args[:7], 100, V(0x2000), _lib.PF_F16, V(0x3000), None) == -1
    assert l.pf_clip_embed(V(0x1004), *args[1:], V(0x3000), None) == -1
    assert l.pf_clip_score(V(0x1000), V(0x2000), 0, 512, V(0x3000), V(0x4000), None) == -1
    assert l.pf_clip_score(V(0x1000), V(0x2000), 2, 512, V(0x3000), V(0x4004), None) == -1
    assert l.pf_clip_prep_taps(0, 5, (C.c_int * 4)()) == -1
    a = _lib.GemmArgs()
    a.A, a.a_rows, a.a_ld, a.B, a.b_ld, a.dtype = 0x10000, 512, 320, 0x20000, 320, 1
    a.M, a.N, a.Kc, a.num_taps, a.out, a.out_ld, a.out_dtype = 512, 320, 320, 1, 0x30000, 320, 1
    a.act = 5
    assert l.pf_gemm_taps(C.byref(a), None) == -1 and b"unknown act" in l.pf_last_error()
    m = CLIPScore(clip=CLIPEncoder(tiny), tokenizer=lambda t, **k: {"input_ids": torch.zeros(len(t), 3, dtype=torch.long)})
    assert m.higher_is_better and not m._update_called
    assert m.score.dtype == torch.float64 and m.n_samples.dtype == torch.int64 and not m.state_dict()
    with pytest.raises(ValueError, match="same"):
        m.update(torch.zeros(2, 3, 8, 8, dtype=torch.uint8), ["a"])
    with pytest.raises(ValueError, match="3d"):
        m.update([torch.zeros(3, 8, 8, dtype=torch.uint8), torch.zeros(8, 8, dtype=torch.uint8)], ["a", "b"])
    with pytest.raises(ValueError, match="pass tokenizer="):
        CLIPScore(clip=CLIPEncoder(tiny))
    with pytest.raises(ValueError, match="CLIPEncoder"):
        CLIPScore(clip=object(), tokenizer=len)
    assert not m._update_called and int(m.n_samples) == 0
