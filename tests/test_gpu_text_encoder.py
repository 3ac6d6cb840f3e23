"""-m gpu: the CLIP text encoder + prompt-embedding cache (panfusion_b200/text_encoder.py) against transformers' own
CLIPTextModel executed on the CPU (oracle/text_encoder.py) — the class the reference instantiates at
models/pano/PanoGenerator.py:117-121 — on seeded weights and token rows. Limits = 2x the measured end-to-end deviation
(16-bit storage between ~140 kernels against an fp32 reference), relative to max|ref|."""
import pytest
import torch

pytestmark = pytest.mark.gpu

# measured on an H100: fp16 2.5e-3 / 2.4e-4, bf16 2.1e-2 / 2.0e-3 (SD-2 size, 23 layers)
LIMITS = {torch.float16: (5e-3, 5e-4), torch.bfloat16: (4.7e-2, 4e-3)}


def _cmp(name, got, ref, dtype):
    scale = ref.abs().max().item()
    d = (got.float().cpu() - ref).abs()
    mx, mean = d.max().item() / scale, d.mean().item() / scale
    print(f"[parity] {name} {dtype}: max {mx:.3e} mean {mean:.3e} (of max|ref|) limits {LIMITS[dtype]}")
    assert mx <= LIMITS[dtype][0] and mean <= LIMITS[dtype][1]


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("config", ["TINY_TEXT_CONFIG", "SD2_TEXT_CONFIG"])
def test_text_encoder_vs_transformers(cuda_device, dtype, config):
    from oracle import text_encoder as ot
    from panfusion_b200.text_encoder import CLIPTextEncoder
    cfg = getattr(ot, config)
    model = ot.build_text_encoder(cfg, seed=0)
    ids = ot.token_ids(3, vocab=cfg["vocab_size"], seed=1)
    ref = ot.encode_text(model, ids)
    enc = CLIPTextEncoder(model, dtype).prepare(cuda_device, dtype)
    got = enc(ids)
    assert got.shape == ref.shape and got.dtype == dtype
    _cmp(f"CLIPTextModel {config}", got, ref, dtype)
    # causal: changing a late token must not change earlier positions (bit-exact), and must change later ones
    ids2 = ids.clone()
    ids2[0, 40] = (ids2[0, 40] + 1) % (cfg["vocab_size"] - 2)
    got2 = enc(ids2)
    assert torch.equal(got2[0, :40], got[0, :40]) and torch.equal(got2[1:], got[1:])
    assert (got2[0, 40:].float() - got[0, 40:].float()).abs().max().item() > 1e-3
    # a shorter sequence (no padding to 77) is the prefix of the same computation
    short = enc(ids[:, :20])
    assert torch.equal(short, got[:, :20])


def test_prompt_embedder_cache_and_cfg_layout(cuda_device):
    """embed_prompt + the [null; text] concatenation of PanFusion.inference (PanFusion.py:45-62,134-138): layout, values,
    and that each distinct token row is encoded once."""
    from oracle import text_encoder as ot
    from panfusion_b200.text_encoder import CLIPTextEncoder, PromptEmbedder
    cfg = ot.TINY_TEXT_CONFIG
    model = ot.build_text_encoder(cfg, seed=0)
    emb = PromptEmbedder(CLIPTextEncoder(model, torch.float16).prepare(cuda_device, torch.float16))
    ids = ot.token_ids(3, vocab=cfg["vocab_size"], seed=2)
    pano_ids, null_ids = ids[:2], ids[2:3]
    m = 4
    pers, pano = emb.embed_prompt(pano_ids, null_ids, m)
    assert pers.shape == (4, m, 77, cfg["hidden_size"]) and pano.shape == (4, 1, 77, cfg["hidden_size"])
    assert emb.misses == 3 and emb.hits == 0
    ref = ot.encode_text(model, ids)
    tol = dict(rtol=0, atol=3e-3 * ref.abs().max().item())
    torch.testing.assert_close(pano[2:, 0].float().cpu(), ref[:2], **tol)       # text half
    torch.testing.assert_close(pano[0, 0].float().cpu(), ref[2], **tol)          # null half
    assert torch.equal(pano[0], pano[1]) and torch.equal(pers[2, 3], pano[2, 0]) and torch.equal(pers[0, 1], pano[0, 0])
    pers2, pano2 = emb.embed_prompt(pano_ids, null_ids, m)                        # second image: all from the cache
    assert emb.misses == 3 and emb.hits == 3 and torch.equal(pano2, pano) and torch.equal(pers2, pers)
    per_view = ot.token_ids(2 * m, vocab=cfg["vocab_size"], seed=3)               # use_pers_prompt
    pers3, _ = emb.embed_prompt(pano_ids, null_ids, m, pers_ids=per_view)
    torch.testing.assert_close(pers3[2:].reshape(2 * m, 77, -1).float().cpu(), ot.encode_text(model, per_view), **tol)
    with pytest.raises(ValueError):
        emb.encoder(torch.zeros((1, 78), dtype=torch.int64))
