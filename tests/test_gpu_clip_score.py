"""GPU: the CLIP score kernels (pf_clip_prep, pf_clip_embed, pf_clip_score, pf_gemm_taps with PF_ACT_QUICK_GELU) and
panfusion_b200.clip_score against the oracle's preprocessing, fp64 torch and tests/golden/clip_score.npz (minted by
oracle/clip_score.py; the seeded weights are regenerated here and their digest is checked on the CPU)."""
import ctypes as C
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import clip_score as oc
from panfusion_b200 import _lib, ops
from panfusion_b200.clip_score import CLIPEncoder, CLIPScore

pytestmark = pytest.mark.gpu
GOLD = np.load(Path(__file__).parent / "golden" / "clip_score.npz")
SIZES = [(512, 1024), (1024, 512), (512, 512), (299, 299), (300, 517), (225, 225), (224, 224), (17, 9)]
# gates: about 2x the values measured on an H100 80GB HBM3 at 700 W (DESIGN.md 5e)
EMB_MAX, EMB_MEAN = 1e-3, 2e-4   # of max|ref|; measured 5.0e-4 / 9.6e-5 (text), 3.6e-4 / 7.0e-5 (image)
SCORE_ABS, COMPUTE_ABS = 0.1, 0.05  # points; measured 0.054 per sample, 0.027 on a set's mean
QUICK_GELU_GEMM = 8e-4  # of max|ref|; measured <= 4.1e-4


def _rows():
    return [r.tolist()[:n] for r, n in zip(GOLD["input_ids"], GOLD["lengths"])]


def tokenizer(text, padding=True, return_tensors="pt"):
    """The golden's synthetic prompts: 'p<i>' -> its token row, padded with EOS like CLIPTokenizer(padding=True)."""
    rows = _rows()
    return {"input_ids": oc.pad_ids([rows[int(t[1:])] for t in text])[0]}


@pytest.fixture(scope="module")
def enc():
    return CLIPEncoder(oc.seeded_state(int(GOLD["seed"])), oc.clip_config())


@pytest.fixture(scope="module")
def imgs():
    return oc.golden_images(int(GOLD["seed"]))


def _prep(x, out_dtype):
    l = _lib.lib()
    B, _, H, W = x.shape
    n = int(l.pf_clip_prep_taps_ints(H, W))
    taps = torch.empty(n, dtype=torch.int32)
    _lib.check(l.pf_clip_prep_taps(H, W, C.c_void_p(taps.data_ptr())))
    taps = taps.to(x.device)
    out = torch.empty(B * 196, 768, device=x.device, dtype=out_dtype)
    _lib.check(l.pf_clip_prep(C.c_void_p(x.data_ptr()), int(x.dtype == torch.uint8), B, H, W, C.c_void_p(taps.data_ptr()),
                              C.c_void_p(out.data_ptr()), _lib.dtype_code(out_dtype), C.c_void_p(_lib.stream_ptr())))
    return out


@pytest.mark.parametrize("hw", SIZES)
@pytest.mark.parametrize("kind", ["uint8", "float32"])
def test_prep_bit_equal_to_oracle(hw, kind, cuda_device):
    """The uint8 crop and the fp32 pixel values equal the oracle's (PIL.Image.resize, numpy) bit for bit; the fp16
    rows are those values rounded once."""
    x = oc.structured_images(7 + hw[0], 2, *hw)
    if kind == "float32":
        x = (x.float() / 255 + 0.003 * torch.rand(x.shape, generator=torch.Generator().manual_seed(3))).clamp(0, 1)
    crops, pv = zip(*(oc.preprocess(i) for i in x))
    ref = oc.patch_rows(np.stack(pv))
    got = _prep(x.contiguous().to(cuda_device), torch.float32).cpu().numpy()
    assert got.view(np.uint32).tobytes() == ref.view(np.uint32).tobytes()
    # the uint8 crop: pixel values are an injective function of the uint8 level
    levels = ((np.arange(256, dtype=np.float64) * (1 / 255)).astype(np.float32)[None, :] - oc.MEAN[:, None]) / oc.STD[:, None]
    u8 = np.stack([np.searchsorted(levels[c], got.reshape(2, 14, 14, 3, 16, 16)[:, :, :, c]) for c in range(3)], -1)
    u8 = u8.transpose(0, 1, 3, 2, 4, 5).reshape(2, 224, 224, 3)
    assert np.array_equal(u8, np.stack(crops))
    half = _prep(x.contiguous().to(cuda_device), torch.float16).cpu()
    assert torch.equal(half, torch.from_numpy(ref).half())


@pytest.mark.parametrize("M,K,N,k_splits", [(197 * 2, 768, 3072, 1), (77 * 2, 512, 2048, 1), (40, 768, 3072, 3),
                                            (197, 768, 768, 2)])
def test_quick_gelu_gemm_vs_fp64(M, K, N, k_splits, cuda_device):
    """fc1 + quick_gelu at the tower shapes (in-kernel epilogue) and through the split-K reduce."""
    g = torch.Generator().manual_seed(M + N)
    a = torch.randn(M, K, generator=g).half()
    w = (torch.randn(N, K, generator=g) / K ** 0.5).half()
    b = 0.1 * torch.randn(N, generator=g)
    out = torch.empty(M, N, device=cuda_device, dtype=torch.float16)
    ops.gemm_taps(a.to(cuda_device), w.to(cuda_device), out, M=M, Kc=K, bias=b.to(cuda_device),
                  act=ops.PF_ACT_QUICK_GELU, k_splits=k_splits)
    z = a.double() @ w.double().T + b.double()
    ref = z * torch.sigmoid(1.702 * z)
    err = (out.double().cpu() - ref).abs().max().item() / ref.abs().max().item()
    print(f"quick_gelu GEMM M={M} K={K} N={N} k_splits={k_splits}: {err:.2e} of max|ref|")
    assert err < QUICK_GELU_GEMM


def test_clip_embed_vs_fp64(cuda_device):
    g = torch.Generator().manual_seed(5)
    B, Cc = 3, 768
    patches = torch.randn(B * 196, Cc, generator=g)
    cls, pos = torch.randn(Cc, generator=g), 0.5 * torch.randn(197, Cc, generator=g)
    gam, bet = 1 + 0.1 * torch.randn(Cc, generator=g), 0.05 * torch.randn(Cc, generator=g)
    dp, dc, dpos, dg, db = (t.to(cuda_device).contiguous() for t in (patches, cls, pos, gam, bet))
    out = torch.empty(B * 197, Cc, device=cuda_device, dtype=torch.float16)
    st = torch.empty(B * 197, 2, 2, device=cuda_device)
    Cv = C.c_void_p
    _lib.check(_lib.lib().pf_clip_embed(Cv(dp.data_ptr()), Cv(dc.data_ptr()), Cv(dpos.data_ptr()), Cv(dg.data_ptr()),
                                        Cv(db.data_ptr()), C.c_float(1e-5), B, Cc, Cv(out.data_ptr()), _lib.PF_F16,
                                        Cv(st.data_ptr()), Cv(_lib.stream_ptr())))
    torch.cuda.synchronize()
    e = torch.cat([cls.double()[None].expand(B, 1, Cc), patches.double().reshape(B, 196, Cc)], 1) + pos.double()
    ref = torch.nn.functional.layer_norm(e, (Cc,), gam.double(), bet.double(), 1e-5).reshape(B * 197, Cc)
    got = out.double().cpu()
    assert (got - ref).abs().max().item() < 2 * 2 ** -11 * ref.abs().max().item()
    s = st.double().cpu()
    assert torch.allclose(s[:, 0, 0], got.sum(1), rtol=1e-5, atol=1e-3)
    assert torch.allclose(s[:, 0, 1], (got * got).sum(1), rtol=1e-5)
    assert not s[:, 1].any()


def test_clip_score_kernel_vs_fp64(cuda_device):
    g = torch.Generator().manual_seed(9)
    B, D = 37, 512
    img, txt = torch.randn(B, D, generator=g), torch.randn(B, D, generator=g) + 0.5 * torch.randn(B, D, generator=g)
    state = torch.full((), 1.25, dtype=torch.float64, device=cuda_device)
    scores = torch.empty(B, device=cuda_device)
    Cv = C.c_void_p
    i, t = img.to(cuda_device), txt.to(cuda_device)
    _lib.check(_lib.lib().pf_clip_score(Cv(i.data_ptr()), Cv(t.data_ptr()), B, D, Cv(scores.data_ptr()),
                                        Cv(state.data_ptr()), Cv(_lib.stream_ptr())))
    ref = 100 * torch.nn.functional.cosine_similarity(img.double(), txt.double(), dim=-1)
    assert (scores.double().cpu() - ref).abs().max().item() < 1e-4
    acc = 1.25 + sum(float(v) for v in scores.cpu().double())
    assert float(state) == acc


def _golden_embeddings(enc, imgs, dev):
    img_e, txt_e = [], []
    rows = _rows()
    for s, i, p in GOLD["pairs"]:
        img_e.append(enc.encode_image(imgs[oc.ORDER[s]][i:i + 1].to(dev)))
        txt_e.append(enc.encode_text(oc.pad_ids([rows[p][:77]])[0], dev))
    return torch.cat(img_e).double().cpu(), torch.cat(txt_e).double().cpu()


def test_embeddings_and_scores_vs_golden(enc, imgs, cuda_device):
    img, txt = _golden_embeddings(enc, imgs, cuda_device)
    for name, got, ref in (("image", img, GOLD["img_emb"]), ("text", txt, GOLD["txt_emb"])):
        ref = torch.from_numpy(ref)
        scale = ref.abs().max().item()
        mx, mean = (got - ref).abs().max().item() / scale, (got - ref).abs().mean().item() / scale
        print(f"{name} embeddings: max {mx:.2e}, mean {mean:.2e} of max|ref|")
        assert mx < EMB_MAX and mean < EMB_MEAN
    m = CLIPScore(clip=enc, tokenizer=tokenizer, device=cuda_device)
    scores = []
    for s, i, p in GOLD["pairs"]:
        m.update(imgs[oc.ORDER[s]][i].to(cuda_device), f"p{p}")
        scores.append(m.last_scores.cpu())
    d = (torch.cat(scores).double() - torch.from_numpy(GOLD["scores"])).abs().max().item()
    print(f"per-sample scores: max |err| {d:.2e} points")
    assert d < SCORE_ABS


@pytest.mark.parametrize("which", ["pos", "neg"])
def test_compute_vs_golden(enc, imgs, which, cuda_device):
    """compute() of a set with a clearly positive mean and of one with a negative mean (clamped to 0)."""
    m = CLIPScore(clip=enc, tokenizer=tokenizer, device=cuda_device)
    assert not m._update_called
    for k in GOLD[f"set_{which}"]:
        s, i, p = GOLD["pairs"][k]
        m.update(imgs[oc.ORDER[s]][i:i + 1].to(cuda_device), [f"p{p}"])
    v = m.compute()
    assert v.is_cuda and v.dtype == torch.float32 and v.dim() == 0 and m._update_called
    mean = float(m.score) / int(m.n_samples)
    print(f"compute {which}: {float(v):.4f} (golden {float(GOLD[f'compute_{which}']):.4f}), mean {mean:.4f} "
          f"(golden {float(GOLD[f'mean_{which}']):.4f})")
    assert abs(float(v) - float(GOLD[f"compute_{which}"])) < COMPUTE_ABS
    assert abs(mean - float(GOLD[f"mean_{which}"])) < COMPUTE_ABS
    if which == "neg":
        assert float(v) == 0.0 and mean < -5
    m.reset()
    assert not m._update_called and float(m.score) == 0 and int(m.n_samples) == 0


def test_repeatable_and_batch_invariant(enc, imgs, cuda_device):
    pano = imgs["pano"].to(cuda_device)
    x = torch.cat([pano] * 4)  # batch 8
    a, b = enc.encode_image(x), enc.encode_image(x)
    assert torch.equal(a, b)
    one = torch.cat([enc.encode_image(x[k:k + 1]) for k in range(8)])
    assert torch.equal(one, a)
    rows = _rows()
    ids = oc.pad_ids([rows[k][:77] for k in range(8)])[0]
    t8 = enc.encode_text(ids, cuda_device)
    t1 = torch.cat([enc.encode_text(oc.pad_ids([rows[k][:77]])[0], cuda_device) for k in range(8)])
    assert torch.equal(t8, enc.encode_text(ids, cuda_device))
    assert torch.equal(t1, t8)  # padding follows the EOS row and the mask is causal
    m1 = CLIPScore(clip=enc, tokenizer=tokenizer, device=cuda_device)
    m2 = CLIPScore(clip=enc, tokenizer=tokenizer, device=cuda_device)
    for m in (m1, m2):
        m.update(x, [f"p{k}" for k in range(8)])
    assert torch.equal(m1.score, m2.score) and torch.equal(m1.compute(), m2.compute())


def test_eval_pano_gen_usage(enc, imgs, cuda_device):
    """EvalPanoGen: four metrics in an nn.ModuleDict sharing one encoder, built on the CPU, requires_grad_(False),
    moved with .to(device), fed what models/pano/EvalPanoGen.py:87,97,159,169 pass."""
    from panfusion_b200 import geometry
    d = torch.nn.ModuleDict({k: CLIPScore("openai/clip-vit-base-patch16", clip=enc, tokenizer=tokenizer)
                             for k in ("CS", "rot_CS", "mv_CS", "pers_CS")})
    d.requires_grad_(False)
    pano_gen = imgs["pano"]
    pano_prompt = ["p0", "p8"]
    with pytest.raises(ValueError, match="move the metric"):
        d["CS"].update(pano_gen.to(cuda_device), pano_prompt)
    d.to(cuda_device)
    assert all(m.score.is_cuda and m.n_samples.is_cuda for m in d.values())
    pano_gen = pano_gen.to(cuda_device)
    with pytest.warns(UserWarning, match="longer than"):
        d["CS"].update(pano_gen, pano_prompt)
    d["rot_CS"].update(torch.roll(pano_gen, pano_gen.shape[3] // 2, 3), pano_prompt)
    views = pano_gen.float() / 255
    pers_gen = torch.cat([geometry.e2p(views, 90, u, 0, (299, 299)) for u in (0, 90, 180, 270)]).contiguous()
    pers_prompt = [f"p{k}" for k in range(8)]
    d["mv_CS"].update(pers_gen, pers_prompt)
    images_pred = imgs["pers"].repeat(4, 1, 1, 1).to(cuda_device)
    d["pers_CS"].update(images_pred, pers_prompt)
    ref = CLIPScore(clip=enc, tokenizer=tokenizer, device=cuda_device)
    ref.update((pers_gen * 255).to(torch.uint8), pers_prompt)  # the float path is uint8(x * 255)
    assert torch.equal(ref.score, d["mv_CS"].score)
    for k, n in (("CS", 2), ("rot_CS", 2), ("mv_CS", 8), ("pers_CS", 8)):
        v = d[k].compute()
        assert int(d[k].n_samples) == n and v.is_cuda and v.dtype == torch.float32 and torch.isfinite(v)
    with pytest.raises(ValueError, match="same"):
        d["CS"].update(pano_gen, ["p0"])
    with pytest.raises(ValueError, match="3d"):
        d["CS"].update([pano_gen[0], pano_gen], ["p0", "p1"])
