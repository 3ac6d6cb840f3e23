"""CLIP score oracle: torchmetrics 1.3.2's CLIPScore update / compute, transformers 4.26.1's CLIPImageProcessor and the
CLIP ViT-B/16 towers, as models/pano/EvalPanoGen.py:33-46 builds them (`CLIPScore('openai/clip-vit-base-patch16')`).

Sources and what is pinned:
- The towers are the installed transformers' own `CLIPModel`, run in fp64 from a seeded `CLIPConfig` with the ViT-B/16
  geometry. transformers 5.x pools the text tower at the first `eos_token_id` unless `eos_token_id == 2`, in which case
  it pools at `input_ids.argmax(-1)`, which is what 4.26.1 always does [3P-mem]; the config sets `eos_token_id=2`.
- The preprocessing is restated on `PIL.Image.resize`, numpy and 4.26.1's order [3P-mem]: short side to 224 and long
  side to int(224 * long / short) (no resample when the short side is 224), BICUBIC by Pillow on uint8 HWC, centre crop
  at ((h - 224) // 2, (w - 224) // 2), rescale in float64 then float32, normalise in float32. A float image reaches
  Pillow as (x * 255).astype(uint8) (4.26.1's to_pil_image; unpinned [3P-mem]). The installed transformers' processor is
  not used: its resize differs from Pillow's uint8 path by up to one level.
- `resize_u8` restates Pillow's 8-bit bicubic resample from its behaviour (separable, horizontal first, coefficients in
  double normalised to 22-bit fixed point, int32 accumulation from 1 << 21); tests pin it bit-exactly against
  `PIL.Image.resize`. `tap_table` is the same computation in pf_clip_prep_taps' layout.
- `clip_score_update` / `clip_score_compute` restate torchmetrics 1.3.2 [3P-mem] (neither torchmetrics nor 4.26.1 is
  installed here).

`python -m oracle.clip_score` mints tests/golden/clip_score.npz from seeded weights (the seed and a SHA-256 of the
weight bytes are stored, not the weights), seeded images and synthetic token ids.
"""
from __future__ import annotations

import hashlib
import math
import warnings
from pathlib import Path

import numpy as np
import torch
from PIL import Image

GOLDEN = Path(__file__).resolve().parent.parent / "tests" / "golden" / "clip_score.npz"
SEED = 1616
SIZE = 224
MEAN = np.array([0.48145466, 0.4578275, 0.40821073], dtype=np.float32)
STD = np.array([0.26862954, 0.26130258, 0.27577711], dtype=np.float32)
BOS, EOS = 49406, 49407  # CLIP's <|startoftext|>, <|endoftext|> (also the pad token)
MAX_LEN = 77
# visual_projection and text_projection share a rank-one component of gain PROJ_GAIN: without it every image-text cosine
# of random towers sits near 0 and the clamp of compute() hides any error. With it per-sample scores spread over tens of
# points of both signs (recorded in DESIGN.md 5e).
PROJ_GAIN = 1.5


# ---- preprocessing ---------------------------------------------------------------------------------------------------

def resized_size(h: int, w: int) -> tuple[int, int]:
    """CLIPImageProcessor.resize's output (height, width) for shortest_edge 224 (get_resize_output_image_size)."""
    short, long = (w, h) if w <= h else (h, w)
    if short == SIZE:
        return h, w
    new_short, new_long = SIZE, int(SIZE * long / short)
    return (new_long, new_short) if w <= h else (new_short, new_long)


def _bicubic(x: float) -> float:
    a = -0.5
    x = abs(x)
    if x < 1.0:
        return ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    if x < 2.0:
        return (((x - 5) * x + 8) * x - 4) * a
    return 0.0


def axis_coeffs(n_in: int, n_out: int) -> tuple[int, list[tuple[int, int, list[int]]]]:
    """Pillow's bicubic taps of an n_in -> n_out axis: (ksize, [(start, count, 22-bit fixed-point coefficients)])."""
    scale = n_in / n_out
    fs = max(scale, 1.0)
    support = 2.0 * fs
    ksize = int(math.ceil(support)) * 2 + 1
    out = []
    for xx in range(n_out):
        center = (xx + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        xmax = min(int(center + support + 0.5), n_in) - xmin
        k = [_bicubic((x + xmin - center + 0.5) / fs) for x in range(xmax)]
        ww = 0.0
        for w in k:
            ww += w
        if ww != 0.0:
            k = [w / ww for w in k]
        fixed = [int(-0.5 + w * (1 << 22)) if w < 0 else int(0.5 + w * (1 << 22)) for w in k]
        out.append((xmin, xmax, fixed))
    return ksize, out


def _pass(x: np.ndarray, taps) -> np.ndarray:
    """One resample pass along axis 0 of int64 x [n_in, ...] -> uint8-valued int64 [n_out, ...]."""
    _, rows = taps
    out = np.empty((len(rows),) + x.shape[1:], dtype=np.int64)
    for i, (s, n, k) in enumerate(rows):
        acc = np.full(x.shape[1:], 1 << 21, dtype=np.int64)
        for j in range(n):
            acc += x[s + j] * k[j]
        out[i] = np.clip(acc >> 22, 0, 255)
    return out


def resize_u8(img: np.ndarray, h_out: int, w_out: int) -> np.ndarray:
    """Pillow's 8-bit bicubic Image.resize of a uint8 [H, W, C] image, restated: the horizontal pass when the width
    changes, then the vertical pass when the height changes, each on uint8 values."""
    x = img.astype(np.int64)
    h, w = x.shape[:2]
    if w_out != w:
        x = _pass(x.transpose(1, 0, 2), axis_coeffs(w, w_out)).transpose(1, 0, 2)
    if h_out != h:
        x = _pass(x, axis_coeffs(h, h_out))
    return x.astype(np.uint8)


def tap_table(h: int, w: int) -> np.ndarray:
    """pf_clip_prep_taps(h, w): {Kx, Ky, 0, 0}, then (start, count, Kx coefficients) per kept column, then (start, count,
    Ky coefficients) per kept row, as int32."""
    hr, wr = resized_size(h, w)
    blocks = []
    ks = []
    for n_in, n_out in ((w, wr), (h, hr)):
        k, rows = axis_coeffs(n_in, n_out)
        first = (n_out - SIZE) // 2
        t = np.zeros((SIZE, 2 + k), dtype=np.int32)
        for i in range(SIZE):
            s, n, c = rows[first + i]
            t[i, 0], t[i, 1] = s, n
            t[i, 2:2 + n] = c
        blocks.append(t.ravel())
        ks.append(k)
    return np.concatenate([np.array([ks[0], ks[1], 0, 0], dtype=np.int32)] + blocks)


def to_uint8_hwc(img: torch.Tensor) -> np.ndarray:
    """One CHW image as 4.26.1's to_pil_image sees it: uint8 as is, a float image as (x * 255).astype(uint8)."""
    a = img.detach().cpu().numpy().transpose(1, 2, 0)
    if a.dtype != np.uint8:
        a = (a.astype(np.float32) * np.float32(255)).astype(np.uint8)
    return np.ascontiguousarray(a)


def preprocess(img: torch.Tensor) -> tuple[np.ndarray, np.ndarray]:
    """One CHW image -> (the uint8 224x224x3 crop, pixel_values float32 [3, 224, 224])."""
    a = to_uint8_hwc(img)
    h, w = a.shape[:2]
    hr, wr = resized_size(h, w)
    if (hr, wr) != (h, w):
        a = np.asarray(Image.fromarray(a).resize((wr, hr), resample=Image.BICUBIC))
    top, left = (hr - SIZE) // 2, (wr - SIZE) // 2
    crop = a[top:top + SIZE, left:left + SIZE]
    x = (crop.astype(np.float64) * (1 / 255)).astype(np.float32)
    x = (x - MEAN) / STD
    return crop, x.transpose(2, 0, 1)


def patch_rows(pixel_values: np.ndarray) -> np.ndarray:
    """float32 [B, 3, 224, 224] -> [B * 196, 768] rows in the (c, kh, kw) order of patch_embedding.weight.reshape(768, -1)
    (pf_clip_prep's output layout)."""
    b = pixel_values.shape[0]
    p = pixel_values.reshape(b, 3, 14, 16, 14, 16).transpose(0, 2, 4, 1, 3, 5)
    return np.ascontiguousarray(p.reshape(b * 196, 768))


# ---- model -----------------------------------------------------------------------------------------------------------

def clip_config():
    """CLIPConfig of openai/clip-vit-base-patch16's geometry, with eos_token_id = 2 for 4.26.1's argmax pooling."""
    from transformers import CLIPConfig
    cfg = CLIPConfig(
        text_config=dict(vocab_size=49408, hidden_size=512, intermediate_size=2048, num_hidden_layers=12,
                         num_attention_heads=8, max_position_embeddings=MAX_LEN, hidden_act="quick_gelu",
                         layer_norm_eps=1e-5, eos_token_id=2, bos_token_id=0, pad_token_id=1),
        vision_config=dict(hidden_size=768, intermediate_size=3072, num_hidden_layers=12, num_attention_heads=12,
                           image_size=224, patch_size=16, num_channels=3, hidden_act="quick_gelu", layer_norm_eps=1e-5),
        projection_dim=512)
    cfg._attn_implementation = "eager"
    cfg.text_config._attn_implementation = "eager"
    cfg.vision_config._attn_implementation = "eager"
    return cfg


def seeded_state(seed: int = SEED) -> dict[str, torch.Tensor]:
    """fp32 state dict with CLIPModel's key names: linears N(0, 1/fan_in), biases N(0, 0.02), LayerNorm gamma
    1 + N(0, 0.1) and beta N(0, 0.05), embeddings N(0, 0.5) (class embedding N(0, 1)), and projections that share one
    rank-one component (PROJ_GAIN)."""
    from transformers import CLIPModel
    g = torch.Generator().manual_seed(seed)
    names = CLIPModel(clip_config()).state_dict()
    sd = {}
    for k in sorted(names):
        shape = tuple(names[k].shape)
        if k == "logit_scale":
            sd[k] = torch.tensor(math.log(1 / 0.07))
        elif k.endswith("projection.weight"):
            continue
        elif "norm" in k and k.endswith(".weight"):
            sd[k] = 1 + 0.1 * torch.randn(shape, generator=g)
        elif "norm" in k and k.endswith(".bias"):
            sd[k] = 0.05 * torch.randn(shape, generator=g)
        elif k.endswith(".bias"):
            sd[k] = 0.02 * torch.randn(shape, generator=g)
        elif k.endswith("class_embedding"):
            sd[k] = torch.randn(shape, generator=g)
        elif "embedding" in k and k.endswith("weight") and "patch" not in k:
            sd[k] = 0.5 * torch.randn(shape, generator=g)
        else:
            fan_in = int(np.prod(shape[1:]))
            sd[k] = torch.randn(shape, generator=g) / math.sqrt(fan_in)
    u = torch.randn(512, generator=g)
    u /= u.norm()
    noise = {k: torch.randn(512, d, generator=g) / math.sqrt(d)
             for k, d in (("visual_projection.weight", 768), ("text_projection.weight", 512))}
    # the shared component reads each tower's pooled feature along its main direction of variation over the golden
    # inputs (orthogonal to their mean): random towers map every input to nearly the same pooled vector
    model = build_model({**sd, **noise})
    imgs, prompts = golden_images(seed), golden_prompts(seed)
    with torch.no_grad():
        pv = torch.from_numpy(np.stack([preprocess(imgs[s][i])[1] for s in ORDER for i in range(len(imgs[s]))]))
        hv = model.vision_model(pixel_values=pv.double()).pooler_output
        ids, mask = pad_ids(prompts)
        ht = model.text_model(input_ids=ids[:, :MAX_LEN], attention_mask=mask[:, :MAX_LEN]).pooler_output
    for k, h in (("visual_projection.weight", hv), ("text_projection.weight", ht)):
        m = h.mean(0)
        a = torch.linalg.svd(h - m, full_matrices=False)[2][0]
        a = a - (a @ m) / (m @ m) * m
        z = h @ a
        r = (h @ noise[k].double().T).norm(dim=1).median()
        sd[k] = noise[k] + (PROJ_GAIN * r / z.std()) * u[:, None] * a[None, :].float()
    return {k: v.float().contiguous() for k, v in sd.items()}


def state_sha256(sd: dict[str, torch.Tensor]) -> str:
    h = hashlib.sha256()
    for k in sorted(sd):
        h.update(k.encode())
        h.update(sd[k].float().contiguous().numpy().tobytes())
    return h.hexdigest()


def build_model(sd: dict[str, torch.Tensor]):
    from transformers import CLIPModel
    m = CLIPModel(clip_config())
    m.load_state_dict(sd, strict=False)
    return m.double().eval()


# ---- torchmetrics 1.3.2 ----------------------------------------------------------------------------------------------

def pad_ids(rows: list[list[int]]) -> tuple[torch.Tensor, torch.Tensor]:
    """padding=True: pad to the longest row with the pad token (EOS); -> (input_ids, attention_mask) int64."""
    n = max(len(r) for r in rows)
    ids = torch.full((len(rows), n), EOS, dtype=torch.int64)
    mask = torch.zeros((len(rows), n), dtype=torch.int64)
    for i, r in enumerate(rows):
        ids[i, :len(r)] = torch.tensor(r)
        mask[i, :len(r)] = 1
    return ids, mask


@torch.no_grad()
def clip_score_update(images, text, model, tokenize) -> tuple[torch.Tensor, int, torch.Tensor, torch.Tensor]:
    """torchmetrics' _clip_score_update with `tokenize(list[str]) -> list of id rows`: -> (per-sample scores, n,
    normalised image features, normalised text features), fp64."""
    if not isinstance(images, list):
        images = [images] if images.ndim == 3 else list(images)
    if not all(i.ndim == 3 for i in images):
        raise ValueError("Expected all images to be 3d but found image that has either more or less")
    if not isinstance(text, list):
        text = [text]
    if len(text) != len(images):
        raise ValueError(
            f"Expected the number of images and text examples to be the same but got {len(images)} and {len(text)}")
    pixel_values = torch.from_numpy(np.stack([preprocess(i)[1] for i in images]))
    ids, mask = pad_ids(tokenize(text))
    if mask.shape[-1] > MAX_LEN:
        warnings.warn(f"Encountered caption longer than max_position_embeddings={MAX_LEN}. Will truncate captions to "
                      "this length.", UserWarning)
        ids, mask = ids[..., :MAX_LEN], mask[..., :MAX_LEN]
    img = model.get_image_features(pixel_values.double()).pooler_output
    img = img / img.norm(p=2, dim=-1, keepdim=True)
    txt = model.get_text_features(ids, mask).pooler_output
    txt = txt / txt.norm(p=2, dim=-1, keepdim=True)
    return 100 * (img * txt).sum(axis=-1), len(text), img, txt


def clip_score_compute(score_sum: float, n_samples: int) -> float:
    return max(score_sum / n_samples, 0.0)


# ---- golden ----------------------------------------------------------------------------------------------------------

def structured_images(seed: int, n: int, h: int, w: int) -> torch.Tensor:
    """uint8 [n, 3, h, w]: smooth colour fields with seeded bands and blobs (not white noise: the resize and the towers
    see edges and gradients)."""
    g = torch.Generator().manual_seed(seed)
    yy, xx = torch.meshgrid(torch.linspace(0, 1, h, dtype=torch.float64), torch.linspace(0, 1, w, dtype=torch.float64),
                            indexing="ij")
    out = torch.empty(n, 3, h, w, dtype=torch.uint8)
    for i in range(n):
        p = torch.rand(3, 8, generator=g, dtype=torch.float64)
        img = torch.empty(3, h, w, dtype=torch.float64)
        for c in range(3):
            f = 0.5 + 0.25 * torch.sin(2 * math.pi * (p[c, 0] * 3 * xx + p[c, 1] * 2 * yy + p[c, 2]))
            f = f + 0.2 * torch.exp(-((xx - p[c, 3]) ** 2 + (yy - p[c, 4]) ** 2) / (0.01 + 0.05 * p[c, 5]))
            f = f + 0.1 * ((xx * (4 + 8 * p[c, 6])).floor() % 2) * p[c, 7]
            img[c] = f
        img = img + 0.03 * torch.randn(3, h, w, generator=g, dtype=torch.float64)
        out[i] = (img.clamp(0, 1) * 255).round().to(torch.uint8)
    return out


def golden_images(seed: int = SEED) -> dict[str, torch.Tensor]:
    """The image sets EvalPanoGen feeds CLIPScore: uint8 512x1024 panoramas (CS), their roll(W/2) (rot_CS), fp32 [0, 1]
    299^2 crops (mv_CS), uint8 512^2 perspective images (pers_CS), and one uint8 image already 224^2."""
    pano = structured_images(seed, 2, 512, 1024)
    crops = structured_images(seed + 1, 2, 299, 299).float() / 255
    crops = (crops + 0.002 * torch.rand(crops.shape, generator=torch.Generator().manual_seed(seed + 2))).clamp(0, 1)
    return {"pano": pano, "rot": torch.roll(pano, pano.shape[3] // 2, 3), "crop": crops,
            "pers": structured_images(seed + 3, 2, 512, 512), "sq224": structured_images(seed + 4, 1, 224, 224)}


def golden_prompts(seed: int = SEED) -> list[list[int]]:
    """Synthetic token rows (BOS, ids, EOS) of varied length, the last one 90 tokens long without an EOS in its first 77."""
    g = torch.Generator().manual_seed(seed + 5)
    rows = []
    for n in (5, 12, 20, 7, 33, 9, 15, 3):
        rows.append([BOS] + torch.randint(1, BOS, (n,), generator=g).tolist() + [EOS])
    rows.append([BOS] + torch.randint(1, BOS, (88,), generator=g).tolist() + [EOS])
    return rows


ORDER = ("pano", "rot", "crop", "pers", "sq224")


def image_digest(imgs: dict[str, torch.Tensor]) -> str:
    h = hashlib.sha256()
    for k in ORDER:
        h.update(k.encode())
        h.update(imgs[k].contiguous().numpy().tobytes())
    return h.hexdigest()


def golden_pairs() -> list[tuple[str, int, int]]:
    """(set, image index, prompt index) of the 9 golden samples, in order."""
    return [("pano", 0, 0), ("pano", 1, 8), ("rot", 0, 0), ("rot", 1, 8), ("crop", 0, 1), ("crop", 1, 2),
            ("pers", 0, 3), ("pers", 1, 4), ("sq224", 0, 5)]


def mint() -> dict[str, np.ndarray]:
    sd = seeded_state(SEED)
    model = build_model(sd)
    imgs = golden_images(SEED)
    prompts = golden_prompts(SEED)
    names = {f"p{i}": r for i, r in enumerate(prompts)}
    tok = lambda text: [names[t] for t in text]
    scores, img_f, txt_f = [], [], []
    for s, i, p in golden_pairs():
        sc, _, fi, ft = clip_score_update(imgs[s][i], f"p{p}", model, tok)
        scores.append(sc)
        img_f.append(fi)
        txt_f.append(ft)
    scores = torch.cat(scores)
    img_raw, txt_raw = [], []  # unnormalised projections (the towers' outputs)
    with torch.no_grad():
        for s, i, p in golden_pairs():
            pv = torch.from_numpy(preprocess(imgs[s][i])[1][None]).double()
            img_raw.append(model.get_image_features(pv).pooler_output)
            ids, mask = pad_ids([prompts[p]])
            txt_raw.append(model.get_text_features(ids[:, :MAX_LEN], mask[:, :MAX_LEN]).pooler_output)
    pos = [k for k in range(len(scores)) if scores[k] > 0]
    neg = [k for k in range(len(scores)) if scores[k] < 0]
    ids, _ = pad_ids(prompts)
    out = dict(
        seed=np.int64(SEED), weights_sha256=np.array(state_sha256(sd)), images_sha256=np.array(image_digest(imgs)),
        input_ids=ids.numpy(), lengths=np.array([len(r) for r in prompts], dtype=np.int64),
        pairs=np.array([(ORDER.index(s), i, p) for s, i, p in golden_pairs()], dtype=np.int64),
        img_emb=torch.cat(img_raw).numpy(), txt_emb=torch.cat(txt_raw).numpy(), scores=scores.numpy(),
        set_pos=np.array(pos, dtype=np.int64), set_neg=np.array(neg, dtype=np.int64),
        compute_pos=np.float64(clip_score_compute(float(scores[pos].sum()), len(pos))),
        compute_neg=np.float64(clip_score_compute(float(scores[neg].sum()), len(neg))),
        mean_pos=np.float64(scores[pos].mean()), mean_neg=np.float64(scores[neg].mean()))
    return out


if __name__ == "__main__":
    g = mint()
    GOLDEN.parent.mkdir(parents=True, exist_ok=True)
    with open(GOLDEN, "wb") as f:
        np.savez_compressed(f, **g)
    print(f"{GOLDEN}: {GOLDEN.stat().st_size} bytes; scores {np.round(g['scores'], 2).tolist()}; "
          f"compute pos {float(g['compute_pos']):.3f} (mean {float(g['mean_pos']):.3f}), "
          f"neg {float(g['compute_neg']):.3f} (mean {float(g['mean_neg']):.3f})")
