"""EvalPanoGen oracle: the reference's own models/pano/EvalPanoGen.py test_step, executed by path with metrics that only
record their update calls (oracle/shims/recording.py), then the oracle's seeded networks (oracle/inception.py,
oracle/clip_score.py, oracle/faed.py) turning the recorded images into per-slot features and the final values.

Executing the reference pins what the driver must reproduce: the order of the metric calls, the RNG draws and the
cameras (the reference's random_sample_camera on the global numpy RandomState), the e2p crops (CPU e2p through the kornia
shim) and every dtype conversion. A "slot" is one update call of one metric: `<key>#<call>`.

`python -m oracle.eval_pano` mints tests/golden/eval_pano.npz (build container only: it needs the reference). The
golden holds the seeds, the drawn cameras, per slot the image count, the real flag and a SHA-256 of every image (uint8,
as the metric sees it; reference_crops makes the crops again and the digests pin them), the oracle's pool3 / logits /
CLIP scores / FAED features of every image of step 0 and of the first image of each later slot (`_rows` of them), the
unclamped mean CLIP scores and the final values of on_test_end over every image (the IS values after
torch.manual_seed(IS_SEED), drawn in the metrics' order), and cv2.resize(INTER_AREA) by 2 of seeded images. The
golden stays small: the crops are made again rather than stored, and the outputs of step 1 past each slot's first
image enter only through the final values.
"""
from __future__ import annotations

import hashlib
import importlib
import importlib.util
import sys
import types
from pathlib import Path

import numpy as np
import torch

from oracle import clip_score as oc
from oracle import faed as of
from oracle import inception as oi

GOLDEN = Path(__file__).resolve().parent.parent / "tests" / "golden" / "eval_pano.npz"
SHIMS = Path(__file__).resolve().parent / "shims"
SEED = 4242          # np.random.seed before the first test_step
IS_SEED = 77         # torch.manual_seed before on_test_end
STEPS = 2            # two test_steps, so the RNG carry-over between steps is pinned
PANO_HW = (128, 256)  # pano_height 128: FAED pools 4 latitude rows, two of them with weight 0.87
VIEW_HW = (32, 32)
NUM_EVAL_CROPS = 2
KEYS = ("FID", "IS", "CS", "rot_FID", "rot_IS", "rot_CS", "crop_FID", "crop_IS", "seam_FID", "seam_IS", "mv_FID",
        "mv_IS", "mv_CS", "pers_FID", "pers_IS", "pers_CS", "FAED")  # EvalPanoGen.eval_metrics' order, without layout


# ---- seeded batches and prompts -------------------------------------------------------------------------------------

def batch(step: int) -> dict:
    """The test batch of step `step` in the reference's layout: uint8 pano / pano_pred [1, 1, 3, H, W], images_pred
    [1, 8, 3, h, w], pano_prompt [1], prompt collated view-major (8 sequences of 1)."""
    base = SEED + 10 * step
    return dict(
        pano=oc.structured_images(base, 1, *PANO_HW)[:, None],
        pano_pred=oc.structured_images(base + 1, 1, *PANO_HW)[:, None],
        images_pred=oc.structured_images(base + 2, 8, *VIEW_HW)[None],
        pano_prompt=[f"a panorama of room {step}"],
        prompt=[[f"view {i} of room {step}"] for i in range(8)],
        pano_id=[f"scene_{step}"])


def token_rows(text: list[str]) -> list[list[int]]:
    """A deterministic stand-in for CLIPTokenizer: BOS, one id per byte, EOS."""
    return [[oc.BOS] + [1 + (b * 131 + i) % (oc.BOS - 1) for i, b in enumerate(t.encode())] + [oc.EOS] for t in text]


def tokenizer(text, padding=True, return_tensors="pt"):
    """token_rows as the callable CLIPScore takes (padded with EOS like CLIPTokenizer(padding=True))."""
    return {"input_ids": oc.pad_ids(token_rows(list(text)))[0]}


# ---- the reference's test_step over recording metrics ---------------------------------------------------------------

def _module_from(path: Path, name: str):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    sys.modules[name] = mod
    spec.loader.exec_module(mod)
    return mod


def load_reference():
    """models/pano/EvalPanoGen.py by path, its metrics resolved to recording stand-ins."""
    from oracle import ref_loader
    ref_loader.load()
    fid = importlib.import_module("torchmetrics.image.fid")
    from oracle.shims.recording import RecordingMetric
    fid.FrechetInceptionDistance = type("FrechetInceptionDistance", (RecordingMetric,), {})
    for pkg in ("models.faed", "models.horizonnet"):
        m = types.ModuleType(pkg)
        m.__path__ = []
        sys.modules[pkg] = m
    _module_from(SHIMS / "models" / "faed" / "FAED.py", "models.faed.FAED")
    _module_from(SHIMS / "models" / "horizonnet" / "HorizonNet.py", "models.horizonnet.HorizonNet")
    _module_from(SHIMS / "models" / "pano" / "PanoGenerator.py", "models.pano.PanoGenerator")
    return importlib.import_module("models.pano.EvalPanoGen")


def run_reference():
    """-> (EvalPanoGen with recorded calls, the cameras random_sample_camera returned (radians, float64), in order)."""
    mod = load_reference()
    draws = []
    sample = mod.random_sample_camera

    def recording_sample(n):
        theta, phi = sample(n)
        draws.append((theta.copy(), phi.copy()))
        return theta, phi

    mod.random_sample_camera = recording_sample
    ev = mod.EvalPanoGen(num_eval_crops=NUM_EVAL_CROPS, pano_height=PANO_HW[0], log_test_samples=0)
    np.random.seed(SEED)
    with torch.no_grad():
        for s in range(STEPS):
            ev.test_step(batch(s), s)
    return ev, draws


def as_uint8(imgs: torch.Tensor, normalize: bool) -> torch.Tensor:
    """The uint8 image a metric sees: torchmetrics' normalize=True is (x * 255).byte()."""
    return (imgs * 255).byte() if normalize else imgs


def digest(img: torch.Tensor) -> str:
    return hashlib.sha256(img.contiguous().numpy().tobytes()).hexdigest()


def slots(ev) -> list[tuple[str, int, dict]]:
    """(key, call index, {images uint8, real, text, step}) of every recorded update, in key then call order."""
    out = []
    for key in KEYS:
        m = ev.eval_metrics[key]
        per_step = len(m.calls) // STEPS
        for c, (args, kwargs) in enumerate(m.calls):
            imgs = as_uint8(args[0], bool(m.init_kwargs.get("normalize", False)))
            out.append((key, c, dict(images=imgs, real=kwargs.get("real"), text=args[1] if len(args) > 1 else None,
                                     step=c // per_step)))
    return out


def crop_slots(gold):
    """(FID slot tag, uint8 panorama [1, 3, H, W], theta, phi (fp32 degrees), crop size, normalize) of every crop set
    the reference's test_step made, from the golden's cameras: crop_ and seam_ (theta 180) from the recorded draws,
    mv_ and pers_ from the 8 horizon cameras; real and generated side (pers_'s generated images are images_pred)."""
    mv = (np.rad2deg(np.linspace(0, 2 * np.pi, 8, endpoint=False)).astype(np.float32), np.zeros(8, np.float32))
    for s in range(int(gold["steps"])):
        b = batch(s)
        crop = tuple(gold[f"draw{2 * s}_deg32"])
        seam = (np.full_like(gold[f"draw{2 * s + 1}_deg32"][0], 180.0), gold[f"draw{2 * s + 1}_deg32"][1])
        for prefix, (theta, phi), hw, normalize in (("crop", crop, (299, 299), True), ("seam", seam, (299, 299), True),
                                                    ("mv", mv, (299, 299), True),
                                                    ("pers", mv, tuple(gold["view_hw"]), False)):
            for real, key in ((True, "pano"), (False, "pano_pred")):
                if prefix != "pers" or real:
                    yield f"{prefix}_FID#{2 * s + (not real)}", b[key][:, 0], theta, phi, hw, normalize


def reference_crops(pano: torch.Tensor, theta, phi, hw, normalize: bool) -> torch.Tensor:
    """The uint8 crops the reference's test_step hands its metrics, made again on the CPU with oracle/geometry.py's
    e2p (the reference's CPU e2p restated; the golden's digests pin the result): uint8 pano [1, 3, H, W] and fp32
    angles in degrees -> `(e2p(pano.float() / 255, ...) * 255).byte()`, or `e2p(pano.float(), ...).to(torch.uint8)`."""
    from oracle import geometry as og
    theta, phi = torch.as_tensor(theta, dtype=torch.float32), torch.as_tensor(phi, dtype=torch.float32)
    x = pano.float()
    x = (x / 255 if normalize else x).expand(theta.numel(), -1, -1, -1)
    v = og.e2p(x, 90, theta, phi, tuple(hw))
    return as_uint8(v, True) if normalize else v.to(torch.uint8)


# ---- final values from per-slot features ---------------------------------------------------------------------------

def inception_score_perm(logits: torch.Tensor, idx: torch.Tensor, splits: int = 10) -> tuple[float, float]:
    """InceptionScore.compute after its randperm `idx` (oracle/inception.py's reduction without the reseed)."""
    f = logits.double()[idx]
    prob, log_prob = f.softmax(dim=1), f.log_softmax(dim=1)
    kl = []
    for p, lp in zip(prob.chunk(splits, dim=0), log_prob.chunk(splits, dim=0)):
        m = p.mean(dim=0, keepdim=True)
        kl.append((p * (lp - m.log())).sum(dim=1).mean().exp())
    kl = torch.stack(kl)
    return float(kl.mean()), float(kl.std())


def final_values(per_slot: list[tuple[str, int, dict]], is_seed: int = IS_SEED) -> dict[str, float]:
    """on_test_end over per-slot outputs: {key: real, pool3 | logits | scores | faed}. FID and FAED are the fp64
    distance with clamped symmetric eigensolvers (oracle/faed.py faed_eigh); the IS randperms are drawn in key order
    after torch.manual_seed(is_seed)."""
    by_key: dict[str, list[dict]] = {}
    for key, _, s in per_slot:
        by_key.setdefault(key, []).append(s)
    torch.manual_seed(is_seed)
    out = {}
    for key in KEYS:
        if key not in by_key:
            continue
        calls = by_key[key]
        if key.endswith("IS"):
            logits = torch.cat([torch.as_tensor(s["logits"]) for s in calls])
            out[key], out[f"{key}_std"] = inception_score_perm(logits, torch.randperm(logits.shape[0]))
        elif key.endswith("CS"):
            sc = torch.cat([torch.as_tensor(s["scores"]).double() for s in calls])
            out[key] = oc.clip_score_compute(float(sc.sum()), sc.numel())
        else:
            f = "faed" if key == "FAED" else "pool3"
            st = [of.stats([torch.as_tensor(s[f]) for s in calls if bool(s["real"]) == side]) for side in (True, False)]
            out[key] = of.faed_eigh(*st[0], *st[1])
    return out


# ---- cv2.resize(INTER_AREA) by 2 of the stitched ground truth (dataset/PanoDataset.py:140) --------------------------

RESIZE_CASES = [(8, 2048), (6, 2046), (10, 30), (1024, 2048)]  # (H, W) of seeded uint8 [H, W, 3] images, seed 500 + i
RESIZE_FULL = 3  # the cases from here on keep a digest of the output, not the output


def resize_input(i: int) -> np.ndarray:
    g = torch.Generator().manual_seed(500 + i)
    return torch.randint(0, 256, (*RESIZE_CASES[i], 3), generator=g, dtype=torch.uint8).numpy()


def resize_golden() -> dict:
    import cv2
    out = {}
    for i, (h, w) in enumerate(RESIZE_CASES):
        r = cv2.resize(resize_input(i), (w // 2, h // 2), interpolation=cv2.INTER_AREA)
        if i < RESIZE_FULL:
            out[f"resize{i}"] = r
        else:
            out[f"resize{i}_sha256"] = np.array(hashlib.sha256(np.ascontiguousarray(r).tobytes()).hexdigest())
    return out


# ---- minting -------------------------------------------------------------------------------------------------------

def mint() -> dict:
    torch.set_num_threads(8)
    ev, draws = run_reference()
    isd, csd, fsd = oi.synth_state(), oc.seeded_state(), of.synth_state()
    net = oi.network().double()
    net.load_state_dict(isd)
    clip = oc.build_model(csd)
    cache: dict[str, tuple[torch.Tensor, torch.Tensor]] = {}

    def inception(imgs):
        for x in imgs:
            if digest(x) not in cache:
                p, l = oi.features(net, x[None], torch.float64)
                cache[digest(x)] = (p[0].float(), l[0].float())
        return (torch.stack([cache[digest(x)][0] for x in imgs]), torch.stack([cache[digest(x)][1] for x in imgs]))

    gold = {"seed": np.int64(SEED), "is_seed": np.int64(IS_SEED), "steps": np.int64(STEPS),
            "pano_hw": np.array(PANO_HW), "view_hw": np.array(VIEW_HW), "num_eval_crops": np.int64(NUM_EVAL_CROPS),
            "inception_sha256": np.array(oi.state_sha256(isd)), "clip_sha256": np.array(oc.state_sha256(csd)),
            "faed_sha256": np.array(of.state_sha256(fsd)),
            "batches_sha256": np.array([digest(torch.cat([batch(s)[k].reshape(-1) for k in ("pano", "pano_pred",
                                                                                               "images_pred")]))
                                        for s in range(STEPS)])}
    # the cameras: random_sample_camera's radians and the fp32 degrees e2p receives
    for i, (theta, phi) in enumerate(draws):
        gold[f"draw{i}_rad"] = np.stack([theta, phi])
        gold[f"draw{i}_deg32"] = np.stack([np.rad2deg(theta), np.rad2deg(phi)]).astype(np.float32)
    per_slot, names = [], []
    for key, c, s in slots(ev):
        imgs, tag = s["images"], f"{key}#{c}"
        names.append(tag)
        rec = {"real": s["real"]}
        rows = imgs.shape[0] if s["step"] == 0 else 1  # outputs kept: every image of step 0, the first of step 1
        gold[f"{tag}_n"] = np.int64(imgs.shape[0])
        gold[f"{tag}_rows"] = np.int64(rows)
        gold[f"{tag}_hw"] = np.array(imgs.shape[-2:])
        gold[f"{tag}_digests"] = np.array([digest(x) for x in imgs])
        if s["real"] is not None:
            gold[f"{tag}_real"] = np.bool_(s["real"])
        if key == "FAED":
            rec["faed"] = of.features(fsd, imgs, torch.float64)
            gold[f"{tag}_faed"] = rec["faed"][:rows].numpy()
        elif key.endswith("CS"):
            sc, _, _, _ = oc.clip_score_update(imgs, list(s["text"]), clip, token_rows)
            rec["scores"] = sc
            gold[f"{tag}_scores"] = sc[:rows].numpy()
            gold[f"{tag}_text"] = np.array(list(s["text"]))
        else:
            p, l = inception(imgs)
            rec["pool3" if key.endswith("FID") else "logits"] = p if key.endswith("FID") else l
            gold[f"{tag}_{'pool3' if key.endswith('FID') else 'logits'}"] = (p if key.endswith("FID") else l)[:rows].numpy()
        per_slot.append((key, c, rec))
    gold["slots"] = np.array(names)
    gold.update(resize_golden())
    for k, v in final_values(per_slot).items():
        gold[f"final_{k}"] = np.float64(v)
    for key in ("CS", "rot_CS", "mv_CS", "pers_CS"):  # before compute()'s clamp at 0
        gold[f"mean_{key}"] = np.float64(torch.cat([r["scores"] for k, _, r in per_slot if k == key]).double().mean())
    return gold


if __name__ == "__main__":
    g = mint()
    np.savez_compressed(GOLDEN, **g)
    print(GOLDEN, GOLDEN.stat().st_size, "bytes,", len(g["slots"]), "slots")
    for k in sorted(g):
        if k.startswith("final_"):
            print(k, float(g[k]))
