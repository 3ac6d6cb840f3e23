"""FAED oracle: a torch restatement of the FAED encoder (models/faed/modules.py:5-36,176-264), its features
(models/faed/FAED.py:69-78), statistics (FAED.py:80-90) and distance (FAED.py:92-103 + torchmetrics' _compute_fid), and
`python -m oracle.faed`, which mints tests/golden/faed.npz by executing the reference's own modules.py and FAED.py by
path through oracle/ref_loader.py (build container only; torchmetrics, lightning and wandb resolve to oracle/shims).

The golden holds the weight seed and a SHA-256 of the weight bytes (not the weights), per-image features at 64x128,
128x256 and 512x1024, the features and fp64 statistics of a real and a fake set (two update calls each) for a
rank-deficient case (128x256, n = 6 < d = 512) and a full-rank case (32x64, n = 136 > d = 128), and the reference's
FAED of both. The full-rank case runs at 32x64 so that its features fit in the file. At H <= 64 (H/32 <= 2) the
latitude weight is cos(fp32 +-pi/2) = -4.4e-8 on every row, which scales the features but not the relative error of
the distance. A second full-rank case at 128x256 (n = 520 > d = 512, latitude weights 0, 0.87, 0.87, 0) stores the
statistics' sums, diagonals and Frobenius norms and the FAED, not the features (they would not fit).
"""
from __future__ import annotations

import hashlib
import importlib
import math
from pathlib import Path

import numpy as np
import torch
import torch.nn.functional as F

from oracle.shims.torchmetrics.image.fid import _compute_fid as compute_fid  # [3P-mem], restated once

GOLDEN = Path(__file__).resolve().parent.parent / "tests" / "golden" / "faed.npz"
SEED = 20240
BN_EPS = 1e-5

# (prefix, Cin, Cout, k) of every modules.Conv2d in Encoder, with its BatchNorm (None for downconv1 and fuse)
_RES = [("downres1_rgb", 32, 9), ("downres2_rgb", 64, 7), ("downres3_rgb", 128, 5), ("downres4_rgb", 128, 3),
        ("downres5_rgb", 128, 3)]
_DOWN = [("downconv2_rgb", 32, 64), ("downconv3_rgb", 64, 128), ("downconv4_rgb", 128, 128),
         ("downconv5_rgb", 128, 128), ("downconv6_rgb", 128, 128)]


def conv_specs():
    specs = [("downconv1_rgb", 3, 32, 9, None), ("fuse", 128, 128, 3, None)]
    for name, c, k in _RES:
        specs += [(f"{name}.conv1", c, c, k, f"{name}.batchnorm1"), (f"{name}.conv2", c, c, k, f"{name}.batchnorm2")]
    for name, ci, co in _DOWN:
        specs.append((f"{name}.conv1", ci, co, 4, f"{name}.batchnorm1"))
    return specs


def synth_state(seed: int = SEED) -> dict[str, torch.Tensor]:
    """Seeded encoder weights with the reference's state-dict names. BN running mean / var, gamma and beta are drawn
    away from the identity."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for conv, ci, co, k, bn in conv_specs():
        sd[f"{conv}.conv2d.weight"] = torch.randn(co, ci, k, k, generator=g) * math.sqrt(1.0 / (ci * k * k))
        sd[f"{conv}.conv2d.bias"] = 0.05 * torch.randn(co, generator=g)
        if bn is not None:
            sd[f"{bn}.weight"] = 0.8 + 0.4 * torch.rand(co, generator=g)
            sd[f"{bn}.bias"] = 0.1 * torch.randn(co, generator=g)
            sd[f"{bn}.running_mean"] = 0.1 * torch.randn(co, generator=g)
            sd[f"{bn}.running_var"] = 0.5 + torch.rand(co, generator=g)
            sd[f"{bn}.num_batches_tracked"] = torch.tensor(0)
    return sd


def state_sha256(sd: dict[str, torch.Tensor]) -> str:
    h = hashlib.sha256()
    for k in sorted(sd):
        h.update(k.encode())
        h.update(sd[k].contiguous().numpy().tobytes())
    return h.hexdigest()


def images(shape, dist: str, seed: int) -> torch.Tensor:
    """Seeded uint8 panoramas [B, 3, H, W]: 'real' uniform over 0..255, 'fake' a clamped Gaussian around 128."""
    g = torch.Generator().manual_seed(seed)
    if dist == "real":
        return torch.randint(0, 256, shape, generator=g, dtype=torch.uint8)
    return (128 + 40 * torch.randn(shape, generator=g)).round().clamp(0, 255).to(torch.uint8)


# ---- restatement ------------------------------------------------------------------------------------------------

def circular_pad(x: torch.Tensor, p: int) -> torch.Tensor:
    """Rows zero-padded by p, columns wrapped by p, corners zero (modules.py:5-19)."""
    if p == 0:
        return x
    x = F.pad(x, (0, 0, p, p))
    return torch.cat([x[..., -p:], x, x[..., :p]], dim=-1)


def _conv(sd, name, x, stride, pad, bn=None, dtype=torch.float32):
    y = F.conv2d(circular_pad(x, pad), sd[f"{name}.conv2d.weight"].to(dtype), sd[f"{name}.conv2d.bias"].to(dtype),
                 stride=stride)
    if bn is not None:
        y = F.batch_norm(y, sd[f"{bn}.running_mean"].to(dtype), sd[f"{bn}.running_var"].to(dtype),
                         sd[f"{bn}.weight"].to(dtype), sd[f"{bn}.bias"].to(dtype), False, 0.0, BN_EPS)
    return y


def encoder(sd, x: torch.Tensor) -> torch.Tensor:
    """Encoder.forward (modules.py:248-264) in x's dtype, eval-mode BatchNorm."""
    dt = x.dtype
    x = _conv(sd, "downconv1_rgb", x[:, :3], 1, 4, dtype=dt)
    for (r, _, k), (d, _, _) in zip(_RES, _DOWN):
        y = F.relu(_conv(sd, f"{r}.conv1", x, 1, k // 2, f"{r}.batchnorm1", dt))
        x = _conv(sd, f"{r}.conv2", y, 1, k // 2, f"{r}.batchnorm2", dt) + x
        x = F.relu(_conv(sd, f"{d}.conv1", x, 2, 1, f"{d}.batchnorm1", dt))
    return _conv(sd, "fuse", x, 1, 1, dtype=dt)


def features(sd, imgs: torch.Tensor, dtype=torch.float32) -> torch.Tensor:
    """FAED.get_activation (FAED.py:69-78)."""
    x = imgs.to(torch.float32) / 127.5 - 1
    f = encoder(sd, x.to(dtype)).to(torch.float32)
    m = f.mean(dim=3)
    w = torch.cos(torch.linspace(math.pi / 2, -math.pi / 2, m.shape[-1]))
    return (w * m).reshape(m.shape[0], -1)


def stats(feature_batches) -> tuple[torch.Tensor, torch.Tensor, int]:
    """fp64 (sum, cov_sum, n) after one update per batch (FAED.py:80-90)."""
    d = feature_batches[0].shape[1]
    s, c, n = torch.zeros(d, dtype=torch.float64), torch.zeros(d, d, dtype=torch.float64), 0
    for f in feature_batches:
        f = torch.as_tensor(f).double()
        s += f.sum(dim=0)
        c += f.t().mm(f)
        n += f.shape[0]
    return s, c, n


def covariances(s, c, n):
    mu = (s / n).unsqueeze(0)
    return mu.squeeze(0), (c - n * mu.t().mm(mu)) / (n - 1)


def faed(s1, c1, n1, s2, c2, n2) -> float:
    """FrechetAutoEncoderDistance.compute (FAED.py:92-103)."""
    mu1, S1 = covariances(s1, c1, n1)
    mu2, S2 = covariances(s2, c2, n2)
    return float(compute_fid(mu1, S1, mu2, S2))


def faed_eigh(s1, c1, n1, s2, c2, n2) -> float:
    """The same distance through symmetric eigensolvers: tr sqrt(S1^1/2 S2 S1^1/2), eigenvalues clamped at 0."""
    mu1, S1 = covariances(s1, c1, n1)
    mu2, S2 = covariances(s2, c2, n2)
    lam, U = torch.linalg.eigh(S1)
    R = U * lam.clamp_min(0).sqrt() @ U.t()
    e = torch.linalg.eigvalsh(R @ S2 @ R).clamp_min(0).sqrt().sum()
    return float((mu1 - mu2).square().sum() + S1.trace() + S2.trace() - 2 * e)


# ---- cases shared by the golden and the tests ---------------------------------------------------------------------

FEATURE_SIZES = [(64, 128), (128, 256), (512, 1024)]  # two images each, 'real' distribution, seed 100 + index
RANK_DEFICIENT = dict(hw=(128, 256), batches=(3, 3))   # per side; real seeds 200.., fake seeds 300..
FULL_RANK = dict(hw=(32, 64), batches=(68, 68))
FULL_RANK_LAT = dict(hw=(128, 256), batches=(130, 130, 130, 130))  # statistics only in the golden


def feature_images(i: int) -> torch.Tensor:
    return images((2, 3, *FEATURE_SIZES[i]), "real", 100 + i)


def set_images(case: dict, side: str) -> list[torch.Tensor]:
    base = (200 if side == "real" else 300) + {"rd": 0, "fr": 50, "frl": 70}[case_tag(case)]
    return [images((b, 3, *case["hw"]), side, base + j) for j, b in enumerate(case["batches"])]


def case_tag(case: dict) -> str:
    return {id(RANK_DEFICIENT): "rd", id(FULL_RANK): "fr", id(FULL_RANK_LAT): "frl"}[id(case)]


def images_sha256(imgs: list[torch.Tensor]) -> str:
    h = hashlib.sha256()
    for x in imgs:
        h.update(x.numpy().tobytes())
    return h.hexdigest()


# ---- minting ------------------------------------------------------------------------------------------------------

def _load_reference():
    """The reference's models/faed/modules.py and FAED.py, loaded through oracle/ref_loader.py's package stubs and
    sys.path (models/faed has no __init__.py, so it resolves under the `models` stub)."""
    from oracle import ref_loader
    ref_loader.load()
    return importlib.import_module("models.faed.modules"), importlib.import_module("models.faed.FAED")


def mint() -> dict:
    mods, fa = _load_reference()
    sd = synth_state()
    enc = mods.Encoder()
    enc.load_state_dict(sd)
    enc.eval()
    gold = {"seed": np.int64(SEED), "weights_sha256": np.array(state_sha256(sd))}
    with torch.no_grad():
        for i, (h, w) in enumerate(FEATURE_SIZES):
            m = fa.FrechetAutoEncoderDistance(h)
            m.encoder = enc
            gold[f"features_{h}"] = m.get_activation(feature_images(i)).numpy()
        for tag, case in (("rd", RANK_DEFICIENT), ("fr", FULL_RANK), ("frl", FULL_RANK_LAT)):
            m = fa.FrechetAutoEncoderDistance(case["hw"][0])
            m.encoder = enc
            for side in ("real", "fake"):
                imgs = set_images(case, side)
                gold[f"{tag}_{side}_images_sha256"] = np.array(images_sha256(imgs))
                feats = []
                for x in imgs:
                    if tag != "frl":
                        feats.append(m.get_activation(x))
                    m.update(x, real=side == "real")
                if tag != "frl":
                    gold[f"{tag}_{side}_features"] = torch.cat(feats).numpy()
                gold[f"{tag}_{side}_sum"] = getattr(m, f"{side}_features_sum").numpy()
                c = getattr(m, f"{side}_features_cov_sum")
                gold[f"{tag}_{side}_cov_sum_diag"] = torch.diagonal(c).numpy()
                gold[f"{tag}_{side}_cov_sum_fro"] = np.float64(c.norm())
                gold[f"{tag}_{side}_num_samples"] = np.int64(getattr(m, f"{side}_features_num_samples"))
            gold[f"{tag}_faed"] = np.float64(m.compute())
            st = [(getattr(m, f"{side}_features_sum"), getattr(m, f"{side}_features_cov_sum"),
                   int(getattr(m, f"{side}_features_num_samples"))) for side in ("real", "fake")]
            gold[f"{tag}_faed_eigh"] = np.float64(faed_eigh(*st[0], *st[1]))
    return gold


if __name__ == "__main__":
    gold = mint()
    np.savez_compressed(GOLDEN, **gold)
    print(GOLDEN, GOLDEN.stat().st_size, "bytes")
    for k in ("rd", "fr", "frl"):
        print(k, "faed", float(gold[f"{k}_faed"]), "eigh", float(gold[f"{k}_faed_eigh"]))
