"""FID / Inception Score oracle: torch-fidelity's FeatureExtractorInceptionV3 (the network of torchmetrics'
NoTrainInceptionV3), its TF1-style resize, and torchmetrics' FrechetInceptionDistance update / compute and
InceptionScore compute, restated from memory [3P-mem] (neither package is installed here).

The network is torchvision's `Inception3(aux_logits=False)` built from torchvision's own `BasicConv2d` and `Inception*`
classes, with the four FID deviations overriding `forward`: Mixed_5b..5d, 6b..6e and 7b average-pool with
count_include_pad=False, Mixed_7c max-pools its pool branch, and the head is fc 2048 -> 1008 read without its bias
(`logits_unbiased = pool3 @ fc.weight^T`). `fid=False` keeps torchvision's blocks, which pins the graph, the key names
and the BN eps against executable code.

`python -m oracle.inception` mints tests/golden/inception.npz from seeded weights (the seed and a SHA-256 of the weight
bytes are stored, not the weights) and seeded structured images.
"""
from __future__ import annotations

import math
import sys
from pathlib import Path

import numpy as np
import torch
import torch.nn.functional as F
from torchvision.models import inception as tvi

from oracle import faed as of

GOLDEN = Path(__file__).resolve().parent.parent / "tests" / "golden" / "inception.npz"
SEED = 2015
SIZE = 299
# fc rows have norm ~FC_GAIN and are orthogonal to the (fp16-rounded) pool3 of a mid-gray image: a seeded deep ReLU
# network answers every image mostly along that one direction, and without this every image gets the same class and
# IS is ~1. With it softmax is neither one-hot nor uniform and IS is well above 1 (asserted from the golden).
FC_GAIN = 12.0


# ---- network ------------------------------------------------------------------------------------------------------

class FIDInceptionA(tvi.InceptionA):
    def forward(self, x):
        b1 = self.branch1x1(x)
        b5 = self.branch5x5_2(self.branch5x5_1(x))
        b3 = self.branch3x3dbl_3(self.branch3x3dbl_2(self.branch3x3dbl_1(x)))
        bp = self.branch_pool(F.avg_pool2d(x, 3, stride=1, padding=1, count_include_pad=False))
        return torch.cat([b1, b5, b3, bp], 1)


class FIDInceptionC(tvi.InceptionC):
    def forward(self, x):
        b1 = self.branch1x1(x)
        b7 = self.branch7x7_3(self.branch7x7_2(self.branch7x7_1(x)))
        bd = self.branch7x7dbl_1(x)
        for m in (self.branch7x7dbl_2, self.branch7x7dbl_3, self.branch7x7dbl_4, self.branch7x7dbl_5):
            bd = m(bd)
        bp = self.branch_pool(F.avg_pool2d(x, 3, stride=1, padding=1, count_include_pad=False))
        return torch.cat([b1, b7, bd, bp], 1)


class FIDInceptionE1(tvi.InceptionE):
    """Mixed_7b: average pool without the padded zeros."""
    max_pool = False

    def forward(self, x):
        b1 = self.branch1x1(x)
        t = self.branch3x3_1(x)
        b3 = torch.cat([self.branch3x3_2a(t), self.branch3x3_2b(t)], 1)
        d = self.branch3x3dbl_2(self.branch3x3dbl_1(x))
        bd = torch.cat([self.branch3x3dbl_3a(d), self.branch3x3dbl_3b(d)], 1)
        if self.max_pool:
            p = F.max_pool2d(x, 3, stride=1, padding=1)
        else:
            p = F.avg_pool2d(x, 3, stride=1, padding=1, count_include_pad=False)
        return torch.cat([b1, b3, bd, self.branch_pool(p)], 1)


class FIDInceptionE2(FIDInceptionE1):
    """Mixed_7c: max pool."""
    max_pool = True


def network(fid: bool = True, num_classes: int = 1008) -> torch.nn.Module:
    blocks = [tvi.BasicConv2d, tvi.InceptionA, tvi.InceptionB, tvi.InceptionC, tvi.InceptionD, tvi.InceptionE,
              tvi.InceptionAux]
    if fid:
        blocks[1], blocks[3], blocks[5] = FIDInceptionA, FIDInceptionC, FIDInceptionE1
    net = tvi.Inception3(num_classes=num_classes, aux_logits=False, transform_input=False, inception_blocks=blocks,
                         init_weights=False)
    if fid:
        net.Mixed_7c = FIDInceptionE2(2048)
    return net.eval()


def synth_state(seed: int = SEED) -> dict[str, torch.Tensor]:
    """Seeded weights under torch-fidelity's names: conv std sqrt(2 / fan_in), BN gamma / beta / running stats drawn
    away from the identity, fc std FC_GAIN / sqrt(2048) projected off the mid-gray response (see FC_GAIN)."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for k, v in network().state_dict().items():
        if k.endswith("num_batches_tracked"):
            sd[k] = torch.tensor(0)
        elif k.endswith("conv.weight"):
            sd[k] = torch.randn(v.shape, generator=g) * math.sqrt(2.0 / v[0].numel())
        elif k.endswith("bn.weight"):
            sd[k] = 0.8 + 0.4 * torch.rand(v.shape, generator=g)
        elif k.endswith("bn.bias"):
            sd[k] = 0.1 * torch.randn(v.shape, generator=g)
        elif k.endswith("running_mean"):
            sd[k] = 0.1 * torch.randn(v.shape, generator=g)
        elif k.endswith("running_var"):
            sd[k] = 0.5 + torch.rand(v.shape, generator=g)
        elif k == "fc.weight":
            sd[k] = torch.randn(v.shape, generator=g, dtype=torch.float64) * (FC_GAIN / math.sqrt(v.shape[1]))
        elif k == "fc.bias":
            sd[k] = 0.1 * torch.randn(v.shape, generator=g)
        else:
            raise KeyError(k)
    net = network().double()
    net.load_state_dict(sd)
    gray, _ = features(net, torch.full((1, 3, SIZE, SIZE), 128, dtype=torch.uint8), torch.float64)
    u = gray[0].half().double()  # rounded, so thread-count-dependent last bits of the forward cannot change it
    w = sd["fc.weight"]
    sd["fc.weight"] = (w - torch.outer(w @ u, u) / (u @ u)).float()
    return sd


def state_sha256(sd: dict[str, torch.Tensor]) -> str:
    return of.state_sha256(sd)


# ---- prep ---------------------------------------------------------------------------------------------------------

def resize_tf1(x: torch.Tensor, size: tuple[int, int]) -> torch.Tensor:
    """torch-fidelity's interpolate_bilinear_2d_like_tensorflow1x(align_corners=False, method='slow') on fp32 NCHW."""
    def axis(n_in, n_out):
        scale = torch.tensor(n_in / n_out, dtype=torch.float32)
        g = torch.arange(n_out, dtype=torch.float32) * scale
        lo = g.long()
        hi = (lo + 1).clamp(max=n_in - 1)
        return lo, hi, g - lo

    y0, y1, dy = axis(x.shape[2], size[0])
    x0, x1, dx = axis(x.shape[3], size[1])
    dx, dy = dx.view(1, 1, 1, -1), dy.view(1, 1, -1, 1)
    a00, a01 = x[:, :, y0][..., x0], x[:, :, y0][..., x1]
    a10, a11 = x[:, :, y1][..., x0], x[:, :, y1][..., x1]
    r0 = a00 + (a01 - a00) * dx
    r1 = a10 + (a11 - a10) * dx
    return r0 + (r1 - r0) * dy


def prep(imgs: torch.Tensor) -> torch.Tensor:
    """FeatureExtractorInceptionV3.forward's input: uint8 [B, 3, H, W] -> fp32 [B, 3, 299, 299] in about [-1, 1]."""
    assert imgs.dtype == torch.uint8 and imgs.dim() == 4 and imgs.shape[1] == 3
    x = resize_tf1(imgs.float(), (SIZE, SIZE))
    return (x - 128) / 128


@torch.no_grad()
def features(net: torch.nn.Module, imgs: torch.Tensor, dtype=torch.float32) -> tuple[torch.Tensor, torch.Tensor]:
    """(pool3 [B, 2048], logits_unbiased [B, 1008]) in `dtype` (net must hold `dtype` weights)."""
    x = prep(imgs).to(dtype)
    for name in ("Conv2d_1a_3x3", "Conv2d_2a_3x3", "Conv2d_2b_3x3", "maxpool1", "Conv2d_3b_1x1", "Conv2d_4a_3x3",
                 "maxpool2", "Mixed_5b", "Mixed_5c", "Mixed_5d", "Mixed_6a", "Mixed_6b", "Mixed_6c", "Mixed_6d",
                 "Mixed_6e", "Mixed_7a", "Mixed_7b", "Mixed_7c"):
        x = getattr(net, name)(x)
    pool3 = x.mean(dim=(2, 3))
    return pool3, pool3 @ net.fc.weight.t()


# ---- torchmetrics -------------------------------------------------------------------------------------------------

def fid_stats(feature_batches):
    """FrechetInceptionDistance.update on each batch: fp64 (sum, cov_sum, n)."""
    return of.stats(feature_batches)


def fid(s1, c1, n1, s2, c2, n2) -> float:
    """FrechetInceptionDistance.compute: the same _compute_fid over the same statistics as FAED."""
    return of.faed(s1, c1, n1, s2, c2, n2)


def chunk_count(n: int, splits: int) -> int:
    return len(torch.arange(n).chunk(splits))


def inception_score(logits: torch.Tensor, splits: int, seed: int) -> tuple[float, float]:
    """InceptionScore.compute with torch.manual_seed(seed) drawn just before it (its randperm)."""
    torch.manual_seed(seed)
    idx = torch.randperm(logits.shape[0])
    f = logits[idx]
    prob, log_prob = f.softmax(dim=1), f.log_softmax(dim=1)
    kl = []
    for p, lp in zip(prob.chunk(splits, dim=0), log_prob.chunk(splits, dim=0)):
        m = p.mean(dim=0, keepdim=True)
        kl.append((p * (lp - m.log())).sum(dim=1).mean().exp())
    kl = torch.stack(kl)
    return float(kl.mean()), float(kl.std())


# ---- seeded structured images -------------------------------------------------------------------------------------

def images(n: int, hw: tuple[int, int], kind: str, seed: int) -> torch.Tensor:
    """uint8 [n, 3, H, W]: a smooth seeded field plus noise. 'real' has strong structure and little noise, 'fake'
    weaker, warmer structure and more noise."""
    g = torch.Generator().manual_seed(seed)
    h, w = hw
    coarse = torch.randn(n, 3, 6, 10, generator=g)
    smooth = F.interpolate(coarse, size=(h, w), mode="bicubic", align_corners=False)
    noise = torch.randn(n, 3, h, w, generator=g)
    if kind == "real":
        x = 128 + 55 * smooth + 8 * noise
    else:
        x = 140 + 30 * smooth + 30 * noise + torch.tensor([12.0, 0.0, -12.0]).view(1, 3, 1, 1)
    return x.round().clamp(0, 255).to(torch.uint8)


FEATURE_SIZES = [(299, 299), (512, 1024), (512, 512)]  # 8 'real' images each, seed 10 + index
RANK_DEFICIENT = dict(hw=(512, 1024), batches=(12, 8))  # per side: n = 20 < d = 2048; real seeds 20.., fake 30..
FULL_RANK = dict(hw=(299, 299), batches=(700, 700, 700))  # per side: n = 2100 > d = 2048; real seeds 40.., fake 50..
IS_CASES = [(40, 10, 7), (25, 10, 8)]  # (n, splits, torch.manual_seed): the first n logits of the rank-deficient set


def feature_images(i: int) -> torch.Tensor:
    return images(8, FEATURE_SIZES[i], "real", 10 + i)


def set_images(case: dict, side: str) -> list[torch.Tensor]:
    base = {id(RANK_DEFICIENT): 20, id(FULL_RANK): 40}[id(case)] + (0 if side == "real" else 10)
    return [images(b, case["hw"], side, base + j) for j, b in enumerate(case["batches"])]


def is_logits_images() -> torch.Tensor:
    """The 40 images whose logits the IS cases use: the rank-deficient set's real then fake images."""
    return torch.cat(set_images(RANK_DEFICIENT, "real") + set_images(RANK_DEFICIENT, "fake"))


# ---- minting ------------------------------------------------------------------------------------------------------

def _net(sd, dtype):
    net = network()
    net.load_state_dict(sd)
    return net.to(dtype)


def _fid_set(net, case, dtype, chunk):
    gold = {}
    st = []
    for side in ("real", "fake"):
        feats = []
        for x in set_images(case, side):
            feats.append(torch.cat([features(net, x[i:i + chunk], dtype)[0] for i in range(0, x.shape[0], chunk)]))
        s, c, n = fid_stats(feats)
        gold[f"{side}_sum"] = s.numpy()
        gold[f"{side}_cov_sum_diag"] = torch.diagonal(c).numpy()
        gold[f"{side}_cov_sum_fro"] = np.float64(c.norm())
        gold[f"{side}_num_samples"] = np.int64(n)
        st.append((s, c, n))
    gold["fid"] = np.float64(fid(*st[0], *st[1]))
    return gold, feats


def mint(full_rank: bool = True) -> dict:
    torch.set_num_threads(8)
    sd = synth_state()
    gold = {"seed": np.int64(SEED), "weights_sha256": np.array(state_sha256(sd)), "fc_gain": np.float64(FC_GAIN)}
    net64 = _net(sd, torch.float64)
    for i, (h, w) in enumerate(FEATURE_SIZES):
        p, l = features(net64, feature_images(i), torch.float64)
        gold[f"pool3_{h}x{w}"], gold[f"logits_{h}x{w}"] = p.float().numpy(), l.float().numpy()
    rd, _ = _fid_set(net64, RANK_DEFICIENT, torch.float64, 4)
    gold.update({f"rd_{k}": v for k, v in rd.items()})
    logits = torch.cat([features(net64, x[i:i + 4], torch.float64)[1] for x in [is_logits_images()]
                        for i in range(0, 40, 4)])
    for n, splits, seed in IS_CASES:
        m, s = inception_score(logits[:n], splits, seed)
        gold[f"is_{n}_mean"], gold[f"is_{n}_std"] = np.float64(m), np.float64(s)
    # non-degeneracy of the seeded network on these images
    p = torch.from_numpy(gold["pool3_299x299"]).double()
    gold["pool3_zero_fraction"] = np.float64((p == 0).double().mean())
    prob = logits.softmax(dim=1)
    gold["softmax_max_mean"] = np.float64(prob.max(dim=1).values.mean())
    if full_rank:
        net32 = _net(sd, torch.float32)
        fr, _ = _fid_set(net32, FULL_RANK, torch.float32, 50)
        gold.update({f"fr_{k}": v for k, v in fr.items()})
    return gold


if __name__ == "__main__":
    gold = mint(full_rank="--no-full-rank" not in sys.argv)
    np.savez_compressed(GOLDEN, **gold)
    print(GOLDEN, GOLDEN.stat().st_size, "bytes")
    for k in sorted(gold):
        if np.asarray(gold[k]).size == 1:
            print(k, gold[k])
