"""GPU: panfusion_b200.evaluate — pf_eval_crops against the composition it replaces and against the reference's crops,
pf_resize_area2_u8 against cv2, and EvalPanoGen end to end against tests/golden/eval_pano.npz (minted by
oracle/eval_pano.py from the reference's own test_step; the seeded networks are those of the inception, CLIP and FAED
goldens, regenerated here)."""
import hashlib
import json
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import clip_score as oc
from oracle import eval_pano as oe
from oracle import faed as of
from oracle import inception as oi
from panfusion_b200 import evaluate, geometry
from panfusion_b200.clip_score import CLIPEncoder
from panfusion_b200.inception import FrechetInceptionDistance, InceptionScore, InceptionV3

pytestmark = pytest.mark.gpu
GOLD = np.load(Path(__file__).parent / "golden" / "eval_pano.npz")
# uint8 crops of the driver against the reference's (kornia on the CPU, e2p grid in numpy): the fp32 bilinear weights
# round differently in a few pixels, which then truncate to the neighbouring level. Gate: about 2x the fraction
# measured on an H100 80GB HBM3 at 700 W (1.45e-5 over every crop of the golden).
CROP_DIFF_FRACTION = 3e-5


@pytest.fixture(scope="module")
def nets(cuda_device):
    return dict(inception=InceptionV3(oi.synth_state(), cuda_device), clip=CLIPEncoder(oc.seeded_state(), oc.clip_config()),
                faed=of.synth_state(), tokenizer=oe.tokenizer)


def _panos(P, H, W, seed):
    return oc.structured_images(seed, P, H, W)


def _cameras(n, seed):
    """n random cameras plus seam, pole and near-pole ones, fp32 degrees."""
    rng = np.random.RandomState(seed)
    cams = evaluate.draw_cameras(1, n, rng)
    return cams["crop"][0] + cams["seam"][0][:4] + [(0.0, 90.0), (45.0, -90.0), (180.0, 89.9), (-180.0, -89.5), (10.0, 0.0)]


def _composition(panos, angles, per, hw, normalize):
    """e2p (pf_e2p) of `pano.float() / 255` (the division on the CPU, as the reference's torch does it) then
    (v * 255).byte(), or of `pano.float()` then .to(torch.uint8)."""
    out = []
    for p in range(panos.shape[0]):
        a = angles[p * per:(p + 1) * per]
        x = panos[p:p + 1].float()
        x = (x / 255 if normalize else x).cuda().expand(len(a), -1, -1, -1).contiguous()
        v = geometry.e2p(x, 90, [t for t, _ in a], [q for _, q in a], hw)
        out.append((v * 255).byte() if normalize else v.to(torch.uint8))
    return torch.cat(out)


@pytest.mark.parametrize("hw", [(299, 299), (256, 256), (37, 53)])
@pytest.mark.parametrize("size", [(512, 1024), (97, 202)])
def test_crops_equal_the_composition(hw, size, cuda_device):
    P = 3
    panos = _panos(P, *size, 60 + size[0])
    per_cams = _cameras(22, 5)
    per = len(per_cams)
    angles = [(t + 7.0 * p, q) for p in range(P) for t, q in per_cams]
    recs = evaluate.camera_records(angles, *hw, cuda_device)
    d = panos.to(cuda_device)
    for normalize in (True, False):
        got = evaluate.eval_crops(d, recs, per, hw, normalize)
        ref = _composition(panos, angles, per, hw, normalize)
        assert got.shape == (P * per, 3, *hw) and got.dtype == torch.uint8
        assert torch.equal(got, ref), (normalize, (got.int() - ref.int()).abs().max().item())


def test_crops_against_the_reference(cuda_device):
    """The driver's crops of the golden's panoramas against the reference's, every crop of every FID slot (made again
    on the CPU by oracle/eval_pano.py and checked against the golden's digests): equal but for uint8 steps of 1 on a
    small fraction of pixels."""
    diff = total = same = n = 0
    for tag, pano, theta, phi, hw, normalize in oe.crop_slots(GOLD):
        ref = oe.reference_crops(pano, theta, phi, hw, normalize)
        assert [oe.digest(x) for x in ref] == [str(h) for h in GOLD[f"{tag}_digests"]], tag
        recs = evaluate.camera_records(list(zip(theta.tolist(), phi.tolist())), *hw, cuda_device)
        got = evaluate.eval_crops(pano.to(cuda_device), recs, len(theta), hw, normalize).cpu()
        d = (got.int() - ref.int()).abs()
        assert d.max().item() <= 1, tag
        diff += int((d > 0).sum())
        total += d.numel()
        same += sum(bool(torch.equal(x, y)) for x, y in zip(got, ref))
        n += len(ref)
    frac = diff / total
    print(f"crops vs reference: {frac:.2e} of the pixels differ by 1; {same}/{n} crops identical")
    assert frac <= CROP_DIFF_FRACTION


@pytest.mark.parametrize("i", range(len(oe.RESIZE_CASES)))
def test_resize_area2_equals_cv2(i, cuda_device):
    h, w = oe.RESIZE_CASES[i]
    x = torch.from_numpy(oe.resize_input(i)).to(cuda_device).permute(2, 0, 1)[None]
    got = evaluate.resize_area2(x, (h // 2, w // 2))[0].permute(1, 2, 0).contiguous().cpu().numpy()
    if i < oe.RESIZE_FULL:
        assert np.array_equal(got, GOLD[f"resize{i}"])
    else:
        assert hashlib.sha256(got.tobytes()).hexdigest() == str(GOLD[f"resize{i}_sha256"])
    assert torch.equal(evaluate.resize_area2(x, (h, w)), x)  # already the target size: unchanged
    with pytest.raises(NotImplementedError, match="factor-2"):
        evaluate.resize_area2(x[..., :h // 3 * 3, :w // 3 * 3], (h // 3, w // 3))


def _spied(ev):
    """Record every per-slot output the driver hands to its metrics, in call order: {key: [dict]}."""
    rec: dict[str, list] = {}
    for key, m in ev.eval_metrics.items():
        if key.endswith("FID"):
            def f(pool3, real, _m=m, _k=key, _orig=m.update_features):
                rec.setdefault(_k, []).append({"pool3": pool3.double().cpu(), "real": real})
                _orig(pool3, real)
            m.update_features = f
        elif key.endswith("IS"):
            def f(logits, _k=key, _orig=m.update_logits):
                rec.setdefault(_k, []).append({"logits": logits.double().cpu(), "real": None})
                _orig(logits)
            m.update_logits = f
        elif key.endswith("CS"):
            def f(images, text, _m=m, _k=key, _orig=m.update):
                _orig(images, text)
                rec.setdefault(_k, []).append({"scores": _m.last_scores.double().cpu(), "real": None})
            m.update = f
        else:
            enc = m.encoder
            feats = []

            def fwd(imgs, _orig=enc.forward, _f=feats):
                out = _orig(imgs)
                _f.append(out.double().cpu())
                return out
            enc.forward = fwd

            def f(imgs, real, _m=m, _orig=m.update, _f=feats):
                _orig(imgs, real)
                rec.setdefault("FAED", []).append({"faed": _f.pop(), "real": real})
            m.update = f
    return rec


def _run_golden(nets, dev):
    ev = evaluate.EvalPanoGen(int(GOLD["num_eval_crops"]), int(GOLD["pano_hw"][0]), device=dev, **nets)
    rec = _spied(ev)
    np.random.seed(int(GOLD["seed"]))
    for s in range(int(GOLD["steps"])):
        ev.test_step(oe.batch(s))
    return ev, rec


def _rel(got, ref):
    d = (got - ref).abs()
    scale = ref.abs().max().item()
    return d.max().item() / scale, d.mean().item() / scale


def test_end_to_end_against_the_golden(nets, cuda_device):
    ev, rec = _run_golden(nets, cuda_device)
    names = [str(t) for t in GOLD["slots"]]
    assert sorted(names) == sorted(f"{k}#{c}" for k, v in rec.items() for c in range(len(v)))
    worst = {}
    for tag in names:
        key, c = tag.split("#")
        mine = rec[key][int(c)]
        if f"{tag}_real" in GOLD:
            assert mine["real"] == GOLD[f"{tag}_real"].item(), tag
        for field in ("pool3", "logits", "scores", "faed"):
            if f"{tag}_{field}" in GOLD:
                ref = torch.from_numpy(GOLD[f"{tag}_{field}"]).double()
                assert mine[field].shape[0] == int(GOLD[f"{tag}_n"]), tag
                mine_rows = mine[field][:int(GOLD[f"{tag}_rows"])]  # the golden keeps step 0 whole, then first rows
                assert mine_rows.shape == ref.shape, tag
                if field == "scores":
                    e = ((mine_rows - ref).abs().max().item(), 0.0)
                else:
                    e = _rel(mine_rows, ref)
                w = worst.setdefault(field, [0.0, 0.0])
                w[0], w[1] = max(w[0], e[0]), max(w[1], e[1])
    print("per-slot max / mean error of max|ref| (scores: points):", {k: [f"{x:.2e}" for x in v] for k, v in worst.items()})
    # the gates of test_gpu_inception.py / test_gpu_clip_score.py, on crops that are themselves within a uint8 step of
    # the reference's
    assert worst["pool3"][0] <= 3e-3 and worst["pool3"][1] <= 5e-4
    assert worst["logits"][0] <= 3e-3 and worst["logits"][1] <= 1e-3
    assert worst["scores"][0] < 0.1
    assert worst["faed"][0] <= 3e-3

    torch.manual_seed(int(GOLD["is_seed"]))
    got = ev.compute()
    want = {k[len("final_"):]: float(GOLD[k]) for k in GOLD.files if k.startswith("final_")}
    assert set(got) == set(want)
    # the composition on its own: the fp64 oracle over the driver's own per-slot outputs
    own = oe.final_values([(k, c, s) for k, v in rec.items() for c, s in enumerate(v)])
    # FID and FAED relative to tr S1 + tr S2: with a few samples against d = 2048 features the statistics are rank
    # deficient, and each of the ~2000 null eigenvalues adds the square root of its rounding to the distance whatever
    # its size (test_gpu_inception.py gates the same quantity). Measured <= 8.1e-7 on an H100; IS and CS <= 5e-8
    comp = {}
    for k in got:
        if k.endswith("FID") or k == "FAED":
            f = "faed" if k == "FAED" else "pool3"
            st = [of.stats([s[f] for s in rec[k] if s["real"] == side]) for side in (True, False)]
            comp[k] = abs(got[k] - own[k]) / sum(float(of.covariances(*x)[1].trace()) for x in st)
        elif not k.endswith("_std"):
            comp[k] = abs(got[k] - own[k]) / max(abs(own[k]), 1e-30)
    print("compute() vs fp64 over the driver's own outputs (FID / FAED: of tr S1 + tr S2):",
          {k: f"{v:.1e}" for k, v in comp.items()})
    for k, v in comp.items():
        assert v <= 1e-6 or (own[k] == 0 and got[k] == 0), (k, got[k], own[k])
    for k in got:
        if k.endswith("_std"):
            assert abs(got[k] - own[k]) <= 1e-6 * max(own[k[:-4]], 1.0), k
    # CLIP scores of random towers are negative here, so compute() clamps them to 0: check the unclamped means too
    for k in ("CS", "rot_CS", "mv_CS", "pers_CS"):
        m = ev.eval_metrics[k]
        mean = float(m.score) / int(m.n_samples)
        ref = float(GOLD[f"mean_{k}"])
        assert abs(mean - ref) < 0.05, (k, mean, ref)
    rel = {k: abs(got[k] - want[k]) / max(abs(want[k]), 1.0) for k in got}
    print("compute() vs golden, relative (of max(|golden|, 1)):", {k: f"{v:.1e}" for k, v in rel.items()})
    # FID / FAED of a few samples against the fp64 reference features, IS over <= 16 logits: measured <= 1.3e-3 (FID)
    # on an H100 80GB HBM3 at 700 W, gated at about 2x
    for k, v in rel.items():
        assert v <= 3e-3, (k, got[k], want[k])


def test_sharing_one_forward_changes_no_number(nets, cuda_device):
    """compute() equals the standalone FrechetInceptionDistance / InceptionScore modules fed the same images, panorama
    by panorama."""
    K, B = 3, 2
    gt, gen = _panos(B, 512, 1024, 90), _panos(B, 512, 1024, 91)
    views = oc.structured_images(92, 8 * B, 256, 256).reshape(B, 8, 3, 256, 256)
    ev = evaluate.EvalPanoGen(K, 512, device=cuda_device, **nets)
    cams = ev.test_step(dict(pano=gt[:, None], pano_pred=gen[:, None], images_pred=views, pano_prompt=["a", "b"],
                             prompt=[[f"v{i}", f"w{i}"] for i in range(8)]), np.random.RandomState(4))
    assert ev.inception_forwards == B * (4 + 2 * (2 * K + 8) + 16)
    torch.manual_seed(5)
    got = ev.compute()
    net = nets["inception"]
    g, f = gt.to(cuda_device), gen.to(cuda_device)

    def crop(x, a, hw, norm):
        return evaluate.eval_crops(x, evaluate.camera_records(a, *hw, cuda_device), len(a), hw, norm)

    def sets(b):
        one = slice(b, b + 1)
        return {"": (g[one], f[one]), "rot_": (torch.roll(g[one], 512, 3), torch.roll(f[one], 512, 3)),
                "crop_": tuple(crop(x[one], cams["crop"][b], (299, 299), True) for x in (g, f)),
                "seam_": tuple(crop(x[one], cams["seam"][b], (299, 299), True) for x in (g, f)),
                "mv_": tuple(crop(x[one], cams["mv"], (299, 299), True) for x in (g, f)),
                "pers_": (crop(g[one], cams["mv"], (256, 256), False), views[b].to(cuda_device))}

    per_b = [sets(b) for b in range(B)]
    torch.manual_seed(5)
    for prefix in per_b[0]:
        fid = FrechetInceptionDistance(inception=net, device=cuda_device)
        iscore = InceptionScore(inception=net, device=cuda_device)
        for s in per_b:
            real, fake = s[prefix]
            fid.update(real, real=True)
            fid.update(fake, real=False)
            iscore.update(fake)
        for k, v in ((f"{prefix}FID", float(fid.compute())), (f"{prefix}IS", float(iscore.compute()[0]))):
            assert abs(got[k] - v) <= 1e-6 * abs(v), (k, got[k], v)


def test_batch_equals_single_steps(nets, cuda_device):
    panos = [(_panos(1, 128, 256, 70 + i), _panos(1, 128, 256, 80 + i)) for i in range(2)]
    views = [oc.structured_images(75 + i, 8, 32, 32) for i in range(2)]

    def batch(idx):
        return dict(pano=torch.cat([panos[i][0] for i in idx])[:, None],
                    pano_pred=torch.cat([panos[i][1] for i in idx])[:, None],
                    images_pred=torch.stack([views[i] for i in idx]), pano_prompt=[f"room {i}" for i in idx],
                    prompt=[[f"view {v} of {i}" for i in idx] for v in range(8)])

    out = []
    for steps in ([[0, 1]], [[0], [1]]):
        ev = evaluate.EvalPanoGen(2, 128, device=cuda_device, **nets)
        rng = np.random.RandomState(11)
        for idx in steps:
            ev.test_step(batch(idx), rng)
        torch.manual_seed(3)
        out.append(ev.compute())
    assert out[0] == out[1]


def _png(path, arr):
    from PIL import Image
    path.parent.mkdir(parents=True, exist_ok=True)
    Image.fromarray(arr).save(path)


def test_command_line(nets, tmp_path, cuda_device):
    """A seeded results directory (one PanFusion result, one MVDiffusion result without pano.png) and data directory."""
    data, results = tmp_path / "data", tmp_path / "results"
    hwc = lambda x: np.ascontiguousarray(x.permute(1, 2, 0).numpy())  # noqa: E731
    for k, (scene, view) in enumerate((("sceneA", "v0"), ("sceneB", "v1"))):
        _png(data / scene / "matterport_stitched_images" / f"{view}.png", hwc(_panos(1, 256, 512, 40 + k)[0]))
        for i in range(8):
            (data / scene / "blip3").mkdir(parents=True, exist_ok=True)
            (data / scene / "blip3" / f"{view}_{i * 45}.txt").write_text(f"view {i} of {scene}\n")
        r = results / f"{scene}_{view}"
        if k == 0:
            _png(r / "pano.png", hwc(_panos(1, 128, 256, 50)[0]))
        for i, v in enumerate(oc.structured_images(60 + k, 8, 32, 32)):
            _png(r / f"{i}.png", hwc(v))
        (r / "prompt.txt").write_text(f"a room in {scene}\nsecond line\n")
    out = tmp_path / "metrics.json"
    argv = ["--results", str(results), "--data", str(data), "--pano-height", "128", "--pers-resolution", "32",
            "--num-eval-crops", "2", "--seed", "3", "--out", str(out), "--device", str(cuda_device)]
    metrics = evaluate.main(argv, **nets)
    written = json.loads(out.read_text())
    assert written == metrics
    keys = {"FID", "IS", "IS_std", "CS", "rot_FID", "rot_IS", "rot_IS_std", "rot_CS", "crop_FID", "crop_IS",
            "crop_IS_std", "seam_FID", "seam_IS", "seam_IS_std", "mv_FID", "mv_IS", "mv_IS_std", "mv_CS", "pers_FID",
            "pers_IS", "pers_IS_std", "pers_CS", "FAED"}
    assert set(written) == keys
    assert all(np.isfinite(v) for k, v in written.items() if not k.endswith("_std"))
    _png(results / "sceneA_v0" / "3.png", np.zeros((40, 40, 3), np.uint8))
    with pytest.raises(ValueError, match="pers-resolution"):
        evaluate.main(argv, **nets)
