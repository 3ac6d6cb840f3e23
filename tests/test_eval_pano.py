"""CPU: the host side of panfusion_b200.evaluate (camera draws, camera records, slot bookkeeping) against
tests/golden/eval_pano.npz, minted by oracle/eval_pano.py from the reference's own EvalPanoGen.test_step; and the
argument checks of pf_eval_crops / pf_resize_area2_u8, which run before any CUDA call."""
import ctypes as C
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import eval_pano as oe
from panfusion_b200 import _lib, evaluate

GOLD = np.load(Path(__file__).parent / "golden" / "eval_pano.npz")


def test_golden_inputs_regenerate():
    """The seeded batches the golden was minted from are regenerated bit for bit here."""
    for s in range(int(GOLD["steps"])):
        b = oe.batch(s)
        got = oe.digest(torch.cat([b[k].reshape(-1) for k in ("pano", "pano_pred", "images_pred")]))
        assert got == str(GOLD["batches_sha256"][s])


def test_reference_crops_regenerate():
    """oracle/eval_pano.py's CPU crops equal the reference's own, crop for crop (the golden's digests), so the GPU test
    can compare the driver's crops with every one of them."""
    n = 0
    for tag, pano, theta, phi, hw, normalize in oe.crop_slots(GOLD):
        ref = oe.reference_crops(pano, theta, phi, hw, normalize)
        assert [oe.digest(x) for x in ref] == [str(h) for h in GOLD[f"{tag}_digests"]], tag
        n += len(ref)
    assert n == 2 * (2 * 2 + 2 * 2 + 2 * 8 + 8)


def test_cameras_match_the_reference_draws():
    """After np.random.seed, two steps draw exactly the reference's cameras: per step crop then seam, the fp32 degrees
    e2p receives, seam theta 180, the 8 horizon cameras."""
    K = int(GOLD["num_eval_crops"])
    np.random.seed(int(GOLD["seed"]))
    for s in range(int(GOLD["steps"])):
        cams = evaluate.draw_cameras(1, K, np.random)
        for j, name in enumerate(("crop", "seam")):
            ref = GOLD[f"draw{2 * s + j}_deg32"]
            got = np.array(cams[name][0], dtype=np.float64).T
            want = ref.astype(np.float64)
            if name == "seam":
                want[0] = 180.0
            assert np.array_equal(got, want), (s, name)
        assert np.array_equal(np.array(cams["mv"]).T[0], np.arange(8) * 45.0)
        assert not np.array(cams["mv"]).T[1].any()


def test_cameras_per_panorama_equal_batch_of_one():
    a = np.random.RandomState(3)
    b = np.random.RandomState(3)
    batched = evaluate.draw_cameras(3, 4, a)
    single = [evaluate.draw_cameras(1, 4, b) for _ in range(3)]
    for k in ("crop", "seam"):
        assert batched[k] == [s[k][0] for s in single]


def test_camera_records_match_oracle_rotations():
    from oracle import geometry as og
    np.random.seed(int(GOLD["seed"]))
    cams = evaluate.draw_cameras(1, int(GOLD["num_eval_crops"]), np.random)
    angles = cams["crop"][0] + cams["seam"][0] + cams["mv"]
    rec = evaluate.camera_records(angles, 299, 299, "cpu").numpy()
    assert rec.shape == (len(angles), _lib.PF_CAM_DOUBLES)
    for r, (t, p) in zip(rec, angles):
        R1, R2 = og.camera_rotations(t, p)
        np.testing.assert_allclose(r[:9].reshape(3, 3), R1, atol=1e-15)
        np.testing.assert_allclose(r[9:18].reshape(3, 3), R2, atol=1e-15)
        assert r[18] == r[19] == np.tan(np.radians(45.0))


def test_slot_counts_match_the_reference_calls():
    """Images per metric and side after the golden's two steps equal what the reference's test_step passed."""
    seen: dict[str, list] = {}
    for tag in GOLD["slots"]:
        key = str(tag).split("#")[0]
        real = GOLD[f"{tag}_real"].item() if f"{tag}_real" in GOLD else None
        seen.setdefault(key, [0, 0])[0 if real in (True, None) else 1] += int(GOLD[f"{tag}_n"])
    want = evaluate.slot_counts(1, int(GOLD["num_eval_crops"]), 8, True)
    assert set(seen) == set(want)
    for key, n in want.items():
        n = tuple(2 * v for v in n) if isinstance(n, tuple) else (2 * n, 0)
        assert tuple(seen[key]) == n, key
    # without views or prompts the reference skips pers_ and the per-view CLIP scores
    assert set(evaluate.slot_counts(1, 20, None, False)) == set(want) - {"mv_CS", "pers_FID", "pers_IS", "pers_CS"}
    assert "pers_FID" not in evaluate.slot_counts(1, 20, 4, True) and "pers_CS" in evaluate.slot_counts(1, 20, 4, True)


def test_inception_forwards_per_panorama():
    """One forward per distinct image: 116 per panorama at 20 crops and 8 views, against the reference's 174 (each
    generated set once for FID and once for IS)."""
    c = evaluate.slot_counts(1, 20, 8, True)
    fid = sum(sum(c[k]) for k in c if k.endswith("FID"))
    assert fid == 116
    assert fid + sum(c[k] for k in c if k.endswith("IS")) == 174


def test_kernel_arguments_are_checked_without_gpu():
    l = _lib.lib()
    rc = l.pf_resize_area2_u8(C.c_void_p(16), 1, 3, 6, 9, 2, 3, C.c_void_p(16), None)
    assert rc == -3 and b"not a factor-2" in l.pf_last_error()
    with pytest.raises(NotImplementedError):
        _lib.check(rc)
    assert l.pf_resize_area2_u8(None, 1, 3, 4, 4, 2, 2, None, None) == -1
    assert l.pf_eval_crops(C.c_void_p(16), 1, 8, 16, 2, 3, 4, 4, C.c_void_p(16), 1, C.c_void_p(16), None) == -1
    assert b"read past" in l.pf_last_error()
    assert l.pf_eval_crops(C.c_void_p(16), 1, 8, 16, 2, 2, 4, 4, C.c_void_p(16), 2, C.c_void_p(16), None) == -1
