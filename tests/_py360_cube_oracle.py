"""Oracle for the cubemap half of py360convert (external/py360convert/c2e.py:6-64, e2c.py:6-40, utils.py:5-64,135-173),
restated in numpy on the reference's own float32 / float64 mix, and the minting of tests/golden/py360_cube.npz by
executing the reference's files by path on seeded inputs. Test infrastructure only.

    python tests/_py360_cube_oracle.py     # needs the reference checkout (oracle/ref_loader.REF); prints the deviation

The restatement samples with scipy.ndimage.map_coordinates (mode='wrap', the legacy period-(n - 1) boundary) exactly as
the reference does. Its padded-face layout comes from panfusion_b200.py360.cube_border (host numpy, no GPU), so the
bit-for-bit match against the golden also pins that table.

The golden keeps the SHA-256 of each reference output (dtype, shape and bytes) rather than the arrays: c2e's float64
bilinear values do not compress, and a digest pins the restatement to the reference bit for bit just as well. The
kernels are then compared with the restatement evaluated on the same seeded inputs. The face-type tables are kept
whole (a few kB compressed).
"""
from __future__ import annotations

import hashlib
import sys
from pathlib import Path

import numpy as np
from scipy.ndimage import map_coordinates

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

from oracle import py360 as op  # noqa: E402  (the e2p oracle's pole-padded 'wrap' sampler, pinned against scipy)
from panfusion_b200 import py360  # noqa: E402

GOLDEN = ROOT / "tests" / "golden" / "py360_cube.npz"

FORMATS = ("dice", "horizon", "list", "dict")


def _product(widths, sizes):
    """Every face width x image size x mode x dtype x channel count; the four cube formats take turns."""
    cases = [(fw, hw, mode, tag, C) for fw in widths for hw in sizes for mode in ("bilinear", "nearest")
             for tag in ("u8", "f32") for C in (1, 3)]
    return [c + (FORMATS[k % 4],) for k, c in enumerate(cases)]


# (face_w, (h, w) of the equirect image, mode, dtype tag, channels, cube_format)
C2E_CASES = _product((64, 48), ((64, 128), (96, 200)))
E2C_CASES = _product((32, 57), ((64, 128), (63, 130)))
FACETYPE_HW = [(64, 128), (96, 200), (33, 64), (100, 40), (512, 1024), (1024, 2048)]


def digest(a) -> str:
    """SHA-256 over an array's dtype, shape and C-order bytes."""
    a = np.ascontiguousarray(a)
    return hashlib.sha256(f"{a.dtype.str}{a.shape}".encode() + a.tobytes()).hexdigest()


def seeded(shape, tag, seed):
    rng = np.random.default_rng(seed)
    if tag == "u8":
        return rng.integers(0, 256, shape).astype(np.uint8)
    return rng.random(shape).astype(np.float32)


def c2e_input(k):
    """Case k's cube in its cube_format (built from a seeded horizon cube with the product's layout helpers)."""
    fw, _, _, tag, C, fmt = C2E_CASES[k]
    cube_h = seeded((fw, 6 * fw, C), tag, 100 + k)
    return py360._FROM_HORIZON[fmt](cube_h)


def e2c_input(k):
    _, (H, W), _, tag, C, _ = E2C_CASES[k]
    return seeded((H, W, C), tag, 200 + k)


def as_horizon(cube, fmt):
    return py360._TO_HORIZON[fmt](cube)


def facetype(h, w):
    """equirect_facetype (utils.py:47-64): side faces 0..3 in quarters, U above each column's ceiling row, D below
    its mirror, everything rolled right by 3w/8."""
    q = w // 4
    ceil = h // 2 - np.round(np.arctan(np.cos(np.linspace(-np.pi, np.pi, q) / 4)) * h / np.pi).astype(int)
    top = np.arange(h)[:, None] < np.tile(ceil, 4)[None, :]
    tp = np.broadcast_to(np.repeat(np.arange(4), q), (h, w)).copy()
    tp[top] = 4
    tp[top[::-1]] = 5
    return np.roll(tp, 3 * w // 8, 1).astype(np.int32)


def padded_face_index(fw):
    """[6, fw + 2, fw + 2] horizon-cube pixel index of every sample of sample_cubefaces' padded faces (-1: zero)."""
    f = np.arange(fw * 6 * fw, dtype=np.int64).reshape(fw, 6, fw).transpose(1, 0, 2).copy()
    f[1], f[2], f[4] = f[1][:, ::-1], f[2][:, ::-1], f[4][::-1]
    bt = py360.cube_border(fw).astype(np.int64)
    P = np.empty((6, fw + 2, fw + 2), np.int64)
    P[:, :fw, :fw] = f
    P[:, fw, :fw], P[:, fw + 1, :fw] = bt[:, :fw], bt[:, fw:2 * fw]
    P[:, :, fw], P[:, :, fw + 1] = bt[:, 2 * fw:3 * fw + 2], bt[:, 3 * fw + 2:]
    return P


def c2e_coords(h, w, fw):
    """(face type, row coordinate, column coordinate) of every equirect pixel in its padded face: float32 trig as
    numpy evaluates c2e.py:40-53, then the float64 clip and scale of c2e.py:56-57."""
    tp = facetype(h, w)
    u = np.broadcast_to(np.linspace(-np.pi, np.pi, w, dtype=np.float32)[None, :], (h, w))
    v = np.broadcast_to((np.linspace(np.pi, -np.pi, h, dtype=np.float32) / 2)[:, None], (h, w))
    cx, cy = np.zeros((h, w)), np.zeros((h, w))
    for k in range(4):
        m = tp == k
        a = u[m] - np.float32(np.pi * k / 2)
        cx[m] = np.float32(0.5) * np.tan(a)
        cy[m] = np.float32(-0.5) * np.tan(v[m]) / np.cos(a)
    for k, sign in ((4, 1), (5, -1)):
        m = tp == k
        c = np.float32(0.5) * np.tan(np.float32(np.pi / 2) - (v[m] if k == 4 else np.abs(v[m])))
        cx[m] = c * np.sin(u[m])
        cy[m] = np.float32(sign) * c * np.cos(u[m])
    return tp, (np.clip(cy, -0.5, 0.5) + 0.5) * fw, (np.clip(cx, -0.5, 0.5) + 0.5) * fw


def c2e(cube_h, h, w, mode="bilinear"):
    """Horizon cube [fw, 6 fw, C] -> float64 [h, w, C] (c2e.py:6-64)."""
    assert w % 8 == 0 and cube_h.shape[0] * 6 == cube_h.shape[1]
    order = {"bilinear": 1, "nearest": 0}[mode]
    fw = cube_h.shape[0]
    tp, Y, X = c2e_coords(h, w, fw)
    P = padded_face_index(fw)
    out = []
    for ch in range(cube_h.shape[2]):
        flat = cube_h[..., ch].reshape(-1).astype(np.float64)
        faces = np.where(P >= 0, flat[np.maximum(P, 0)], 0.0)
        out.append(map_coordinates(faces, [tp, Y, X], order=order, mode="wrap"))
    return np.stack(out, -1)


def e2c_coords(fw, H, W):
    """float32 (column, row) coordinates in the equirect image of every horizon-cube pixel (xyzcube -> xyz2uv ->
    uv2coor, utils.py:5-37,82-114)."""
    rng = np.linspace(-0.5, 0.5, fw, dtype=np.float32)
    a, b = np.broadcast_to(rng[None, :], (fw, fw)), np.broadcast_to(-rng[:, None], (fw, fw))
    half = np.full((fw, fw), 0.5, np.float32)
    faces = [(a, b, half), (half, b, a), (a, b, -half), (-half, b, a), (a, half, b), (a, -half, b)]  # (x, y, z)
    x, y, z = (np.concatenate([f[i] for f in faces], 1) for i in range(3))
    u = np.arctan2(x, z)
    v = np.arctan2(y, np.sqrt(x ** 2 + z ** 2))
    return (u / np.float32(2 * np.pi) + np.float32(0.5)) * np.float32(W) - np.float32(0.5), \
        (-v / np.float32(np.pi) + np.float32(0.5)) * np.float32(H) - np.float32(0.5)


def e2c(e_img, face_w, mode="bilinear"):
    """Equirect [H, W, C] -> horizon cube [face_w, 6 face_w, C] in the image's dtype (e2c.py:6-40)."""
    order = {"bilinear": 1, "nearest": 0}[mode]
    cx, cy = e2c_coords(face_w, *e_img.shape[:2])
    return np.stack([op.sample_equirec(e_img[..., i], cx, cy, order) for i in range(e_img.shape[2])], -1)


def mint():
    """Execute external/py360convert by path on the seeded cases, compare the restatement and write the golden."""
    import importlib
    from oracle import ref_loader
    if str(ref_loader.REF) not in sys.path:
        sys.path.insert(0, str(ref_loader.REF))
    ref = importlib.import_module("external.py360convert")
    out, worst = {}, 0.0
    for k, (fw, (h, w), mode, tag, C, fmt) in enumerate(C2E_CASES):
        cube = c2e_input(k)
        r = ref.c2e(cube, h, w, mode=mode, cube_format=fmt)
        assert r.dtype == np.float64 and r.shape == (h, w, C)
        out[f"c2e{k}_sha256"], out[f"c2e{k}_sum"] = digest(r), r.sum()
        worst = max(worst, float(np.abs(r - c2e(as_horizon(cube, fmt), h, w, mode)).max()))
    for k, (fw, (H, W), mode, tag, C, fmt) in enumerate(E2C_CASES):
        im = e2c_input(k)
        r = ref.e2c(im, face_w=fw, mode=mode, cube_format=fmt)
        r_h = {"horizon": lambda c: c, "list": ref.cube_list2h, "dict": ref.cube_dict2h, "dice": ref.cube_dice2h}[fmt](r)
        assert r_h.dtype == im.dtype and r_h.shape == (fw, 6 * fw, C)
        out[f"e2c{k}_sha256"], out[f"e2c{k}_sum"] = digest(r_h), r_h.astype(np.float64).sum()
        worst = max(worst, float(np.abs(r_h.astype(np.float64) - e2c(im, fw, mode).astype(np.float64)).max()))
        # the layout helpers agree with the reference's on this case's output
        for a, b in zip(ref.cube_h2list(r_h), py360.cube_h2list(r_h)):
            assert np.array_equal(a, b)
        assert np.array_equal(ref.cube_h2dice(r_h), py360.cube_h2dice(r_h))
        assert np.array_equal(ref.cube_dice2h(ref.cube_h2dice(r_h)), py360.cube_dice2h(ref.cube_h2dice(r_h)))
    for h, w in FACETYPE_HW:
        tp = ref.equirect_facetype(h, w)
        out[f"facetype_{h}x{w}"] = tp.astype(np.uint8)
        worst = max(worst, float(np.abs(tp - facetype(h, w)).max()))
    print(f"  py360convert c2e / e2c / equirect_facetype: max |oracle - reference| = {worst:.3e}")
    np.savez_compressed(GOLDEN, **out)
    return worst


if __name__ == "__main__":
    sys.exit(0 if mint() == 0.0 else 1)
