"""`py360convert.e2p` behind its own signature, on the GPU (SURVEY.md 8f rank 2).

Reference: external/py360convert/e2p.py:6-43 (+ utils.py:104-132,231-243), called by `Equirectangular.to_perspective`
(utils/pano.py:160-161) once per view in the dataset (dataset/PanoDataset.py:138: 20 views per panorama on the CPU, scipy
map_coordinates per channel). Here one launch resamples ALL requested views of a panorama; only the three 3x3 rotations per
camera are prepared on the host (29 doubles, cached). numpy in -> numpy out like the reference; a CUDA tensor in -> CUDA
tensor out (no host round trip). There is no CPU fallback.

The cubemap conversions `c2e` / `e2c` (c2e.py:6-64, e2c.py:6-40; `Cubemap.to_equirectangular` / `Equirectangular.to_cubemap`,
utils/pano.py:124-125,146-147) and the cube layout helpers (utils.py:176-228) follow with the reference's signatures, so this
module stands in for all of `external.py360convert` as utils/pano.py imports it.
"""
from __future__ import annotations

import functools

import numpy as np
import torch

from . import _lib


def _rotation_matrix(rad: float, ax) -> np.ndarray:  # utils.py:231-243
    ax = np.array(ax, dtype=np.float64)
    ax = ax / np.sqrt((ax ** 2).sum())
    R = np.diag([np.cos(rad)] * 3)
    R = R + np.outer(ax, ax) * (1.0 - np.cos(rad))
    ax = ax * np.sin(rad)
    return R + np.array([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]])


@functools.lru_cache(maxsize=4096)
def _record(h_fov_deg: float, v_fov_deg: float, u_deg: float, v_deg: float, in_rot_deg: float) -> tuple:
    u, v, in_rot = -u_deg * np.pi / 180, v_deg * np.pi / 180, in_rot_deg * np.pi / 180  # e2p.py:28-29
    Rx = _rotation_matrix(v, [1, 0, 0])
    Ry = _rotation_matrix(u, [0, 1, 0])
    Ri = _rotation_matrix(in_rot, np.array([0, 0, 1.0]).dot(Rx).dot(Ry))
    ext = [np.tan(h_fov_deg * np.pi / 180 / 2), np.tan(v_fov_deg * np.pi / 180 / 2)]
    return tuple(np.concatenate([Rx.reshape(-1), Ry.reshape(-1), Ri.reshape(-1), ext]).tolist())


def _fov_pair(fov_deg):
    try:
        return float(fov_deg[0]), float(fov_deg[1])
    except TypeError:  # the reference's scalar branch is broken (NameError, e2p.py:17-18); a scalar means a square FoV
        return float(fov_deg), float(fov_deg)


def e2p_views(e_img, fov_deg, u_deg, v_deg, out_hw, in_rot_deg=0, mode="bilinear"):
    """All views of one panorama in one launch: u_deg / v_deg sequences of length m -> [m, h, w, C] ([m, h, w] for a 2-D image)."""
    if mode == "bilinear":
        code = 0
    elif mode == "nearest":
        code = 1
    else:
        raise NotImplementedError("unknown mode")
    as_numpy = isinstance(e_img, np.ndarray)
    x = torch.from_numpy(np.ascontiguousarray(e_img)).cuda() if as_numpy else e_img
    _lib.require_cuda(x)
    if x.dim() not in (2, 3):
        raise AssertionError("e_img must be [H, W] or [H, W, C]")
    squeeze = x.dim() == 2
    x = x.contiguous() if not squeeze else x.contiguous()[..., None]
    if x.dtype == torch.uint8:
        is_u8 = 1
    elif x.dtype == torch.float32:
        is_u8 = 0
    else:
        raise TypeError(f"py360 e2p: uint8 or float32 images, got {x.dtype}")
    H, W, C = x.shape
    h, w = int(out_hw[0]), int(out_hw[1])
    hf, vf = _fov_pair(fov_deg)
    us, vs = np.atleast_1d(np.asarray(u_deg, dtype=np.float64)), np.atleast_1d(np.asarray(v_deg, dtype=np.float64))
    rot = np.broadcast_to(np.asarray(in_rot_deg, dtype=np.float64), us.shape)
    recs = torch.tensor([_record(hf, vf, float(a), float(b), float(r)) for a, b, r in zip(us, vs, rot)],
                        dtype=torch.float64).to(x.device)
    out = torch.empty((len(us), h, w, C), dtype=x.dtype, device=x.device)
    Cv = _lib.C.c_void_p
    _lib.check(_lib.lib().pf_e2p_py360(Cv(x.data_ptr()), Cv(out.data_ptr()), is_u8, H, W, C, h, w, Cv(recs.data_ptr()),
                                       len(us), code, Cv(_lib.stream_ptr())))
    if squeeze:
        out = out[..., 0]
    return out.cpu().numpy() if as_numpy else out


def e2p(e_img, fov_deg, u_deg, v_deg, out_hw, in_rot_deg=0, mode="bilinear"):
    """py360convert.e2p(e_img[H, W, *], fov_deg, u_deg, v_deg, out_hw, in_rot_deg, mode) -> [h, w, *] (e2p.py:6-43)."""
    return e2p_views(e_img, fov_deg, [u_deg], [v_deg], out_hw, in_rot_deg, mode)[0]


# ---------------------------------------------------------------------------------------------------------------------
# cubemaps (c2e.py:6-64, e2c.py:6-40). A cube is [face_w, 6 * face_w, C] in horizon order F R B L U D; the layout helpers
# below take and return numpy arrays or torch tensors alike, since they only move faces around.
# ---------------------------------------------------------------------------------------------------------------------
FACE_KEYS = ("F", "R", "B", "L", "U", "D")
_DICE_XY = ((1, 1), (2, 1), (3, 1), (0, 1), (1, 0), (1, 2))  # (column, row) of each face in the 4 x 3 dice


def _flip(x, axis):
    return torch.flip(x, (axis,)) if isinstance(x, torch.Tensor) else np.flip(x, axis)


def _cat(parts, axis):
    return torch.cat(list(parts), axis) if isinstance(parts[0], torch.Tensor) else np.concatenate(parts, axis)


def _dice_face(face, i):
    """Horizon face i <-> its dice orientation (the same flip both ways): R and B mirrored left-right, U upside down."""
    if i in (1, 2):
        return _flip(face, 1)
    return _flip(face, 0) if i == 4 else face


def cube_h2list(cube_h):
    assert cube_h.shape[0] * 6 == cube_h.shape[1]
    fw = cube_h.shape[0]
    return [cube_h[:, k * fw:(k + 1) * fw] for k in range(6)]


def cube_list2h(cube_list):
    assert len(cube_list) == 6
    assert all(tuple(face.shape) == tuple(cube_list[0].shape) for face in cube_list)
    return _cat(cube_list, 1)


def cube_h2dict(cube_h):
    return dict(zip(FACE_KEYS, cube_h2list(cube_h)))


def cube_dict2h(cube_dict, face_k=FACE_KEYS):
    assert len(face_k) == 6
    return cube_list2h([cube_dict[k] for k in face_k])


def cube_h2dice(cube_h):
    assert cube_h.shape[0] * 6 == cube_h.shape[1]
    w = cube_h.shape[0]
    shape = (w * 3, w * 4, cube_h.shape[2])
    if isinstance(cube_h, torch.Tensor):
        dice = torch.zeros(shape, dtype=cube_h.dtype, device=cube_h.device)
    else:
        dice = np.zeros(shape, dtype=cube_h.dtype)
    for i, face in enumerate(cube_h2list(cube_h)):
        sx, sy = _DICE_XY[i]
        dice[sy * w:(sy + 1) * w, sx * w:(sx + 1) * w] = _dice_face(face, i)
    return dice


def cube_dice2h(cube_dice):
    w = cube_dice.shape[0] // 3
    assert cube_dice.shape[0] == w * 3 and cube_dice.shape[1] == w * 4
    return _cat([_dice_face(cube_dice[sy * w:(sy + 1) * w, sx * w:(sx + 1) * w], i)
                 for i, (sx, sy) in enumerate(_DICE_XY)], 1)


_TO_HORIZON = {"horizon": lambda c: c, "list": cube_list2h, "dict": cube_dict2h, "dice": cube_dice2h}
_FROM_HORIZON = {"horizon": lambda c: c, "list": cube_h2list, "dict": cube_h2dict, "dice": cube_h2dice}


def _mode_code(mode):
    if mode == "bilinear":
        return 0
    if mode == "nearest":
        return 1
    raise NotImplementedError("unknown mode")


def _to_device(img, what):
    """(contiguous CUDA tensor, is_u8, came-from-numpy)."""
    as_numpy = isinstance(img, np.ndarray)
    x = torch.from_numpy(np.ascontiguousarray(img)).cuda() if as_numpy else img.contiguous()
    _lib.require_cuda(x)
    if x.dtype not in (torch.uint8, torch.float32):
        raise TypeError(f"py360 {what}: uint8 or float32 images, got {x.dtype}")
    return x, int(x.dtype == torch.uint8), as_numpy


def ceil_rows(h: int, w: int) -> np.ndarray:
    """Ceiling row of each column of one quarter of the panorama (equirect_facetype, utils.py:55-56): columns of face U
    are rows [0, ceil), of face D their mirror image. float64 numpy, as the reference evaluates it, so that no pixel
    lands on a different face."""
    lon = np.linspace(-np.pi, np.pi, w // 4) / 4
    return (h // 2 - np.round(np.arctan(np.cos(lon)) * h / np.pi).astype(int)).astype(np.int32)


def equirect_facetype(h: int, w: int) -> np.ndarray:
    """Face id (0F 1R 2B 3L 4U 5D) of every pixel of an h x w panorama, [h, w] int32: the mapping pf_c2e_py360 applies
    to `ceil_rows` (the four side faces rolled right by 3w/8; U on top of its ceiling row, D below the mirrored one)."""
    xs = (np.arange(w) - 3 * w // 8) % w
    ceil = ceil_rows(h, w)[xs % (w // 4)]
    r = np.arange(h)[:, None]
    tp = np.broadcast_to(xs // (w // 4), (h, w)).astype(np.int32)
    tp = np.where(r < ceil, 4, tp)
    return np.where(h - 1 - r < ceil, 5, tp).astype(np.int32)


def cube_border(face_w: int) -> np.ndarray:
    """[6, 4 * face_w + 4] int32: for each face of sample_cubefaces (utils.py:135-173), the horizon-cube pixel
    (row * 6 * face_w + col) behind each sample of its two pad rows [row fw][fw], [row fw + 1][fw] and two pad columns
    [col fw][fw + 2], [col fw + 1][fw + 2]; -1 where the reference pads with zeros."""
    fw = face_w
    # pixel index of each face sample [face, row, col], with the R / B column flip and the U row flip applied
    f = np.arange(fw * 6 * fw, dtype=np.int64).reshape(fw, 6, fw).transpose(1, 0, 2).copy()
    f[1], f[2], f[4] = f[1][:, ::-1], f[2][:, ::-1], f[4][::-1]
    rows = [(f[5][0], f[4][-1]), (f[5][:, -1], f[4][::-1, -1]), (f[5][-1, ::-1], f[4][0, ::-1]),
            (f[5][::-1, 0], f[4][:, 0]), (f[0][0], f[2][0, ::-1]), (f[2][-1, ::-1], f[0][-1])]
    tall = [np.concatenate([f[k], np.stack(rows[k])]) for k in range(6)]  # [fw + 2, fw]: face + its two pad rows
    z = np.array([-1])
    cols = [(tall[1][:, 0], tall[3][:, -1]), (tall[2][:, 0], tall[0][:, -1]), (tall[3][:, 0], tall[1][:, -1]),
            (tall[0][:, 0], tall[2][:, -1]),
            # U and D: only the inner fw samples are set, taken from pad-row-extended R / L rows 0 and fw
            (np.concatenate([z, tall[1][0, ::-1], z]), np.concatenate([z, tall[3][0], z])),
            (np.concatenate([z, tall[1][fw], z]), np.concatenate([z, tall[3][fw, ::-1], z]))]
    return np.stack([np.concatenate([*rows[k], *cols[k]]) for k in range(6)]).astype(np.int32)


@functools.lru_cache(maxsize=16)
def _c2e_tables(h: int, w: int, face_w: int, device: torch.device):
    return (torch.from_numpy(ceil_rows(h, w)).to(device), torch.from_numpy(cube_border(face_w)).to(device))


def c2e(cubemap, h, w, mode="bilinear", cube_format="dice"):
    """py360convert.c2e(cubemap, h, w, mode, cube_format) -> equirect [h, w, C] float64 (c2e.py:6-64): numpy in ->
    numpy out, CUDA tensor in -> CUDA tensor out. Faces are uint8 or float32, channels-last."""
    code = _mode_code(mode)
    if cube_format not in _TO_HORIZON:
        raise NotImplementedError("unknown cube_format")
    cube = _TO_HORIZON[cube_format](cubemap)
    assert len(cube.shape) == 3
    assert cube.shape[0] * 6 == cube.shape[1]
    assert w % 8 == 0
    x, is_u8, as_numpy = _to_device(cube, "c2e")
    fw, C = x.shape[0], x.shape[2]
    ceil, border = _c2e_tables(int(h), int(w), fw, x.device)
    out = torch.empty((h, w, C), dtype=torch.float64, device=x.device)
    Cv = _lib.C.c_void_p
    _lib.check(_lib.lib().pf_c2e_py360(Cv(x.data_ptr()), Cv(out.data_ptr()), is_u8, fw, C, int(h), int(w),
                                       Cv(ceil.data_ptr()), Cv(border.data_ptr()), code, Cv(_lib.stream_ptr())))
    return out.cpu().numpy() if as_numpy else out


def e2c(e_img, face_w=256, mode="bilinear", cube_format="dice"):
    """py360convert.e2c(e_img[H, W, C], face_w, mode, cube_format) (e2c.py:6-40) -> cubemap in `cube_format`, in the
    image's dtype (uint8 rounded to nearest): numpy in -> numpy out, CUDA tensor in -> CUDA tensor out."""
    assert len(e_img.shape) == 3
    code = _mode_code(mode)
    if cube_format not in _FROM_HORIZON:
        raise NotImplementedError()
    x, is_u8, as_numpy = _to_device(e_img, "e2c")
    H, W, C = x.shape
    out = torch.empty((face_w, 6 * face_w, C), dtype=x.dtype, device=x.device)
    Cv = _lib.C.c_void_p
    _lib.check(_lib.lib().pf_e2c_py360(Cv(x.data_ptr()), Cv(out.data_ptr()), is_u8, H, W, C, int(face_w), code,
                                       Cv(_lib.stream_ptr())))
    return _FROM_HORIZON[cube_format](out.cpu().numpy() if as_numpy else out)
