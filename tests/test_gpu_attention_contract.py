"""-m gpu: every attention launch the models make, against the fp64 restatements of tests/_contract.py: flash attention
(pf_fmha_fwd) on the EPPA bias tables pf_eppa_tables builds for real camera rigs, in the resident form CameraTables
picks, at the levels and widths the UNets run them, sliced per view shard as eppa.py slices them; the text tower's
causal bias; the CLIP vision tower's 197 tokens; the UNet's self and text attention; and the three CPAttn kernels of
MVDiffusion (pf_cpattn_gather, pf_cpattn_attn) at every (C, level) of the SD-2-width forward, with shared and
per-batch camera tables.

Outputs are NaN-filled, so a store outside the contract fails as well. The resident bias forms are checked exactly:
tile flags, the exclusive scan of live tiles, their count and every stored tile. `_Recorder` wraps the library handle
and logs the class of every attention call (the kernel path it takes); `test_attention_call_table_covers_the_models`
runs the models and requires a case for every class they make."""
import ctypes as C
import functools
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

import _contract as ct

pytestmark = pytest.mark.gpu

DTYPES = [torch.float16, torch.bfloat16]
ENTRIES = ("pf_fmha_fwd", "pf_cpattn_gather", "pf_cpattn_attn")
MIN_LOGIT = -1e30  # a bias at or below this becomes -inf in the kernel's fmaf(bias, log2(e), ...)


def _nan(shape, dtype, dev):
    return torch.full(shape, float("nan"), dtype=dtype, device=dev)


def _rand(g, shape, dev, dtype):
    return torch.randn(shape, generator=g).to(dtype).to(dev)


def _vp(t):
    return C.c_void_p(0 if t is None else t.data_ptr())


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


# ---- call classes ---------------------------------------------------------------------------------------------------

class _DeviceArray:
    """Device memory at a raw address (__cuda_array_interface__), only read here: what a recorded call's pointer holds."""

    def __init__(self, ptr, shape, strides, typestr):
        self.__cuda_array_interface__ = dict(shape=tuple(shape), strides=tuple(4 * s for s in strides),
                                             typestr=typestr, data=(int(ptr), False), version=2)


def _view(ptr, shape, strides, typestr="<f4"):
    return torch.as_tensor(_DeviceArray(ptr, shape, strides, typestr), device="cuda")


def _bias_has_min(a) -> bool:
    """Does the bias of FmhaArgs `a` hold an entry the kernel turns into -inf (the text tower's finfo.min)?"""
    if not a.bias:
        return False
    if a.bias_tile_off:
        G, QT, KT = (a.B if a.flags_bstride else 1), -(-a.Lq // 128), -(-a.Lk // 64)
        off = _view(a.bias_tile_off, (G, QT, KT), (a.flags_bstride or QT * a.flags_ld, a.flags_ld, 1), "<i4")
        n = int(off.max()) + 1
        return n > 0 and bool((_view(a.bias, (n * 128 * 64,), (1,)) <= MIN_LOGIT).any())
    G = a.B if a.bias_bstride else 1
    bias = _view(a.bias, (G, a.Lq, a.Lk), (a.bias_bstride or a.Lq * a.bias_ld, a.bias_ld, 1))
    return bool((bias <= MIN_LOGIT).any())


def fmha_class(a):
    """(head dim, bias form, per-batch bias, Lq % 128 != 0, Lk % 64 != 0, strided q/k/v, K/V outside q's buffer,
    bias holding finfo.min) of one pf_fmha_fwd call."""
    hd = a.H * a.head_dim
    if not a.bias:
        form, per_batch = "none", False
    elif a.bias_tile_off:
        form, per_batch = "packed", a.flags_bstride != 0
    else:
        form, per_batch = ("dense+flags" if a.bias_flags else "dense"), a.bias_bstride != 0
    fused = (a.k == a.q + 2 * hd and a.v == a.k + 2 * hd and a.q_ld == a.k_ld == a.v_ld
             and a.q_bstride == a.k_bstride == a.v_bstride)
    return ("pf_fmha_fwd", a.head_dim, form, per_batch, a.Lq % 128 != 0, a.Lk % 64 != 0,
            max(a.q_ld, a.k_ld, a.v_ld) > hd, not fused, _bias_has_min(a))


def call_class(name, args):
    if name == "pf_fmha_fwd":
        return fmha_class(args[0]._obj)
    if name == "pf_cpattn_gather":  # (x, ldx, dtype, B, m, h, w, C, G, ...): 8 key rows per CTA
        _x, ldx, _dt, B, m, h, w, Cc, G = args[:9]
        return (name, G > 1, ldx > Cc, (B * m * h * w * ct.CP_SLOTS) % 8 != 0)
    _q, ldq, _kv, ldkv, _o, ldo, _dt, ntok, Cc = args[:9]  # pf_cpattn_attn: one thread per (token, head), 256 per CTA
    ntok = ntok.value if isinstance(ntok, C.c_longlong) else ntok
    return (name, ldq > Cc or ldkv > 2 * Cc or ldo > Cc, (ntok * (Cc // 32)) % 256 != 0)


class _Recorder:
    """Stands in for the library handle: logs the class of every attention call, then forwards it."""

    def __init__(self, lib):
        self._lib, self.calls = lib, []

    def __getattr__(self, name):
        f = getattr(self._lib, name)
        if name not in ENTRIES:
            return f

        def rec(*args):
            self.calls.append(call_class(name, args))
            return f(*args)
        return rec


@pytest.fixture(scope="module", autouse=True)
def _release_tables():
    """The camera tables are shared by this module's tests only."""
    yield
    _eppa_tables.cache_clear()
    _cp_tables.cache_clear()


@pytest.fixture
def recorder(monkeypatch, cuda_device):
    from panfusion_b200 import _lib
    rec = _Recorder(_lib.lib())
    monkeypatch.setattr(_lib, "lib", lambda: rec)
    return rec


# ---- camera rigs and EPPA tables ------------------------------------------------------------------------------------

def _horizon(m, rot=0.0):
    return np.rad2deg(np.linspace(0, 2 * np.pi, m, endpoint=False)) + rot, np.zeros(m)


def _ico():
    sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
    from bench import icosahedron_cameras
    return icosahedron_cameras()


# rig -> (batch elements b, per-element (theta, phi) in degrees; FoV 90)
RIGS = {
    "c2": lambda: (2, [_horizon(8)] * 2),                      # bench c2: CFG pair, the same 8 horizon views
    "c2 rot90": lambda: (2, [_horizon(8, 90.0)] * 2),          # the sampler's +90 degree rotation phase
    "c2 per-batch": lambda: (2, [_horizon(8), _horizon(8, 45.0)]),  # different cameras per element: G = 2
    "ico20": lambda: (2, [_ico()] * 2),                        # bench c4: 20 icosahedron views
    "tiny m2": lambda: (1, [_horizon(2)]),                     # the tiny-config forwards the models test
    "tiny m2 per-batch": lambda: (2, [_horizon(2), _horizon(2, 45.0)]),
    "tiny m8": lambda: (2, [_horizon(8)] * 2),
}

# EPPA levels (ph, pw, eh, ew, C): views against the panorama, with the channel width the UNet has there
C2_LEVELS = [(32, 32, 32, 64, 320), (16, 16, 16, 32, 640), (8, 8, 8, 16, 1280)]
ICO_LEVEL = (32, 32, 64, 128, 320)
TINY_LEVELS = [(8, 8, 8, 16, 64), (4, 4, 4, 8, 128), (2, 2, 2, 4, 128)]


@functools.lru_cache(maxsize=None)
def _eppa_tables(rig, level):
    """The dense tables (pf_eppa_tables) and the resident forms CameraTables.bias keeps, for one rig and level."""
    from panfusion_b200 import ops
    from panfusion_b200.eppa import CameraTables
    dev = torch.device("cuda:0")
    b, cams = RIGS[rig]()
    theta = np.concatenate([t for t, _ in cams])
    phi = np.concatenate([p for _, p in cams])
    cameras = dict(FoV=torch.full((len(theta),), 90.0), theta=torch.tensor(theta, dtype=torch.float32),
                   phi=torch.tensor(phi, dtype=torch.float32))
    tables = CameraTables()
    key, groups = CameraTables.dedup(CameraTables.camera_key(cameras), b)
    ph, pw, eh, ew, _c = level
    V = len(key[0])
    ce, cp = tables._records(key, V, ph, pw, dev)
    dense1, dense2 = ops.eppa_tables(ce, cp, V // groups, ph, pw, eh, ew)
    resident = tables.bias(key, groups, ph, pw, eh, ew, dev)
    return dict(b=b, m=len(cams[0][0]), groups=groups, dense=(dense1, dense2), resident=resident)


def _eppa_launches(g, dev, dt, rig, level, m_locs=(None,)):
    """The two flash-attention launches of WarpAttn.forward_tokens (eppa.py:262-318) per view shard: q / k / v as
    slices of the fused QKV projections, K / V of a sharded rank from the separate gathered [b, m P, 2C] buffer,
    direction 2's bias sliced to the rank's views. -> [(label, q, k, v, fmha kwargs, dense bias)]"""
    t = _eppa_tables(rig, level)
    b, m = t["b"], t["m"]
    ph, pw, eh, ew, Cc = level
    P, E = ph * pw, eh * ew
    d1, d2 = t["resident"]
    dense1, dense2 = t["dense"]
    kw = dict(heads=Cc // 32, head_dim=32, scale=32 ** -0.5)
    kw1 = dict(kw, **(dict(bias_tiles=(d1[1], d1[2])) if d1[0] == "packed" else dict(bias=d1[1], bias_flags=d1[2])))
    qkv_e = _rand(g, (b, E, 3 * Cc), dev, dt)
    name = f"{rig} {ph}x{pw}/{eh}x{ew} C={Cc}"
    out, gathered = [], False
    for m_loc in m_locs:
        if m_loc is None:
            qkv_p = _rand(g, (b, m * P, 3 * Cc), dev, dt)
            kw2 = dict(kw, **(dict(bias_tiles=(d2[1], d2[2])) if d2[0] == "packed" else dict(bias=d2[1], bias_flags=d2[2])))
            out.append((f"{name} dir1 {d1[0]}", qkv_e[..., :Cc], qkv_p[..., Cc:2 * Cc], qkv_p[..., 2 * Cc:], kw1, dense1))
            out.append((f"{name} dir2 {d2[0]}", qkv_p[..., :Cc], qkv_e[..., Cc:2 * Cc], qkv_e[..., 2 * Cc:], kw2, dense2))
            continue
        if not gathered:
            gathered = True
            kv_all = _rand(g, (b, m * P, 2 * Cc), dev, dt)  # what par.gather_views returns
            out.append((f"{name} dir1 {d1[0]} gathered K|V", qkv_e[..., :Cc], kv_all[..., :Cc], kv_all[..., Cc:], kw1,
                        dense1))
        for v0 in range(0, m, m_loc):
            qkv_p = _rand(g, (b, m_loc * P, 3 * Cc), dev, dt)
            if d2[0] == "packed":
                off2 = d2[2][:, (v0 * P) // 128:((v0 + m_loc) * P) // 128].contiguous()
                kw2 = dict(kw, bias_tiles=(d2[1], off2))
            else:
                bias2 = d2[1][:, v0 * P:(v0 + m_loc) * P]
                flags2 = d2[2][:, (v0 * P) // 128:((v0 + m_loc) * P + 127) // 128].contiguous() \
                    if (v0 * P) % 128 == 0 and (m_loc * P) % 128 == 0 else None
                kw2 = dict(kw, bias=bias2, bias_flags=flags2)
            form = "packed" if d2[0] == "packed" else ("dense+flags" if kw2["bias_flags"] is not None else "dense")
            out.append((f"{name} dir2 {form} views [{v0}, {v0 + m_loc})", qkv_p[..., :Cc], qkv_e[..., Cc:2 * Cc],
                        qkv_e[..., 2 * Cc:], kw2, dense2[:, v0 * P:(v0 + m_loc) * P]))
    return out


# ---- flash-attention cases ------------------------------------------------------------------------------------------

def fcase_eppa_c2(g, dev, dt):
    """bench c2's rig at the three EPPA levels of a 512 x 1024 panorama, shared by the CFG pair (G = 1), at rotation
    phases 0 and +90 degrees: packed where E or P is a multiple of 128, dense + flags at the 8 x 8 views."""
    return [x for rig in ("c2", "c2 rot90") for lv in C2_LEVELS for x in _eppa_launches(g, dev, dt, rig, lv)]


def fcase_eppa_per_batch(g, dev, dt):
    """b = 2 with different cameras per element (G = 2): per-batch packed tables and per-batch dense + flags."""
    return [x for lv in C2_LEVELS for x in _eppa_launches(g, dev, dt, "c2 per-batch", lv)]


def fcase_eppa_shards(g, dev, dt):
    """Every rank of 2, 4 and 8 view shards of the c2 rig: sliced tile-offset tables, dense slices whose flags are
    dropped when v0 P is not a multiple of 128 (8 x 8 views, one view per rank), K / V from the gathered buffer."""
    return [x for lv in C2_LEVELS for x in _eppa_launches(g, dev, dt, "c2", lv, m_locs=(4, 2, 1))]


def fcase_eppa_ico20(g, dev, dt):
    """bench c4's 20 icosahedron views at 32 x 32 against a 64 x 128 panorama: direction 1 has Lk = 20480."""
    return _eppa_launches(g, dev, dt, "ico20", ICO_LEVEL)


def fcase_eppa_tiny(g, dev, dt):
    """The tiny-config levels (8 x 8 .. 2 x 2 views, ragged in both directions, dense + flags) with 2 views, 2 views
    per batch element, and 8 views in 2 and 8 shards."""
    out = []
    for lv in TINY_LEVELS:
        out += _eppa_launches(g, dev, dt, "tiny m2", lv)
        out += _eppa_launches(g, dev, dt, "tiny m2 per-batch", lv)
        out += _eppa_launches(g, dev, dt, "tiny m8", lv, m_locs=(None, 4, 1))
    return out


def fcase_text_tower(g, dev, dt):
    """text_encoder.py:97-99,126: the causal [77, 80] bias (finfo(float32).min above the diagonal) sliced [:Lx], q / k /
    v slices of the fused [B, Lx, 3C] projection, SD-2's width (16 heads of 64), Lx = 77 and a shorter prompt."""
    Cc, L = 1024, 77
    causal = torch.zeros((L, 80))
    causal[:, :L] = torch.full((L, L), torch.finfo(torch.float32).min).triu(1)
    causal = causal.to(dev)
    out = []
    for Lx in (77, 20):
        qkv = _rand(g, (2, Lx, 3 * Cc), dev, dt)
        out.append((f"text Lx={Lx}", qkv[..., :Cc], qkv[..., Cc:2 * Cc], qkv[..., 2 * Cc:],
                    dict(heads=16, head_dim=64, scale=64 ** -0.5, bias=causal[:Lx]), causal[:Lx, :Lx]))
    return out


def fcase_clip_vision(g, dev, dt):
    """clip_score.py encode_image: ViT-B/16, 197 tokens (CLS + 14 x 14 patches), no bias, 12 heads of 64."""
    qkv = _rand(g, (2, 197, 3 * 768), dev, dt)
    return [("vision L=197", qkv[..., :768], qkv[..., 768:1536], qkv[..., 1536:],
             dict(heads=12, head_dim=64, scale=64 ** -0.5), None)]


def fcase_unet(g, dev, dt):
    """engine.py:323,327: self attention over the fused [N, L, 3C] projection at the 64 x 64, 8 x 8 and (tiny config)
    4 x 4 levels; text cross attention with K / V column slices of the hoisted [N, 77, 24960] text K/V."""
    out = []
    for L in (4096, 64, 16):
        qkv = _rand(g, (2, L, 3 * 320), dev, dt)
        out.append((f"self L={L}", qkv[..., :320], qkv[..., 320:640], qkv[..., 640:],
                    dict(heads=5, head_dim=64, scale=64 ** -0.5), None))
    kv = _rand(g, (2, 77, 24960), dev, dt)
    for L in (1024, 64):
        q = _rand(g, (2, L, 640), dev, dt)
        out.append((f"cross L={L}", q, kv[..., 1280:1920], kv[..., 1920:2560],
                    dict(heads=10, head_dim=64, scale=64 ** -0.5), None))
    return out


FMHA_CASES = {
    "eppa_c2": fcase_eppa_c2,
    "eppa_per_batch": fcase_eppa_per_batch,
    "eppa_shards": fcase_eppa_shards,
    "eppa_ico20": fcase_eppa_ico20,
    "eppa_tiny": fcase_eppa_tiny,
    "text_tower": fcase_text_tower,
    "clip_vision": fcase_clip_vision,
    "unet": fcase_unet,
}


def _run_fmha(launch, dt):
    from panfusion_b200 import ops
    _label, q, k, v, kw, _dense = launch
    out = _nan((q.shape[0], q.shape[1], kw["heads"] * kw["head_dim"]), dt, q.device)
    ops.fmha(q, k, v, out, **kw)
    return out


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("case", list(FMHA_CASES))
def test_fmha_contract(cuda_device, case, dtype):
    g = torch.Generator().manual_seed(sum(map(ord, case)))
    worst = 0.0
    for launch in FMHA_CASES[case](g, cuda_device, dtype):
        label, q, k, v, kw, dense = launch
        out = _run_fmha(launch, dtype)
        ref, pv = ct.fmha_ref(q, k, v, heads=kw["heads"], head_dim=kw["head_dim"], scale=kw["scale"], bias=dense)
        r = ct.worst_ratio(out, ref, ct.fmha_bound(ref, pv, dtype))
        print(f"[contract] fmha {case} / {label} {dtype}: worst err/bound {r:.3f}")
        worst = max(worst, r)
        del out, ref, pv
    assert worst <= 1.0, worst


# ---- resident bias forms, exact -------------------------------------------------------------------------------------

TABLE_SPECS = ([(rig, lv) for rig in ("c2", "c2 rot90", "c2 per-batch") for lv in C2_LEVELS] + [("ico20", ICO_LEVEL)]
               + [(rig, lv) for rig in ("tiny m2", "tiny m2 per-batch", "tiny m8") for lv in TINY_LEVELS])


def _tiles(bias):
    """Dense [G, Lq, Lk] -> its 128 x 64 tiles [G * QT * KT, 128, 64], zero past Lq / Lk, and which entries exist."""
    G, Lq, Lk = bias.shape
    QT, KT = -(-Lq // 128), -(-Lk // 64)
    pad = torch.zeros((G, QT * 128, KT * 64), device=bias.device)
    inb = torch.zeros((G, QT * 128, KT * 64), dtype=torch.bool, device=bias.device)
    pad[:, :Lq, :Lk] = bias
    inb[:, :Lq, :Lk] = True
    tile = lambda t: t.reshape(G, QT, 128, KT, 64).permute(0, 1, 3, 2, 4).reshape(G * QT * KT, 128, 64)
    return tile(pad), tile(inb), (G, QT, KT)


def test_table_specs_include_a_multi_chunk_per_batch_scan():
    """The scan walks its flags in chunks of 1024: at least one real per-batch table has more tiles than one chunk."""
    def tiles(rig, lv):  # direction 1: [G, E, m P] in 128 x 64 tiles
        b, cams = RIGS[rig]()
        G = 1 if all(np.array_equal(c[0], cams[0][0]) and np.array_equal(c[1], cams[0][1]) for c in cams) else b
        return G, G * -(-lv[2] * lv[3] // 128) * -(-len(cams[0][0]) * lv[0] * lv[1] // 64)
    assert any(G == 2 and n > 1024 for G, n in (tiles(rig, lv) for rig, lv in TABLE_SPECS))


@pytest.mark.parametrize("rig,level", TABLE_SPECS, ids=[f"{r.replace(' ', '-')}-{lv[0]}x{lv[1]}" for r, lv in TABLE_SPECS])
def test_resident_bias_is_exact(cuda_device, rig, level):
    """pf_bias_tile_flags / pf_bias_tile_scan / pf_bias_tile_pack on both directions' dense tables against a torch
    restatement: flags exact, tile_off the exclusive scan of the live tiles (-1 for the constant ones), n_live their
    count, every stored tile its dense tile zero-padded past Lq / Lk; and CameraTables keeps exactly these."""
    from panfusion_b200 import _lib, ops
    t = _eppa_tables(rig, level)
    lib = _lib.lib()
    for direction, bias, res in zip((1, 2), t["dense"], t["resident"]):
        tiles, inb, (G, QT, KT) = _tiles(bias)
        G_, Lq, Lk = bias.shape
        constant = ((tiles == -1) | ~inb).flatten(1).all(1)
        flags = torch.full((G, QT, KT), 7, dtype=torch.uint8, device=cuda_device)
        _lib.check(lib.pf_bias_tile_flags(_vp(bias), G, Lq, Lk, bias.stride(1), C.c_int64(bias.stride(0)), _vp(flags),
                                          _st()))
        assert torch.equal(flags.reshape(-1), constant.to(torch.uint8)), (rig, direction)
        live = ~constant
        n = int(live.sum())
        off = torch.full((G, QT, KT), -7, dtype=torch.int32, device=cuda_device)
        n_live = torch.full((1,), -7, dtype=torch.int32, device=cuda_device)
        _lib.check(lib.pf_bias_tile_scan(_vp(flags), G * QT * KT, _vp(off), _vp(n_live), _st()))
        want = torch.where(live, torch.cumsum(live.int(), 0) - 1, -1).int()
        assert torch.equal(off.reshape(-1), want), (rig, direction)
        assert int(n_live) == n, (rig, direction, int(n_live), n)
        store = torch.full((max(n, 1), 128 * 64), float("nan"), device=cuda_device)
        _lib.check(lib.pf_bias_tile_pack(_vp(bias), G, Lq, Lk, bias.stride(1), C.c_int64(bias.stride(0)), _vp(off),
                                         _vp(store), _st()))
        stored = store[:n].reshape(n, 4, 16, 32, 4).permute(0, 1, 3, 2, 4).reshape(n, 128, 64)
        assert torch.equal(stored, tiles[live]), (rig, direction)
        if n:
            assert torch.equal(ops.bias_tile_dense(store[n - 1]), tiles[live][-1])
        print(f"[contract] resident bias {rig} {level[:4]} dir{direction} {res[0]}: G={G} {G * QT * KT} tiles, {n} live")
        if res[0] == "packed":
            assert torch.equal(res[2], off) and torch.equal(res[1][:n], store[:n]), (rig, direction)
        else:
            assert torch.equal(res[2], flags) and torch.equal(res[1], bias), (rig, direction)


# ---- CPAttn ---------------------------------------------------------------------------------------------------------

def _cp_rig(m, img, rot, fov=90.0):
    from oracle import mvdiffusion as omv
    KR = [omv.get_K_R(fov, t, 0.0, img) for t in _horizon(m, rot)[0]]
    return torch.from_numpy(np.stack([k for k, _ in KR])), torch.from_numpy(np.stack([r for _, r in KR]))


@functools.lru_cache(maxsize=None)
def _cp_tables(m, h, img, G, fov):
    """pf_cpattn_tables of one horizon rig (G = 1) or of two rigs 20 degrees apart (G = 2)."""
    from panfusion_b200 import ops
    from panfusion_b200.mvdiffusion import homographies
    rigs = [_cp_rig(m, img, 20.0 * gi, fov) for gi in range(G)]
    K, R = torch.stack([k for k, _ in rigs]), torch.stack([r for _, r in rigs])
    hl, hr = homographies(K, R)
    dev = torch.device("cuda:0")
    return ops.cpattn_tables(hl.to(dev).contiguous(), hr.to(dev).contiguous(), h, h, img)


# (C, level side, views, image side, FoV): the SD-2-width MVDiffusion forward's four CP levels (8 views of 512^2), and a
# 3-view 5 x 5 level whose gather and attention grids end in a partial CTA
CPATTN_CASES = [(320, 64, 8, 512, 90.0), (640, 32, 8, 512, 90.0), (1280, 16, 8, 512, 90.0), (1280, 8, 8, 512, 90.0),
                (320, 5, 3, 40, 120.0)]


def _cp_gather(x, B, m, h, Cc, G, pos, mask, freq, dt):
    from panfusion_b200 import _lib
    rows = B * m * h * h * ct.CP_SLOTS
    keys = _nan((rows, Cc), dt, x.device)
    stats = torch.full((rows, 2, 2), float("nan"), device=x.device)
    _lib.check(_lib.lib().pf_cpattn_gather(_vp(x), x.stride(0), _lib.dtype_code(dt), B, m, h, h, Cc, G, _vp(pos),
                                           _vp(mask), _vp(freq), _vp(keys), _vp(stats), _st()))
    return keys, stats


def _cp_attn(q, kv, Cc, dt):
    from panfusion_b200 import _lib
    out = _nan((q.shape[0], Cc), dt, q.device)
    _lib.check(_lib.lib().pf_cpattn_attn(_vp(q), q.stride(0), _vp(kv), kv.stride(0), _vp(out), out.stride(0),
                                         _lib.dtype_code(dt), C.c_longlong(q.shape[0]), Cc, C.c_float(32 ** -0.5), _st()))
    return out


def _cp_launch_all(g, dev, dt, spec, G):
    """Operands of one CPAttn level as mvdiffusion.CPAttn.forward_tokens passes them (B = 2): tokens [B m P, C], the
    cached tables, the frequency table; q [T, C] and the K|V GEMM's [18 T, 2C]. Launches both kernels."""
    from panfusion_b200.mvdiffusion import _PosEmbedding
    Cc, h, m, img, fov = spec
    B = 2
    pos, mask = _cp_tables(m, h, img, G, fov)
    freq = _PosEmbedding(Cc // 4).freq_bands.reshape(-1).to(dev, torch.float32).contiguous()
    x = _rand(g, (B * m * h * h, Cc), dev, dt)
    keys, stats = _cp_gather(x, B, m, h, Cc, G, pos, mask, freq, dt)
    T = B * m * h * h
    q, kv = _rand(g, (T, Cc), dev, dt), _rand(g, (T * ct.CP_SLOTS, 2 * Cc), dev, dt)
    return dict(x=x, pos=pos, mask=mask, freq=freq, keys=keys, stats=stats, q=q, kv=kv, out=_cp_attn(q, kv, Cc, dt))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("G", [1, 2])
@pytest.mark.parametrize("spec", CPATTN_CASES, ids=[f"C{s[0]}-{s[1]}x{s[1]}-m{s[2]}" for s in CPATTN_CASES])
def test_cpattn_contract(cuda_device, spec, G, dtype):
    """pf_cpattn_gather (keys exact-zero where masked, statistics of the stored keys) and pf_cpattn_attn."""
    Cc, h, m, img, _fov = spec
    B, P = 2, h * h
    g = torch.Generator().manual_seed(Cc + h + G)
    r = _cp_launch_all(g, cuda_device, dtype, spec, G)
    torch.cuda.synchronize()
    keys, stats, rows_b = r["keys"], r["stats"], m * P * ct.CP_SLOTS
    worst_k = worst_s = 0.0
    for b in range(B):  # one batch element at a time: the fp64 keys of the 64 x 64 level are 1.5 GB per element
        gb = 0 if G == 1 else b
        ref, bound = ct.cpattn_gather_ref(r["x"][b * m * P:(b + 1) * m * P], 1, m, h, h, Cc, 1, r["pos"][gb:gb + 1],
                                          r["mask"][gb:gb + 1], r["freq"], dtype)
        kb = keys[b * rows_b:(b + 1) * rows_b]
        worst_k = max(worst_k, ct.worst_ratio(kb, ref, bound))
        del ref, bound
        masked = ~r["mask"][gb].bool().reshape(-1)
        assert masked.any() and (kb[masked] == 0).all() and (stats[b * rows_b:(b + 1) * rows_b][masked] == 0).all()
        sref, sbound = ct.cpattn_stats_ref(kb, Cc)
        worst_s = max(worst_s, float(((stats[b * rows_b:(b + 1) * rows_b, 0].double() - sref).abs() / sbound).max()))
    assert (stats[:, 1] == 0).all()
    ref, bound = ct.cpattn_attn_ref(r["q"], r["kv"], Cc, 32 ** -0.5, dtype)
    worst_a = ct.worst_ratio(r["out"], ref, bound)
    label = f"C={Cc} {h}x{h} m={m} G={G} {dtype}"
    print(f"[contract] cpattn gather {label}: worst err/bound {worst_k:.3f}, stats {worst_s:.3f}")
    print(f"[contract] cpattn attn {label}: worst err/bound {worst_a:.3f}")
    assert worst_k <= 1.0 and worst_s <= 1.0 and worst_a <= 1.0, (worst_k, worst_s, worst_a)


# ---- refusals -------------------------------------------------------------------------------------------------------

def test_argument_errors_are_refused(cuda_device):
    """Host-side checks: pf_cpattn_gather with G not in {1, B} or ldx % 8 != 0, pf_fmha_fwd with a tile-packed bias plus
    bias_flags. Each is an argument error and writes nothing."""
    from panfusion_b200 import _lib, ops
    dev, dt = cuda_device, torch.float16
    B, m, h, Cc = 2, 3, 5, 32
    pos, mask = _cp_tables(m, h, 40, 1, 120.0)
    freq = torch.ones(Cc // 4, device=dev)
    x = torch.zeros((B * m * h * h, Cc + 8), dtype=dt, device=dev)
    rows = B * m * h * h * ct.CP_SLOTS
    keys, stats = _nan((rows, Cc), dt, dev), torch.full((rows, 2, 2), float("nan"), device=dev)
    for G, ldx in ((3, Cc), (1, Cc + 4)):
        with pytest.raises(ValueError):
            _lib.check(_lib.lib().pf_cpattn_gather(_vp(x), ldx, _lib.dtype_code(dt), B, m, h, h, Cc, G, _vp(pos),
                                                   _vp(mask), _vp(freq), _vp(keys), _vp(stats), _st()))
    q = torch.zeros((1, 128, 64), dtype=dt, device=dev)
    out = _nan((1, 128, 64), dt, dev)
    bias = torch.full((1, 128, 64), -1.0, device=dev)
    store, off = ops.bias_pack_tiles(bias)
    a = ops.FmhaArgs()
    a.q = a.k = a.v = q.data_ptr()
    a.out, a.dtype, a.B, a.H, a.Lq, a.Lk, a.head_dim = out.data_ptr(), _lib.dtype_code(dt), 1, 2, 128, 128, 32
    a.q_ld = a.k_ld = a.v_ld = a.out_ld = 64
    a.q_bstride = a.k_bstride = a.v_bstride = 128 * 64
    a.scale, a.bias, a.bias_tile_off, a.flags_ld = 1.0, store.data_ptr(), off.data_ptr(), off.stride(1)
    a.bias_flags = ops.bias_tile_flags(bias).data_ptr()
    with pytest.raises(ValueError):
        _lib.check(_lib.lib().pf_fmha_fwd(C.byref(a), _st()))
    torch.cuda.synchronize()
    assert torch.isnan(keys).all() and torch.isnan(stats).all() and torch.isnan(out).all()


# ---- the table covers the models ------------------------------------------------------------------------------------

def _model_calls(dev):
    """The attention calls of: the tiny PanFusion forward with shared cameras and with per-batch rigs; every rank of
    the 1 x 2 and 1 x 8 view-sharded forwards; the tiny MVDiffusion step; the CLIP text encoder (77 tokens and a
    shorter prompt); the CLIP ViT-B/16 image tower."""
    from oracle import clip_score as oc, synth, text_encoder as ot, unet as ou
    from panfusion_b200.clip_score import CLIPEncoder
    from panfusion_b200.text_encoder import CLIPTextEncoder
    from _rank_replay import run_all_ranks, run_unsharded_recording
    from test_gpu_mvdiffusion import _tiny
    from test_gpu_mvgen import _build_mine, _run_mvgen, _to_dev
    cfg, dt = ou.TINY_CONFIG, torch.float16
    _run_mvgen(dev, cfg, (16, 32), (16, 16), dt)
    _, mine = _build_mine(dev, cfg, dt)
    inp = synth.step_inputs(2, (16, 32), (16, 16), cfg["cross_attention_dim"], seed=0, batch=2)
    inp["cameras"]["theta"][1] += 45.0
    mine(**_to_dev(inp, dev))
    inp8 = _to_dev(synth.step_inputs_cfg(8, (16, 32), (16, 16), cfg["cross_attention_dim"], seed=0), dev)
    _, rec = run_unsharded_recording(mine, inp8)
    for layout in ((1, 2), (1, 8)):
        run_all_ranks(mine, inp8, *layout, rec)
    _, mv, _, cu = _tiny(dev, dt)
    mv(**cu)
    tcfg = ot.TINY_TEXT_CONFIG
    enc = CLIPTextEncoder(ot.build_text_encoder(tcfg, seed=0), dt).prepare(dev, dt)
    ids = ot.token_ids(2, vocab=tcfg["vocab_size"], seed=1)
    enc(ids)
    enc(ids[:, :20])
    CLIPEncoder(oc.seeded_state(), oc.clip_config()).encode_image(
        torch.rand(2, 3, 224, 224, generator=torch.Generator().manual_seed(0)).to(dev))
    torch.cuda.synchronize()


def test_attention_call_table_covers_the_models(recorder, cuda_device):
    """Every attention call class the models make is one a case above launches."""
    g = torch.Generator().manual_seed(0)
    dt = torch.float16
    for build in FMHA_CASES.values():
        for launch in build(g, cuda_device, dt):
            _run_fmha(launch, dt)
    for spec in CPATTN_CASES:
        for G in (1, 2):
            _cp_launch_all(g, cuda_device, dt, spec, G)
    torch.cuda.synchronize()
    covered = set(recorder.calls)
    recorder.calls.clear()
    _model_calls(cuda_device)
    seen = set(recorder.calls)
    assert {c[0] for c in seen} == set(ENTRIES), "a model made no call of one of the entry points"
    for c in sorted(seen, key=str):
        print(f"[contract] attention call class {c}{'' if c in covered else '  <- no case'}")
    missing = sorted(seen - covered, key=str)
    assert not missing, f"call classes without a contract case: {missing}"
