"""EPPA block `WarpAttn` behind the reference's interface (models/pano/modules.py:8-59).

Same constructor, sub-module / parameter names (`transformer.attn1.{to_q,to_k,to_v,to_out}`,
`transformer.ff.net.{0.proj,2}`, `transformer.norm1/2`, buffer `pe.freq_bands`) and forward signature
`(pers_x[(b m),c,ph,pw], equi_x[b,c,eh,ew], cameras) -> (pers_x_out, equi_x_out)`, so reference checkpoints load
unchanged. What changes is the execution: the correspondence bias and the spherical PE come from cached
per-camera tables built by two CUDA kernels (csrc/eppa_tables.cu) instead of the one-hot/grid_sample/blur
pipeline of models/pano/utils.py:10-106, the bias is never repeated per head (transformer.py:68), and both
attention directions run as wgmma flash-attention launches over one fused Q/K/V projection per token set.
"""
from __future__ import annotations

import torch
import torch.nn as nn
from torch import Tensor

from . import geometry, ops
from .engine import Img, _Lin, _LinLN, _Norm, img_from_nchw


class _CrossAttention(nn.Module):  # parameters of models/modules/transformer.py:41-56
    def __init__(self, dim, heads):
        super().__init__()
        self.heads = heads
        self.to_q = nn.Linear(dim, dim, bias=False)
        self.to_k = nn.Linear(dim, dim, bias=False)
        self.to_v = nn.Linear(dim, dim, bias=False)
        self.to_out = nn.Linear(dim, dim)
        nn.init.zeros_(self.to_out.weight)
        nn.init.zeros_(self.to_out.bias)


class _GEGLU(nn.Module):  # transformer.py:8-12
    def __init__(self, dim_in, dim_out):
        super().__init__()
        self.proj = nn.Linear(dim_in, dim_out * 2)


class _FeedForward(nn.Module):  # transformer.py:18-35 (glu=True, mult=4)
    def __init__(self, dim):
        super().__init__()
        first = _GEGLU(dim, dim * 4)  # drawn before the output layer, like the reference, so seeds line up
        last = nn.Linear(dim * 4, dim)
        nn.init.zeros_(last.weight)
        nn.init.zeros_(last.bias)
        self.net = nn.Sequential(first, nn.Dropout(0.0), last)


class _Block(nn.Module):  # transformer.py:130-143
    def __init__(self, dim, heads):
        super().__init__()
        self.attn1 = _CrossAttention(dim, heads)
        self.ff = _FeedForward(dim)
        self.norm1 = nn.LayerNorm(dim)
        self.norm2 = nn.LayerNorm(dim)


class _SphericalPE(nn.Module):  # transformer.py:165-183: only the frequency table lives here
    def __init__(self, n_freqs):
        super().__init__()
        base = 2 if n_freqs <= 80 else 5000 ** (1 / (n_freqs / 2.5))
        self.register_buffer("freq_bands", base ** torch.linspace(0, n_freqs - 1, n_freqs))


def pack_block(t: _Block, dev, dt) -> dict:
    """The weights of a _Block packed for the kernels (once per device/dtype)."""
    a = t.attn1
    bn = ops.pick_block_n(t.ff.net[0].proj.weight.shape[0], ops.PF_ACT_GEGLU)
    return dict(
        key=(dev, dt),
        qkv=_Lin(torch.cat([a.to_q.weight, a.to_k.weight, a.to_v.weight], 0), None, dev, dt),
        out=_Lin(a.to_out.weight, a.to_out.bias, dev, dt),
        ff1_bn=bn,
        ff2=_Lin(t.ff.net[2].weight, t.ff.net[2].bias, dev, dt),
        ff1_ln=_LinLN(t.ff.net[0].proj.weight, t.ff.net[0].proj.bias, t.norm2, dev, dt, geglu_bn=bn),
        ln1=_Norm(t.norm1, dev), heads=a.heads)


def block_tail(w: dict, o: Tensor, x_tok: Tensor, rows: int) -> Tensor:
    """to_out(o) + x, then x + FF(norm2(x)) (transformer.py:159-160) on [rows, C] tokens; w = pack_block(...).
    norm2 is folded into the GEGLU projection (engine._LinLN)."""
    C = w["out"].n
    new = lambda r, n: torch.empty((r, n), dtype=x_tok.dtype, device=x_tok.device)
    x1, st = ops.gemm_taps(o, w["out"].w, new(rows, C), M=rows, Kc=C, bias=w["out"].b, residual=x_tok, row_stats=True)
    f = ops.gemm_taps(x1, w["ff1_ln"].w, new(rows, 4 * C), M=rows, Kc=C, bias=w["ff1_ln"].b, act=ops.PF_ACT_GEGLU,
                      block_n=w["ff1_bn"], ln=(st, w["ff1_ln"].colsum, w["ff1_ln"].eps))
    return ops.gemm_taps(f, w["ff2"].w, new(rows, C), M=rows, Kc=4 * C, bias=w["ff2"].b, residual=x1)


class CameraTables:
    """Per (camera set, level) cache of the EPPA bias tables and per (.., freq table) PE tables. The +90 degree
    rotation per step (PanFusion.py:114-123) cycles through a handful of camera sets, and the two CFG halves carry
    identical cameras (PanoGenerator.py:245-246), so after the first few steps every lookup hits."""

    def __init__(self, max_camera_sets: int = 16):
        """max_camera_sets bounds the cache (LRU over camera sets; the fixed predict rig needs 4 — one per rotation
        phase): random rigs (train-mode cam_rot / random_sample_camera, a rot_diff that does not divide 360) would
        otherwise grow device memory without limit (~35-143 MB per set at SD-2 size). Evicted tables stay alive for as
        long as a captured CUDA graph holds them (`tensors_of`)."""
        self._bias = {}
        self._pe = {}
        self._rec = {}
        self.max_camera_sets = max_camera_sets
        self._lru: list = []   # camera keys, least recently used first

    def _touch(self, key) -> None:
        if self._lru and self._lru[-1] == key:
            return
        if key in self._lru:
            self._lru.remove(key)
        self._lru.append(key)
        while len(self._lru) > self.max_camera_sets:
            old = self._lru.pop(0)
            for cache in (self._bias, self._pe, self._rec):
                for k in [k for k in cache if self._key_of(k) == old]:
                    del cache[k]

    @staticmethod
    def _key_of(cache_key):
        return cache_key[2] if cache_key[0] == "local" else cache_key[0]

    def tensors_of(self, key) -> list:
        """Every cached tensor that belongs to camera set `key` (to be held by whoever captured their addresses)."""
        key = self.dedup_any(key)
        out = []

        def collect(v):
            if torch.is_tensor(v):
                out.append(v)
            elif isinstance(v, (tuple, list)):
                for t in v:
                    collect(t)

        for cache in (self._bias, self._pe, self._rec):
            for k, v in cache.items():
                if self._key_of(k) in key:
                    collect(v)
        return out

    @staticmethod
    def dedup_any(key) -> tuple:
        """The camera keys a full (b*m)-camera key can be stored under: itself and every per-batch-element group."""
        n = len(key[0])
        keys = {key}
        for b in range(1, n + 1):
            if n % b == 0:
                keys.add(CameraTables.dedup(key, b)[0])
        return tuple(keys)

    def nbytes(self) -> int:
        """Device bytes held by the cache (bias tables in their resident form, PE tables, camera records)."""
        seen, total = set(), 0

        def walk(v):
            nonlocal total
            if torch.is_tensor(v):
                if v.data_ptr() not in seen:
                    seen.add(v.data_ptr())
                    total += v.numel() * v.element_size()
            elif isinstance(v, (tuple, list)):
                for t in v:
                    walk(t)

        for cache in (self._bias, self._pe, self._rec):
            for v in cache.values():
                walk(v)
        return total

    def clear(self) -> None:
        self._bias.clear()
        self._pe.clear()
        self._rec.clear()
        self._lru.clear()

    @staticmethod
    def camera_key(cameras: dict) -> tuple:
        vals = [cameras[k].detach().reshape(-1).to("cpu", torch.float64).tolist() for k in ("FoV", "theta", "phi")]
        return tuple(map(tuple, vals))

    def _records(self, key, m_total, ph, pw, dev):
        rk = (key, ph, pw)
        if rk not in self._rec:
            fov, theta, phi = (list(v) for v in key)
            ce, _ = geometry.camera_records("e2p", fov, theta, phi, m_total, ph, pw, dev)
            cp, _ = geometry.camera_records("p2e", fov, theta, phi, m_total, ph, pw, dev)
            self._rec[rk] = (ce, cp)
        return self._rec[rk]

    @staticmethod
    def dedup(key: tuple, b: int) -> tuple[tuple, int]:
        """If every batch element carries the same m cameras, keep one group (G = 1)."""
        n = len(key[0])
        m = n // b
        groups = [tuple(tuple(v[g * m:(g + 1) * m]) for v in key) for g in range(b)]
        if all(g == groups[0] for g in groups):
            return groups[0], 1
        return key, b

    def bias(self, key, groups, ph, pw, eh, ew, dev):
        k = (key, groups, ph, pw, eh, ew)
        self._touch(key)
        if k not in self._bias:
            V = len(key[0])
            ce, cp = self._records(key, V, ph, pw, dev)
            b1, b2 = ops.eppa_tables(ce, cp, V // groups, ph, pw, eh, ew)
            # Most (query tile, key tile) pairs have no geometric correspondence at all: the resident form keeps only the
            # ~15 % of 128 x 64 tiles that are not entirely -1 ("packed": store + tile index table). A direction whose
            # per-view query count is not a multiple of the 128-row tile (the 8x8 level) cannot be sliced by view shard and
            # stays dense (it is tiny).
            P, E = ph * pw, eh * ew
            d1 = ("packed", *ops.bias_pack_tiles(b1)) if E % 128 == 0 else ("dense", b1, ops.bias_tile_flags(b1))
            d2 = ("packed", *ops.bias_pack_tiles(b2)) if P % 128 == 0 else ("dense", b2, ops.bias_tile_flags(b2))
            self._bias[k] = (d1, d2)
        return self._bias[k]

    def pe(self, key, ph, pw, eh, ew, freq_bands: Tensor, dev):
        k = (key, ph, pw, eh, ew, freq_bands.numel())  # SphericalPE's table is a function of n_freqs only
        self._touch(key)
        if k not in self._pe:
            ce, _ = self._records(key, len(key[0]), ph, pw, dev)
            self._pe[k] = ops.eppa_pe(ce, ph, pw, eh, ew, freq_bands)
        return self._pe[k]


class WarpAttn(nn.Module):
    kv_tap = None  # test hook: called with the local views' projected K|V [b, m_loc*P, 2C] of every forward

    def __init__(self, dim):
        super().__init__()
        self.dim = dim
        self.transformer = _Block(dim, dim // 32)
        self.pe = _SphericalPE(dim // 4)
        self._packed = None
        self.tables = CameraTables()  # MultiViewBaseModel replaces this with one shared cache

    # ---- weight packing (once per device/dtype) --------------------------------------------------
    def _pack(self, dev, dt):
        if self._packed is None or self._packed["key"] != (dev, dt):
            self._packed = pack_block(self.transformer, dev, dt)
        return self._packed

    def invalidate(self):
        self._packed = None

    # ---- token-level forward used by MultiViewBaseModel -----------------------------------------
    def forward_tokens(self, pers: Img, equi: Img, cam_key: tuple, par=None, side=None, keep=None) -> tuple[Img, Img]:
        """pers: (b*m_loc) images of ph x pw, equi: b images of eh x ew; cam_key = CameraTables.camera_key(cameras)
        of ALL b*m cameras. `par` (parallel.ViewParallel) marks pers as this rank's slice of the views: the K|V of
        the other view shards arrive through one all-gather, everything else is local."""
        dev, dt = pers.t.device, pers.t.dtype
        w = self._pack(dev, dt)
        C = self.dim
        b = equi.N
        m = len(cam_key[0]) // b               # views per batch element, all shards
        m_loc = pers.N // b                    # views held by this rank
        v0 = par.vs * m_loc if par is not None else 0
        ph, pw, eh, ew = pers.H, pers.W, equi.H, equi.W
        P, E = ph * pw, eh * ew
        key, groups = CameraTables.dedup(cam_key, b)
        d1, d2 = self.tables.bias(key, groups, ph, pw, eh, ew, dev)  # direction 1 [G, E, m*P], direction 2 [G, m*P, E]
        pers_pe, equi_pe = self.tables.pe(key, ph, pw, eh, ew, self.pe.freq_bands, dev)  # [G*m*P, C], [E, C]
        kw1 = dict(bias_tiles=(d1[1], d1[2])) if d1[0] == "packed" else dict(bias=d1[1], bias_flags=d1[2])
        if m_loc != m:
            # this rank's views = a contiguous range of direction 2's query rows
            if d2[0] == "packed":
                off2 = d2[2][:, (v0 * P) // 128:((v0 + m_loc) * P) // 128].contiguous()
                kw2 = dict(bias_tiles=(d2[1], off2))
            else:
                bias2 = d2[1][:, v0 * P:(v0 + m_loc) * P]
                # flag rows are 128-query tiles: usable for the local slice only when it starts on a tile boundary
                flags2 = d2[2][:, (v0 * P) // 128:((v0 + m_loc) * P + 127) // 128].contiguous() \
                    if (v0 * P) % 128 == 0 and (m_loc * P) % 128 == 0 else None
                kw2 = dict(bias=bias2, bias_flags=flags2)
            pers_pe = pers_pe.reshape(groups, m * P, C)[:, v0 * P:(v0 + m_loc) * P].reshape(groups * m_loc * P, C)
            pers_pe = pers_pe if pers_pe.is_contiguous() else self._local_pe(pers_pe, (key, ph, pw, v0, m_loc))
        else:
            kw2 = dict(bias_tiles=(d2[1], d2[2])) if d2[0] == "packed" else dict(bias=d2[1], bias_flags=d2[2])
        heads, d = w["heads"], C // w["heads"]
        Tp, Te = b * m_loc * P, b * E
        new = lambda rows, n: torch.empty((rows, n), dtype=dt, device=dev)
        # norm1(x + pe) for both token sets (transformer.py:153-158: query_pe added to the query, context carries its
        # own pe, both through the SAME norm1), then one fused q/k/v projection each
        ap = ops.layernorm(pers.t, w["ln1"].g, w["ln1"].b, w["ln1"].eps, pers_pe)
        ae = ops.layernorm(equi.t, w["ln1"].g, w["ln1"].b, w["ln1"].eps, equi_pe)
        qkv_p = ops.gemm_taps(ap, w["qkv"].w, new(Tp, 3 * C), M=Tp, Kc=C).reshape(b, m_loc * P, 3 * C)
        qkv_e = ops.gemm_taps(ae, w["qkv"].w, new(Te, 3 * C), M=Te, Kc=C).reshape(b, E, 3 * C)
        scale = d ** -0.5
        if WarpAttn.kv_tap is not None:
            WarpAttn.kv_tap(qkv_p[..., C:])
        if m_loc != m:
            # the one collective of the block: K|V of every view shard (bf16, 2C per token) over NVLink
            kv_loc = new(Tp, 2 * C)
            ops.copy2d(qkv_p.reshape(Tp, 3 * C)[:, C:], kv_loc)
            kv_all = par.gather_views(kv_loc.reshape(b, m_loc * P, 2 * C))
            k_all, v_all = kv_all[..., :C], kv_all[..., C:]
        else:
            k_all, v_all = qkv_p[..., C:2 * C], qkv_p[..., 2 * C:]

        finish = lambda o, x_tok, rows: block_tail(w, o, x_tok, rows)

        # The two directions only share their inputs: direction 1 (few pano tokens, under-filled launches) runs on the
        # panorama branch's side stream, concurrently with direction 2 on the caller's stream. Its result is consumed
        # by the panorama branch on that same stream, so no join is needed here; the shared inputs produced on the
        # caller's stream are parked in `keep` until the branches next join.
        main = torch.cuda.current_stream()
        two = side is not None and side is not main
        if two:
            side.wait_event(main.record_event())
            if keep is not None:
                keep.extend([qkv_p, qkv_e, k_all, v_all, equi.t])
        # direction 1 (modules.py:44-48): pano pixels query every view's pixels
        with torch.cuda.stream(side if two else main):
            o1 = torch.empty((b, E, C), dtype=dt, device=dev)
            ops.fmha(qkv_e[..., :C], k_all, v_all, o1, heads=heads, head_dim=d, scale=scale, **kw1)
            equi_out = finish(o1.reshape(Te, C), equi.t, Te)
        # direction 2 (modules.py:51-55): view pixels query the pano; reads the INPUT features
        o2 = torch.empty((b, m_loc * P, C), dtype=dt, device=dev)
        ops.fmha(qkv_p[..., :C], qkv_e[..., C:2 * C], qkv_e[..., 2 * C:], o2, heads=heads, head_dim=d, scale=scale, **kw2)
        pers_out = finish(o2.reshape(Tp, C), pers.t, Tp)
        return Img(pers_out, b * m_loc, ph, pw), Img(equi_out, b, eh, ew)

    def _local_pe(self, pe_view: Tensor, key) -> Tensor:
        cache = self.tables._pe
        k = ("local", self.dim) + key
        if k not in cache:
            cache[k] = pe_view.contiguous()
        return cache[k]

    # ---- reference signature (NCHW in / out) -------------------------------------------------------
    def forward(self, pers_x: Tensor, equi_x: Tensor, cameras: dict, compute_dtype: torch.dtype | None = None):
        dt = compute_dtype or (pers_x.dtype if pers_x.dtype in (torch.float16, torch.bfloat16) else torch.bfloat16)
        po, eo = self.forward_tokens(img_from_nchw(pers_x, dt), img_from_nchw(equi_x, dt),
                                     CameraTables.camera_key(cameras))
        return po.nchw().to(pers_x.dtype).contiguous(), eo.nchw().to(equi_x.dtype).contiguous()
