"""-m gpu: the panorama branch's conv_out and copy2d (pf_copy2d) against plain PyTorch fp32 on the same 16-bit-rounded
inputs, pad_pano (pf_pad_pano) bit for bit, and the EPPA tables (pf_eppa_tables, pf_eppa_pe) against the oracle's
get_masks / get_coords / SphericalPE (models/pano/utils.py:10-106, transformer.py:185-201). conv_in is held to its fp64
contract in test_gpu_elementwise_contract.py; GroupNorm, LayerNorm, CFG + DDIM and the timestep embedding in
test_gpu_norm_contract.py."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("circ", [False, True])
def test_branch_conv_out(cuda_device, circ):
    from panfusion_b200 import engine
    from panfusion_b200.packing import pack_conv3x3
    from oracle.eppa import pad_pano, unpad_pano
    g = torch.Generator().manual_seed(4)
    N, H, W, C = 2, 16, 32, 320
    conv = lambda x, w, b: unpad_pano(F.conv2d(pad_pano(x, 1), w, b, padding=1), 1) if circ else F.conv2d(x, w, b, padding=1)
    # conv_norm_out -> SiLU -> conv_out, as Branch.conv_out runs it: pf_gn_prep, then the 64-wide tap-GEMM
    x = torch.randn(N, C, H, W, generator=g).half()
    gamma, beta = torch.randn(C, generator=g), torch.randn(C, generator=g)
    w_out, b_out = torch.randn(4, C, 3, 3, generator=g) * 0.05, torch.randn(4, generator=g)
    ref = conv(F.silu(F.group_norm(x.float(), 32, gamma, beta, 1e-5)), w_out, b_out)
    # the fields of engine.UNetPack that Branch.conv_out reads: 4 output channels zero-padded to one 64-wide tile
    wpad, bpad = torch.zeros(64, C, 3, 3), torch.zeros(64)
    wpad[:4], bpad[:4] = w_out, b_out
    norm = SimpleNamespace(weight=gamma, bias=beta, eps=1e-5, num_groups=32)
    pack = SimpleNamespace(dt=torch.float16, groups=32, norm_out=engine._Norm(norm, cuda_device), conv_out_c=4,
                           conv_out_packed=pack_conv3x3(wpad).to(cuda_device, torch.float16).contiguous(),
                           conv_out_bpad=bpad.to(cuda_device))
    br = engine.Branch(pack, circular=circ)
    got = br.conv_out(engine.img_from_nchw(x.to(cuda_device), torch.float16))
    # the prepared activations and the packed weights are rounded to fp16
    torch.testing.assert_close(got.cpu(), ref, rtol=2e-3, atol=3e-3)


def test_copy2d(cuda_device):
    from panfusion_b200 import ops
    src = torch.randn(50, 64).half().to(cuda_device)
    dst = torch.zeros(50, 192, dtype=torch.float16, device=cuda_device)
    ops.copy2d(src, dst[:, 64:128])
    assert torch.equal(dst[:, 64:128], src) and dst[:, :64].abs().sum() == 0 and dst[:, 128:].abs().sum() == 0


def _cams(n, seed=0):
    rng = np.random.default_rng(seed)
    return dict(FoV=torch.tensor(rng.uniform(70, 100, n), dtype=torch.float32),
                theta=torch.tensor(rng.uniform(0, 360, n), dtype=torch.float32),
                phi=torch.tensor(rng.uniform(-60, 60, n), dtype=torch.float32))


@pytest.mark.parametrize("ph,pw,eh,ew,V,m", [(8, 8, 8, 16, 3, 3), (16, 16, 16, 32, 4, 2), (8, 8, 16, 32, 2, 1),
                                            (32, 32, 32, 64, 2, 2)])
def test_eppa_tables_vs_oracle(cuda_device, ph, pw, eh, ew, V, m):
    """Bias tables == get_masks (utils.py:10-84) rearranged like modules.py:46,53; PE == SphericalPE(get_coords)."""
    from oracle import eppa as oe
    from panfusion_b200 import geometry as pg, ops
    cams = _cams(V, seed=ph + V)
    if ph == 32:  # the reference's own rig: horizon cameras
        cams = dict(FoV=torch.tensor([90.0, 90.0]), theta=torch.tensor([0.0, 180.0]), phi=torch.zeros(2))
    pm, em = oe.get_masks(ph, pw, eh, ew, cams)
    P, E = ph * pw, eh * ew
    ref1 = pm.reshape(V // m, m, E, P).permute(0, 2, 1, 3).reshape(V // m, E, m * P)
    ref2 = em.reshape(V // m, m * P, E)
    ce, _ = pg.camera_records("e2p", cams["FoV"], cams["theta"], cams["phi"], V, ph, pw, cuda_device)
    cp, _ = pg.camera_records("p2e", cams["FoV"], cams["theta"], cams["phi"], V, ph, pw, cuda_device)
    b1, b2 = ops.eppa_tables(ce, cp, m, ph, pw, eh, ew)
    torch.testing.assert_close(b1.cpu(), ref1, rtol=1e-5, atol=2e-6)
    torch.testing.assert_close(b2.cpu(), ref2, rtol=1e-5, atol=2e-6)
    for dim in (320, 640):
        pe_mod = oe.SphericalPE(dim // 4)
        pc, ec = oe.get_coords(ph, pw, eh, ew, cams)
        rp, re = pe_mod(pc).reshape(V * P, dim), pe_mod(ec).reshape(E, dim)
        gp, ge = ops.eppa_pe(ce, ph, pw, eh, ew, pe_mod.freq_bands)
        # sin/cos of arguments up to 2^79: both sides are correctly-rounded-ish fp32 libm results of the SAME fp32
        # argument; allow a few ulp
        torch.testing.assert_close(gp.cpu(), rp, rtol=0, atol=5e-6)
        torch.testing.assert_close(ge.cpu(), re, rtol=0, atol=5e-6)


def test_eppa_tables_vs_reference_goldens(cuda_device):
    """The CUDA bias tables against the goldens minted by executing the reference's get_masks (not the oracle):
    the 3-camera rig of tests/golden/eppa_geometry.npz and BASELINE config 4's geometry (ph != eh, icosahedron rings)."""
    from pathlib import Path
    import numpy as np
    from panfusion_b200 import geometry as pg, ops
    gdir = Path(__file__).parent / "golden"
    cases = [("eppa_geometry.npz", (8, 8, 8, 16), dict(FoV=torch.tensor([90.0, 75.0, 100.0]),
                                                       theta=torch.tensor([0.0, 45.0, 200.0]),
                                                       phi=torch.tensor([0.0, 30.0, -60.0]))),
             ("eppa_geometry_c4.npz", (8, 8, 16, 32), dict(FoV=torch.full((4,), 90.0),
                                                           theta=torch.tensor([-144.0, 72.0, -180.0, 36.0]),
                                                           phi=torch.tensor([52.6226, 10.8123, -10.8123, -52.6226])))]
    for fname, (ph, pw, eh, ew), cams in cases:
        gold = np.load(gdir / fname)
        V, P, E = len(cams["FoV"]), ph * pw, eh * ew
        pm, em = torch.from_numpy(gold["pers_masks"]), torch.from_numpy(gold["equi_masks"])
        ref1 = pm.reshape(1, V, E, P).permute(0, 2, 1, 3).reshape(1, E, V * P)   # modules.py:46
        ref2 = em.reshape(1, V * P, E)                                           # modules.py:53
        ce, _ = pg.camera_records("e2p", cams["FoV"], cams["theta"], cams["phi"], V, ph, pw, cuda_device)
        cp, _ = pg.camera_records("p2e", cams["FoV"], cams["theta"], cams["phi"], V, ph, pw, cuda_device)
        b1, b2 = ops.eppa_tables(ce, cp, V, ph, pw, eh, ew)
        torch.testing.assert_close(b1.cpu(), ref1, rtol=1e-5, atol=2e-6)
        torch.testing.assert_close(b2.cpu(), ref2, rtol=1e-5, atol=2e-6)


def test_eppa_tables_config4_level_size_vs_reference_golden(cuda_device):
    """pf_eppa_tables at config 4's real first EPPA level (32x32 views / 64x128 pano, icosahedron rings) against the
    reference-run golden: a strided subset of the query rows element-wise, the key-sum of EVERY row."""
    from pathlib import Path
    import numpy as np
    from oracle.make_golden import C4GEO_LEVEL, _cams_ico
    from panfusion_b200 import geometry as pg, ops
    gold = np.load(Path(__file__).parent / "golden" / "eppa_geometry_c4_level.npz")
    ph, pw, eh, ew = C4GEO_LEVEL
    cams = _cams_ico()
    V, P, E = len(cams["FoV"]), ph * pw, eh * ew
    ce, _ = pg.camera_records("e2p", cams["FoV"], cams["theta"], cams["phi"], V, ph, pw, cuda_device)
    cp, _ = pg.camera_records("p2e", cams["FoV"], cams["theta"], cams["phi"], V, ph, pw, cuda_device)
    b1, b2 = ops.eppa_tables(ce, cp, V, ph, pw, eh, ew)          # [1, E, V*P], [1, V*P, E]
    pm = b1.reshape(eh, ew, V, ph, pw).permute(2, 0, 1, 3, 4)     # -> pers_masks [V, eh, ew, ph, pw] (modules.py:46)
    em = b2.reshape(V, ph, pw, eh, ew)                            # -> equi_masks [V, ph, pw, eh, ew] (modules.py:53)
    torch.testing.assert_close(pm[:, ::7, ::9].cpu(), torch.from_numpy(gold["pers_rows"]), rtol=1e-5, atol=2e-6)
    torch.testing.assert_close(em[:, ::5, ::5].cpu(), torch.from_numpy(gold["equi_rows"]), rtol=1e-5, atol=2e-6)
    torch.testing.assert_close(pm.double().sum((-1, -2)).cpu(), torch.from_numpy(gold["pers_rowsum"]), rtol=0, atol=2e-3)
    torch.testing.assert_close(em.double().sum((-1, -2)).cpu(), torch.from_numpy(gold["equi_rowsum"]), rtol=0, atol=2e-3)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.uint8])
def test_pad_pano_bit_exact(cuda_device, dtype):
    """pad_pano / unpad_pano (utils/pano.py:74-105): 4-D and 5-D, every dtype width, against the oracle restatement
    (itself pinned to the reference in tests/test_oracle_golden.py)."""
    from oracle.eppa import pad_pano as ref_pad
    from panfusion_b200.pano import pad_pano, unpad_pano
    g = torch.Generator().manual_seed(3)
    for shape in ((2, 3, 5, 16), (2, 2, 3, 4, 12)):
        x = (torch.rand(shape, generator=g) * 200).to(dtype)
        for p in (1, 2, 8):
            got = pad_pano(x.to(cuda_device), p)
            ref = ref_pad(x.float(), p).to(dtype)
            assert got.shape == ref.shape and torch.equal(got.cpu(), ref)
            assert torch.equal(unpad_pano(got, p).cpu(), x)
    xd = x.to(cuda_device)
    assert pad_pano(xd, 0) is xd and unpad_pano(xd, 0) is xd
    with pytest.raises(NotImplementedError):
        pad_pano(torch.zeros(3, 4, 5, device=cuda_device), 1)
