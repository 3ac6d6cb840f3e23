"""CPU (-m "not gpu"): the FID InceptionV3 oracle (oracle/inception.py) against torchvision's Inception3 and
tests/golden/inception.npz; the TF1 resize; BN folding, packing and the state-dict loader of panfusion_b200.inception;
the IS chunking; the seeded network's non-degeneracy; the metrics' module behaviour and argument checks."""
from pathlib import Path

import numpy as np
import pytest
import torch
from torchvision.models import inception as tvi

from oracle import inception as oi

GOLD = np.load(Path(__file__).parent / "golden" / "inception.npz")


@pytest.fixture(scope="module")
def sd():
    return oi.synth_state(int(GOLD["seed"]))


def test_golden_weights_regenerate(sd):
    assert str(GOLD["weights_sha256"]) == oi.state_sha256(sd)


def test_graph_matches_torchvision_without_fid_deviations(sd):
    """With the four FID deviations off, the oracle's forward is torchvision's Inception3(aux_logits=False) at pool3.
    The strict state-dict load pins torch-fidelity's key names on torchvision's modules."""
    ref = tvi.Inception3(num_classes=1008, aux_logits=False, init_weights=False).eval()
    ref.load_state_dict(sd)
    seen = {}
    ref.avgpool.register_forward_hook(lambda m, i, o: seen.setdefault("pool3", o.flatten(1)))
    x = oi.feature_images(0)[:1]
    with torch.no_grad():
        ref(oi.prep(x))
    net = oi.network(fid=False)
    net.load_state_dict(sd)
    got, _ = oi.features(net, x)
    want = seen["pool3"]
    assert (got - want).abs().max() <= 1e-5 * want.abs().max()
    fid_net = oi._net(sd, torch.float32)
    assert not torch.equal(oi.features(fid_net, x)[0], got)  # the deviations do change the features


def test_conv_table_matches_torchvision():
    from panfusion_b200.inception import CONVS
    net = oi.network()
    convs = [n[:-len(".conv")] for n, m in net.named_modules() if isinstance(m, torch.nn.Conv2d)]
    assert list(CONVS) == convs and len(convs) == 94
    for name, (cin, cout, kh, kw, s, ph, pw) in CONVS.items():
        m = net.get_submodule(name).conv
        assert (m.in_channels, m.out_channels, m.kernel_size, m.stride, m.padding) == \
            (cin, cout, (kh, kw), (s, s), (ph, pw)), name


def test_oracle_matches_golden(sd):
    net = oi._net(sd, torch.float64)
    p, l = oi.features(net, oi.feature_images(0), torch.float64)
    for name, got in (("pool3", p), ("logits", l)):
        ref = GOLD[f"{name}_299x299"].astype(np.float64)
        assert np.abs(got.numpy() - ref).max() <= 1e-6 * np.abs(ref).max(), name


def test_resize_identity_and_hand_examples():
    x = torch.rand(2, 3, 299, 299) * 255
    assert torch.equal(oi.resize_tf1(x, (299, 299)), x)
    a = torch.tensor([10.0, 20.0, 50.0]).view(1, 1, 1, 3)
    # 3 -> 2: scale 1.5, g = [0, 1.5]
    assert torch.allclose(oi.resize_tf1(a, (1, 2)), torch.tensor([10.0, 35.0]).view(1, 1, 1, 2))
    b = torch.tensor([10.0, 20.0]).view(1, 1, 2, 1)
    # 2 -> 5: scale 0.4, g = [0, .4, .8, 1.2, 1.6]; rows past the last input row clamp to it
    want = torch.tensor([10.0, 14.0, 18.0, 20.0, 20.0]).view(1, 1, 5, 1)
    assert torch.allclose(oi.resize_tf1(b, (5, 1)), want, atol=1e-5)


def test_bn_folding_and_packing(sd):
    from panfusion_b200 import inception
    name = "Mixed_6b.branch7x7_2"
    x = torch.randn(2, 128, 9, 9, dtype=torch.float64)
    m = oi.network().get_submodule(name).double()
    m.load_state_dict({k[len(name) + 1:]: v for k, v in sd.items() if k.startswith(name + ".")})
    with torch.no_grad():
        ref = m.eval()(x)
    w, b = inception.fold_bn(sd, name)
    got = torch.nn.functional.conv2d(x, w, b, padding=(0, 3)).relu()
    assert (got - ref).abs().max() <= 1e-12 * ref.abs().max()
    p = inception.pack_weight(w, 128)
    assert p.shape == (7, 128, 128) and p.dtype == torch.float16 and p[5, 11, 7] == w[7, 11, 0, 5].half()
    p = inception.pack_weight(inception.fold_bn(sd, "Mixed_5b.branch5x5_1")[0], 192)
    assert p.shape == (1, 192, 64) and not p[..., 48:].any()  # Cout 48 padded to one 64-wide tile
    p = inception.pack_weight(inception.fold_bn(sd, "Conv2d_1a_3x3")[0], 16)
    assert p.shape == (9, 16, 32) and not p[:, 3:].any()
    assert [inception.packed_cout(c) for c in (32, 48, 80, 192, 448)] == [32, 64, 128, 192, 448]


def test_loader_rejects_missing_and_misshaped_keys(sd, tmp_path):
    from panfusion_b200 import inception
    bad = dict(sd)
    del bad["Mixed_6c.branch7x7dbl_3.bn.running_var"]
    with pytest.raises(ValueError, match="Mixed_6c.branch7x7dbl_3.bn.running_var"):
        inception.InceptionV3(bad)
    bad = dict(sd)
    bad["fc.weight"] = torch.zeros(1000, 2048)
    with pytest.raises(ValueError, match="fc.weight"):
        inception.InceptionV3(bad)
    path = tmp_path / "pt_inception-2015-12-05-6726825d.pth"
    torch.save(sd, path)
    net = inception.InceptionV3(str(path))
    assert net.fc_w.shape == (1008, 2048) and net.Conv2d_1a_3x3_w.shape == (9, 16, 32)


def test_inception_score_chunks():
    assert oi.chunk_count(25, 10) == 9 and oi.chunk_count(40, 10) == 10 and oi.chunk_count(7, 1) == 1
    m, s = oi.inception_score(torch.randn(7, 1008, dtype=torch.float64), 1, 0)
    assert m > 1 and np.isnan(s)  # one chunk: std is nan, as torch gives


def test_seeded_network_is_not_degenerate():
    assert float(GOLD["pool3_zero_fraction"]) < 0.5
    assert 0.05 < float(GOLD["softmax_max_mean"]) < 0.9  # neither uniform (1/1008) nor one-hot
    for n, _, _ in oi.IS_CASES:
        assert float(GOLD[f"is_{n}_mean"]) > 1.03 and float(GOLD[f"is_{n}_std"]) > 0
    for tag in ("rd", "fr"):
        tr = 0.0
        for side in ("real", "fake"):
            n, s = int(GOLD[f"{tag}_{side}_num_samples"]), GOLD[f"{tag}_{side}_sum"]
            tr += (GOLD[f"{tag}_{side}_cov_sum_diag"].sum() - (s * s).sum() / n) / (n - 1)
        assert float(GOLD[f"{tag}_fid"]) > tr, tag  # far from 0: larger than tr S1 + tr S2


def test_golden_statistics_are_consistent():
    for tag in ("rd", "fr"):
        for side in ("real", "fake"):
            n = int(GOLD[f"{tag}_{side}_num_samples"])
            assert n == {"rd": 20, "fr": 2100}[tag]
            assert GOLD[f"{tag}_{side}_sum"].shape == (2048,) and GOLD[f"{tag}_{side}_cov_sum_diag"].shape == (2048,)
            assert float(GOLD[f"{tag}_{side}_cov_sum_fro"]) >= np.abs(GOLD[f"{tag}_{side}_cov_sum_diag"]).max()


def test_metrics_are_modules_like_torchmetrics(sd):
    from panfusion_b200 import inception
    net = inception.InceptionV3(sd)
    d = torch.nn.ModuleDict({"FID": inception.FrechetInceptionDistance(inception=net),
                             "FID_crop": inception.FrechetInceptionDistance(normalize=True, inception=net),
                             "IS": inception.InceptionScore(inception=net)})
    d.requires_grad_(False)
    m = d["FID"]
    assert m.inception is d["IS"].inception and not m._update_called
    bufs = dict(m.named_buffers())
    for side in ("real", "fake"):
        assert bufs[f"{side}_features_sum"].shape == (2048,) and bufs[f"{side}_features_sum"].dtype == torch.float64
        assert bufs[f"{side}_features_cov_sum"].shape == (2048, 2048)
        assert bufs[f"{side}_features_num_samples"].dtype == torch.int64
    assert bufs["inception.fc_w"].dtype == torch.float32 and bufs["inception.Mixed_7c_branch_pool_w"].dtype == torch.float16
    assert not d.state_dict()  # states and packed weights are non-persistent, like torchmetrics' states
    with pytest.raises(ValueError, match="uint8"):
        m.update(torch.rand(2, 3, 64, 64), real=True)
    with pytest.raises(ValueError, match="float32"):
        d["FID_crop"].update(torch.zeros(2, 3, 64, 64, dtype=torch.uint8), real=True)
    with pytest.raises(Exception):
        m.update(torch.zeros(2, 3, 64, 64, dtype=torch.uint8), real=True)  # CPU images: no CPU path
    assert not m._update_called
    m.reset()
    d["IS"].reset()
    assert not d["IS"]._update_called and d["IS"].features == []
    with pytest.raises(ValueError):
        inception.FrechetInceptionDistance(feature=768, inception=net)
    with pytest.raises(ValueError):
        inception.InceptionScore(feature="logits", inception=net)
    with pytest.raises(RuntimeError, match="More than one sample"):
        m.compute()


def test_inception_entry_points_reject_bad_arguments():
    import ctypes as C
    from panfusion_b200 import _lib
    l = _lib.lib()
    assert l.pf_inception_prep(None, 1, 1, 64, 64, None, None) == -1
    assert l.pf_conv2d_nhwc(1, 1, 8, 8, 24, 1, 1, 32, 3, 3, 1, 1, 1, 1, 1, 1, 32, 0, None) == -1  # Cin % 16
    assert l.pf_conv2d_nhwc(1, 1, 8, 8, 32, 1, 1, 32, 9, 9, 1, 4, 4, 1, 1, 1, 32, 0, None) == -1  # 9x9
    assert l.pf_conv2d_nhwc(1, 1, 8, 8, 32, 1, 1, 32, 3, 3, 1, 1, 1, 1, 1, 1, 40, 16, None) == -1  # slice overflow
    assert l.pf_conv2d_nhwc(1, 1, 8, 8, 32, 1, 1, 32, 3, 3, 1, 1, 1, 1, 1, 2, 32, 0, None) == -1  # bf16 output
    assert l.pf_pool2d_nhwc(1, 1, 8, 8, 64, 5, 1, 1, 1, 64, 0, None) == -1
    assert l.pf_pool2d_nhwc(1, 1, 8, 8, 60, 0, 1, 1, 1, 64, 0, None) == -1
    assert l.pf_inception_head(None, 1, 64, 2048, 1, 1008, 1, 1, None) == -1
    assert l.pf_inception_score(1, 1, 0, 1008, 10, 1, 1, None) == -1
    assert [l.pf_conv2d_packed_cout(c) for c in (32, 48, 80, 384)] == [32, 64, 128, 384]
    l.pf_inception_score_ws_doubles.restype = C.c_longlong
    assert l.pf_inception_score_ws_doubles(25, 1008, 10) == 2 * 25 * 1008 + 10 * 1009
