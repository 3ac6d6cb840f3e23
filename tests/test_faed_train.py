"""CPU: the FAED training restatement and host code (panfusion_b200.faed_train, panfusion_b200.train_faed)."""
from pathlib import Path

import numpy as np
import pytest
import torch
from PIL import Image

from oracle import faed_train as of
from panfusion_b200 import faed_train as ft, train_faed

GOLD = np.load(Path(__file__).parent / "golden" / "faed_train.npz")
N_PARAMS = 5166019


def test_init_matches_reference_hash_and_names():
    """tests/golden/faed_train.npz holds the SHA-256 and key list of the reference's `torch.manual_seed(0);
    AutoEncoder()` state dict; the oracle's module-free initialisation and the trainer's module reproduce both."""
    sd = ft.init_state(int(GOLD["seed"]))
    assert list(sd) == list(GOLD["keys"])
    assert of.state_sha256(sd) == str(GOLD["init_sha256"])
    assert of.state_sha256(of.init_state(int(GOLD["seed"]))) == str(GOLD["init_sha256"])
    net = ft.AutoEncoder()
    assert sum(p.numel() for p in net.parameters()) == N_PARAMS
    assert sum(isinstance(m, torch.nn.Conv2d) for m in net.modules()) == 30
    state = torch.random.get_rng_state()
    ft.init_state(1)
    assert torch.equal(state, torch.random.get_rng_state())  # the global RNG is left alone


def test_oracle_restatement_matches_golden():
    """Three fp64 training steps (forward, autograd backward, Adam restated op by op) against the reference's
    modules.py and torch.optim.Adam."""
    err, where = of.max_rel_error(GOLD, of.restated_run(of.init_state(int(GOLD["seed"]))))
    assert err <= 1e-10, (err, where)


def test_trainer_module_matches_golden():
    """faed_train.AutoEncoder (the GPU tests' fp64 reference) with torch.optim.Adam reproduces the golden."""
    net = ft.AutoEncoder().double().train()
    net.load_state_dict(ft.init_state(int(GOLD["seed"])))
    opt = torch.optim.Adam(net.parameters(), lr=of.LR, foreach=False)
    run = {}
    for s in range(of.STEPS):
        x = of.panos(s)
        opt.zero_grad()
        loss = (net(x) - x).abs().mean()
        loss.backward()
        grads = [(n, p.grad.clone()) for n, p in net.named_parameters()]
        opt.step()
        run[f"step{s}/loss"] = loss.item()
        bufs = {f"step{s}/{k}": v for k, v in net.state_dict().items() if "running" in k}
        for k, v in of.digests(grads, bufs).items():
            run[k if k.startswith("step") else f"step{s}/{k}"] = v
    err, where = of.max_rel_error(GOLD, run)
    assert err <= 1e-10, (err, where)


def test_circular_pad():
    x = torch.arange(2 * 4 * 6, dtype=torch.float64).reshape(1, 2, 4, 6)
    y = ft.circular_pad(x, 2)
    assert y.shape == (1, 2, 8, 10)
    assert torch.equal(y[..., 2:6, 2:8], x)
    assert torch.equal(y[..., 2:6, :2], x[..., -2:]) and torch.equal(y[..., 2:6, -2:], x[..., :2])
    assert not y[..., :2, :].any() and not y[..., -2:, :].any()


def test_host_data_path(tmp_path):
    rng = np.random.default_rng(0)
    for i in range(5):
        Image.fromarray(rng.integers(0, 256, (40, 80, 3), dtype=np.uint8)).save(tmp_path / f"p{i}.png")
    Image.fromarray(rng.integers(0, 256, (40, 80, 4), dtype=np.uint8), "RGBA").save(tmp_path / "rgba.png")
    a = train_faed.load_pano(str(tmp_path / "p0.png"), 32, False)
    f = train_faed.load_pano(str(tmp_path / "p0.png"), 32, True)
    assert a.shape == (3, 32, 64) and a.dtype == np.float32 and -1 <= a.min() and a.max() <= 1
    src = np.array(Image.open(tmp_path / "p0.png"))
    import cv2
    ref = cv2.resize(src, (64, 32), interpolation=cv2.INTER_AREA).astype(np.float32) / 127.5 - 1
    np.testing.assert_array_equal(a, ref.transpose(2, 0, 1))
    ref_f = cv2.resize(np.ascontiguousarray(src[:, ::-1]), (64, 32), interpolation=cv2.INTER_AREA)
    np.testing.assert_array_equal(f, (ref_f.astype(np.float32) / 127.5 - 1).transpose(2, 0, 1))
    assert train_faed.load_pano(str(tmp_path / "rgba.png"), 32, False).shape == (3, 32, 64)
    import random
    from concurrent.futures import ThreadPoolExecutor
    paths = sorted(str(p) for p in tmp_path.glob("*.png"))
    with ThreadPoolExecutor(2) as pool:
        bs = list(train_faed.batches(paths, 32, 4, random.Random(0), pool))
    assert len(bs) == 1 and bs[0].shape == (4, 3, 32, 64) and bs[0].dtype == torch.float32
    with pytest.raises(SystemExit):
        train_faed.main(["--images", str(tmp_path / "*.png"), "--pano-height", "40"])
    with pytest.raises(SystemExit):
        train_faed.main(["--images", str(tmp_path / "none*.png")])
