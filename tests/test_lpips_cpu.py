"""LPIPS (VGG) and SSIM without a GPU: the fp64 oracle against the reference golden, the bf16-emulating oracle against
fp64 (the precision decision's regression guard), strict state-dict loading, the checkpoint-file mapping and the
argument rules of gaussiananything_b200/lpips.py."""
import json
import os

import numpy as np
import pytest
import torch

from gaussiananything_b200 import lpips as lp
from oracle import lpips_oracle as lo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "lpips_small.npz")
KEYS = os.path.join(ROOT, "tests", "golden", "lpips_vgg_keys.json")
SIZES = ("64x64", "50x70")
# bf16 convolutions against fp64, absolute on the LPIPS value: rounding noise enters squared, so near-identical pairs
# have a large relative but a tiny absolute error; 1e-3 is below the third decimal LPIPS is reported at
BF16_ABS = 1e-3


@pytest.fixture(scope="module")
def golden():
    with np.load(GOLDEN) as z:
        g = {k: z[k] for k in z.files}
    sd = lo.random_state_dict(int(g["seed"]))
    for k, v in sd.items():                  # the stored weights are regenerated from the seed: check they are the same
        assert float(v.double().sum()) == pytest.approx(float(g["sum/" + k]), rel=1e-12, abs=1e-12), k
        assert np.array_equal(v.reshape(-1)[:4].numpy(), g["first/" + k]), k
    return g, sd


def _pair(g, size):
    return torch.from_numpy(g[size + "/in0"]), torch.from_numpy(g[size + "/in1"])


@pytest.mark.parametrize("size", SIZES)
def test_fp64_oracle_reproduces_reference_golden(golden, size):
    g, sd = golden
    a, b = _pair(g, size)
    r = lo.lpips(sd, a, b)
    per, val = torch.from_numpy(g[size + "/per_tap"]).double(), torch.from_numpy(g[size + "/value"]).double()
    assert float(((r["per_tap"] - per).abs() / per.abs()).max()) <= 1e-5
    assert float(((r["value"] - val).abs() / val.abs()).max()) <= 1e-5
    s = lo.ssim((a + 1) / 2, (b + 1) / 2)
    assert float((s - torch.from_numpy(g[size + "/ssim"]).double()).abs().max()) <= 1e-6


def test_bf16_oracle_within_abs_tolerance_of_fp64(golden):
    """The golden pairs (another view, noise sigma 0.05, blur, 2-pixel shift) plus near-identical pairs (noise sigma
    0.01 and 0.002 on [0, 1]) and an identical pair."""
    g, sd = golden
    worst = 0.0
    for size in SIZES:
        a, b = _pair(g, size)
        gen = torch.Generator().manual_seed(5)
        near = [(a[:1] + s * 2 * torch.randn(a[:1].shape, generator=gen)).clamp(-1, 1) for s in (0.01, 0.002)]
        a2, b2 = torch.cat([a, a[:1], a[:1], a[:1]]), torch.cat([b, near[0], near[1], a[:1]])
        e = lo.lpips(sd, a2, b2, emulate_bf16=True)["value"]
        f = lo.lpips(sd, a2, b2)["value"]
        err = (e - f).abs()
        print(size, "lpips fp64", f.tolist(), "bf16 - fp64", (e - f).tolist())
        assert float(e[-1]) == 0.0
        worst = max(worst, float(err.max()))
    assert worst <= BF16_ABS, worst


def test_key_table_matches_reference_module():
    with open(KEYS) as f:
        want = {k: tuple(v) for k, v in json.load(f).items()}
    assert lp.state_dict_shapes() == want


def test_strict_state_dict_loading():
    sd = lo.random_state_dict(0)
    lp.check_state_dict(sd)
    lp.check_state_dict({k: v for k, v in sd.items() if not k.startswith("scaling_layer.")})     # optional buffers
    with pytest.raises(RuntimeError, match="net.slice3.12.bias"):
        lp.check_state_dict({k: v for k, v in sd.items() if k != "net.slice3.12.bias"})
    with pytest.raises(RuntimeError, match="lin5.model.1.weight"):
        lp.check_state_dict(dict(sd, **{"lin5.model.1.weight": torch.zeros(1, 8, 1, 1)}))
    with pytest.raises(RuntimeError, match="lin0.model.1.weight"):
        lp.check_state_dict(dict(sd, **{"lin0.model.1.weight": torch.zeros(1, 32, 1, 1)}))


def _write_checkpoints(d, sd):
    vgg = {"features.%d.%s" % (i, p): sd["net.slice%d.%d.%s" % (k + 1, i, p)] for k, i, _, _ in lp.CONVS
           for p in ("weight", "bias")}
    vgg["classifier.0.weight"] = torch.zeros(4, 4)
    lin = {"lin%d.model.1.weight" % k: sd["lin%d.model.1.weight" % k] for k in range(5)}
    torch.save(vgg, os.path.join(d, lp.VGG_FILE))
    torch.save(lin, os.path.join(d, lp.LIN_FILE))


def test_state_dict_from_files(tmp_path):
    sd = lo.random_state_dict(3)
    _write_checkpoints(str(tmp_path), sd)
    got = lp.state_dict_from_files(str(tmp_path / lp.VGG_FILE), str(tmp_path / lp.LIN_FILE))
    lp.check_state_dict(got)
    assert set(got) == {k for k in sd if not k.startswith("scaling_layer.")}
    assert all(torch.equal(got[k], sd[k]) for k in got)


def test_default_weight_files_and_missing_files(tmp_path, monkeypatch):
    monkeypatch.setattr(torch.hub, "get_dir", lambda: str(tmp_path))
    with pytest.raises(RuntimeError, match="vgg16-397923af.pth.*checkpoints"):
        lp.LPIPS()
    os.makedirs(tmp_path / "checkpoints")
    sd = lo.random_state_dict(1)
    _write_checkpoints(str(tmp_path / "checkpoints"), sd)
    os.remove(tmp_path / "checkpoints" / lp.LIN_FILE)
    with pytest.raises(RuntimeError, match="vgg.pth"):
        lp.state_dict_from_files()
    _write_checkpoints(str(tmp_path / "checkpoints"), sd)
    got = lp.state_dict_from_files()
    assert all(torch.equal(got[k], sd[k]) for k in got)


def test_argument_rules():
    for kw in ({"net": "alex"}, {"net": "squeeze"}, {"version": "0.0"}, {"spatial": True}):
        with pytest.raises(NotImplementedError):
            lp.LPIPS(state_dict=lo.random_state_dict(0), **kw)
    m = lp.LPIPS.__new__(lp.LPIPS)                # the input rules are checked before anything touches a device
    x = torch.zeros(2, 3, 32, 32)
    for a, b in ((x, torch.zeros(2, 3, 32, 33)), (x, torch.zeros(1, 3, 32, 32)), (torch.zeros(2, 4, 32, 32),) * 2,
                 (torch.zeros(2, 3, 15, 32),) * 2, (torch.zeros(2, 3, 32, 8),) * 2, (torch.zeros(0, 3, 32, 32),) * 2,
                 (torch.zeros(3, 32, 32),) * 2):
        with pytest.raises(ValueError):
            m.forward(a, b)
    with pytest.raises(NotImplementedError):
        lp.ssim(x, x, window_size=7)
    with pytest.raises(ValueError):
        lp.ssim(x, torch.zeros(2, 1, 32, 32))
    with pytest.raises(RuntimeError, match="CUDA"):
        lp.ssim(x, x)


def test_window_is_create_window():
    w = lp.gaussian_window()
    assert w.dtype == torch.float32 and tuple(w.shape) == (11, 11)
    assert torch.equal(w, lo.gaussian_window())
    assert abs(float(w.double().sum()) - 1.0) < 1e-6 and torch.equal(w, w.t())
