"""CPU checks of the DINOv2 image conditioner (SURVEY.md 8f row N3): the oracle's precision, the hub key table,
strict loading, weights without a network, the embedder's scope and the conditioner's key and zeroing rules."""
import json
import math
import os

import pytest
import torch

from gaussiananything_b200 import dino
from oracle import dino_oracle as do

KEYS = os.path.join(os.path.dirname(__file__), "golden", "dinov2_vitl14_reg4_keys.json")


def rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


def _img(B, H, W, seed):
    return torch.rand(B, 3, H, W, generator=torch.Generator().manual_seed(seed)) * 2 - 1


def _small_sd(depth=2, seed=0):
    return dino.random_state_dict(depth, seed=seed)


@pytest.mark.parametrize("H,W", [(518, 518), (256, 256), (700, 400)])
def test_oracle_fp32_matches_fp64(H, W):
    """The restatement in fp32 against itself in fp64: the preprocess (identity, upscale, blur + downscale) and a
    2-block encoder."""
    img = _img(1, H, W, H + W)
    p32, p64 = do.preprocess(img), do.preprocess(img.double(), dtype=torch.float64)
    # the resize computes its source coordinates in the working precision: fp32 puts them ~1e-7 x 518 px off
    assert p32.shape == (1, 3, 518, 518) and rel(p32, p64) < 5e-5
    if (H, W) == (518, 518):
        # the identity resize: preprocess is only the two normalisation steps
        assert torch.equal(p32, ((img + 1.0) / 2.0 - torch.tensor(do.MEAN).view(1, 3, 1, 1)) / torch.tensor(do.STD).view(1, 3, 1, 1))
    sd = _small_sd()
    o32, o64 = do.forward(sd, img), do.forward(sd, img.double(), dtype=torch.float64)
    assert o32["x_norm_patchtokens"].shape == (1, 1369, 1024) and o32["x_norm_clstoken"].shape == (1, 1024)
    for k in ("x_norm_patchtokens", "x_norm_clstoken"):
        assert rel(o32[k], o64[k]) < 1e-4, k


def test_oracle_blur_parameters_and_border():
    """kornia's antialias rule: no blur when upscaling, sigma = (factor - 1) / 2 floored at 0.001, odd kernel >= 3;
    the taps are normalised and the reflect border keeps a constant image constant."""
    assert do.blur_params(1024, 518) == pytest.approx((0.4884, 3), abs=1e-4)
    assert do.blur_params(4096, 518)[1] == 13 and do.blur_params(400, 518) == (0.001, 3)
    t = do.gaussian_taps(13, 3.45, torch.float64)
    assert float(t.sum()) == pytest.approx(1.0) and torch.equal(t, t.flip(0))
    x = torch.full((1, 3, 700, 600), 0.25, dtype=torch.float64)
    assert torch.allclose(do.resize(x), torch.full((1, 3, 518, 518), 0.25, dtype=torch.float64))


def test_random_state_dict_matches_hub_key_table():
    table = {k: tuple(v) for k, v in json.load(open(KEYS)).items()}
    sd = dino.random_state_dict(24, seed=0)
    assert {k: tuple(v.shape) for k, v in sd.items()} == table
    assert dino.expected_shapes(24) == table
    assert dino.check_state_dict(sd) == 24
    g = sd["blocks.3.ls1.gamma"]
    assert float(g.min()) >= 0.1 and float(g.max()) <= 1.0


def test_strict_loading_names_missing_and_extra_keys():
    sd = _small_sd(1)
    bad = dict(sd)
    del bad["blocks.0.attn.proj.bias"]
    with pytest.raises(RuntimeError, match=r"missing keys \['blocks.0.attn.proj.bias'\]"):
        dino.check_state_dict(bad)
    bad = dict(sd, **{"blocks.0.attn.q_norm.weight": torch.ones(64)})
    with pytest.raises(RuntimeError, match=r"unexpected keys \['blocks.0.attn.q_norm.weight'\]"):
        dino.check_state_dict(bad)
    bad = dict(sd, pos_embed=torch.zeros(1, 257, 1024))                   # a 224^2 model
    with pytest.raises(RuntimeError, match="pos_embed"):
        dino.check_state_dict(bad)


class _RecordingEncoder:
    """Stands in for the CUDA encoder on a CPU-only machine: checks the weights it is given, returns fixed tensors
    and counts calls."""
    made = []

    def __init__(self, state_dict, device="cuda:0"):
        self.depth = dino.check_state_dict(state_dict)
        self.calls = 0
        _RecordingEncoder.made.append(self)

    def encode(self, img):
        self.calls += 1
        B = img.shape[0]
        g = torch.Generator().manual_seed(int(img.float().sum() * 1000) % 1000)
        return {"x_norm_clstoken": torch.randn(B, 1024, generator=g) + 1.0,
                "x_norm_patchtokens": torch.randn(B, 1369, 1024, generator=g) + 1.0}


@pytest.fixture
def offline(monkeypatch, tmp_path):
    """Any attempt to reach the network fails the test; the hub directory is an empty temporary one."""
    import urllib.request

    def refuse(*a, **k):
        raise AssertionError("network access attempted")
    monkeypatch.setattr(torch.hub, "load", refuse)
    monkeypatch.setattr(torch.hub, "load_state_dict_from_url", refuse)
    monkeypatch.setattr(torch.hub, "download_url_to_file", refuse)
    monkeypatch.setattr(urllib.request, "urlopen", refuse)
    monkeypatch.setattr(torch.hub, "get_dir", lambda: str(tmp_path))
    monkeypatch.setattr(dino, "Dinov2Encoder", _RecordingEncoder)
    return tmp_path


def test_embedder_weights_never_come_from_the_network(offline):
    e = dino.FrozenDinov2ImageEmbedder(arch="vitl", inp_size=518, output_cls=True, state_dict=_small_sd(1))
    assert isinstance(e.encoder, _RecordingEncoder) and e.encoder.depth == 1
    want = os.path.join(str(offline), "checkpoints", "dinov2_vitl14_reg4_pretrain.pth")
    with pytest.raises(RuntimeError, match="dinov2_vitl14_reg4_pretrain.pth") as ei:
        dino.FrozenDinov2ImageEmbedder(arch="vitl", inp_size=518, output_cls=True)
    assert want in str(ei.value) and "state_dict=" in str(ei.value)
    # the local file, once placed there, is what loads
    os.makedirs(os.path.dirname(want))
    torch.save(_small_sd(2, seed=3), want)
    e = dino.FrozenDinov2ImageEmbedder(arch="vitl", inp_size=518, output_cls=True)
    assert e.encoder.depth == 2


def test_embedder_scope_raises_not_implemented(offline):
    sd = _small_sd(1)
    with pytest.raises(NotImplementedError, match="vitl"):
        dino.FrozenDinov2ImageEmbedder(arch="vitg", inp_size=518, state_dict=sd)
    with pytest.raises(NotImplementedError, match="518"):
        dino.FrozenDinov2ImageEmbedder(arch="vitl", state_dict=sd)                 # the reference default inp_size=224
    with pytest.raises(NotImplementedError, match="518"):
        dino.FrozenDinov2ImageEmbedder(arch="vitl", inp_size=448, state_dict=sd)


def test_random_weights_make_attention_selective():
    """Block 0's attention on a noise image is far from uniform: mean row entropy < 0.9 ln N."""
    ent = do.block0_attention_entropy(_small_sd(1), _img(1, 518, 518, 7))
    assert ent < 0.9 * math.log(1374), ent


def _conditioner(stage2, calls):
    enc = _RecordingEncoder(_small_sd(1))
    calls.append(enc)
    emb = dino.FrozenDinov2ImageEmbedder(arch="vitl", inp_size=518, output_cls=True, encoder=enc)
    cfgs = [emb]
    emb.input_key, emb.ucg_rate = "img", 0.1
    if stage2:
        cfgs.append({"is_trainable": False, "input_key": "fps-xyz", "ucg_rate": 0.0,
                     "target": "sgm.modules.encoders.modules.PCD_Scaler",
                     "params": {"scaling_factor": 0.45, "perturb_pcd_scale": 0.0}})
    return dino.GeneralConditioner(cfgs)


def test_conditioner_keys_and_zeroing_rules():
    calls = []
    img = _img(2, 518, 518, 3).bfloat16()
    # stage 1: the trainer zeroes its conditioning key 'img' in uc
    cond = _conditioner(False, calls)
    c, uc = cond.get_unconditional_conditioning({"img": img}, force_uc_zero_embeddings=["img"])
    assert sorted(c) == sorted(uc) == ["img_crossattn", "img_vector"]
    assert c["img_crossattn"].shape == (2, 1369, 1024) and c["img_vector"].shape == (2, 1024)
    assert c["img_crossattn"].dtype == torch.bfloat16 and c["img_vector"].dtype == torch.bfloat16
    assert float(uc["img_crossattn"].abs().max()) == 0 and float(uc["img_vector"].abs().max()) == 0
    assert float(c["img_crossattn"].abs().max()) > 0 and float(c["img_vector"].abs().max()) > 0
    assert calls[-1].calls == 1                                   # encoder ran once for c and uc
    assert cond.embedders[0].ucg_rate == 0.1                      # the rate is restored afterwards
    # stage 2: conditioning key 'img-xyz' names no embedder, so uc == c
    cond = _conditioner(True, calls)
    xyz = torch.rand(2, 768, 3) * 0.9 - 0.45
    c, uc = cond.get_unconditional_conditioning({"img": img, "fps-xyz": xyz}, force_uc_zero_embeddings=["img-xyz"])
    assert sorted(c) == sorted(uc) == ["fps-xyz", "img_crossattn", "img_vector"]
    assert all(torch.equal(c[k], uc[k]) for k in c)
    assert torch.equal(c["fps-xyz"], xyz / 0.45)
    assert calls[-1].calls == 1
    # a separate batch_uc runs the embedders again
    c, uc = cond.get_unconditional_conditioning({"img": img, "fps-xyz": xyz}, {"img": img, "fps-xyz": xyz})
    assert calls[-1].calls == 3 and all(torch.equal(c[k], uc[k]) for k in c)
    # forward with force_zero_embeddings, and the output key of an embedder whose key is not 'img'
    out = cond({"img": img, "fps-xyz": xyz}, force_zero_embeddings=["fps-xyz"])
    assert float(out["fps-xyz"].abs().max()) == 0


def test_embedder_forward_order_dtype_and_dropout():
    calls = []
    enc = _RecordingEncoder(_small_sd(1))
    calls.append(enc)
    emb = dino.FrozenDinov2ImageEmbedder(arch="vitl", inp_size=518, output_cls=True, encoder=enc)
    img = _img(3, 518, 518, 5).bfloat16()
    tokens, z = emb(img)
    assert tokens.shape == (3, 1369, 1024) and z.shape == (3, 1024)
    assert tokens.dtype == z.dtype == torch.bfloat16
    emb.ucg_rate = 1.0                                            # every sample dropped ...
    tokens, z = emb(img)
    assert float(tokens.abs().max()) == 0 and float(z.abs().max()) == 0
    tokens, z = emb(img, no_dropout=True)                         # ... unless dropout is off
    assert float(tokens.abs().max()) > 0
    emb.output_cls = False
    assert emb(img, no_dropout=True).shape == (3, 1369, 1024)


def test_install_shims_replaces_conditioner_classes():
    import sys
    import types
    import gaussiananything_b200 as ga
    names = ("sgm", "sgm.modules", "sgm.modules.encoders", "sgm.modules.encoders.modules")
    saved = {k: sys.modules.get(k) for k in names + ("diff_surfel_rasterization", "transport", "transport.transport",
                                                     "transport.path", "transport.integrators")}
    try:
        for n in names:
            sys.modules[n] = types.ModuleType(n)
        ga.install_shims()
        for n in ("sgm.modules.encoders.modules", "sgm.modules"):
            m = sys.modules[n]
            assert m.FrozenDinov2ImageEmbedder is dino.FrozenDinov2ImageEmbedder
            assert m.PCD_Scaler is dino.PCD_Scaler and m.GeneralConditioner is dino.GeneralConditioner
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


def test_encoder_refuses_cpu():
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        dino.Dinov2Encoder(_small_sd(1), device="cpu")
