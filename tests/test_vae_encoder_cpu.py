"""3D VAE encoder, CPU side: the fp32 oracle against the golden made by the reference's own encoder classes, FPS
indices, the strict key table, and SurfelAE without an encoder behaving as before."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import vae_encoder_oracle as vo

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return float((a - b).norm() / b.norm())


@pytest.fixture(scope="module")
def golden():
    z = dict(np.load(os.path.join(GOLDEN, "vae_encoder_small.npz")))
    z.update(np.load(os.path.join(GOLDEN, "vae_encoder_small.part2.npz")))
    return {k: torch.from_numpy(v) for k, v in z.items()}


@pytest.fixture(scope="module")
def oracle_run(golden):
    from gaussiananything_b200.vae_encoder import random_state_dict
    seed, B, V, H, NP, K = (int(v) for v in golden["cfg"])
    sd = random_state_dict(seed=seed)
    acts = {}
    out = vo.encode(sd, golden["img"], golden["pcd"], V, K, golden["start"], acts=acts)
    post = vo.posterior(sd, out["h"], golden["eps"])
    return out, post, acts


def test_oracle_matches_reference_golden(golden, oracle_run):
    out, post, acts = oracle_run
    for k in ("level0", "level1", "level2"):
        assert rel(acts[k][:, :, ::2, ::2], golden["act_" + k]) <= 1e-5, k
    for k in ("level3", "attn_1", "agg_ca", "srt"):
        assert rel(acts[k], golden["act_" + k]) <= 1e-5, k
    assert rel(out["h"], golden["h"]) <= 1e-5
    for k in ("mean", "logvar", "latent_normalized"):
        assert rel(post[k], golden[k]) <= 1e-5, k


def test_fps_indices_match_golden(golden, oracle_run):
    out, _, _ = oracle_run
    assert torch.equal(out["query_pcd_xyz"], golden["query_pcd_xyz"])
    assert int(out["fps_idx"][0, 0]) == int(golden["start"][0])


def test_fps_ties_go_to_lowest_index():
    pcd = torch.tensor([[[0.0, 0, 0], [1, 0, 0], [-1, 0, 0], [1, 0, 0], [0, 2, 0]]])
    _, idx = vo.fps(pcd, 4, torch.tensor([0]))
    assert idx.tolist() == [[0, 4, 1, 2]]                 # 1 and 3 tie with 2 after step 2: lowest index first


def test_key_table_matches_reference():
    from gaussiananything_b200.vae_encoder import _expected_keys, random_state_dict
    ref = json.load(open(os.path.join(GOLDEN, "vae_encoder_keys.json")))
    ours = {k: list(v) for k, v in _expected_keys().items()}
    assert ours == ref
    sd = random_state_dict()
    assert {k: list(v.shape) for k, v in sd.items()} == ref


def test_strict_loading_names_the_key():
    from gaussiananything_b200.vae_encoder import check_state_dict, random_state_dict
    sd = random_state_dict()
    check_state_dict(dict(sd, **{"decoder.superresolution.conv_sr.weight": torch.zeros(1)}))   # other AE keys pass
    bad = dict(sd)
    del bad["encoder.mid.attn_1.proj_in.weight"]
    with pytest.raises(KeyError, match="encoder.mid.attn_1.proj_in.weight"):
        check_state_dict(bad)
    bad = dict(sd, **{"encoder.extra.weight": torch.zeros(3)})
    with pytest.raises(KeyError, match="encoder.extra.weight"):
        check_state_dict(bad)
    bad = dict(sd, **{"encoder.agg_ca.q_norm.weight": torch.zeros(32)})
    with pytest.raises(KeyError, match="encoder.agg_ca.q_norm.weight"):
        check_state_dict(bad)


def test_surfel_ae_without_encoder_raises_as_before():
    from gaussiananything_b200.vae_decoder import SurfelAE
    ae = SurfelAE(decoder=None, renderer=object())
    for b in ("enc", "encoder_vae", "enc_dec_wo_triplane", "enc_dec"):
        with pytest.raises(NotImplementedError, match="outside the decode / render path"):
            ae(img=None, behaviour=b)


def test_encode_flops_estimate():
    from gaussiananything_b200.vae_encoder import encode_flops
    assert 4.0e12 < encode_flops() < 4.2e12
    assert encode_flops(B=2) == pytest.approx(2 * encode_flops(B=1), rel=1e-9)
