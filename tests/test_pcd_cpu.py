"""Surface point clouds without a GPU: known answers of the FPS rule the kernels follow (through
oracle/vae_encoder_oracle.fps), the chunk keep rule on the committed chunk against the reference's shipped cloud,
the PLY writer, and the GPU-only entry points refusing CPU input."""
import os

import numpy as np
import pytest
import torch

from oracle import vae_encoder_oracle as vo
from tests import pcd_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHUNK = os.path.join(ROOT, "tests", "golden", "gbuffer_chunk")
PLY = os.path.join(CHUNK, "fps-4096.ply")


def test_fps_on_a_line():
    x = torch.tensor([0.0, 1.0, 2.0, 3.0, 10.0])
    pcd = torch.stack([x, torch.zeros(5), torch.zeros(5)], -1)[None]
    _, idx = vo.fps(pcd, 5, torch.tensor([0]))
    assert idx[0].tolist() == [0, 4, 3, 1, 2]        # 10, then 3 (9 from 0), then 1 and 2 tie at 1: lowest index
    _, idx = vo.fps(pcd, 3, torch.tensor([2]))      # explicit start
    assert idx[0].tolist() == [2, 4, 0]


def test_fps_cube_corners_and_k_equal_n():
    c = torch.tensor([[i >> 2 & 1, i >> 1 & 1, i & 1] for i in range(8)], dtype=torch.float32)[None]
    xyz, idx = vo.fps(c, 8, torch.tensor([0]))
    assert idx[0, 1] == 7                            # the opposite corner
    assert sorted(idx[0].tolist()) == list(range(8))  # K = N: a permutation
    assert torch.equal(xyz[0], c[0][idx[0]])
    _, one = vo.fps(c, 1, torch.tensor([5]))
    assert one.tolist() == [[5]]


def test_fps_duplicates_tie_to_the_lowest_index():
    pcd = torch.tensor([[0.0, 0, 0], [1, 1, 1], [1, 1, 1], [0, 0, 0], [1, 1, 1]])[None]
    _, idx = vo.fps(pcd, 5, torch.tensor([0]))
    assert idx[0].tolist()[:2] == [0, 1]
    # every point at distance 0 after the two distinct ones: the lowest index again (0, already chosen)
    assert idx[0].tolist()[2:] == [0, 0, 0]


def test_fps_padded_past_the_length():
    g = torch.Generator().manual_seed(0)
    pcd = torch.rand(2, 10, 3, generator=g)
    xyz, idx = pcd_ref.fps_padded(pcd, torch.tensor([4, 10]), 6, torch.tensor([1, 0]))
    assert idx[0, 4:].tolist() == [-1, -1] and float(xyz[0, 4:].abs().max()) == 0
    assert sorted(idx[0, :4].tolist()) == [0, 1, 2, 3] and idx[0, 0] == 1
    assert torch.equal(idx[1], vo.fps(pcd[1:], 6, torch.tensor([0]))[1][0])


@pytest.fixture(scope="module")
def chunk():
    from gaussiananything_b200 import gbuffer
    return gbuffer.read_chunk(CHUNK)


def test_keep_rule_on_the_chunk_against_the_shipped_cloud(chunk):
    """The reference's rules (alpha == 255, depth >= 1.05, inside the clip) in fp32, as its torch code computes them:
    254 899 points, each within 0.1 of the shipped fps-4096.ply (made from views this chunk lacks), and the median
    shipped point within 0.02 of the fused cloud.  Views 13-15 repeat 5-7, so the cloud holds exact duplicates."""
    from scipy.spatial import cKDTree
    from gaussiananything_b200 import gbuffer
    pts = pcd_ref.surface_points(chunk, dtype=torch.float32).numpy()
    assert pts.shape == (254899, 3)
    assert float(np.abs(pts).max()) < 0.45 and bool((pts != 0).all())
    ref = gbuffer.read_fps_pcd(PLY)
    d_fused, _ = cKDTree(ref).query(pts)
    d_ref, _ = cKDTree(pts).query(ref)
    print("fused -> shipped max %.4f; shipped -> fused median %.4f" % (d_fused.max(), np.median(d_ref)))
    assert d_fused.max() < 0.1 and np.median(d_ref) < 0.02
    assert len(np.unique(pts, axis=0)) < len(pts)
    # the fp64 yardstick keeps almost the same pixels
    p64 = pcd_ref.surface_points(chunk, dtype=torch.float64)
    assert abs(p64.shape[0] - pts.shape[0]) <= 10


def test_write_ply_round_trips(tmp_path):
    from gaussiananything_b200 import gbuffer, pcd
    g = torch.Generator().manual_seed(3)
    xyz = torch.randn(1000, 3, generator=g)
    xyz[5] = torch.tensor([float("inf"), -0.0, 1e-40])
    f = os.path.join(tmp_path, "fps-1000.ply")
    pcd.write_ply(f, xyz)
    back = gbuffer.read_fps_pcd(f)
    assert back.dtype == np.float32 and back.view(np.uint32).tobytes() == xyz.numpy().view(np.uint32).tobytes()
    pcd.write_ply(f, np.zeros((0, 3), np.float32))
    assert gbuffer.read_fps_pcd(f).shape == (0, 3)
    with pytest.raises(ValueError):
        pcd.write_ply(f, np.zeros((4, 2)))


def test_cpu_input_is_refused(chunk):
    from gaussiananything_b200 import pcd
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        pcd.sample_farthest_points(torch.rand(1, 10, 3), K=4)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        pcd.chunk_surface_points(chunk, device="cpu")
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        pcd.gaussians_pcd(torch.rand(1, 10, 13), K=4)
