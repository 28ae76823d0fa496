"""Multi-GPU plumbing for the render stage of the cascade (SURVEY.md 8e): one process per GPU,
samples decoded where they were sampled, ONE all-gather of the decoded surfels, then every rank renders
an interleaved share of all (sample, view) pairs.  No collective inside any kernel.

The reference has no multi-GPU inference at all (scripts/gradio_app_cascaded.py:96-100 pins world size 1);
this is the GPU-native addition BASELINE.json's north_star asks for.  Works with NCCL (GPU) and gloo
(CPU, used by the tests for the host logic)."""
from typing import List, Tuple

import torch
import torch.distributed as dist


def shard_pairs(num_samples: int, views: int, world: int, rank: int) -> List[Tuple[int, int]]:
    """(sample, view) pairs owned by `rank`: pair q = sample*views + view goes to rank q % world, so ranks get
    equal counts (+-1) and each rank touches several samples (balances per-sample cost differences)."""
    if not (0 <= rank < world):
        raise ValueError("rank out of range")
    return [(q // views, q % views) for q in range(num_samples * views) if q % world == rank]


def all_gather_surfels(local: torch.Tensor, group=None) -> torch.Tensor:
    """local [S_local, P, 13] on every rank (same shape) -> [world*S_local, P, 13], rank-major.
    Single collective (NCCL all-gather over NVLink on GPU)."""
    if not dist.is_available() or not dist.is_initialized() or dist.get_world_size(group) == 1:
        return local
    world = dist.get_world_size(group)
    local = local.contiguous()
    out = torch.empty((world * local.shape[0],) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
    dist.all_gather_into_tensor(out, local, group=group)
    return out


def group_pairs_by_sample(pairs):
    """[(b, v), ...] -> {b: [v, ...]} keeping order; one batched rasteriser call per distinct sample."""
    out = {}
    for b, v in pairs:
        out.setdefault(b, []).append(v)
    return out


def render_sharded(renderer, local_surfels, cam_view, cam_view_proj, cam_pos, tanfov, group=None, **kw):
    """local_surfels [S_local, P, 13] (this rank's decoded samples); cameras [S, V, ...] for ALL samples (replicated).
    Returns {(b, v): dict of [C,H,W] tensors} for the pairs this rank owns.

    The all-gather is the only collective; afterwards the rank's pairs are rendered with ONE batched rasteriser
    call per distinct views-per-sample count (normally one call in total: samples that own the same number of
    views form one [B', V'] batch of the kernels' (batch item, view) grid)."""
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    surfels = all_gather_surfels(local_surfels, group)            # [S, P, 13]
    S, V = cam_view.shape[:2]
    by_sample = group_pairs_by_sample(shard_pairs(S, V, world, rank))
    buckets = {}
    for b, vs in by_sample.items():
        buckets.setdefault(len(vs), []).append(b)
    result = {}
    for nv, samples in buckets.items():
        bi = torch.tensor(samples, device=cam_view.device)
        vi = torch.tensor([by_sample[b] for b in samples], device=cam_view.device)          # [B', nv]
        rows = bi[:, None].expand(-1, nv)
        out = renderer.render(surfels[bi], cam_view[rows, vi], cam_view_proj[rows, vi], cam_pos[rows, vi], tanfov, **kw)
        for i, b in enumerate(samples):
            for j, v in enumerate(by_sample[b]):
                result[(b, v)] = {k: t[i, j] for k, t in out.items()}
    return result
