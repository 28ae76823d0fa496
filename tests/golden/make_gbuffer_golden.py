"""Writes tests/golden/gbuffer_small.npz from the reference's own chunk reader and post-processing, run on the chunk
folder committed beside it (tests/golden/gbuffer_chunk: Animals/0/10075 chunk 2 of the reference's
assets/demo-image-for-i23d/for-vae-reconstruction, with that object's FPS_PCD_for_vae fps-4096.ply).

ChunkObjaverseDataset.read_chunk (datasets/g_buffer_objaverse.py:3225-3302) is called unbound on a stand-in `self`
with the attributes it reads at the vae-3d.sh flags (img_ext 'jpg', chunk_size 16, read_normal); PostProcess is
constructed with the arguments ChunkObjaverseDataset.__init__ passes for those flags (:3189-3206: reso = reso_encoder =
512, imgnet_normalize=True as load_eval_data leaves it, plucker_embedding, append_xyz, frame_0_as_canonical=False,
split_chunk_size 16) and _post_process_sample_batch (:481-702) is run on the chunk's 16 views in stored order, as
paired_post_process_chunk does for a 16-view chunk.  CPU, fp32.  imageio is absent here: imageio.v3.imread is stood
in for by PIL's decoder (np.asarray(Image.open(path))); the other absent third-party imports are never reached.

Stored: rows OFFSET::STRIDE and columns OFFSET::STRIDE of img_to_encoder [16, 15, 512, 512], img, alpha and depth; c;
and, at every pixel, which xyz values (channels 12-14) are exactly zero, as np.packbits of the [16, 3, 512, 512]
mask.  The file stays below 1 MB.

    python tests/golden/make_gbuffer_golden.py
"""
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import _ref_stubs  # noqa: E402

STRIDE, OFFSET = 11, 3
CHUNK = os.path.join(HERE, "gbuffer_chunk")
OUT = os.path.join(HERE, "gbuffer_small.npz")


def main():
    from PIL import Image
    _ref_stubs.mod("imageio")
    _ref_stubs.mod("imageio.v3", imread=lambda p: np.asarray(Image.open(p)))
    import nsr  # noqa: F401  (first: nsr and datasets import each other, and only this order resolves)
    from datasets.g_buffer_objaverse import ChunkObjaverseDataset, PostProcess
    reader = types.SimpleNamespace(img_ext="jpg", chunk_size=16, read_normal=True)
    sample = ChunkObjaverseDataset.read_chunk(reader, CHUNK)
    pp = PostProcess(512, 512, imgnet_normalize=True, plucker_embedding=True, decode_encode_img_only=False,
                     mv_input=True, split_chunk_input=16, duplicate_sample=True, append_depth=False, append_xyz=True,
                     gs_cam_format=True, orthog_duplicate=False, frame_0_as_canonical=False, pcd_path=CHUNK,
                     load_pcd=True, split_chunk_size=16)
    enc, img, alpha, depth, c, _bbox = pp._post_process_sample_batch(list(sample[:-2]))
    assert tuple(enc.shape) == (16, 15, 512, 512), enc.shape
    sub = lambda t: np.ascontiguousarray(t.numpy()[..., OFFSET::STRIDE, OFFSET::STRIDE])
    np.savez_compressed(OUT, img_to_encoder=sub(enc), img=sub(img), alpha=sub(alpha), depth=sub(depth), c=c.numpy(),
                        xyz_zero_bits=np.packbits(enc[:, 12:15].numpy() == 0), stride=np.int64(STRIDE), offset=np.int64(OFFSET))
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
