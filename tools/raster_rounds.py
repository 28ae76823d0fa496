"""CPU estimate (from the oracle's tile lists of the C2 scene) of how many evaluation rounds a warp needs per chunk
under different lane mappings of the composite kernels:
  forward : one surfel per warp round (GS=32) | two 4x4 half-warp groups (GS=16) | four 4x2 groups (GS=8) | one list per lane
  backward: per-lane lists synchronised every 32 surfels (round 1) | per-lane lists over a whole group of 128
and the totals of the forward's split mapping (csrc/raster_render.cu) beside those of the GS=8 mapping it replaced:
  phase 1: (instance, pixel) pairs inside the clipped cull boxes, packed 32 per warp iteration, per window of FWD_PAIRS
  phase 2: per warp and window, the largest number of box pairs of one of its pixels (an upper bound: only the pairs
           that reach alpha >= 1/255 are composited)
and the backward's phase B: serial record iterations per window (the longest walk of one lane) when every instance
gets two lanes, sorted by record count with 16 instances per warp (csrc/raster_render.cu), and when the window's
records are spread evenly over the 256 lanes, for windows of 4096 and 3072 records.  A record is a box pixel in front of the pixel's last
contributor, an upper bound on the forward's contributions.
Cull boxes are approximated by the low-pass disc.  Counts, not timings.
    python tools/raster_rounds.py [tiles per view, or 0 for all] [views]"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests.helpers import cameras, oracle_view, scene  # noqa: E402

CHUNK, FWD_PAIRS = 256, 4096


def windows(cc, limit):
    """Splits a chunk's per-slot counts into windows of consecutive slots whose counts fit `limit`."""
    incl = np.cumsum(cc)
    t0, base = 0, 0
    while t0 < len(cc):
        t1 = t0 + int(((incl - base <= limit) & (np.arange(len(cc)) >= t0)).sum())
        yield t0, t1
        base, t0 = int(incl[t1 - 1]), t1


def phase_b_pairs(c):
    """Two lanes per instance, instances sorted by count, 16 per warp and 128 per round: the slowest warp's iterations."""
    c = np.sort(c[c > 0])[::-1]
    per_warp = np.zeros(8, np.int64)
    for b0 in range(0, len(c), 128):
        rnd = -(-c[b0:b0 + 128] // 2)
        for w in range(8):
            if 16 * w < len(rnd):
                per_warp[w] += rnd[16 * w:16 * w + 16].max()
    return int(per_warp.max())


def main():
    ntiles = int(sys.argv[1]) if len(sys.argv) > 1 else 200
    nviews = int(sys.argv[2]) if len(sys.argv) > 2 else 1
    P, H, W = 100000, 512, 512
    g = scene(P, 40)
    vs, ps, _, _ = cameras(6)
    tot = dict(gs32=0, gs16=0, gs8=0, lane=0, lane_sub32=0, lane_grp128=0, useful=0)
    split = dict(gs8_rounds=0, pairs=0, phase1_warp_iters=0, phase2_rounds=0, windows=0, chunks=0, max_chunk_pairs=0)
    # phase B: (records per window, windows, serial iterations) per scheme; instances per window and records per instance
    pb = {"pairs 4096": [4096, 0, 0], "pairs 3072": [3072, 0, 0], "even 4096": [4096, 0, 0], "even 3072": [3072, 0, 0]}
    pb_records, pb_inst, pb_inst_max, pb_rec_max = 0, 0, 0, 0
    nw = 0
    for view in range(nviews):
        o = oracle_view(g, vs[view], ps[view], [1, 1, 1], H, W)
        xy, opa = o["xy"], g[:, 3]
        tau = 2 * np.log(np.maximum(255 * opa, 1.0)) * 1.001 + 1e-3
        r2 = np.sqrt(0.5 * tau) + 0.51                  # the low-pass disc of K1's cull box (the 3-D part is tiny here)
        bx0, bx1, by0, by1 = xy[:, 0] - r2, xy[:, 0] + r2, xy[:, 1] - r2, xy[:, 1] + r2
        ids, rng, last = o["ids"], o["ranges"], o["n_contrib"][0]
        tiles = np.arange(len(rng)) if ntiles <= 0 else np.random.default_rng(0).choice(len(rng), ntiles, replace=False)
        for t in tiles:
            a, b = rng[t]
            if b <= a:
                continue
            sid = ids[a:b].astype(int)
            ty, tx = divmod(int(t), W // 16)
            ox, oy = tx * 16, ty * 16
            X0, X1, Y0, Y1 = bx0[sid], bx1[sid], by0[sid], by1[sid]
            valid = opa[sid] * 255 >= 1

            def hits(x0, y0, w, h):
                return valid & ~((X1 < ox + x0) | (X0 > ox + x0 + w - 1) | (Y1 < oy + y0) | (Y0 > oy + y0 + h - 1))
            pix = np.stack([hits(x, y, 1, 1) for y in range(16) for x in range(16)])       # [256 pixels, n]
            for wp in range(8):
                nw += 1
                lx0, ly0 = (wp & 1) * 8, (wp >> 1) * 4
                tot["gs32"] += hits(lx0, ly0, 8, 4).sum()
                tot["gs16"] += max(hits(lx0, ly0, 4, 4).sum(), hits(lx0 + 4, ly0, 4, 4).sum())
                gs8 = max(hits(lx0 + 4 * (k & 1), ly0 + 2 * (k >> 1), 4, 2).sum() for k in range(4))
                tot["gs8"] += gs8
                split["gs8_rounds"] += gs8
                pl = np.stack([pix[(ly0 + (l >> 3)) * 16 + lx0 + (l & 7)] for l in range(32)])   # [32 lanes, n]
                tot["lane"] += pl.sum(1).max()
                tot["useful"] += pl.sum()
                n = pl.shape[1]
                tot["lane_sub32"] += sum(pl[:, s:s + 32].sum(1).max() for s in range(0, n, 32))
                tot["lane_grp128"] += sum(pl[:, s:s + 128].sum(1).max() for s in range(0, n, 128))
            # split mapping: per chunk, windows of consecutive instances whose pairs fit FWD_PAIRS
            cnt = pix.sum(0)                                                                # pairs per instance
            warp_pix = [np.array([(ly0 + (l >> 3)) * 16 + lx0 + (l & 7) for l in range(32)])
                        for lx0, ly0 in (((wp & 1) * 8, (wp >> 1) * 4) for wp in range(8))]
            for c0 in range(0, len(sid), CHUNK):
                cc = cnt[c0:c0 + CHUNK]
                split["chunks"] += 1
                split["max_chunk_pairs"] = max(split["max_chunk_pairs"], int(cc.sum()))
                incl = np.cumsum(cc)
                t0, base = 0, 0
                while t0 < len(cc):
                    t1 = t0 + int(((incl - base <= FWD_PAIRS) & (np.arange(len(cc)) >= t0)).sum())
                    wpairs = int(incl[t1 - 1] - base)
                    split["windows"] += 1
                    split["pairs"] += wpairs
                    split["phase1_warp_iters"] += -(-wpairs // 32)
                    per_pix = pix[:, c0 + t0:c0 + t1].sum(1)
                    split["phase2_rounds"] += sum(int(per_pix[wpx].max()) for wpx in warp_pix)
                    base, t0 = int(incl[t1 - 1]), t1
            # backward: slot t of a chunk is list position hi - 1 - t, chunks from the tile's deepest contributor down
            lc = last[oy:oy + 16, ox:ox + 16].reshape(256)
            recs = (pix & (np.arange(len(sid))[None, :] < lc[:, None])).sum(0)
            for hi in range(int(lc.max()), 0, -CHUNK):
                cc = recs[max(0, hi - CHUNK):hi][::-1]
                pb_records += int(cc.sum())
                for key, v in pb.items():
                    for t0, t1 in windows(cc, v[0]):
                        w = cc[t0:t1]
                        v[1] += 1
                        v[2] += phase_b_pairs(w) if key.startswith("pairs") else -(-int(w.sum()) // 256)
                        if key == "pairs 4096":
                            pb_inst += int((w > 0).sum())
                            pb_inst_max = max(pb_inst_max, int((w > 0).sum()))
                            pb_rec_max = max(pb_rec_max, int(w.max()))
    print("rounds per warp (C2 scene, %s tiles x %d views): " % ("all" if ntiles <= 0 else ntiles, nviews)
          + ", ".join("%s %.1f" % (k, v / nw) for k, v in tot.items()))
    print("split forward totals (FWD_PAIRS %d): " % FWD_PAIRS + ", ".join("%s %d" % kv for kv in split.items()))
    nwin = pb["pairs 4096"][1]
    print("backward phase B (%d records; with 4096 records per window: %d windows, instances per window mean %.1f max %d, "
          "records per instance mean %.1f max %d): " % (pb_records, nwin, pb_inst / nwin, pb_inst_max,
                                                        pb_records / max(pb_inst, 1), pb_rec_max)
          + ", ".join("%s: %d windows, serial iterations %.1f per window, %d in all" % (k, v[1], v[2] / v[1], v[2])
                      for k, v in pb.items()))


if __name__ == "__main__":
    main()
