"""Golden fixtures larger than 1 MB are committed in parts: <name>.npz plus <name>.part2.npz.
save_parts() writes them, load_parts() reads every part back into one mapping."""
import os

import numpy as np


def save_parts(path, arrays, second_part_keys):
    """Writes `arrays` to `path`, the keys in `second_part_keys` to <name>.part2.npz (both compressed)."""
    second = {k: v for k, v in arrays.items() if k in second_part_keys}
    first = {k: v for k, v in arrays.items() if k not in second_part_keys}
    np.savez_compressed(path, **first)
    if second:
        np.savez_compressed(path[:-len(".npz")] + ".part2.npz", **second)


def load_parts(path):
    """{key: array} of `path` and all of its parts."""
    out = {}
    stem, k = path[:-len(".npz")], 1
    part = path
    while os.path.exists(part):
        with np.load(part) as z:
            for key in z.files:
                out[key] = z[key]
        k += 1
        part = "%s.part%d.npz" % (stem, k)
    if not out:
        raise FileNotFoundError(path)
    return out
