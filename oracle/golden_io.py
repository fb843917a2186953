"""Golden files on disk: one `name.npz`, or - when that would exceed PART_LIMIT - `name.part<k>.npz` pieces holding
disjoint subsets of the arrays.  load() gives the same dict either way."""
import glob
import io
import os

import numpy as np

PART_LIMIT = 900 * 1024       # bytes per stored file (no file in the repository above 1 MB)


def _packed(arrays):
    buf = io.BytesIO()
    np.savez_compressed(buf, **arrays)
    return buf.getvalue()


def save(path, arrays):
    """Write `arrays` to `path` (…/name.npz), split greedily in key order into parts of at most PART_LIMIT bytes."""
    stem = path[:-len(".npz")]
    for old in [path] + glob.glob(stem + ".part*.npz"):
        if os.path.exists(old):
            os.remove(old)
    blob = _packed(arrays)
    if len(blob) <= PART_LIMIT:
        with open(path, "wb") as f:
            f.write(blob)
        return [path]
    parts, cur = [], {}
    for k, v in arrays.items():
        if cur and len(_packed(dict(cur, **{k: v}))) > PART_LIMIT:
            parts.append(cur)
            cur = {}
        cur[k] = v
    parts.append(cur)
    names = []
    for i, part in enumerate(parts):
        blob = _packed(part)
        assert len(blob) <= PART_LIMIT, "array %r alone exceeds the part limit" % list(part)
        names.append("%s.part%d.npz" % (stem, i))
        with open(names[-1], "wb") as f:
            f.write(blob)
    return names


def load(path):
    if os.path.exists(path):
        return dict(np.load(path, allow_pickle=False))
    parts = sorted(glob.glob(path[:-len(".npz")] + ".part*.npz"))
    if not parts:
        raise FileNotFoundError(path)
    out = {}
    for p in parts:
        out.update(np.load(p, allow_pickle=False))
    return out
