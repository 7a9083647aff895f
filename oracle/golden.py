"""Golden fixtures under tests/golden: compressed .npz files of at most ~1 MB each.

A record too large for one file (trained checkpoint weights) is stored as `<name>.npz`, `<name>.1.npz`, ...;
an array larger than one part is cut into row blocks stored as `<key>@@<i>`.  `load()` reassembles the record.
"""
import glob
import os

import numpy as np

PART_BYTES = 900 * 1024


def save(path, **rec):
    """np.savez_compressed(path, **rec), split into parts of <= PART_BYTES of raw array data."""
    pieces = []
    for k, v in rec.items():
        v = np.asarray(v)
        if v.nbytes <= PART_BYTES or v.ndim == 0:
            pieces.append((k, v))
            continue
        rows = max(1, PART_BYTES // max(1, v.nbytes // v.shape[0]))
        for i, r0 in enumerate(range(0, v.shape[0], rows)):
            pieces.append(('%s@@%d' % (k, i), v[r0:r0 + rows]))
    parts, cur, size = [], {}, 0
    for k, v in pieces:
        if cur and size + v.nbytes > PART_BYTES:
            parts.append(cur)
            cur, size = {}, 0
        cur[k] = v
        size += v.nbytes
    parts.append(cur)
    base = path[:-4] if path.endswith('.npz') else path
    for i, p in enumerate(parts):
        np.savez_compressed(base + ('.npz' if i == 0 else '.%d.npz' % i), **p)


class Record(dict):
    """dict of arrays with the `files` attribute of an np.load() result."""

    @property
    def files(self):
        return list(self)


def load(path):
    """The record written by save() (or by a plain np.savez) as a Record of arrays."""
    base = path[:-4] if path.endswith('.npz') else path
    files = [base + '.npz'] + sorted(glob.glob(base + '.[0-9]*.npz'), key=lambda f: int(f.split('.')[-2]))
    out, split = Record(), {}
    for f in files:
        if not os.path.exists(f):
            raise FileNotFoundError(f)
        with np.load(f) as z:
            for k in z.files:
                if '@@' in k:
                    name, i = k.rsplit('@@', 1)
                    split.setdefault(name, {})[int(i)] = z[k]
                else:
                    out[k] = z[k]
    for name, blocks in split.items():
        out[name] = np.concatenate([blocks[i] for i in sorted(blocks)], axis=0)
    return out
