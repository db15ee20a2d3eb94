"""ORACLE - TEST INFRASTRUCTURE ONLY.  The format of the fixtures under tests/golden/: one compressed .npz of named numpy
arrays and, where the fixture has one, a `meta` entry holding a JSON object as uint8 bytes (seeds, sizes, settings)."""
import json

import numpy as np


def save(path, arrays, meta=None):
    blob = dict(arrays)
    if meta is not None:
        blob["meta"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
    np.savez_compressed(path, **blob)


def load(path):
    """-> ({name: numpy array} without `meta`, the meta dict or {} where the fixture has none)"""
    with np.load(path) as z:
        arrays = {k: z[k] for k in z.files}
    meta = arrays.pop("meta", None)
    return arrays, ({} if meta is None else json.loads(meta.tobytes().decode()))
