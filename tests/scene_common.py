"""The scene fixtures tests/golden/scene_*.npz (oracle/gen_golden_scene.py: the reference's own eval loader and file
writers on small seeded scene folders): the folder rebuilt from its stored bytes, and the reference's items."""
import functools
import os

import numpy as np

from oracle import fixture as F
from tests.common import GOLDEN

CASES = ("dtu", "tt_identity", "tt_short_range", "eth3d")


@functools.lru_cache(maxsize=None)
def fixture(name):
    """-> (arrays, meta)"""
    return F.load(os.path.join(GOLDEN, f"scene_{name}.npz"))


def write_folder(name, root):
    """writes the case's scene folder under root; -> the loader's datapath"""
    blob, meta = fixture(name)
    for i, rel in enumerate(meta["files"]):
        p = os.path.join(root, rel)
        os.makedirs(os.path.dirname(p), exist_ok=True)
        with open(p, "wb") as f:
            f.write(blob[f"file_{i}"].tobytes())
    return os.path.join(root, "test")


def load_args(meta):
    """load_scene's arguments after datapath"""
    return dict(scan=meta["scan"], dataset=meta["dataset"], nviews=meta["nviews"], ndepths=meta["ndepths"],
                interval_scale=meta["interval_scale"], max_h=meta["max_h"], max_w=meta["max_w"],
                use_short_range=meta["use_short_range"])


def reference_item(name, k):
    """-> (imgs [V,3,H,W], {stage1..4: [V,2,4,4]}, depth_values [D]) of MVSDataset[k], numpy"""
    blob, meta = fixture(name)
    imgs = np.stack([blob[f"img_{v}"] for v in meta["items"][k]])
    return imgs, {f"stage{s}": blob[f"proj_{k}_stage{s}"] for s in range(1, 5)}, blob[f"dv_{k}"]
