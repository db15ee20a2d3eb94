"""Shared helpers of the depth-map fusion tests: fixture loading and the mask rule."""
import os

import numpy as np
import torch

from oracle import fixture
from oracle import fusion as OF
from tests.common import GOLDEN

FIXTURES = ("fusion_n6_40x72", "fusion_n11_32x48")
MARGIN = 1e-4        # a comparison this close (relative) to its threshold in fp64 may fall on either side in fp32
MAX_DISAGREE = 1e-3  # and that may happen to this fraction of a view's pixels at most


def load_fixture(name):
    """-> scene dict (float32 CPU tensors, images back in [0,1]), meta, raw arrays"""
    z, meta = fixture.load(os.path.join(GOLDEN, name + ".npz"))
    scene = dict(depths=torch.from_numpy(z["depths"]), confs=torch.from_numpy(z["confs"]), cams=torch.from_numpy(z["cams"]),
                 images=torch.from_numpy(z["images"]).float() / 255.0, pairs=[(r, s) for r, s in meta["pairs"]])
    return scene, meta, z


def fixture_view(z, meta, method, r):
    H, W = meta["H"], meta["W"]
    mask = torch.from_numpy(np.unpackbits(z[f"{method}_mask_{r}"])[:H * W].reshape(H, W).astype(bool))
    return mask, torch.from_numpy(z[f"{method}_depth_{r}"]), torch.from_numpy(z[f"{method}_points_{r}"])


def check_view(mask, avg, ref, srcs, scene, method, points=None, inv=None, **kw):
    """The mask rule for one reference view: `mask` may differ from the fp32 oracle's only at pixels where the fp64 oracle
    has a comparison within MARGIN of its threshold, and at fewer than MAX_DISAGREE of the pixels; at the other pixels
    the averaged depth agrees to 1e-5 relative and (where both keep the pixel) the points [H,W,3] to 1e-3 absolute.
    inv: the camera inverses the checked path used (the kernels'), given to the fp32 oracle so that both start from the
    same numbers.  -> dict(disagree_fraction, worst_margin, depth_rel, points_abs)"""
    d, c, k = scene["depths"], scene["confs"], scene["cams"]
    m32, a32, _ = OF.filter_view(ref, srcs, d, c, k, method, inv=inv, **kw)
    _, _, margin = OF.filter_view(ref, srcs, d, c, k, method, dtype=torch.float64, **kw)
    mask, avg = mask.cpu(), avg.cpu()
    bad = mask != m32
    worst = float(margin[bad].max()) if bad.any() else 0.0
    assert worst < MARGIN, f"{int(bad.sum())} pixels disagree with the fp32 oracle, one with fp64 margin {worst:.3e}"
    frac = float(bad.float().mean())
    assert frac < MAX_DISAGREE, f"{frac:.3e} of the pixels disagree with the fp32 oracle"
    clear = (margin >= MARGIN) & torch.isfinite(a32)
    rel = float(((avg - a32).abs() / a32.abs().clamp_min(1e-12))[clear].max()) if clear.any() else 0.0
    assert rel < 1e-5, f"averaged depth differs by {rel:.3e} relative"
    out = dict(disagree_fraction=frac, worst_margin=worst, depth_rel=rel)
    if points is not None:
        both = mask & m32 & clear
        ref_pts = OF.view_points(ref, a32, k, inv=inv)
        out["points_abs"] = float((points.cpu() - ref_pts)[both].abs().max()) if both.any() else 0.0
        assert out["points_abs"] < 1e-3, f"points differ by {out['points_abs']:.3e}"
    return out


def scatter_points(mask, pts):
    """[M,3] points of the masked pixels in row-major order -> [H,W,3] (zeros elsewhere)"""
    full = torch.zeros(*mask.shape, 3, dtype=pts.dtype)
    full[mask.cpu()] = pts.cpu()
    return full
