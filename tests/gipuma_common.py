"""Shared helpers of the gipuma fusion tests: the reference-executed fixture and the per-view comparison rule."""
import os

import torch

from oracle import fixture
from oracle import gipuma as OG
from tests.common import GOLDEN

FIXTURE = "gipuma_n8_40x72"
MARGIN = 1e-4          # a decision may differ from the oracle's only this close (relative) to its boundary ...
MAX_DISAGREE = 1e-3    # ... and on fewer than this share of a view's pixels


def load_fixture():
    """-> scene dict (depths, confs = conf_u8 / 255 in fp32, cams, images in [0,1]), meta, the raw arrays"""
    z, meta = fixture.load(os.path.join(GOLDEN, FIXTURE + ".npz"))
    scene = dict(depths=torch.from_numpy(z["depths"]), confs=torch.from_numpy(z["conf_u8"]).float() / 255,
                 cams=torch.from_numpy(z["cams"]), images=torch.from_numpy(z["images"]).float() / 255)
    return scene, meta, z


def compare_step(got_keep, got_xyz, got_rgb, got_used, want, truth):
    """One view's step against the fp32 oracle's `want` from the same used state; `truth` is the fp64 oracle's step (with
    footprint_below=MARGIN) for the margins.  Emit decisions may differ only at pixels of fp64 margin < MARGIN and on fewer
    than MAX_DISAGREE of the pixels; used marks only inside the footprint of such pixels; points agree to 1e-3 and
    colours exactly where both emit.  -> dict of the numbers"""
    keep = want["keep"]
    dis = got_keep != keep
    frac = float(dis.float().mean())
    assert frac < MAX_DISAGREE, f"{frac:.2e} of the pixels disagree"
    if dis.any():
        assert float(truth["margin"][dis].max()) < MARGIN, "an emit decision far from its boundary differs"
    udis = got_used != want["used"]
    if udis.any():
        assert bool(truth["footprint"][udis].all()), "a used mark no near-boundary decision explains differs"
    both = got_keep & keep
    gi = torch.cumsum(got_keep.reshape(-1).long(), 0)[both.reshape(-1)] - 1
    wi = torch.cumsum(keep.reshape(-1).long(), 0)[both.reshape(-1)] - 1
    err = float((got_xyz[gi] - want["xyz"][wi].float()).abs().max()) if len(gi) else 0.0
    assert err < 1e-3, err
    assert torch.equal(got_rgb[gi], want["rgb"][wi])
    return dict(disagree=frac, used_disagree=int(udis.sum()), xyz_err=err, points=int(got_keep.sum()))


def oracle_steps(ref, D, table, cams, images, used, disp, nc, range_margin=None):
    """-> (fp32 step on `table` (the kernel's own), fp64 step on the fp64 table of `cams` with margins and footprint),
    both from `used`"""
    want = OG.step(ref, D, table, images, used, disp, nc, torch.float32, range_margin)
    truth = OG.step(ref, D, OG.camera_table(cams, torch.float64), images, used, disp, nc, torch.float64, range_margin,
                    footprint_below=MARGIN)
    return want, truth
