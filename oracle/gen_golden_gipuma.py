"""ORACLE - TEST INFRASTRUCTURE ONLY.  Generates the gipuma fusion fixture by executing the REFERENCE's own input stage of
gipuma_filter (misc/gipuma.py and datasets/data_io.py, loaded read-only by oracle/reference.py) on a
seeded scene of synth.make_fusion_scene, written to disk the way test.py saves a scan:

  depth_est/<view>.pfm          datasets/data_io.save_pfm (test.py:278)
  confidence/<view>.npy         uint8(conf * 255) (test.py:285-286)
  cams/<view>_cam.txt           the extrinsic / intrinsic text format of test.py:149-166
  images/<view>.jpg             names only: probability_filter and mvsnet_to_gipuma list the folder

then misc/gipuma.probability_filter (-> depth_est/<view>_prob_filtered.pfm, read back with data_io.read_pfm) and
misc/gipuma.mvsnet_to_gipuma_cam (-> the 3x4 P text file, parsed in fp64).  fusibile itself is not part of the reference,
so the fixture holds the inputs it would get.  Writes only

  tests/golden/gipuma_n8_40x72.npz   depths, conf_u8, cams, images (uint8), filtered (the prob_filtered depths), P [N,3,4]
                                     fp64, meta (N, H, W, seed, prob_threshold, and the disp_threshold / num_consistent the
                                     tests use at this size)

Re-run:  python oracle/gen_golden_gipuma.py
"""
import os
import sys
import tempfile

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

from mvsformerplusplus_b200 import synth  # noqa: E402
from oracle import fixture, reference  # noqa: E402

NAME = "gipuma_n8_40x72"
# f b / depth is ~0.108 at this size (f ~ 130 px, depth ~ 650), so a disparity threshold of the order of the synthetic
# depth noise (0.0015 ~ 1.4 % in depth) makes the consistency test go both ways
CASE = dict(N=8, H=40, W=72, seed=81, n_src=7, prob_threshold=0.5, disp_threshold=0.0015, num_consistent=2)


def reference_gipuma_modules():
    """(misc/gipuma.py, datasets/data_io.py) of the reference as modules, or None where the reference is not available"""
    if reference.root("misc/gipuma.py", "datasets/data_io.py") is None:
        return None
    return reference.module("misc/gipuma.py"), reference.module("datasets/data_io.py")


def write_cam(path, cam):
    """the cam text file of test.py:149-166: extrinsic 4x4, intrinsic 3x3, then the depth line of slot 1's last row"""
    E, K = cam[0], cam[1]
    lines = ["extrinsic"] + [" ".join(str(v) for v in E[i]) + " " for i in range(4)] + ["", "intrinsic"]
    lines += [" ".join(str(v) for v in K[i, :3]) + " " for i in range(3)]
    lines += ["", " ".join(str(v) for v in K[3])]
    with open(path, "w") as f:
        f.write("\n".join(lines) + "\n")


def reference_inputs(gipuma, data_io, depths, conf_u8, cams, prob_threshold):
    """-> filtered depths [N,H,W] fp32 and P [N,3,4] fp64, through the reference's own functions on files"""
    N = depths.shape[0]
    with tempfile.TemporaryDirectory() as d:
        for sub in ("depth_est", "confidence", "cams", "images"):
            os.makedirs(os.path.join(d, sub))
        for n in range(N):
            v = f"{n:08d}"
            data_io.save_pfm(os.path.join(d, "depth_est", v + ".pfm"), np.ascontiguousarray(depths[n]))
            np.save(os.path.join(d, "confidence", v + ".npy"), conf_u8[n])
            write_cam(os.path.join(d, "cams", v + "_cam.txt"), cams[n])
            open(os.path.join(d, "images", v + ".jpg"), "wb").close()
        gipuma.probability_filter(d, prob_threshold)
        filtered, P = [], []
        for n in range(N):
            v = f"{n:08d}"
            filtered.append(np.ascontiguousarray(data_io.read_pfm(os.path.join(d, "depth_est", v + "_prob_filtered.pfm"))[0]))
            out = os.path.join(d, v + ".P")
            gipuma.mvsnet_to_gipuma_cam(os.path.join(d, "cams", v + "_cam.txt"), out)
            with open(out) as f:
                P.append(np.array([[float(x) for x in line.split()] for line in f.read().split("\n") if line.strip()]))
    return np.stack(filtered).astype(np.float32), np.stack(P).astype(np.float64)


def scene():
    """the fixture's scene as the reference would have saved it: depths, uint8 confidences, cams, uint8 images"""
    sc = synth.make_fusion_scene(CASE["N"], CASE["H"], CASE["W"], seed=CASE["seed"], n_src=CASE["n_src"])
    conf_u8 = (sc["confs"].numpy() * 255).astype(np.uint8)   # test.py:285-286
    images = torch.round(sc["images"] * 255).to(torch.uint8).numpy()
    return sc["depths"].numpy(), conf_u8, sc["cams"].numpy(), images


def main():
    mods = reference_gipuma_modules()
    if mods is None:
        raise SystemExit("reference sources not found")
    depths, conf_u8, cams, images = scene()
    filtered, P = reference_inputs(*mods, depths, conf_u8, cams, CASE["prob_threshold"])
    print(NAME, "valid after probability_filter", float((filtered > 0).mean()))
    path = os.path.join(REPO, "tests", "golden", NAME + ".npz")
    fixture.save(path, dict(depths=depths, conf_u8=conf_u8, cams=cams, images=images, filtered=filtered, P=P), CASE)
    print(NAME, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
