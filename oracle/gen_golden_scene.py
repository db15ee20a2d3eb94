"""ORACLE - TEST INFRASTRUCTURE ONLY.  Generates the scene fixtures by executing the REFERENCE's own eval loader
(datasets/general_eval.MVSDataset, loaded read-only by oracle/reference.py) on small seeded scene
folders in the MVSNet layout, and the reference's own file writers (datasets/data_io.save_pfm, and write_cam as test.py
and test_tt.py define it, taken from their source at run time) on a fixed depth map and camera.

A case's folder, written to a temporary directory under <root>/test (dtu's ground truth under <root>/mvs_training, where
the loader opens it):
  {scan}/images/%08d.jpg     PIL JPEGs of synth.make_images
  {scan}/cams/%08d_cam.txt   look-at cameras (synth.lookat_camera) at the source size; line 11 in the case's forms
  {scan}/cams_1/...          dtu, view 0 only: the loader's depth interval 2.5
  short_range_cameras/cams_{scan}/...   T&T with use_short_range
  {scan}/pair.txt            view sets with fewer sources than nviews - 1 and one view without sources

Writes tests/golden/scene_<case>.npz:
  file_<i>              the bytes of every file of the folder (meta["files"][i] names it, relative to <root>)
  decoded_<vid>         PIL's uint8 [h,w,3] of each image (what the loader decodes)
  img_<vid>             the loader's normalised image [3,H,W] fp32 of each view (asserted equal in every item naming it)
  proj_<k>_stage<s>     item k's proj_matrices[stage s] [V,2,4,4] fp32;   dv_<k>: item k's depth_values [D] fp32
  pfm_bytes, cam_bytes  save_pfm of a fixed depth map, write_cam of item 0's stage4 reference camera (test_tt.py's form,
                        with its depth range, for tt)
  meta                  the case, the files, the items' view ids

Re-run:  python oracle/gen_golden_scene.py
"""
import io
import os
import sys
import tempfile

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

from mvsformerplusplus_b200 import synth  # noqa: E402
from oracle import fixture, reference  # noqa: E402

# sizes are (h, w) of the source JPEGs and (max_h, max_w) of the prepared images, multiples of 32 so that the model runs
CASES = {
    "dtu": dict(dataset="dtu", scan="scan1", src=(152, 200), max_h=96, max_w=128, nviews=4, ndepths=48, interval_scale=1.06,
                use_short_range=False, pairs={0: [1, 2, 3], 1: [0, 2, 3, 4], 2: [3], 3: [2, 1, 0], 4: []}, seed=501),
    "tt_identity": dict(dataset="tt", scan="Family", src=(56, 96), max_h=64, max_w=96, nviews=3, ndepths=32,
                        interval_scale=1.0, use_short_range=False, pairs={0: [1, 2], 1: [0, 2], 2: [1]}, seed=511),
    "tt_short_range": dict(dataset="tt", scan="Horse", src=(90, 150), max_h=64, max_w=96, nviews=3, ndepths=32,
                           interval_scale=1.0, use_short_range=True, pairs={0: [2, 1], 1: [0], 2: [0, 1]}, seed=521),
    "eth3d": dict(dataset="eth3d", scan="courtyard", src=(100, 160), max_h=64, max_w=96, nviews=3, ndepths=32,
                  interval_scale=1.0, use_short_range=False, pairs={0: [1, 2], 1: [2, 0], 2: [0, 1]}, seed=531),
}


def depth_line(case, vid):
    """line 11 of a cam file: dtu alternates the 2-token and the 4-token form, T&T uses 4 tokens (num_depth), eth3d
    gives depth_min and depth_max"""
    if case["dataset"] == "dtu":
        return "425.0 2.65" if vid % 2 == 0 else "425.0 2.65 192 933.8"
    if case["dataset"] == "tt":
        return "480.5 1.7 256 915.7"
    return "520.25 842.5"


def cam_text(E, K, line11):
    rows = ["extrinsic"] + [" ".join(f"{v:.6f}" for v in E[i]) for i in range(4)] + ["", "intrinsic"]
    rows += [" ".join(f"{v:.6f}" for v in K[i]) for i in range(3)] + ["", line11]
    return "\n".join(rows) + "\n"


def scene_files(case):
    """{path relative to root: bytes} of a case's folder"""
    from PIL import Image
    h, w = case["src"]
    scan, ds = case["scan"], case["dataset"]
    views = sorted(case["pairs"])
    files = {}
    imgs = synth.make_images(len(views), h, w, seed=case["seed"])
    for n, v in enumerate(views):
        u8 = (imgs[n] * 40.0 + 128.0).clamp(0, 255).round().byte().permute(1, 2, 0).contiguous().numpy()
        buf = io.BytesIO()
        Image.fromarray(u8).save(buf, "JPEG", quality=90)
        files[f"test/{scan}/images/{v:08d}.jpg"] = buf.getvalue()
        E, K = synth.lookat_camera(synth.VIEW_ORDER[n], h, w, theta_step=0.12)
        text = cam_text(E.numpy(), K.numpy(), depth_line(case, v)).encode()
        if ds == "tt" and case["use_short_range"]:
            files[f"test/short_range_cameras/cams_{scan.lower()}/{v:08d}_cam.txt"] = text
        else:
            files[f"test/{scan}/cams/{v:08d}_cam.txt"] = text
        if ds == "dtu" and v == 0:
            files[f"test/{scan}/cams_1/{v:08d}_cam.txt"] = text
        if ds == "dtu":
            buf = io.BytesIO()
            Image.fromarray(np.full((8, 8), 200, np.uint8)).save(buf, "PNG")
            files[f"mvs_training/Depths_raw/{scan}/depth_visual_{v:04d}.png"] = buf.getvalue()
            files[f"mvs_training/Depths_raw/{scan}/depth_map_{v:04d}.pfm"] = b"Pf\n8 8\n-1.000000\n" + np.ones(64, "<f4").tobytes()
    lines = [str(len(views))]
    for v in views:
        srcs = case["pairs"][v]
        lines += [str(v), " ".join([str(len(srcs))] + [f"{s} {100.0 - k:.1f}" for k, s in enumerate(srcs)])]
    files[f"test/{scan}/pair.txt"] = ("\n".join(lines) + "\n").encode()
    return files


def write_files(root, files):
    for rel, data in files.items():
        p = os.path.join(root, rel)
        os.makedirs(os.path.dirname(p), exist_ok=True)
        with open(p, "wb") as f:
            f.write(data)
    return os.path.join(root, "test")


def reference_datasets():
    """(general_eval, data_io) of the reference as modules, or None where the reference is not available"""
    if reference.root("datasets/general_eval.py", "datasets/data_io.py") is None:
        return None
    return reference.module("datasets/general_eval.py"), reference.module("datasets/data_io.py")


def generate(name, case, ge, data_io):
    from PIL import Image
    files = scene_files(case)
    with tempfile.TemporaryDirectory() as d:
        datapath = write_files(d, files)
        ds = ge.MVSDataset(datapath, [case["scan"]], "test", case["nviews"], ndepths=case["ndepths"],
                           interval_scale=case["interval_scale"], max_h=case["max_h"], max_w=case["max_w"],
                           dataset=case["dataset"], use_short_range=case["use_short_range"])
        blob, items, imgs = {}, [], {}
        for k in range(len(ds)):
            _, ref, srcs, _ = ds.metas[k]
            sample = ds[k]
            ids = [ref] + list(srcs)
            items.append(ids)
            for j, v in enumerate(ids):
                x = sample["imgs"][j].numpy()
                assert v not in imgs or np.array_equal(imgs[v], x), (name, v)
                imgs[v] = x
            for s in range(1, 5):
                blob[f"proj_{k}_stage{s}"] = sample["proj_matrices"][f"stage{s}"]
            blob[f"dv_{k}"] = sample["depth_values"]
        for v, x in imgs.items():
            blob[f"img_{v}"] = x
            p = os.path.join(datapath, "{}/images/{:0>8}.jpg".format(case["scan"], v))
            blob[f"decoded_{v}"] = np.asarray(Image.open(p).convert("RGB"))
        # the writers, on a fixed depth map and item 0's stage4 reference camera
        g = np.random.default_rng(case["seed"])
        depth = (400 + 500 * g.random((case["max_h"], case["max_w"]))).astype(np.float32)
        data_io.save_pfm(os.path.join(d, "d.pfm"), depth)
        cam = blob["proj_0_stage4"][0]
        if case["dataset"] == "tt":
            dv = blob["dv_0"]
            reference.function("test_tt.py", "write_cam")(os.path.join(d, "c.txt"), cam, [dv[0], dv[-1]])
        else:
            reference.function("test.py", "write_cam")(os.path.join(d, "c.txt"), cam)
        blob["pfm_depth"] = depth
        blob["pfm_bytes"] = np.frombuffer(open(os.path.join(d, "d.pfm"), "rb").read(), np.uint8)
        blob["cam_bytes"] = np.frombuffer(open(os.path.join(d, "c.txt"), "rb").read(), np.uint8)
    names = sorted(files)
    for i, rel in enumerate(names):
        blob[f"file_{i}"] = np.frombuffer(files[rel], np.uint8)
    meta = dict(case, pairs={str(k): v for k, v in case["pairs"].items()}, files=names, items=items)
    path = os.path.join(REPO, "tests", "golden", f"scene_{name}.npz")
    fixture.save(path, blob, meta)
    print(name, len(items), "items", os.path.getsize(path), "bytes")


def main():
    mods = reference_datasets()
    if mods is None:
        raise SystemExit("reference sources not found")
    for name, case in CASES.items():
        generate(name, case, *mods)


if __name__ == "__main__":
    main()
