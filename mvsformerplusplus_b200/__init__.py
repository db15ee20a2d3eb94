"""CUDA-native (H100, sm_90a) depth-inference hot path of MVSFormer++ (FMT -> warp/group-correlation/visibility aggregation ->
cost regularisation -> soft-argmax, 4-stage cascade) behind the reference's Python seams.  See DESIGN.md."""
from .config import default_args, load_args, validate_args  # noqa: F401

__all__ = ["default_args", "load_args", "validate_args", "StageNet", "FMT_with_pathway", "HotPathNet", "install",
           "cascade_forward", "homo_warping_3D_with_mask", "FPNEncoder", "FPNDecoder", "CrossVITDecoder",
           "DinoVisionTransformer", "vit_base", "DINOv2MVSNet", "filter_view", "fuse_scene", "fuse_scene_gipuma", "write_ply",
           "read_pair_file", "load_scene", "reconstruct_scene"]


def __getattr__(name):  # hotpath imports torch + ctypes; keep `import mvsformerplusplus_b200` light
    if name in ("StageNet", "FMT_with_pathway", "HotPathNet", "install", "cascade_forward", "to_nhwc", "to_nchw",
                "homo_warping_3D_with_mask", "FPNEncoder", "FPNDecoder",
                "CrossVITDecoder", "DinoVisionTransformer", "vit_base", "DINOv2MVSNet"):
        from . import hotpath
        return getattr(hotpath, name)
    if name in ("filter_view", "fuse_scene", "fuse_scene_gipuma", "write_ply", "read_pair_file"):
        from . import fusion
        return getattr(fusion, name)
    if name in ("load_scene", "reconstruct_scene"):
        from . import scene
        return getattr(scene, name)
    raise AttributeError(name)
