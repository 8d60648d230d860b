"""Drop the heal_b200 mirrors into an importable `opencood` tree so that the reference's own entry points
(opencood/tools/train_utils.create_model -> importlib `opencood.models.<core_method>`, heter_pyramid_collab's
`opencood.models.heter_encoders` lookup) resolve to the B200 implementations.  See INTEGRATION.md."""
import importlib
import sys

_MAP = {
    "opencood.models.heter_pyramid_collab": "heal_b200.models.heter_pyramid_collab",
    "opencood.models.heter_model_baseline": "heal_b200.models.heter_model_baseline",
    "opencood.models.heter_model_baseline_ms": "heal_b200.models.heter_model_baseline_ms",
    "opencood.models.heter_model_late": "heal_b200.models.heter_model_late",
    "opencood.models.heter_pyramid_single": "heal_b200.models.heter_pyramid_single",
    "opencood.models.point_pillar": "heal_b200.models.point_pillar",
    "opencood.models.heter_encoders": "heal_b200.models.heter_encoders",
    "opencood.models.fuse_modules.pyramid_fuse": "heal_b200.models.fuse_modules.pyramid_fuse",
    "opencood.models.sub_modules.pillar_vfe": "heal_b200.models.sub_modules.pillar_vfe",
    "opencood.models.sub_modules.point_pillar_scatter": "heal_b200.models.sub_modules.point_pillar_scatter",
    "opencood.models.sub_modules.mean_vfe": "heal_b200.models.sub_modules.mean_vfe",
    "opencood.models.sub_modules.sparse_backbone_3d": "heal_b200.models.sub_modules.sparse_backbone_3d",
    "opencood.models.sub_modules.height_compression": "heal_b200.models.sub_modules.height_compression",
    "opencood.models.sub_modules.base_bev_backbone": "heal_b200.models.sub_modules.base_bev_backbone",
    "opencood.models.sub_modules.base_bev_backbone_resnet": "heal_b200.models.sub_modules.base_bev_backbone_resnet",
    "opencood.models.sub_modules.resblock": "heal_b200.models.sub_modules.resblock",
    "opencood.models.sub_modules.downsample_conv": "heal_b200.models.sub_modules.downsample_conv",
    "opencood.models.sub_modules.naive_compress": "heal_b200.models.sub_modules.naive_compress",
}


def install_gpu_postprocessor():
    """Opt-in: make the reference's post-processor registry (opencood/data_utils/post_processor/__init__.py `__all__`) hand out a
    SUBCLASS of its own VoxelPostprocessor whose `post_process` runs on the GPU for early, intermediate and late fusion (one cav or
    up to 16 cavs with one head geometry, with or without iou_preds) and falls back to the reference implementation for everything
    else (CPU tensors, anchor-free heads, cavs whose head maps differ in size).  All label / collate / gt-box methods
    the datasets call are inherited unchanged."""
    from .data_utils.post_processor.voxel_postprocessor import make_reference_subclass
    reg = importlib.import_module("opencood.data_utils.post_processor")
    ref_cls = importlib.import_module("opencood.data_utils.post_processor.voxel_postprocessor").VoxelPostprocessor
    cls = make_reference_subclass(ref_cls)
    reg.__all__["VoxelPostprocessor"] = cls
    return cls


CAMERA_DATASETS = (
    "opencood.data_utils.datasets.intermediate_fusion_dataset",
    "opencood.data_utils.datasets.intermediate_2stage_fusion_dataset",
    "opencood.data_utils.datasets.intermediate_heter_fusion_dataset",
    "opencood.data_utils.datasets.late_fusion_dataset",
    "opencood.data_utils.datasets.late_heter_fusion_dataset",
    "opencood.data_utils.datasets.heter_infer.intermediate_heter_infer_fusion_dataset",
)


def install_gpu_camera_input(modules=CAMERA_DATASETS):
    """Opt-in: rebind `img_transform` and `normalize_img` in the reference's dataset modules that import them, so that the camera
    branch of an inference batch (flip False, rotate 0, no depth image) carries each decoded frame as a uint8 (H0, W0, 3) tensor
    with the reference's own post_rot / post_tran; LiftSplatShoot then resizes, crops and normalises every camera of a modality in
    one heal_camera_input launch.  Every other case runs the reference's functions.  Returns the modules it changed."""
    from .data_utils.camera_input import reference_pair
    done = []
    for name in modules:
        mod = importlib.import_module(name)
        ref_t = getattr(mod.img_transform, "reference", mod.img_transform)
        ref_n = getattr(mod.normalize_img, "reference", mod.normalize_img)
        mod.img_transform, mod.normalize_img = reference_pair(ref_t, ref_n)
        done.append(name)
    return done


def install_gpu_eval():
    """Opt-in: rebind `opencood.utils.eval_utils.caluclate_tp_fp` to heal_b200.utils.eval_utils.caluclate_tp_fp, which matches a
    frame's detections to its GT boxes on the GPU when both are CUDA fp32 (N, 8, 3) tensors and calls the reference function
    (kept as `.reference`) otherwise.  inference.py, inference_w_noise.py and inference_heter_in_order.py all call it through the
    module, so this covers the three.  Returns the new function."""
    from .utils import eval_utils as ours
    mod = importlib.import_module("opencood.utils.eval_utils")
    cur = mod.caluclate_tp_fp
    if cur is not ours.caluclate_tp_fp:
        ours.caluclate_tp_fp.reference = cur
    mod.caluclate_tp_fp = ours.caluclate_tp_fp
    return ours.caluclate_tp_fp


def install_into_opencood(only=None):
    """Alias the mirrors under their opencood module names (call BEFORE opencood.tools imports the models)."""
    done = []
    for ref_name, ours in _MAP.items():
        if only is not None and ref_name not in only:
            continue
        sys.modules[ref_name] = importlib.import_module(ours)
        done.append(ref_name)
    return done
