"""Golden vectors of the camera input stage (TEST INFRASTRUCTURE ONLY): the UNMODIFIED reference's sample_augmentation
(is_train False), img_transform (PIL resize + crop) and normalize_img (ToTensor + Normalize) on seeded uint8 frames.

    python -m oracle.make_golden_camera_input        (needs the reference package: oracle/_ref or HEAL_REFERENCE_ROOT, and Pillow)

Writes tests/golden/camera_input.pt: per case the data_aug_conf, the frames (n, H0, W0, 3) uint8, the reference's images
(n, 3, fH, fW) fp32, resize_dims, crop, post_rot and post_tran.  The cases are small: a downscale whose crop starts above the
resized frame (as every shipped conf's does), an upscale, and a frame whose size differs from the conf's H / W (PIL resizes the
frame it is given)."""
import os
import sys

import numpy as np
import torch

from oracle import ref_shim

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "camera_input.pt")

CASES = (
    ({"H": 60, "W": 80, "final_dim": [40, 48], "bot_pct_lim": [0.0, 0.05]}, (60, 80), 101),
    ({"H": 30, "W": 40, "final_dim": [48, 56], "bot_pct_lim": [0.0, 0.05]}, (30, 40), 102),
    ({"H": 60, "W": 80, "final_dim": [32, 40], "bot_pct_lim": [0.0, 0.05]}, (45, 70), 103),
)
FRAMES_PER_CASE = 2


def reference_case(cu, conf, frames):
    """The reference's camera branch for each frame (intermediate_heter_fusion_dataset.py:199-242, no depth image)."""
    from PIL import Image
    imgs, out = [], {}
    for f in frames:
        resize, resize_dims, crop, flip, rotate = cu.sample_augmentation(conf, False)
        img_src, post_rot2, post_tran2 = cu.img_transform([Image.fromarray(f)], torch.eye(2), torch.zeros(2), resize=resize,
                                                          resize_dims=resize_dims, crop=crop, flip=flip, rotate=rotate)
        imgs.append(cu.normalize_img(img_src[0]))
        out.update(resize_dims=tuple(resize_dims), crop=tuple(crop), post_rot=post_rot2, post_tran=post_tran2)
    out["imgs"] = torch.stack(imgs)
    return out


def main():
    ref_shim.install()
    import opencood.utils.camera_utils as cu
    cases = []
    for conf, (H0, W0), seed in CASES:
        frames = np.random.default_rng(seed).integers(0, 256, (FRAMES_PER_CASE, H0, W0, 3), dtype=np.uint8)
        r = reference_case(cu, conf, frames)
        cases.append({"conf": conf, "frames": torch.from_numpy(frames), **r})
        print(f"conf {conf} frame {H0}x{W0}: resize_dims {r['resize_dims']} crop {r['crop']} -> {tuple(r['imgs'].shape)}")
    torch.save({"cases": cases}, OUT)
    print(f"wrote {OUT} ({os.path.getsize(OUT)} bytes)")


if __name__ == "__main__":
    sys.exit(main())
