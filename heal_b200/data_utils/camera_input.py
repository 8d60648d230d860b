"""Host plan of the camera agent's image stage on the GPU (SURVEY.md 8f-4).

The reference prepares every camera frame on the host, in its DataLoader workers (intermediate_heter_fusion_dataset.py:199-246):
`sample_augmentation(data_aug_conf, is_train=False)` picks a resize and a crop (opencood/utils/camera_utils.py:33-59),
`img_transform` applies them with PIL and updates the post-homography (:62-91), and `normalize_img` is ToTensor + Normalize
(:120-125).  Here the frames stay uint8 until `heal_camera_input` (csrc/camera_input.cu) resamples them on the GPU, bit for bit:

    plan = inference_plan(data_aug_conf, H0, W0)        # resize_dims, crop, post_rot, post_tran of the reference
    imgs = ops.camera_input(frames, plan, "nchw")       # frames uint8 (n, H0, W0, 3) -> fp32 (n, 3, fH, fW)

`resize_dims` comes from the conf's H / W, as the reference computes it; the coefficients come from the real frame size (H0, W0),
because PIL resizes the image it is given.  The device tables are cached per (H0, W0, resize_dims, crop, device), so a captured
graph replays without host work.

`reference_pair` makes the drop-in replacements of `img_transform` / `normalize_img` that heal_b200.install.install_gpu_camera_input
puts into the reference's datasets: in the inference case they ship the decoded frame as a uint8 (H0, W0, 3) tensor instead of the
normalised image."""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np
import torch

PRECISION_BITS = 22          # Pillow's fixed-point precision for 8-bit images
TILE_ROWS = 32               # output rows per CTA of k_camera_input (csrc/camera_input.cu TH)


@dataclass(frozen=True)
class CameraPlan:
    """The reference's inference augmentation of one camera frame of size (H0, W0)."""
    H0: int
    W0: int
    final_dim: tuple            # (fH, fW)
    resize: float
    resize_dims: tuple          # (newW, newH), as PIL's resize takes it
    crop: tuple                 # (left, top, right, bottom) in the resized frame; may lie outside it
    post_rot: torch.Tensor      # (2, 2) fp32, as img_transform returns it
    post_tran: torch.Tensor     # (2,) fp32

    def post_rot3(self) -> torch.Tensor:
        """The dataset's 3x3 form (intermediate_heter_fusion_dataset.py:233-236)."""
        r = torch.eye(3)
        r[:2, :2] = self.post_rot
        return r

    def post_tran3(self) -> torch.Tensor:
        t = torch.zeros(3)
        t[:2] = self.post_tran
        return t

    def tables(self, device):
        """(col_table, col_taps, row_table, row_taps, span_rows) on `device` for heal_camera_input, cached."""
        dev = torch.device(device)
        key = (self.H0, self.W0, self.resize_dims, self.crop, dev)
        hit = _TABLES.get(key)
        if hit is None:
            l, t, r, b = self.crop
            newW, newH = self.resize_dims
            cols = axis_table(self.W0, newW, l, r - l)
            rows = axis_table(self.H0, newH, t, b - t)
            hit = (torch.from_numpy(cols).to(dev), cols.shape[1] - 2, torch.from_numpy(rows).to(dev), rows.shape[1] - 2,
                   span_rows(rows))
            _TABLES[key] = hit
        return hit


_TABLES = {}


def inference_plan(data_aug_conf, H0: int, W0: int) -> CameraPlan:
    """sample_augmentation(data_aug_conf, is_train=False) and img_transform's post_rot / post_tran (flip False, rotate 0), with the
    reference's arithmetic: python floats for the resize and the crop, fp32 torch for the matrices."""
    missing = [k for k in ('H', 'W', 'final_dim', 'bot_pct_lim') if k not in data_aug_conf]
    if missing:
        raise ValueError(f"raw camera frames need data_aug_conf {missing} (the reference's sample_augmentation reads them)")
    H, W = data_aug_conf['H'], data_aug_conf['W']
    fH, fW = data_aug_conf['final_dim']
    resize = max(fH / H, fW / W)
    resize_dims = (int(W * resize), int(H * resize))
    newW, newH = resize_dims
    crop_h = int((1 - np.mean(data_aug_conf['bot_pct_lim'])) * newH) - fH
    crop_w = int(max(0, newW - fW) / 2)
    crop = (crop_w, crop_h, crop_w + fW, crop_h + fH)
    post_rot = torch.eye(2)
    post_rot *= resize
    post_tran = torch.zeros(2) - torch.Tensor(crop[:2])
    A = torch.Tensor([[np.cos(0.0), np.sin(0.0)], [-np.sin(0.0), np.cos(0.0)]])     # get_rot(0)
    c = torch.Tensor([crop[2] - crop[0], crop[3] - crop[1]]) / 2
    c = A.matmul(-c) + c
    post_rot = A.matmul(post_rot)
    post_tran = A.matmul(post_tran) + c
    return CameraPlan(int(H0), int(W0), (int(fH), int(fW)), resize, resize_dims, crop, post_rot, post_tran)


def _bicubic(x):
    """Pillow's bicubic kernel (a = -0.5) in double, elementwise."""
    a = -0.5
    x = np.abs(x)
    near = ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    far = (((x - 5) * x + 8) * x - 4) * a
    return np.where(x < 1.0, near, np.where(x < 2.0, far, 0.0))


def axis_table(in_size: int, out_size: int, first: int, n: int) -> np.ndarray:
    """int32 (n, 2 + K): for output index first + i of an axis resized from in_size to out_size, Pillow's 8-bit bicubic window
    (first source index, tap count, K taps in 22-bit fixed point, zero-padded).  Indices outside [0, out_size) get a count of 0 (the
    crop's black border); an axis that keeps its size gets one tap of 1.0 (Pillow skips that pass, and one unit tap reproduces it)."""
    idx = first + np.arange(n)
    inside = (idx >= 0) & (idx < out_size)
    if in_size == out_size:
        tab = np.zeros((n, 3), dtype=np.int64)
        tab[:, 0] = np.where(inside, idx, 0)
        tab[:, 1] = inside
        tab[:, 2] = np.where(inside, 1 << PRECISION_BITS, 0)
        return tab.astype(np.int32)
    scale = float(in_size) / out_size
    filterscale = max(scale, 1.0)
    support = 2.0 * filterscale
    center = (idx.astype(np.float64) + 0.5) * scale
    lo = np.maximum(np.trunc(center - support + 0.5), 0).astype(np.int64)
    hi = np.minimum(np.trunc(center + support + 0.5), in_size).astype(np.int64)
    count = np.where(inside, hi - lo, 0)
    K = max(int(count.max()), 1)
    k = np.arange(K)
    live = k[None, :] < count[:, None]
    w = np.where(live, _bicubic((k[None, :] + lo[:, None] - center[:, None] + 0.5) / filterscale), 0.0)
    ww = np.zeros(n)
    for j in range(K):                               # Pillow adds the weights one after the other
        ww = ww + w[:, j]
    w = np.where(ww[:, None] != 0.0, w / np.where(ww == 0.0, 1.0, ww)[:, None], w)
    q = np.trunc(np.where(w < 0, -0.5 + w * (1 << PRECISION_BITS), 0.5 + w * (1 << PRECISION_BITS))).astype(np.int64)
    tab = np.zeros((n, 2 + K), dtype=np.int64)
    tab[:, 0] = np.where(inside, lo, 0)
    tab[:, 1] = count
    tab[:, 2:] = np.where(live, q, 0)
    return tab.astype(np.int32)


def span_rows(row_table: np.ndarray) -> int:
    """The most source rows one band of TILE_ROWS output rows reads (the kernel's shared tile height)."""
    span = 1
    for y0 in range(0, row_table.shape[0], TILE_ROWS):
        band = row_table[y0:y0 + TILE_ROWS]
        live = np.nonzero(band[:, 1] > 0)[0]
        if live.size:
            a, b = band[live[0]], band[live[-1]]
            span = max(span, int(b[0] + b[1] - a[0]))
    return span


def reference_pair(img_transform, normalize_img):
    """Drop-in replacements of the reference's `img_transform` and `normalize_img` for the datasets' camera branch.  For one RGB PIL
    image with flip False and rotate 0 (the inference augmentation, no depth image), `img_transform` returns the decoded frame as a
    uint8 (H0, W0, 3) tensor with the reference's own post_rot / post_tran, and `normalize_img` passes that tensor through, so the
    batch carries raw frames that LiftSplatShoot resamples on the GPU with its own data_aug_conf.  Anything else goes to the
    originals.  Meant for datasets built with train=False: a training crop is random and only the inference plan runs on the GPU."""

    def gpu_img_transform(imgs, post_rot, post_tran, resize, resize_dims, crop, flip, rotate):
        if flip or rotate != 0 or len(imgs) != 1 or getattr(imgs[0], "mode", None) != "RGB":
            return img_transform(imgs, post_rot, post_tran, resize=resize, resize_dims=resize_dims, crop=crop, flip=flip,
                                 rotate=rotate)
        frame = torch.from_numpy(np.array(imgs[0], dtype=np.uint8))
        _, post_rot2, post_tran2 = img_transform([], post_rot, post_tran, resize=resize, resize_dims=resize_dims, crop=crop,
                                                 flip=flip, rotate=rotate)
        return [frame], post_rot2, post_tran2

    def gpu_normalize_img(img):
        if isinstance(img, torch.Tensor) and img.dtype == torch.uint8:
            return img
        return normalize_img(img)

    gpu_img_transform.reference = img_transform
    gpu_normalize_img.reference = normalize_img
    return gpu_img_transform, gpu_normalize_img
