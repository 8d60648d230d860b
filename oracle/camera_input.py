"""ORACLE — TEST INFRASTRUCTURE ONLY.  numpy restatement of the reference's inference image path for one RGB frame:
`normalize_img(Image.fromarray(frame).resize(resize_dims).crop(crop))` (opencood/utils/camera_utils.py:62-91, :120-125).

Pillow's 8-bit resize with its default filter (antialiased bicubic, a = -0.5):
  - per axis, scale = in / out and support = 2 * max(scale, 1); output index x has the window centre (x + 0.5) * scale, the first
    tap max(int(centre - support + 0.5), 0) and the last min(int(centre + support + 0.5), in) - 1; weights are the bicubic kernel at
    (tap - centre + 0.5) / max(scale, 1) in double, divided by their sum, then rounded away from zero to 22-bit integers;
  - sums are integers starting at 1 << 21, shifted right by 22 and clipped to [0, 255];
  - the horizontal pass runs first and is clipped to uint8 before the vertical pass; an axis that keeps its size is not resampled.
`crop` fills pixels outside the resized frame with 0.  `normalize_img` is ToTensor (u / 255 in fp32) then
Normalize((x - mean) / std in fp32).

No PIL here: the GPU tests compare against this module on the GPU machine.  tests/test_camera_input_cpu.py pins it to PIL and
torchvision bit for bit."""
import numpy as np

PRECISION_BITS = 22
MEAN = np.array([0.485, 0.456, 0.406], dtype=np.float32)
STD = np.array([0.229, 0.224, 0.225], dtype=np.float32)


def _bicubic(x):
    a = -0.5
    x = abs(x)
    if x < 1.0:
        return ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    if x < 2.0:
        return (((x - 5) * x + 8) * x - 4) * a
    return 0.0


def coefficients(in_size: int, out_size: int):
    """Per output index: (first tap, int32 weights) of Pillow's 8-bit bicubic resample of one axis."""
    scale = float(in_size) / out_size
    filterscale = max(scale, 1.0)
    support = 2.0 * filterscale
    out = []
    for x in range(out_size):
        center = (x + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        xmax = min(int(center + support + 0.5), in_size) - xmin
        w = [_bicubic((i + xmin - center + 0.5) / filterscale) for i in range(xmax)]
        ww = sum(w)
        w = [v / ww if ww != 0.0 else v for v in w]
        q = [int(-0.5 + v * (1 << PRECISION_BITS)) if v < 0 else int(0.5 + v * (1 << PRECISION_BITS)) for v in w]
        out.append((xmin, np.array(q, dtype=np.int64)))
    return out


def _pass(img, coeffs, axis):
    """One resample pass along `axis` (0 rows, 1 columns) of a uint8 (H, W, 3) image."""
    src = np.moveaxis(img.astype(np.int64), axis, 0)
    res = np.empty((len(coeffs),) + src.shape[1:], dtype=np.int64)
    for o, (start, w) in enumerate(coeffs):
        acc = np.full(src.shape[1:], 1 << (PRECISION_BITS - 1), dtype=np.int64)
        for k, wk in enumerate(w):
            acc += src[start + k] * wk
        res[o] = np.clip(acc >> PRECISION_BITS, 0, 255)
    return np.moveaxis(res.astype(np.uint8), 0, axis)


def resize(frame, dims):
    """uint8 (H0, W0, 3) -> uint8 (H, W, 3), dims = (W, H) as PIL takes it."""
    W, H = dims
    H0, W0 = frame.shape[:2]
    img = frame
    if W != W0:
        img = _pass(img, coefficients(W0, W), 1)
    if H != H0:
        img = _pass(img, coefficients(H0, H), 0)
    return img


def crop(img, box):
    """PIL crop (l, t, r, b): pixels outside the image are 0."""
    l, t, r, b = box
    H, W = img.shape[:2]
    out = np.zeros((b - t, r - l, 3), dtype=np.uint8)
    y0, y1, x0, x1 = max(t, 0), min(b, H), max(l, 0), min(r, W)
    if y0 < y1 and x0 < x1:
        out[y0 - t:y1 - t, x0 - l:x1 - l] = img[y0:y1, x0:x1]
    return out


def normalize(u8):
    """uint8 (H, W, 3) -> fp32 (3, H, W): (u / 255 - mean) / std, each step rounded to fp32."""
    x = np.ascontiguousarray(u8.transpose(2, 0, 1)).astype(np.float32) / np.float32(255)
    return (x - MEAN[:, None, None]) / STD[:, None, None]


def camera_input(frame, dims, box):
    """The reference's resize -> crop -> normalize_img of one frame: fp32 (3, b - t, r - l)."""
    return normalize(crop(resize(frame, dims), box))


def to_s2d(chw):
    """fp32 (3, H, W) -> the ResNet-101 stem's space-to-depth input (H/4, W/4, 64): channel c*16 + dy*4 + dx, c == 3 zero."""
    _, H, W = chw.shape
    x4 = np.zeros((4, H, W), dtype=np.float32)
    x4[:3] = chw
    return np.ascontiguousarray(x4.reshape(4, H // 4, 4, W // 4, 4).transpose(1, 3, 0, 2, 4).reshape(H // 4, W // 4, 64))
