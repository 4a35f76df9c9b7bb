"""numpy restatement of the reference's Cityscapes-3D sample transform (TP/data/cityscapes3d.py:117-233 with
is_transform=True, augmentations=None, tasks semseg / depth), as mtt_cityscapes_targets and preprocess_image compute it.

PIL NEAREST rule (Pillow 12.2, Image.resize -> ImagingScaleAffine, modes 'F' and 'L' alike), checked exhaustively by
tests/test_cityscapes.py against PIL itself: with s = n_src / n_dst formed in double, the source coordinate of output
index d is the running sum c_0 = s * 0.5, c_{d+1} = c_d + s, every addition rounded to double, and the source index is
trunc(c_d). It is NOT floor((d + 0.5) * s): the accumulated rounding can land just below an integer, e.g. 2 -> 7 picks
source 0 at d = 3 where (3.5 * 2 / 7) is exactly 1. np.cumsum adds sequentially, so it reproduces the sum.

Order: the reference converts the disparity (:151-160), encodes the label ids (:186), then casts to float, resizes and
casts back (:206-221). Every step but the resize is pointwise, so each output pixel is the encoded / converted value of
its nearest-sampled source pixel. The image is cv2.imread (uint8 BGR) -> float32 -> RGB -> uint8 (exact) -> ToTensor
(x / 255) -> Normalize ((x - mean) / std), all IEEE fp32.
"""
import numpy as np

VOID = (0, 1, 2, 3, 4, 5, 6, 9, 10, 14, 15, 16, 18, 29, 30)            # cityscapes3d.py:92 (-1 never matches uint8)
VALID = (7, 8, 11, 12, 13, 17, 19, 20, 21, 22, 23, 24, 25, 26, 27, 28, 31, 32, 33)   # :93
IGNORE = 255
N_CLASSES = 19
ORI_SIZE = (1024, 2048)    # :102: dd_label_map_size equal to this skips the resize
MEAN = np.array([0.485, 0.456, 0.406], np.float32)
STD = np.array([0.229, 0.224, 0.225], np.float32)
SKY_ID = 10                # the reference's `sky_mask = lbl == 10` (:159); Cityscapes id 10 is rail track, sky is 23


def encode_lut():
    """encode_segmap (:235-241) as a 256-entry table over uint8 ids."""
    lut = np.arange(256, dtype=np.int64)
    lut[list(VOID)] = IGNORE
    lut[list(VALID)] = np.arange(N_CLASSES)
    return lut


def pil_nearest_index(n_src, n_dst):
    """Source index of each of n_dst outputs under PIL's NEAREST resize of an axis of n_src pixels."""
    s = n_src / n_dst
    c = np.cumsum(np.concatenate([[s * 0.5], np.full(n_dst - 1, s)]))
    return np.minimum(c.astype(np.int64), n_src - 1)


def out_size(hw, dd_label_map_size):
    """The label / depth map size the reference produces for a raw h x w sample."""
    return tuple(hw) if tuple(dd_label_map_size) == ORI_SIZE else tuple(int(v) for v in dd_label_map_size)


def sample_grid(hw, out_hw):
    """(row index [H], column index [W]) of the source pixels; the identity when nothing is resized."""
    return pil_nearest_index(hw[0], out_hw[0]), pil_nearest_index(hw[1], out_hw[1])


def targets(ids, disparity, dd_label_map_size):
    """One sample: ids uint8 [h,w], disparity uint16 [h,w] or None -> (semseg int64 [H,W], depth fp32 [1,H,W] or None)."""
    H, W = out_size(ids.shape, dd_label_map_size)
    ys, xs = sample_grid(ids.shape, (H, W))
    raw = ids[ys][:, xs]
    semseg = encode_lut()[raw]
    depth = None
    if disparity is not None:
        d = disparity[ys][:, xs].astype(np.float32)
        # :153 then :156 on one array: d == 1 first becomes 0, then -1 like d == 0
        depth = np.where(d > 1, (d - np.float32(1)) / np.float32(256), np.float32(-1)).astype(np.float32)
        depth[raw == SKY_ID] = 0
        depth = depth[None]
    return semseg, depth


def invalid_sampled(ids, dd_label_map_size):
    """The reference's check (:223-226) on the resized map: an encoded value other than 255 that is >= 19. Those are
    exactly the raw ids 34..254 (0..33 are all void or valid), so only the sampled pixels matter."""
    H, W = out_size(ids.shape, dd_label_map_size)
    ys, xs = sample_grid(ids.shape, (H, W))
    raw = ids[ys][:, xs]
    return bool(((raw >= 34) & (raw != IGNORE)).any())


def image(img_bgr):
    """cv2.imread's uint8 BGR [h,w,3] -> the reference's fp32 [3,h,w]."""
    x = img_bgr[..., ::-1].astype(np.float32) / np.float32(255)
    return np.ascontiguousarray(((x - MEAN) / STD).transpose(2, 0, 1))


def reference_sample_work(img_bgr, ids, disparity, dd_label_map_size):
    """The reference's per-sample host work in its own order (float image, 35 numpy passes of encode_segmap, the
    disparity conversion, two PIL resizes, the validity check, normalisation), for timing against the device path."""
    from PIL import Image

    img = img_bgr.astype(np.float32)[..., ::-1]
    lbl = ids.copy()
    depth = disparity.astype(np.float32)
    depth[depth > 0] = (depth[depth > 0] - 1) / 256
    depth[depth == 0] = -1
    depth[lbl == SKY_ID] = 0
    for c in VOID:
        lbl[lbl == c] = IGNORE
    old = lbl.copy()
    for i, c in enumerate(VALID):
        lbl[old == c] = i
    size = tuple(dd_label_map_size)
    if size != ORI_SIZE:
        lbl = np.array(Image.fromarray(lbl.astype(float)).resize((size[1], size[0]), Image.NEAREST))
        depth = np.array(Image.fromarray(depth).resize((size[1], size[0]), Image.NEAREST))
    lbl = lbl.astype(int)
    if not np.all(np.unique(lbl[lbl != IGNORE]) < N_CLASSES):
        raise ValueError("Segmentation map contained invalid class values")
    x = img.astype(np.uint8).astype(np.float32) / np.float32(255)
    return ((x - MEAN) / STD).transpose(2, 0, 1), lbl, depth[None]
