"""Pure-numpy restatement of the reference's PASCAL-Context / NYUD train and validation transform chains
(TP/utils/common_config.py:96-121; TP/data/transforms.py) with the random draws given as an explicit record.

The record of one sample (what augment.make_collate draws, and what the golden script records from the real chain):
  scale      float; 1.0 = RandomScaling leaves the sample unchanged (transforms.py:50-52)
  crops      None when the scaled size equals the crop size (no draws, :174-175), else 11 (oh, ow) candidates: the first
             of 0..9 whose semseg crop passes the cat_max_ratio test is used, the 11th when none does (:196-205)
  flip       bool (:224)
  bright     None or the brightness beta (:342-346)
  f_mode     bool (:392)
  contrast   None or the contrast alpha (:350-354)
  sat        None or the saturation alpha (:358-365)
  hue        None or the hue shift in [-18, 17] (:369-373)

cv2 is restated, not called, and every rule below was checked bit for bit against cv2 4.13 (tests/test_augment.py):
  INTER_LINEAR, float32: source coordinate (d + 0.5) * (n_src / n_dst) - 0.5 in double, clamped at both edges, fraction
    rounded to float32; each output is fma(v1 - v0, t, v0) in float32, horizontally first, then vertically.
  INTER_NEAREST: src = floor(d * (1 / (n_dst / n_src))) in double, clamped to n_src - 1.
  COLOR_RGB2HSV (uint8): the fixed-point table algorithm (12-bit shifts, H in 0..179).
  COLOR_HSV2RGB (uint8): float32 with s = S * (1/255), v = V * (1/255), h = H * (6/180); sector tab entries v, v(1-s),
    v * fma(-s, h, 1), v * fma(-s, 1 - h, 1); the output x * 255 is TRUNCATED in cv2's vector loop, which covers the
    first floor(width / 32) * 32 pixels of each row (x86-64, AVX2 dispatch), and ROUNDED (half to even) in its scalar
    tail, so a pixel's result depends on its column and the row width.
fma is emulated in float64 (the float32 product is exact there); over every input the tests enumerate it matches.
"""
import numpy as np

F32 = np.float32
MEAN = np.array([0.485, 0.456, 0.406], dtype=F32)   # common_config.py:108
STD = np.array([0.229, 0.224, 0.225], dtype=F32)
LABEL_FILL = {"semseg": 255.0, "human_parts": 255.0, "sal": 255.0, "edge": 255.0, "normals": 0.0, "depth": 0.0}  # :94-100
CAT_MAX_RATIO = 0.75      # common_config.py:105
N_CANDIDATES = 11


def _fma(a, b, c):
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(F32)


# ---- cv2.resize ------------------------------------------------------------------------------------------------
def linear_coords(n_dst, n_src):
    d = np.arange(n_dst, dtype=np.float64)
    fx = (d + 0.5) * (n_src / n_dst) - 0.5
    i0 = np.floor(fx).astype(np.int64)
    t = fx - i0
    t = np.where(i0 < 0, 0.0, t)
    i0 = np.maximum(i0, 0)
    t = np.where(i0 >= n_src - 1, 0.0, t)
    i0 = np.minimum(i0, n_src - 1)
    return i0, np.minimum(i0 + 1, n_src - 1), t.astype(F32)


def nearest_index(n_dst, n_src):
    f = 1.0 / (n_dst / n_src)
    return np.minimum(np.floor(np.arange(n_dst, dtype=np.float64) * f).astype(np.int64), n_src - 1)


def resize_linear(img, dh, dw):
    """cv2.resize(img, (dw, dh), interpolation=cv2.INTER_LINEAR) for float32 [h, w] or [h, w, C]."""
    h, w = img.shape[:2]
    if (dh, dw) == (h, w):
        return img.copy()
    y0, y1, ty = linear_coords(dh, h)
    x0, x1, tx = linear_coords(dw, w)
    ext = (1,) * (img.ndim - 2)
    tx = tx.reshape((1, dw) + ext)
    ty = ty.reshape((dh, 1) + ext)
    r0, r1 = img[:, x0], img[:, x1]
    rows = _fma((r1 - r0).astype(F32), np.broadcast_to(tx, r0.shape), r0)
    v0, v1 = rows[y0], rows[y1]
    return _fma((v1 - v0).astype(F32), np.broadcast_to(ty, v0.shape), v0)


def resize_nearest(img, dh, dw):
    h, w = img.shape[:2]
    if (dh, dw) == (h, w):
        return img.copy()
    return img[nearest_index(dh, h)][:, nearest_index(dw, w)]


# ---- cv2.cvtColor on uint8 --------------------------------------------------------------------------------------
def _hsv_tables():
    i = np.arange(256, dtype=np.float64)
    safe = np.where(i == 0, 1.0, i)
    sdiv = np.where(i == 0, 0, np.rint((255 << 12) / safe)).astype(np.int64)
    hdiv = np.where(i == 0, 0, np.rint((180 << 12) / (6.0 * safe))).astype(np.int64)
    return sdiv, hdiv


_SDIV, _HDIV = _hsv_tables()
_SECTOR = np.array([[1, 3, 0], [1, 0, 2], [3, 0, 1], [0, 2, 1], [0, 1, 3], [2, 1, 0]])   # (b, g, r) tab indices


def rgb2hsv(rgb):
    r, g, b = (rgb[..., k].astype(np.int64) for k in range(3))
    v = np.maximum(np.maximum(b, g), r)
    diff = v - np.minimum(np.minimum(b, g), r)
    s = (diff * _SDIV[v] + (1 << 11)) >> 12
    h = np.where(v == r, g - b, np.where(v == g, b - r + 2 * diff, r - g + 4 * diff))
    h = (h * _HDIV[diff] + (1 << 11)) >> 12
    h = np.where(h < 0, h + 180, h)
    return np.stack([h, s, v], -1).astype(np.uint8)


HSV_VEC_PIXELS = 32


def hsv2rgb(hsv):
    inv255 = F32(1.0 / 255.0)
    hh = (hsv[..., 0].astype(F32) * (F32(6.0) / F32(180.0))).astype(F32)
    s = (hsv[..., 1].astype(F32) * inv255).astype(F32)
    v = (hsv[..., 2].astype(F32) * inv255).astype(F32)
    sector = np.floor(hh).astype(np.int64)
    h = (hh - sector.astype(F32)).astype(F32)
    bad = (sector < 0) | (sector >= 6)
    sector, h = np.where(bad, 0, sector), np.where(bad, F32(0), h)
    one = np.ones_like(s)
    tab = np.stack([v, (v * (F32(1) - s)).astype(F32), (v * _fma(-s, h, one)).astype(F32),
                    (v * _fma(-s, (F32(1) - h).astype(F32), one)).astype(F32)], -1)
    bgr = np.take_along_axis(tab, _SECTOR[sector], -1)
    bgr = np.where((s == 0)[..., None], v[..., None], bgr)
    x = (bgr * F32(255)).astype(F32)
    width = hsv.shape[-2]
    vec = (np.arange(width) < width // HSV_VEC_PIXELS * HSV_VEC_PIXELS)[:, None]
    out = np.clip(np.where(vec, np.trunc(x), np.rint(x)), 0, 255).astype(np.uint8)
    return out[..., ::-1].copy()


# ---- the chain ------------------------------------------------------------------------------------------------
def scaled_size(h, w, scale):
    return (h, w) if scale == 1.0 else (int(h * scale), int(w * scale))     # transforms.py:50-54


def cat_ratio_ok(seg):
    """RandomCrop's acceptance test (transforms.py:201-203)."""
    labels, cnt = np.unique(seg, return_counts=True)
    cnt = cnt[labels != 255]
    return len(cnt) > 1 and np.max(cnt) / np.sum(cnt) < CAT_MAX_RATIO


def chosen_candidate(scaled_semseg, crops, crop_hw):
    if crops is None:
        return None
    for k in range(N_CANDIDATES - 1):
        oh, ow = crops[k]
        if cat_ratio_ok(scaled_semseg[oh:oh + crop_hw[0], ow:ow + crop_hw[1]]):
            return k
    return N_CANDIDATES - 1


def _convert(x, alpha=1, beta=0):                     # transforms.py:334-338
    return np.clip(x.astype(F32) * F32(alpha) + F32(beta), 0, 255).astype(np.uint8)


def photometric(img_u8, rec):
    """PhotoMetricDistortion (transforms.py:376-407) after the uint8 cast, on uint8 RGB."""
    img = img_u8
    if rec["bright"] is not None:
        img = _convert(img, beta=rec["bright"])
    if rec["f_mode"] and rec["contrast"] is not None:
        img = _convert(img, alpha=rec["contrast"])
    if rec["sat"] is not None:
        hsv = rgb2hsv(img)
        hsv[..., 1] = _convert(hsv[..., 1], alpha=rec["sat"])
        img = hsv2rgb(hsv)
    if rec["hue"] is not None:
        hsv = rgb2hsv(img)
        hsv[..., 0] = (hsv[..., 0].astype(np.int64) + rec["hue"]) % 180
        img = hsv2rgb(hsv)
    if not rec["f_mode"] and rec["contrast"] is not None:
        img = _convert(img, alpha=rec["contrast"])
    return img


def normalize(img):
    return ((img.astype(F32) / F32(255.0)) - MEAN) / STD          # transforms.py:246-251


def pad(x, size, fill):
    h, w = x.shape[:2]
    H, W = max(size[0], h), max(size[1], w)
    out = np.full((H, W, x.shape[2]), fill, dtype=F32)
    dh, dw = (H - h) // 2, (W - w) // 2                              # transforms.py:104-114
    out[dh:dh + h, dw:dw + w] = x
    return out


def add_ignore_regions(key, x):                                      # transforms.py:279-299
    if key == "normals":
        sq = [(x[..., c] * x[..., c]).astype(F32) for c in range(3)]
        norm = np.sqrt(((sq[0] + sq[1]).astype(F32) + sq[2]).astype(F32))
        x = x.copy()
        x[norm == 0, :] = 255
    elif key == "human_parts":
        if ((x == 0) | (x == 255)).all():
            x = np.full(x.shape, 255, dtype=x.dtype)
    elif key == "depth":
        x = np.where(x == 0, F32(-1), x).astype(F32)
    return x


def train_transform(sample, rec, crop_hw, return_stages=False):
    """sample: {'image': float32 [h,w,3], task: float32 [h,w,C], ...}; returns {key: float32 CHW}. With
    return_stages, also the uint8 image that enters PhotoMetricDistortion and the chosen crop candidate."""
    img = sample["image"]
    h, w = img.shape[:2]
    sh, sw = scaled_size(h, w, rec["scale"])
    keys = [k for k in sample if k not in ("image", "meta")]
    sc = {"image": resize_linear(img, sh, sw)}
    for k in keys:
        v = resize_nearest(sample[k], sh, sw)
        if k == "depth" and rec["scale"] != 1.0:
            v = (v / F32(rec["scale"])).astype(F32)
        sc[k] = v
    k_sel = chosen_candidate(sc["semseg"], rec["crops"], crop_hw)
    if k_sel is not None:
        oh, ow = rec["crops"][k_sel]
        sc = {k: v[oh:oh + crop_hw[0], ow:ow + crop_hw[1]] for k, v in sc.items()}
    if rec["flip"]:
        sc = {k: v[:, ::-1].copy() for k, v in sc.items()}
        if "normals" in sc:
            sc["normals"][..., 0] *= -1
    u8 = sc["image"].astype(np.uint8)
    out = {"image": pad(normalize(photometric(u8, rec)), crop_hw, 0.0)}
    for k in keys:
        out[k] = add_ignore_regions(k, pad(sc[k], crop_hw, LABEL_FILL[k]))
    out = {k: np.ascontiguousarray(v.transpose(2, 0, 1)) for k, v in out.items()}
    if return_stages:
        return out, {"u8": u8, "chosen": k_sel}
    return out


def valid_transform(sample, size):
    """valid_transforms (common_config.py:115-120): Normalize, PadImage(size), AddIgnoreRegions, ToTensor."""
    out = {"image": pad(normalize(sample["image"]), size, 0.0)}
    for k in sample:
        if k not in ("image", "meta"):
            out[k] = add_ignore_regions(k, pad(sample[k], size, LABEL_FILL[k]))
    return {k: np.ascontiguousarray(v.transpose(2, 0, 1)) for k, v in out.items()}
