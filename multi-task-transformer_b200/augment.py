"""The reference's PASCAL-Context / NYUD transform chains (TP/utils/common_config.py:96-121) on the device.

Build the dataset with ``transform=None`` so it yields raw float32 HWC samples, and load it with
``collate_fn=make_collate(p)`` and ``pin_memory=True``. The collate runs in the DataLoader worker: it draws every random
parameter of the train chain with Python ``random`` (the reference draws them in that same worker, under the same
per-worker seeding) and packs the batch into one flat CPU buffer. ``DeviceTransforms(p)(raw)`` then issues one
non-blocking host-to-device copy and the three ``mtt_augment`` launches, and returns the batch in the format
``collate_mil`` gives for the reference transforms.

Draw order: the reference's (RandomScaling, RandomCrop, flip, PhotoMetricDistortion), except that all 11 crop
candidates are drawn up front where the reference draws them lazily until one passes the cat_max_ratio test; the
device picks the first passing one. So each sample's augmentation has the reference's distribution, but not the
reference's random stream.
"""
import ctypes as C
import random

import numpy as np
import torch

from . import lib as _L
from . import ops

_SUPPORTED = ("PASCALContext", "NYUD")
_CHANNELS = {"normals": 3}
_ALIGN = 256


def _cfg(p, *keys):
    for k in keys:
        p = p[k]
    return p


def _check_db(p):
    if p["train_db_name"] not in _SUPPORTED:
        raise NotImplementedError(f"device transforms cover {_SUPPORTED}, not {p['train_db_name']!r}")


def draw_params(h, w, crop_hw, rng=random):
    """One sample's random draws of the train chain (transforms.py), in the reference's call order."""
    scale = rng.uniform(0.5, 2.0)                                        # RandomScaling :38
    sh, sw = (h, w) if scale == 1.0 else (int(h * scale), int(w * scale))
    crops = None
    if (sh, sw) != tuple(crop_hw):                                       # RandomCrop :174-181
        crops = [(rng.randint(0, max(sh - crop_hw[0], 0)), rng.randint(0, max(sw - crop_hw[1], 0)))
                 for _ in range(_L.AUG_CANDIDATES)]
    flip = rng.random() < 0.5                                            # :224
    bright = rng.uniform(-32, 32) if rng.random() < 0.5 else None        # :342-346
    f_mode = rng.random() < 0.5                                          # :392
    contrast = None
    if f_mode:
        contrast = rng.uniform(0.5, 1.5) if rng.random() < 0.5 else None  # :350-354
    sat = rng.uniform(0.5, 1.5) if rng.random() < 0.5 else None          # :358-365
    hue = rng.randint(-18, 17) if rng.random() < 0.5 else None           # :369-373
    if not f_mode:
        contrast = rng.uniform(0.5, 1.5) if rng.random() < 0.5 else None
    return dict(scale=scale, crops=crops, flip=flip, bright=bright, f_mode=f_mode, contrast=contrast, sat=sat, hue=hue)


def _record(rec, h, w, offsets):
    r = _L.AugmentSample()
    for i, o in enumerate(offsets):
        r.off[i] = o
    scale = rec["scale"]
    sh, sw = (h, w) if scale == 1.0 else (int(h * scale), int(w * scale))
    if sh <= 0 or sw <= 0:
        raise ValueError(f"scale {scale} shrinks a {h}x{w} sample to nothing")
    r.h, r.w, r.sh, r.sw = h, w, sh, sw
    r.lin_y, r.lin_x = h / sh, w / sw
    r.nn_y, r.nn_x = 1.0 / (sh / h), 1.0 / (sw / w)
    r.scaled = int(scale != 1.0)
    r.depth_scale = scale
    if rec["crops"] is not None:
        r.ncand = _L.AUG_CANDIDATES
        for k, (oy, ox) in enumerate(rec["crops"]):
            r.cand[2 * k], r.cand[2 * k + 1] = oy, ox
    r.flip = int(bool(rec["flip"]))
    r.bright_on, r.beta = rec["bright"] is not None, rec["bright"] or 0.0
    r.f_mode = int(bool(rec["f_mode"]))
    r.contrast_on, r.alpha = rec["contrast"] is not None, rec["contrast"] or 0.0
    r.sat_on, r.sat_alpha = rec["sat"] is not None, rec["sat"] or 0.0
    r.hue_on, r.hue_delta = rec["hue"] is not None, rec["hue"] or 0
    return r


_IDENTITY = dict(scale=1.0, crops=None, flip=False, bright=None, f_mode=False, contrast=None, sat=None, hue=None)


def _collate_meta(metas):
    """collate_mil (TP/utils/custom_collate.py) on the datasets' meta dicts: names as a list, sizes as LongTensors,
    numpy arrays stacked (Cityscapes-3D's scale_factor)."""
    out = {}
    for k in metas[0]:
        vals = [m[k] for m in metas]
        if isinstance(vals[0], np.ndarray):
            out[k] = torch.stack([torch.from_numpy(v) for v in vals], 0)
        else:
            out[k] = [torch.LongTensor(list(v)) for v in vals] if isinstance(vals[0], (tuple, list)) else vals
    return out


def pack(samples, tasks, crop_hw, records):
    """Packs raw samples (dicts of float32 HWC arrays) and their parameter records into one flat CPU uint8 buffer:
    B mtt_augment_sample records, then (at a 256-byte boundary) each sample's image and task maps as float32."""
    B = len(samples)
    recs = (_L.AugmentSample * B)()
    arrays, off = [], 0
    for b, s in enumerate(samples):
        img = s["image"]
        h, w = img.shape[:2]
        offsets = []
        for key in ("image",) + tuple(tasks):
            a = np.ascontiguousarray(s[key], dtype=np.float32)
            c = 3 if key == "image" else _CHANNELS.get(key, 1)
            if a.shape[:2] != (h, w) or a.size != h * w * c:
                raise ValueError(f"sample {b}: {key} has shape {a.shape}, expected ({h}, {w}, {c})")
            offsets.append(off)
            arrays.append(a.reshape(-1))
            off += a.size
        recs[b] = _record(records[b], h, w, offsets)
    head = (C.sizeof(recs) + _ALIGN - 1) // _ALIGN * _ALIGN
    buf = torch.empty(head + 4 * off, dtype=torch.uint8)
    np_buf = buf.numpy()
    np_buf[:C.sizeof(recs)] = np.frombuffer(bytes(recs), dtype=np.uint8)
    data = np_buf[head:].view(np.float32)
    pos = 0
    for a in arrays:
        data[pos:pos + a.size] = a
        pos += a.size
    return buf, head


def make_collate(p, train=True):
    """collate_fn for a DataLoader over a PASCALContext / NYUD dataset built with transform=None."""
    _check_db(p)
    tasks = [t for t in _cfg(p, "TASKS", "NAMES") if t in _L.AUG_TASK_KIND]
    size = tuple(_cfg(p, "TRAIN" if train else "TEST", "SCALE"))

    def collate(batch):
        names = [t for t in tasks if t in batch[0]]
        if train:
            records = [draw_params(s["image"].shape[0], s["image"].shape[1], size) for s in batch]
            H, W = size
        else:
            records = [_IDENTITY] * len(batch)
            hw = {(max(size[0], s["image"].shape[0]), max(size[1], s["image"].shape[1])) for s in batch}
            if len(hw) != 1:
                raise ValueError(f"validation samples pad to different sizes {sorted(hw)}; they cannot be stacked")
            H, W = hw.pop()
        buf, head = pack(batch, names, size, records)
        out = {"buf": buf, "head": head, "B": len(batch), "H": H, "W": W, "tasks": names, "records": records}
        if "meta" in batch[0]:
            out["meta"] = _collate_meta([s["meta"] for s in batch])
        return out

    return collate


class DeviceTransforms:
    """__call__(raw) with raw from make_collate(p, train): {'image': [B,3,H,W], task: [B,C,H,W], 'meta': ...} on the
    current CUDA device, enqueued on the current stream without a host synchronisation."""

    def __init__(self, p, train=True, device=None):
        _check_db(p)
        self.train = bool(train)
        self.size = tuple(_cfg(p, "TRAIN" if train else "TEST", "SCALE"))
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self._ws = None
        self.last_chosen = None   # int32 [B] device view of the chosen crop candidates of the last call (-1: none)

    def __call__(self, raw):
        B, H, W, head = raw["B"], raw["H"], raw["W"], raw["head"]
        dev = raw["buf"].to(self.device, non_blocking=True)
        nbytes = ops.augment_workspace_bytes(B)
        if self._ws is None or self._ws.numel() * 4 < nbytes:
            self._ws = torch.empty((nbytes + 3) // 4, dtype=torch.int32, device=self.device)
        out = {"image": torch.empty(B, 3, H, W, dtype=torch.float32, device=self.device)}
        for t in raw["tasks"]:
            out[t] = torch.empty(B, _CHANNELS.get(t, 1), H, W, dtype=torch.float32, device=self.device)
        ops.augment(dev[:head], dev[head:].view(torch.float32), B=B, H=H, W=W, train=self.train, crop_hw=self.size,
                    tasks=raw["tasks"], task_out=[out[t] for t in raw["tasks"]], image_out=out["image"],
                    workspace=self._ws)
        self.last_chosen = self._ws[B * _L.AUG_CANDIDATES:B * (_L.AUG_CANDIDATES + 1)]
        if "meta" in raw:
            out["meta"] = raw["meta"]
        return out
