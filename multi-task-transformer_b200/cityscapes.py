"""The reference's Cityscapes-3D samples (TP/data/cityscapes3d.py, CITYSCAPES3D with is_transform=True and no
augmentations -- common_config.py:150-153, 189-192) on the device, for the semseg and depth tasks.

The reference has no transform chain for this dataset: __getitem__ / transform convert each 1024 x 2048 sample on the
CPU (float image, 35 numpy passes of encode_segmap, the disparity conversion, two PIL NEAREST resizes of the label maps
to dd_label_map_size, normalisation). Here:

* ``RawCityscapes3D(p, root, split, task_list)`` lists the same files and returns the raw arrays: the image as
  cv2.imread gives it (uint8 BGR), the label ids (uint8) and the disparity (uint16), plus the reference's ``meta``.
* ``make_collate(p)`` (in the DataLoader worker) checks the batch, raises the reference's invalid-class ValueError
  where the reference raises it, and packs the batch into one flat uint8 buffer.
* ``DeviceTransforms(p)(raw)`` issues one non-blocking host-to-device copy, one ``preprocess_image`` launch (at
  identity size it is exactly ToTensor + Normalize) and one ``mtt_cityscapes_targets`` launch, and returns
  ``{'image', 'semseg', 'depth', 'meta'}`` in collate_mil's format: fp32 [B,3,h,w], int64 [B,H,W], fp32 [B,1,H,W].

The same batches serve training, since the reference applies no augmentation to this dataset (augmentations=None).
"""
import copy
import json
import os

import numpy as np
import torch

from . import ops
from .augment import _ALIGN, _collate_meta

ORI_SIZE = (1024, 2048)          # cityscapes3d.py:102
EVAL_LABELS = ("car", "truck", "bus", "train", "motorcycle", "bicycle")   # :27, the 3D-detection classes
_TASKS = ("semseg", "depth")


def _get(p, *keys):
    for k in keys:
        try:
            p = p[k]
        except (KeyError, TypeError):
            p = getattr(p, k)
    return p


def _check_tasks(task_list):
    tasks = list(task_list)
    if "3ddet" in tasks:
        raise NotImplementedError("task '3ddet' needs mmdet3d (the FCOS3D detection head and its targets), which "
                                  "mtt_b200 does not provide")
    if "depth" in tasks and "semseg" not in tasks:
        raise ValueError("Cityscapes-3D depth needs the semseg label ids: the reference masks the disparity with them "
                         "(cityscapes3d.py:159)")
    if "semseg" not in tasks:
        raise ValueError(f"Cityscapes-3D device batches need the semseg task, got {tasks}")
    other = [t for t in tasks if t not in _TASKS]
    if other:
        raise NotImplementedError(f"Cityscapes-3D tasks {other} are not supported (semseg, depth)")
    return [t for t in _TASKS if t in tasks]


def recursive_glob(rootdir=".", suffix=""):
    """cityscapes3d.py:36-43: every file under rootdir ending in suffix, in os.walk order."""
    return [os.path.join(looproot, filename)
            for looproot, _, filenames in os.walk(rootdir) for filename in filenames if filename.endswith(suffix)]


def pil_nearest_index(n_src, n_dst):
    """Source index of each of n_dst outputs of Pillow's NEAREST resize of an axis of n_src pixels: the running sum
    c_0 = s * 0.5, c_{d+1} = c_d + s with s = n_src / n_dst in double, truncated (oracle/cityscapes_ref.py)."""
    s = n_src / n_dst
    c = np.cumsum(np.concatenate([[s * 0.5], np.full(n_dst - 1, s)]))
    return np.minimum(c.astype(np.int64), n_src - 1)


def label_size(hw, dd_label_map_size):
    """The size of the semseg / depth maps the reference makes from an h x w sample: no resize when
    dd_label_map_size equals (1024, 2048) (:210, :216)."""
    dd = tuple(int(v) for v in dd_label_map_size)
    return tuple(int(v) for v in hw) if dd == ORI_SIZE else dd


class RawCityscapes3D(torch.utils.data.Dataset):
    """The file list of CITYSCAPES3D.__init__ (:53-106) without any decoding arithmetic. Sample: {'image': uint8 BGR
    [h,w,3], 'label_ids': uint8 [h,w], 'disparity': uint16 [h,w] (with depth), 'meta': as :140-144}.

    The image is never resized: the reference resizes it only when img_size (p.TRAIN / TEST.SCALE) differs from
    1024 x 2048, which no reference config does, so any other SCALE raises NotImplementedError. meta['img_name'] is the
    file's base name up to its first '.', which is the reference's value unless a directory of the path holds a '.'.
    For the train split,
    samples whose gtBbox3d file has no object of the 3D-detection classes are dropped as :243-288 drops them (the
    reference's CS3D_bad_samples_* side files are not written)."""

    def __init__(self, p, root, split=("train",), task_list=("semseg", "depth")):
        self.tasks = _check_tasks(task_list)
        split = [split] if isinstance(split, str) else sorted(split)
        self.split, self.root, self.split_text = split, root, "+".join(split)
        scale = tuple(int(v) for v in _get(p, "TRAIN" if self.split_text == "train" else "TEST", "SCALE"))
        if scale != ORI_SIZE:
            raise NotImplementedError(f"Cityscapes-3D with image scale {scale}: the reference's PIL bilinear image "
                                      f"resize (cityscapes3d.py:203-204) is not implemented; use {ORI_SIZE}")
        self.img_size = scale
        self.dd_label_map_size = _get(p, "dd_label_map_size")
        self.files = []
        for s in split:                       # as the reference: the annotation bases are the LAST split's
            self.images_base = os.path.join(root, "leftImg8bit", s)
            self.annotations_base = os.path.join(root, "gtFine", s)
            self.files += recursive_glob(rootdir=self.images_base, suffix=".png")
            self.depth_base = os.path.join(root, "disparity", s)
            self.det_base = os.path.join(root, "gtBbox3d", s)
        if self.split_text == "train":
            self.files = self._without_detection_free(self.files)
        if len(self.files) < 2:
            raise FileNotFoundError(f"No files for split=[{self.split_text}] found in {self.images_base}")

    def _path(self, img_path, base, suffix):
        return os.path.join(base, img_path.split(os.sep)[-2], os.path.basename(img_path)[:-15] + suffix)

    def _without_detection_free(self, files):
        keep = copy.copy(files)
        for img_path in files:
            with open(self._path(img_path.rstrip(), self.det_base, "gtBbox3d.json")) as f:
                objects = json.load(f)["objects"]
            if not any(o["label"] in EVAL_LABELS for o in objects):
                keep.remove(img_path)
        return keep

    def __len__(self):
        return len(self.files)

    def __getitem__(self, index):
        import cv2

        img_path = self.files[index].rstrip()
        img = cv2.imread(img_path)
        if img is None:
            raise FileNotFoundError(img_path)
        sample = {"image": img}
        # The reference takes img_path.split('.')[0].split('/')[-1], which cuts at the first '.' of the WHOLE path: under
        # a directory with a '.' in its name it yields a piece of that directory, the same for every sample. The base
        # name up to its first '.' is what it gives for paths without dots, and stays the file's name otherwise.
        sample["meta"] = {"img_name": os.path.basename(img_path).split(".")[0],
                          "img_size": (img.shape[0], img.shape[1]),
                          "dd_label_map_size": self.dd_label_map_size,
                          "scale_factor": np.array([self.img_size[1] / img.shape[1], self.img_size[0] / img.shape[0]])}
        if "semseg" in self.tasks:
            sample["label_ids"] = _read(self._path(img_path, self.annotations_base, "gtFine_labelIds.png"), np.uint8)
        if "depth" in self.tasks:
            sample["disparity"] = _read(self._path(img_path, self.depth_base, "disparity.png"), np.uint16)
        return sample


def _read(path, dtype):
    import cv2

    a = cv2.imread(path, cv2.IMREAD_UNCHANGED)
    if a is None:
        raise FileNotFoundError(path)
    if a.ndim != 2 or a.dtype != dtype:
        raise ValueError(f"{path}: expected a one-channel {np.dtype(dtype).name} PNG, got {a.dtype} {a.shape}")
    return a


def _align(n):
    return (n + _ALIGN - 1) // _ALIGN * _ALIGN


def invalid_sampled_ids(ids, out_hw):
    """True when a label id that the reference's check rejects (:223-226) lands on a sampled pixel: encoded values
    other than 255 must be < 19, and ids 0..33 all encode to 255 or 0..18, so the rejected ids are 34..254."""
    ys, xs = pil_nearest_index(ids.shape[0], out_hw[0]), pil_nearest_index(ids.shape[1], out_hw[1])
    raw = ids[ys[:, None], xs[None, :]]
    return bool(((raw >= 34) & (raw != 255)).any())


def make_collate(p):
    """collate_fn for a DataLoader over RawCityscapes3D: one CPU uint8 buffer holding the images [B,h,w,3], then the
    label ids [B,h,w], then the disparity [B,h,w] (uint16), each block at a 256-byte boundary."""
    tasks = _check_tasks(_get(p, "TASKS", "NAMES"))
    dd = _get(p, "dd_label_map_size")

    def collate(batch):
        B = len(batch)
        h, w = batch[0]["image"].shape[:2]
        keys = ["image", "label_ids"] + (["disparity"] if "depth" in tasks else [])
        for b, s in enumerate(batch):
            for k in keys:
                want = (h, w, 3) if k == "image" else (h, w)
                if k not in s or s[k].shape != want:
                    got = s[k].shape if k in s else "missing"
                    raise ValueError(f"sample {b}: {k} is {got}, expected {want}; samples of one batch must share one "
                                     "size (the reference's torch.stack fails otherwise)")
        H, W = label_size((h, w), dd)
        for s in batch:
            if invalid_sampled_ids(s["label_ids"], (H, W)):
                raise ValueError("Segmentation map contained invalid class values")
        n = B * h * w
        offsets = [0, _align(3 * n)]
        end = offsets[1] + n
        if "disparity" in keys:
            offsets.append(_align(end))
            end = offsets[2] + 2 * n
        buf = torch.empty(end, dtype=torch.uint8)
        np_buf = buf.numpy()
        for k, off, item in zip(keys, offsets, (3, 1, 2)):
            block = np_buf[off:off + item * n]
            view = block.view(np.uint16) if k == "disparity" else block
            for b, s in enumerate(batch):
                size = view.size // B
                view[b * size:(b + 1) * size] = s[k].reshape(-1)
        out = {"buf": buf, "offsets": offsets, "B": B, "h": h, "w": w, "H": H, "W": W, "tasks": tasks}
        if "meta" in batch[0]:
            out["meta"] = _collate_meta([s["meta"] for s in batch])
        return out

    return collate


class DeviceTransforms:
    """__call__(raw) with raw from make_collate(p): {'image': fp32 [B,3,h,w], 'semseg': int64 [B,H,W], 'depth': fp32
    [B,1,H,W] (with depth), 'meta': ...} on the current CUDA device, enqueued on the current stream (one copy, two
    launches) without a host synchronisation."""

    def __init__(self, p, device=None):
        _check_tasks(_get(p, "TASKS", "NAMES"))
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())

    def __call__(self, raw):
        B, h, w, H, W = raw["B"], raw["h"], raw["w"], raw["H"], raw["W"]
        n = B * h * w
        dev = raw["buf"].to(self.device, non_blocking=True)
        o = raw["offsets"]
        out = {"image": ops.preprocess_image(dev[o[0]:o[0] + 3 * n].view(B, h, w, 3), (h, w))}
        ids = dev[o[1]:o[1] + n].view(B, h, w)
        out["semseg"] = torch.empty(B, H, W, dtype=torch.int64, device=self.device)
        disp, depth = None, None
        if "depth" in raw["tasks"]:
            disp = dev[o[2]:o[2] + 2 * n].view(torch.uint16).view(B, h, w)
            depth = out["depth"] = torch.empty(B, 1, H, W, dtype=torch.float32, device=self.device)
        ops.cityscapes_targets(ids, disp, (H, W), semseg=out["semseg"], depth=depth)
        if "meta" in raw:
            out["meta"] = raw["meta"]
        return out
