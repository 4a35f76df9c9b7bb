"""Writes tests/golden/augment.pt.xz: the REAL reference train / validation transform chains (TP/data/transforms.py, composed
as TP/utils/common_config.py:102-120 does) run on small synthetic PASCAL-Context- and NYUD-like samples, with `random`
replaced by a scripted source whose every draw is recorded.

Each case fixes a parameter record (augment.draw_params' format) chosen to reach a branch: scale below / above / exactly
1, flip and no flip, each photometric branch under both f_mode values, the first / a later / no crop candidate
accepted (the 11th used), an image smaller than the crop in one and in both dimensions, an all-0/255 human_parts map,
zero normals and zero depth. The scripted source serves the record's values in whatever order the reference asks for
them, so the crop candidates are consumed lazily exactly as the reference draws them; `consumed` records how many.

    python -m oracle.make_augment_golden
"""
import io
import lzma
import os
import random

import numpy as np
import torch

from oracle import ref_loader

F32 = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "augment.pt.xz")   # torch.save blob, xz-compressed
CROP = (20, 40)    # wider than 32 pixels: cv2's HSV2RGB takes its vector loop and its scalar tail on one row
VALID = (24, 44)
PASCAL = ("semseg", "human_parts", "sal", "edge", "normals")
NYUD = ("semseg", "depth", "normals", "edge")


class Scripted:
    """Stands in for the `random` module: serves a record's draws and logs every call."""

    def __init__(self, rec):
        self.uni = [rec["scale"]]
        self.rnd = [0.25 if rec["flip"] else 0.75, 0.25 if rec["bright"] is not None else 0.75]
        if rec["bright"] is not None:
            self.uni.append(rec["bright"])
        self.rnd.append(0.25 if rec["f_mode"] else 0.75)
        order = ["contrast", "sat", "hue"] if rec["f_mode"] else ["sat", "hue", "contrast"]
        for k in order:
            self.rnd.append(0.25 if rec[k] is not None else 0.75)
        self.order = order
        self.rec = rec
        self.crops = [c for pair in (rec["crops"] or []) for c in pair]
        self.log = []
        self.crop_draws = 0

    def uniform(self, a, b):
        v = self.uni.pop(0)   # scale, beta, then the contrast / saturation alphas in the reference's order
        self.log.append(("uniform", a, b, v))
        return v

    def random(self):
        v = self.rnd.pop(0)
        self.log.append(("random", v))
        return v

    def randint(self, a, b):
        if (a, b) == (-18, 17):
            v = self.rec["hue"]
        else:
            v = self.crops.pop(0)
            self.crop_draws += 1
            assert 0 <= v <= b, (v, a, b)
        self.log.append(("randint", a, b, v))
        return v


def _alphas_in_order(rec):
    order = ["contrast", "sat", "hue"] if rec["f_mode"] else ["sat", "hue", "contrast"]
    return [rec[k] for k in order if k != "hue" and rec[k] is not None]


def run_reference(sample, rec, train=True):
    ref_loader._activate("TaskPrompter")
    import data.transforms as T

    chain = ([T.RandomScaling(scale_factors=[0.5, 2.0], discrete=False), T.RandomCrop(size=CROP, cat_max_ratio=0.75),
              T.RandomHorizontalFlip(p=0.5), T.PhotoMetricDistortion()] if train else [])
    chain += [T.Normalize(mean=[0.485, 0.456, 0.406], std=[0.229, 0.224, 0.225]),
              T.PadImage(size=CROP if train else VALID), T.AddIgnoreRegions(), T.ToTensor()]
    src = Scripted(rec if train else dict(scale=1.0, crops=None, flip=False, bright=None, f_mode=True, contrast=None,
                                          sat=None, hue=None))
    src.uni += _alphas_in_order(src.rec)
    saved = T.random
    T.random = src
    try:
        out = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in sample.items()}
        for t in chain:
            out = t(out)
    finally:
        T.random = saved
    assert not train or (not src.uni and not src.rnd), (src.uni, src.rnd)
    return {k: v for k, v in out.items() if k != "meta"}, src


def _labels(rng, h, w, kind):
    if kind == "mixed":
        return rng.integers(0, 4, (h, w, 1)).astype(np.float32)
    if kind == "uniform":           # one label: every crop fails cat_max_ratio
        m = np.full((h, w, 1), 7, np.float32)
        m[: h // 6, : w // 6] = 255
        return m
    if kind == "left_uniform":      # uniform on the left, mixed on the right
        m = np.full((h, w, 1), 2, np.float32)
        m[:, w // 2:] = rng.integers(0, 5, (h, w - w // 2, 1))
        return m
    raise ValueError(kind)


def make_sample(rng, h, w, tasks, seg="mixed", parts_ignore=False, zero_normals=False, zero_depth=False):
    s = {"image": rng.integers(0, 256, (h, w, 3)).astype(np.float32), "semseg": _labels(rng, h, w, seg)}
    for t in tasks:
        if t == "human_parts":
            s[t] = (np.where(rng.random((h, w, 1)) < 0.5, 0, 255) if parts_ignore
                    else rng.integers(0, 7, (h, w, 1))).astype(np.float32)
        elif t in ("sal", "edge"):
            s[t] = (rng.random((h, w, 1)) < 0.3).astype(np.float32)
        elif t == "normals":
            n = rng.standard_normal((h, w, 3))
            n /= np.linalg.norm(n, axis=2, keepdims=True)
            # as the datasets decode them from 8-bit PNGs: 2 * q / 255 - 1 in float32 (NYUD nyud.py:207)
            n = F32(2) * np.rint((n + 1) * 127.5).astype(F32) / F32(255) - F32(1)
            if zero_normals:
                n[h // 3: h // 2] = 0
            n[0, 0, 0] = 0.0   # an x of 0 becomes -0.0 when flipped
            s[t] = n.astype(F32)
        elif t == "depth":
            d = (rng.random((h, w, 1)) * 9 + 0.5).astype(np.float32)
            if zero_depth:
                d[:, : w // 4] = 0
            s[t] = d
    s = {k: s[k] for k in ("image",) + tuple(tasks)}
    s["meta"] = {"img_name": "synthetic", "img_size": (h, w)}
    return s


def cases():
    base = dict(scale=1.3, crops=None, flip=False, bright=None, f_mode=True, contrast=None, sat=None, hue=None)

    def rec(rng, h, w, **kw):
        r = dict(base, **kw)
        sh, sw = (h, w) if r["scale"] == 1.0 else (int(h * r["scale"]), int(w * r["scale"]))
        if "crops" not in kw and (sh, sw) != CROP:
            r["crops"] = [(int(rng.integers(0, max(sh - CROP[0], 0) + 1)), int(rng.integers(0, max(sw - CROP[1], 0) + 1)))
                          for _ in range(11)]
        return r

    rng = np.random.default_rng(11)
    out = []
    # (sample kwargs, record kwargs)
    out.append(("first accepted, scale < 1, flip, brightness",
                dict(h=31, w=58, tasks=PASCAL), dict(scale=0.83, flip=True, bright=17.3)))
    out.append(("scale > 1, f_mode contrast first, saturation, hue",
                dict(h=19, w=29, tasks=PASCAL), dict(scale=1.71, contrast=1.37, sat=0.61, hue=-13)))
    out.append(("scale exactly 1, contrast last, hue only",
                dict(h=23, w=47, tasks=NYUD), dict(scale=1.0, f_mode=False, contrast=0.58, hue=16)))
    out.append(("all rejected (11th used), NYUD zero depth, zero normals, flip",
                dict(h=26, w=50, tasks=NYUD, seg="uniform", zero_depth=True, zero_normals=True),
                dict(scale=1.12, flip=True, bright=-25.0, sat=1.44)))
    out.append(("smaller than the crop in one dimension, all-0/255 human parts",
                dict(h=15, w=50, tasks=PASCAL, parts_ignore=True), dict(scale=1.05, f_mode=False, sat=1.2, hue=-18,
                                                                          contrast=1.45)))
    out.append(("smaller than the crop in both dimensions, flip",
                dict(h=18, w=40, tasks=PASCAL), dict(scale=0.9, flip=True, bright=31.0, contrast=0.7)))
    out.append(("scaled size equals the crop size (no crop draws)",
                dict(h=10, w=20, tasks=NYUD), dict(scale=2.0, hue=3, sat=0.5)))
    out.append(("saturation and hue, f_mode False, all photometric", dict(h=24, w=44, tasks=PASCAL),
                dict(scale=1.5, f_mode=False, bright=-3.5, contrast=1.1, sat=1.33, hue=-1)))
    samples, records, names = [], [], []
    for name, skw, rkw in out:
        s = make_sample(rng, **skw)
        r = rec(rng, skw["h"], skw["w"], **rkw)
        samples.append(s)
        records.append(r)
        names.append(name)
    # the k-th candidate accepted: candidates 0..3 in the uniform left half, then one over the mixed half
    s = make_sample(rng, 32, 100, PASCAL, seg="left_uniform")
    r = rec(rng, 32, 100, scale=1.0, flip=True, sat=0.8)
    r["crops"] = [(int(rng.integers(0, 13)), int(rng.integers(0, 11))) for _ in range(4)] + \
                 [(int(rng.integers(0, 13)), 60) for _ in range(7)]
    samples.append(s)
    records.append(r)
    names.append("5th candidate accepted")
    return names, samples, records


def _encode(dicts):
    """Arrays whose values are all integers in 0..255 (images, most label maps) are stored as uint8: exact, and a
    quarter of the bytes."""
    out = []
    for d in dicts:
        e = {}
        for k, v in d.items():
            if isinstance(v, np.ndarray) and np.array_equal(v, np.clip(np.rint(v), 0, 255)) and not np.signbit(v).any():
                v = v.astype(np.uint8)
            e[k] = v
        out.append(e)
    return out


def load(path=OUT):
    """The golden blob with every array as float32 again."""
    with lzma.open(path, "rb") as f:
        blob = torch.load(io.BytesIO(f.read()), weights_only=False)
    for key in ("samples", "outputs", "valid_samples", "valid_outputs"):
        blob[key] = [{k: (v.astype(np.float32) if isinstance(v, np.ndarray) else v) for k, v in d.items()}
                     for d in blob[key]]
    return blob


def main():
    names, samples, records = cases()
    outs, consumed = [], []
    for s, r in zip(samples, records):
        o, src = run_reference(s, r)
        outs.append({k: v.numpy().copy() for k, v in o.items()})
        consumed.append(src.crop_draws // 2)
    rng = np.random.default_rng(5)
    valid_samples = [make_sample(rng, 20, 40, PASCAL), make_sample(rng, 24, 30, NYUD, zero_depth=True, zero_normals=True),
                     make_sample(rng, 15, 17, PASCAL, parts_ignore=True)]
    valid_outs = [{k: v.numpy().copy() for k, v in run_reference(s, None, train=False)[0].items()}
                  for s in valid_samples]
    blob = dict(crop=CROP, valid_size=VALID, names=names, samples=_encode(samples), records=records,
                outputs=_encode(outs), consumed=consumed, valid_samples=_encode(valid_samples),
                valid_outputs=_encode(valid_outs))
    raw = io.BytesIO()
    torch.save(blob, raw)
    with lzma.open(OUT, "wb", preset=9 | lzma.PRESET_EXTREME) as f:
        f.write(raw.getvalue())
    print(f"wrote {OUT} ({os.path.getsize(OUT) / 1e6:.2f} MB): {len(samples)} train and {len(valid_samples)} "
          f"validation samples; crop candidates consumed {consumed}")


if __name__ == "__main__":
    random.seed(0)
    main()
