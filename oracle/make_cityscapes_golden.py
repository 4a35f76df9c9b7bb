"""Writes tests/golden/cityscapes.pt.xz: the UNMODIFIED reference CITYSCAPES3D (TP/data/cityscapes3d.py, is_transform=True,
no augmentations, tasks semseg + depth) and collate_mil run over small synthetic Cityscapes trees.

Each case is one tree written with cv2 into a temporary directory: leftImg8bit / gtFine labelIds / disparity PNGs under
<split>/<city>/. PNG is lossless, so the raw arrays stored here rebuild the same files anywhere. Cases:
  * every id 0..33 and 255, id 10 over positive, zero and maximal disparity, disparity 1 under id 10 and under other
    ids, at 37 x 53 -> 16 x 24 (odd ratios)
  * up-sampling 5 x 12 -> 12 x 29, and 2 x 7 -> 7 x 7 where the accumulated PIL coordinate falls below an integer
  * 32 x 64 -> 16 x 32, the 2:1 ratio of the real 1024 x 2048 -> 512 x 1024
  * dd_label_map_size (1024, 2048): the reference's no-resize branch, at 20 x 30
  * an invalid id (34..254) on a sampled pixel (the reference raises) and on an unsampled one (it does not)
  * the train split, whose samples without a 3D-detection object are dropped

The reference is given img_size=[1024, 2048] as a list, so its image-resize branch (:203) stays off for the small
images, as it is for real 1024 x 2048 images (the configs' tuple compares unequal to the reference's list, and Pillow then
returns an unchanged copy). The reference's imageio.imread comes from a PIL reader installed on the oracle's imageio
shim here (imageio v2 result types: uint8 for 8-bit PNGs), and cityscapesscripts from oracle/shim (import-only).

    python -m oracle.make_cityscapes_golden
"""
import collections
import collections.abc
import io
import json
import lzma
import os
import tempfile

import numpy as np
import torch

from oracle import ref_loader

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "cityscapes.pt.xz")
GOOD_IDS = np.array(list(range(34)) + [255], np.uint8)


def _imread(uri, *args, **kwargs):
    from PIL import Image

    with Image.open(uri) as im:
        a = np.array(im)
        if im.mode.startswith("I;16"):
            a = a.astype(np.uint16)
    return a


def write_tree(root, split, samples, det=None):
    """samples: list of dicts with city, stem, image (uint8 BGR), label_ids (uint8), disparity (uint16);
    det: {stem: list of object labels} for the gtBbox3d files."""
    import cv2

    for s in samples:
        for kind, suffix, key in (("leftImg8bit", "leftImg8bit.png", "image"),
                                  ("gtFine", "gtFine_labelIds.png", "label_ids"),
                                  ("disparity", "disparity.png", "disparity")):
            d = os.path.join(root, kind, split, s["city"])
            os.makedirs(d, exist_ok=True)
            assert cv2.imwrite(os.path.join(d, f"{s['stem']}_{suffix}"), s[key])
        if det is not None:
            d = os.path.join(root, "gtBbox3d", split, s["city"])
            os.makedirs(d, exist_ok=True)
            with open(os.path.join(d, f"{s['stem']}_gtBbox3d.json"), "w") as f:
                json.dump({"objects": [{"label": lab} for lab in det[s["stem"]]]}, f)


def make_sample(rng, city, idx, h, w, ids=None):
    s = {"city": city, "stem": f"{city}_{idx:06d}_000019", "image": rng.integers(0, 256, (h, w, 3), dtype=np.uint8),
         "label_ids": GOOD_IDS[rng.integers(0, len(GOOD_IDS), (h, w))] if ids is None else ids,
         "disparity": rng.integers(0, 65536, (h, w), dtype=np.uint16)}
    zero = rng.random((h, w)) < 0.2
    s["disparity"][zero] = 0
    return s


def cases(rng):
    out = []
    # every id with id 10 over positive / zero / maximal disparity
    a, b = make_sample(rng, "aachen", 0, 37, 53), make_sample(rng, "bochum", 1, 37, 53)
    for s in (a, b):
        s["label_ids"][::3, ::2] = 10
        s["disparity"][::3, ::4] = 0
        s["disparity"][1::3, 1::4] = 65535
        s["label_ids"][1::3, 1::4] = 10
        s["disparity"][::6, ::2] = 1          # disparity 1 under id 10 ...
        s["disparity"][2::3, ::2] = 1         # ... and under other ids (the reference turns it into -1)
    a["label_ids"][0, :35] = GOOD_IDS
    out.append(dict(name="all ids, 37x53 -> 16x24", dd=[16, 24], samples=[a, b]))
    out.append(dict(name="up-sampling 5x12 -> 12x29", dd=[12, 29],
                    samples=[make_sample(rng, "cologne", i, 5, 12) for i in range(2)]))
    out.append(dict(name="2x7 -> 7x7 (accumulated coordinate below an integer)", dd=[7, 7],
                    samples=[make_sample(rng, "cologne", i, 2, 7) for i in range(2)]))
    out.append(dict(name="2:1, 32x64 -> 16x32", dd=[16, 32],
                    samples=[make_sample(rng, "darmstadt", i, 32, 64) for i in range(3)]))
    out.append(dict(name="no resize (dd_label_map_size 1024x2048) at 20x30", dd=[1024, 2048],
                    samples=[make_sample(rng, "erfurt", i, 20, 30) for i in range(2)]))
    from oracle.cityscapes_ref import pil_nearest_index
    ys, xs = pil_nearest_index(37, 16), pil_nearest_index(53, 24)
    unsampled_y = sorted(set(range(37)) - set(ys.tolist()))[0]
    bad = [make_sample(rng, "hamburg", i, 37, 53) for i in range(2)]
    bad[1]["label_ids"][unsampled_y, 3] = 40
    out.append(dict(name="invalid id on an unsampled pixel", dd=[16, 24], samples=bad))
    worse = [make_sample(rng, "hanover", i, 37, 53) for i in range(2)]
    worse[0]["label_ids"][ys[5], xs[7]] = 200
    out.append(dict(name="invalid id on a sampled pixel", dd=[16, 24], samples=worse, raises=True))
    return out


def run_reference(root, split, dd, tasks=("semseg", "depth")):
    ref_loader._activate("TaskPrompter")
    import imageio
    imageio.imread = _imread
    if not hasattr(collections, "Mapping"):      # collate_mil uses the pre-3.10 aliases
        collections.Mapping, collections.Sequence = collections.abc.Mapping, collections.abc.Sequence
    from easydict import EasyDict
    from data.cityscapes3d import CITYSCAPES3D
    from utils.custom_collate import collate_mil

    p = EasyDict(dd_label_map_size=list(dd))
    cwd = os.getcwd()
    os.chdir(root)            # find_bad_samples writes its side files into the working directory
    try:
        ds = CITYSCAPES3D(p, root, split=[split], is_transform=True, img_size=[1024, 2048], augmentations=None,
                          task_list=list(tasks))
    finally:
        os.chdir(cwd)
    return ds, collate_mil


def _batch_arrays(batch):
    return {"image": batch["image"].numpy(), "semseg": batch["semseg"].numpy(), "depth": batch["depth"].numpy(),
            "meta": batch["meta"]}


def main():
    rng = np.random.default_rng(23)
    blob = {"cases": []}
    with tempfile.TemporaryDirectory() as tmp:
        for k, case in enumerate(cases(rng)):
            root = os.path.join(tmp, f"case{k}")
            write_tree(root, "val", case["samples"])
            ds, collate = run_reference(root, "val", case["dd"])
            order = [os.path.basename(f)[:-len("_leftImg8bit.png")] for f in ds.files["val"]]
            rec = dict(name=case["name"], dd=case["dd"], samples=case["samples"], order=order)
            try:
                rec["batch"] = _batch_arrays(collate([ds[i] for i in range(len(ds))]))
            except ValueError as e:
                assert case.get("raises"), (case["name"], e)
                rec["raises"] = str(e)
            else:
                assert not case.get("raises"), case["name"]
            blob["cases"].append(rec)
        # train split: the sample without a 3D-detection object is dropped
        root = os.path.join(tmp, "train")
        samples = [make_sample(rng, "jena", i, 8, 12) for i in range(4)]
        det = {samples[0]["stem"]: ["car", "person"], samples[1]["stem"]: ["rider", "person"],
               samples[2]["stem"]: [], samples[3]["stem"]: ["bicycle"]}
        write_tree(root, "train", samples, det)
        ds, _ = run_reference(root, "train", [4, 6])
        blob["train"] = dict(samples=samples, det=det, dd=[4, 6],
                             kept=sorted(os.path.basename(f)[:-len("_leftImg8bit.png")] for f in ds.files["train"]))
    raw = io.BytesIO()
    torch.save(blob, raw)
    with lzma.open(OUT, "wb", preset=9 | lzma.PRESET_EXTREME) as f:
        f.write(raw.getvalue())
    print(f"wrote {OUT} ({os.path.getsize(OUT) / 1e6:.2f} MB): {len(blob['cases'])} cases, train kept "
          f"{blob['train']['kept']}")


def load(path=OUT):
    with lzma.open(path, "rb") as f:
        return torch.load(io.BytesIO(f.read()), weights_only=False)


if __name__ == "__main__":
    main()
