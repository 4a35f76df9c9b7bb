"""Writes tests/golden/export.pt.xz: the UNMODIFIED reference functions that save and draw predictions, run through
ref_loader on seeded logits, and the files they wrote, read back:
  - TaskPrompter's save_model_pred_for_one_task (TP/evaluation/evaluate_utils.py:69-151; for semseg it raises an
    AttributeError, recorded as None, because :77-79 convert the map to numpy before :150 calls .cpu()) and InvPT's
    (IP/evaluation/evaluate_utils.py:69-105) on PASCAL-like (edge, semseg 21, human_parts 7, sal), NYUD-like (semseg
    40) and Cityscapes-like (semseg 19, TaskPrompter with semseg_save_train_class False) batches: padded predictions,
    ragged image sizes with odd pad deltas, one image whose label is all ignore;
  - TaskPrompter's vis_pred_for_one_task (TP/utils/visualization_utils.py:80-199) on PASCAL (semseg, normals, sal,
    edge, human_parts), NYUD (semseg, depth, normals) and Cityscapes (semseg, and a depth map that is constant after
    get_output's clamp).
imageio and matplotlib come from oracle/shim (imageio.imwrite writes through PIL; matplotlib is import-only). The
reference's save function moves sample['image'] to CUDA only to read its batch size, so the batch carries a CPU
stand-in with .cuda() and .size(). Every logit lies on the fp16 grid and is stored as fp16.

    python -m oracle.make_export_golden
"""
import io
import lzma
import os
import tempfile

import cv2
import numpy as np
import torch
from PIL import Image

from oracle import ref_loader

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "export.pt.xz")

PASCAL = {"edge": 1, "semseg": 21, "human_parts": 7, "sal": 2}
EXPORT_CASES = [   # (name, database, channels per task, padded size, image sizes, all-ignore image, save_train_class)
    ("pascal", "PASCALContext", PASCAL, (22, 27), [(22, 27), (19, 24), (17, 26), (21, 23)], 2, True),
    ("nyud", "NYUD", {"edge": 1, "semseg": 40}, (18, 23), [(15, 20), (18, 23), (13, 21)], None, True),
    ("cityscapes", "Cityscapes3D", {"semseg": 19}, (20, 24), [(17, 21), (20, 23)], None, False),
]
VIS_CASES = [      # (name, database, channels per task, logits size, batch, image size)
    ("pascal", "PASCALContext", {"semseg": 21, "normals": 3, "sal": 2, "edge": 1, "human_parts": 7}, (24, 30), 2,
     (21, 37)),
    ("nyud", "NYUD", {"semseg": 40, "depth": 1, "normals": 3}, (16, 24), 2, (23, 19)),
    ("cityscapes", "Cityscapes3D", {"semseg": 19, "depth": 1}, (16, 32), 1, (13, 29)),
]


class _Image:
    """sample['image'] for the save function: .cuda() returns itself, .size() the batch shape."""

    def __init__(self, B):
        self.B = B

    def cuda(self, non_blocking=False):
        return self

    def size(self):
        return torch.Size([self.B, 3, 1, 1])


def _logits(g, B, C, hw, scale=3.0):
    return (torch.randn((B, C) + tuple(hw), generator=g) * scale).half()


def _p(db, save_train_class=True):
    from easydict import EasyDict
    return EasyDict(train_db_name=db, ignore_index=255, semseg_save_train_class=save_train_class)


def export_cases():
    g = torch.Generator().manual_seed(17)
    out = []
    for name, db, chans, hw, sizes, ignore_img, stc in EXPORT_CASES:
        B = len(sizes)
        logits = {t: _logits(g, B, c, hw) for t, c in chans.items()}
        labels = {}
        for t in chans:
            lab = torch.where(torch.rand((B, 1) + hw, generator=g) < 0.3, 1.0, 0.0)
            lab[torch.rand((B, 1) + hw, generator=g) < 0.1] = 255.0
            if ignore_img is not None:
                lab[ignore_img] = 255.0
            labels[t] = lab.to(torch.uint8)
        meta = {"img_name": [f"{name}_{i:03d}" for i in range(B)], "img_size": [list(s) for s in sizes]}
        out.append(dict(name=name, db=db, save_train_class=stc, logits=logits, labels=labels, meta=meta))
    return out


def vis_cases():
    g = torch.Generator().manual_seed(23)
    out = []
    for name, db, chans, hw, B, size in VIS_CASES:
        logits = {t: _logits(g, B, c, hw) for t, c in chans.items()}
        if db == "Cityscapes3D":
            logits["depth"] = torch.full((B, 1) + hw, -0.5, dtype=torch.float16)   # clamps to a constant 0
        meta = {"img_name": [f"{name}_{i:03d}" for i in range(B)], "img_size": [list(size)] * B}
        out.append(dict(name=name, db=db, logits=logits, meta=meta))
    return out


def run_export(case, reference):
    ref_loader._activate(reference)
    from evaluation.evaluate_utils import save_model_pred_for_one_task
    p = _p(case["db"], case["save_train_class"])
    B = len(case["meta"]["img_name"])
    sample = {"image": _Image(B), "meta": case["meta"]}
    sample.update({t: v.float() for t, v in case["labels"].items()})
    output = {t: v.float() for t, v in case["logits"].items()}
    files = {}
    with tempfile.TemporaryDirectory() as d:
        for t in case["logits"]:
            if reference == "InvPT" and case["db"] == "Cityscapes3D":
                continue
            sd = {t: os.path.join(d, t)}
            os.makedirs(sd[t])
            if reference == "TaskPrompter":
                try:
                    save_model_pred_for_one_task(p, 0, sample, output, sd, t, epoch=0)
                except AttributeError:   # semseg: the prediction is already numpy when :150 calls .cpu() on it
                    assert t == "semseg"
                    files[t] = None
                    continue
            else:
                save_model_pred_for_one_task(p, sample, output, sd, t, epoch=0)
            files[t] = {f: np.array(Image.open(os.path.join(sd[t], f))) for f in sorted(os.listdir(sd[t]))}
    return files


def run_vis(case):
    ref_loader._activate("TaskPrompter")
    from utils.visualization_utils import vis_pred_for_one_task
    p = _p(case["db"])
    B = len(case["meta"]["img_name"])
    sample = {"image": torch.zeros(B, 3, 1, 1), "meta": case["meta"]}
    files = {}
    with tempfile.TemporaryDirectory() as d:
        for t in case["logits"]:
            output = {k: v.float() for k, v in case["logits"].items()}
            sd = os.path.join(d, t)
            os.makedirs(sd)
            vis_pred_for_one_task(p, sample, output, sd, t)
            files[t] = {f: cv2.imread(os.path.join(sd, f), cv2.IMREAD_UNCHANGED) for f in sorted(os.listdir(sd))}
    return files


def load(path=OUT):
    with lzma.open(path, "rb") as f:
        return torch.load(io.BytesIO(f.read()), weights_only=False)


def main():
    ex = export_cases()
    for c in ex:
        c["files"] = {r: run_export(c, r) for r in ("TaskPrompter", "InvPT")}
    vi = vis_cases()
    for c in vi:
        c["files"] = run_vis(c)
    blob = dict(export=ex, vis=vi)
    raw = io.BytesIO()
    torch.save(blob, raw)
    with lzma.open(OUT, "wb", preset=9 | lzma.PRESET_EXTREME) as f:
        f.write(raw.getvalue())
    n = sum(len(v) for c in ex for r in c["files"].values() for v in r.values() if v is not None) + \
        sum(len(v) for c in vi for v in c["files"].values())
    print(f"wrote {OUT} ({os.path.getsize(OUT) / 1e3:.0f} KB): {n} files")


if __name__ == "__main__":
    main()
