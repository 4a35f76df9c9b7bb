"""CPU restatement of the reference's prediction export and inference visualisation, with the reference's loops, crop
rule, skip rule, palettes and JET normalisation:
  save_preds  save_model_pred_for_one_task (TP/evaluation/evaluate_utils.py:69-151, IP/evaluation/evaluate_utils.py:
              69-105) for the 2-D tasks: {file name: uint8 array as written}
  vis_preds   vis_pred_for_one_task's parallel branch (TP/utils/visualization_utils.py:144-199): {file name: uint8
              array as cv2.imwrite gets it (BGR or gray)}
  encode      the encodings alone, on get_output-domain maps (numpy float32 / int64)
The palettes come from mtt_b200.export, which tests/test_export.py checks against the reference's own tables.
"""
import numpy as np
import torch
import torch.nn.functional as F

from mtt_b200 import export as E


def get_output(x, task, semseg_save_train_class=True):
    """TP/utils/utils.py:27-63 for the 2-D tasks (CPU torch)."""
    if task == "normals":
        x = x.permute(0, 2, 3, 1)
        return (F.normalize(x, p=2, dim=3) + 1.0) * 255 / 2.0
    if task in ("semseg", "human_parts"):
        _, x = torch.max(x.permute(0, 2, 3, 1), dim=3)
        if task == "semseg" and not semseg_save_train_class:
            m = x.clone()
            for c, cid in enumerate(E.CS_VALID_CLASSES):
                m[x == c] = cid
            x = m
        return x
    if task == "edge":
        x = x.permute(0, 2, 3, 1)
        return torch.squeeze(255 * 1 / (1 + torch.exp(-x)), dim=3)
    if task == "sal":
        return F.softmax(x.permute(0, 2, 3, 1), dim=3)[:, :, :, 1] * 255
    if task == "depth":
        return x.clamp(min=0.).permute(0, 2, 3, 1)
    raise ValueError(task)


def resize(x, hw):
    return F.interpolate(x, tuple(int(v) for v in hw), mode="bilinear")


def _get(p, k, default=None):
    try:
        return p[k]
    except (KeyError, TypeError):
        return getattr(p, k, default)


def save_preds(p, sample, output, task, reference="TaskPrompter", predicted=False):
    """The files save_model_pred_for_one_task writes for a 2-D task, as {name + '.png': uint8 array}. predicted: the
    output holds predict()'s maps, where get_output is already applied."""
    meta = sample["meta"]
    if predicted:
        out = output[task]
    elif task == "semseg" and reference == "TaskPrompter" and not _get(p, "semseg_save_train_class", True) \
            and _get(p, "train_db_name") == "Cityscapes3D":
        out = get_output(output[task], task, semseg_save_train_class=False)
    else:
        out = get_output(output[task], task)
    files = {}
    for jj in range(int(out.shape[0])):
        lab = sample[task][jj]
        if len(lab.unique()) == 1 and lab.unique() == _get(p, "ignore_index"):
            continue
        h, w = int(meta["img_size"][jj][0]), int(meta["img_size"][jj][1])
        pred = out[jj]
        if (h, w) != tuple(pred.shape[:2]):
            dh, dw = max(pred.shape[0] - h, 0), max(pred.shape[1] - w, 0)
            if dh > 0 or dw > 0:
                pred = pred[dh // 2:dh // 2 + h, dw // 2:dw // 2 + w]
        assert tuple(pred.shape[:2]) == (h, w)
        if pred.ndim == 3:
            raise ValueError("3-D prediction")
        files[str(meta["img_name"][jj]) + ".png"] = pred.cpu().numpy().astype(np.uint8)
    return files


def jet(arr):
    """visualization_utils.py:174-177: min/max normalisation in float32, truncation, cv2's JET (BGR)."""
    import cv2
    arr = np.asarray(arr, dtype=np.float32)
    with np.errstate(invalid="ignore", divide="ignore"):
        a = (arr - arr.min()) / (arr.max() - arr.min()) * 255
        idx = a.astype(np.uint8)
    return cv2.applyColorMap(idx, cv2.COLORMAP_JET)


def encode(arr, task, p):
    """One image's get_output map -> the array vis_pred_for_one_task hands to cv2.imwrite."""
    if task == "depth":
        return jet(np.asarray(arr).squeeze())
    if task == "semseg":
        arr = E.vis_encoding(p, task)[1][arr]
    elif task == "human_parts":
        arr = E.labelcolormap(7)[arr]
    with np.errstate(invalid="ignore"):
        a = np.asarray(arr).astype(np.uint8)
    return a[:, :, [2, 1, 0]] if a.ndim == 3 else a


def vis_preds(p, sample, output, task):
    """The files vis_pred_for_one_task writes, as {'{img_name}_{task}.png': array given to cv2.imwrite}."""
    meta = sample["meta"]
    h, w = int(meta["img_size"][0][0]), int(meta["img_size"][0][1])
    out = get_output(resize(output[task], (h, w)), task).cpu().numpy()
    return {f"{meta['img_name'][jj]}_{task}.png": encode(out[jj], task, p) for jj in range(out.shape[0])}
