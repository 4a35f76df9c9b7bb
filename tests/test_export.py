"""Prediction export and visualisation, CPU side: the oracle (oracle/export_ref.py) against the reference's files in
tests/golden/export.pt.xz and against the live reference, the restated palettes and the JET table, the host logic of
mtt_b200.export, and the PredictionWriter ring with an injected slow encoder."""
import os
import threading
import time

import cv2
import numpy as np
import pytest
import torch

import mtt_b200  # noqa: F401
from mtt_b200 import export as E
from oracle import export_ref as R
from oracle import make_export_golden as G
from oracle import ref_loader

PROJECTS = ("TaskPrompter", "InvPT")


def _gold():
    return G.load()


def _p(db, stc=True):
    return dict(train_db_name=db, ignore_index=255, semseg_save_train_class=stc)


def _sample(case):
    s = {"meta": case["meta"]}
    s.update({t: v.float() for t, v in case["labels"].items()})
    return s


def _oracle_export(case, task, reference):
    out = {t: v.float() for t, v in case["logits"].items()}
    return R.save_preds(_p(case["db"], case["save_train_class"]), _sample(case), out, task, reference)


def _assert_files_equal(got, ref):
    assert sorted(got) == sorted(ref)
    for f in ref:
        assert got[f].dtype == np.uint8 and np.array_equal(got[f], ref[f]), f


def test_oracle_export_matches_golden():
    n = 0
    for case in _gold()["export"]:
        for reference in PROJECTS:
            for task, files in case["files"][reference].items():
                if files is None:    # TaskPrompter's semseg branch raises (evaluate_utils.py:77-79,150)
                    assert reference == "TaskPrompter" and task == "semseg"
                    continue
                _assert_files_equal(_oracle_export(case, task, reference), files)
                n += len(files)
    assert n > 20


def test_golden_export_skips_the_all_ignore_image_and_crops_the_padding():
    case = _gold()["export"][0]
    files = case["files"]["InvPT"]["edge"]
    names = case["meta"]["img_name"]
    assert names[2] + ".png" not in files and len(files) == len(names) - 1
    for i, (h, w) in enumerate(case["meta"]["img_size"]):
        if i != 2:
            assert files[names[i] + ".png"].shape == (h, w)


def test_oracle_vis_matches_golden():
    for case in _gold()["vis"]:
        out = {t: v.float() for t, v in case["logits"].items()}
        for task, files in case["files"].items():
            got = R.vis_preds(_p(case["db"]), {"meta": case["meta"]}, out, task)
            _assert_files_equal(got, files)
    cs = _gold()["vis"][2]["files"]["depth"]
    assert all((a == a.reshape(-1, 3)[0]).all() for a in cs.values())   # constant depth: one JET colour


@pytest.mark.skipif(not ref_loader.available(), reason="reference tree not present")
def test_oracle_matches_live_reference():
    g = _gold()
    case = g["export"][1]
    for reference in PROJECTS:
        live = G.run_export(case, reference)
        for task, files in live.items():
            if files is not None:
                _assert_files_equal(_oracle_export(case, task, reference), files)
    vcase = g["vis"][1]
    live = G.run_vis(vcase)
    out = {t: v.float() for t, v in vcase["logits"].items()}
    for task, files in live.items():
        _assert_files_equal(R.vis_preds(_p(vcase["db"]), {"meta": vcase["meta"]}, out, task), files)


@pytest.mark.skipif(not ref_loader.available(), reason="reference tree not present")
def test_palettes_equal_the_reference():
    ref_loader._activate("TaskPrompter")
    from utils import visualization_utils as V
    for n in (7, 21, 40, 256):
        assert np.array_equal(E.labelcolormap(n), V.labelcolormap(n)), n
    assert np.array_equal(E.cityscapes_colormap(), V.create_cityscapes_label_colormap())
    from utils.utils import CS_class_map
    assert [CS_class_map[i] for i in range(19)] == list(E.cityscapes_id_table()[:19])


def test_jet_table_equals_cv2():
    ref = cv2.applyColorMap(np.arange(256, dtype=np.uint8), cv2.COLORMAP_JET).reshape(256, 3)
    assert np.array_equal(E.jet_bgr(), ref)


def test_numpy_nan_cast_is_zero():
    """The constant-depth rule of mtt_render: numpy's float32 -> uint8 cast sends NaN to 0 on x86-64."""
    with np.errstate(invalid="ignore"):
        assert np.array([np.nan], dtype=np.float32).astype(np.uint8)[0] == 0


def test_crop_window_and_offsets():
    assert E.crop_window((26, 31), (23, 28)) == (1, 1, 23, 28)       # odd deltas: delta // 2
    assert E.crop_window((26, 31), (26, 31)) == (0, 0, 26, 31)
    assert E.crop_window((512, 512), (375, 500)) == (68, 6, 375, 500)
    with pytest.raises(ValueError):
        E.crop_window((26, 31), (27, 31))                              # the reference's assert
    with pytest.raises(ValueError):
        E.crop_window((26, 31), (20, 32))
    offs, total = E.pack_offsets([(2, 3), (4, 5), (1, 1)], 3)
    assert offs == [0, 18, 78] and total == 81
    offs, total = E.pack_offsets([(2, 3), (4, 5)], 1)
    assert offs == [0, 6] and total == 26


def test_encodings_and_refusals():
    p = _p("PASCALContext")
    assert E.export_encoding(p, "edge") == ("u8", None)
    assert E.export_encoding(p, "semseg")[0] == "class" and E.export_encoding(p, "semseg")[1] is None
    enc, table = E.export_encoding(_p("Cityscapes3D", stc=False), "semseg")
    assert enc == "class" and list(table[:19]) == E.CS_VALID_CLASSES and table[200] == 200
    assert E.export_encoding(_p("Cityscapes3D", stc=False), "semseg", "InvPT")[1] is None
    for t in ("normals", "depth"):
        with pytest.raises(ValueError, match="3-D"):
            E.export_encoding(p, t)
    for fn in (lambda: E.export_encoding(p, "3ddet"), lambda: E.vis_encoding(p, "3ddet")):
        with pytest.raises(NotImplementedError, match="mmdet3d"):
            fn()
    assert E.vis_encoding(p, "depth") == ("jet", None)
    assert E.vis_encoding(p, "normals") == ("normals_bgr", None)
    assert np.array_equal(E.vis_encoding(_p("NYUD"), "semseg")[1], E.labelcolormap(40))
    with pytest.raises(ValueError):
        E.PredictionWriter(p, ["edge"], {"edge": "/nonexistent"}, reference="MTI-Net")


class SlowEncoder:
    """Stands in for the device: renders a slot's jobs with the oracle after checking the slot is free, and makes
    the writer threads wait before they see the bytes."""

    def __init__(self, delay=0.05):
        self.delay, self.encoded, self.lock = delay, [], threading.Lock()

    def encode(self, slot, jobs):
        assert slot.future is None or slot.future.done(), "slot reused before its files were written"
        parts, base, fbase = [], 0, 0
        for j in jobs:
            x = j.src
            maps = R.get_output(x, j.task) if j.postproc is not None else x
            blob = []
            for jj, (y0, x0, h, w) in enumerate(j.crops):
                a = maps[jj][y0:y0 + h, x0:x0 + w].numpy().astype(np.uint8)
                assert j.offsets[jj] == sum(b.size for b in blob)
                blob.append(a.reshape(-1))
            j.base = (base, fbase)
            data = np.concatenate(blob)
            assert data.size == j.total
            parts.append(data)
            base += data.size
            fbase += len(j.names)
        slot.host = np.concatenate(parts)
        slot.flags_host = np.zeros(fbase, np.int32)
        with self.lock:
            self.encoded.append(id(slot))

    def wait(self, slot):
        time.sleep(self.delay)
        return slot.host, slot.flags_host


def test_writer_ring_with_a_slow_encoder(tmp_path):
    case = _gold()["export"][0]
    enc = SlowEncoder()
    written = []

    def imwrite(path, arr):
        written.append(path)
        cv2.imwrite(path, arr)

    dirs = {t: str(tmp_path / t) for t in ("edge", "sal")}
    w = E.PredictionWriter(_p("PASCALContext"), ["edge", "sal"], dirs, "InvPT", slots=2, workers=2, encoder=enc,
                           imwrite=imwrite)
    names = case["meta"]["img_name"]
    expected = {}
    for k in range(5):
        meta = {"img_name": [f"b{k}_{n}" for n in names], "img_size": case["meta"]["img_size"]}
        sample = dict(_sample(case), meta=meta)
        logits = {t: case["logits"][t].float() for t in ("edge", "sal")}
        w.update(logits, sample, meta)
        for t in ("edge", "sal"):
            for f, a in R.save_preds(_p("PASCALContext"), dict(sample, meta=meta), logits, t, "InvPT").items():
                expected[os.path.join(dirs[t], f)] = a
    w.close()
    assert len(enc.encoded) == 5 and len(set(enc.encoded)) == 2
    assert sorted(written) == sorted(expected)
    for path, a in expected.items():
        assert np.array_equal(cv2.imread(path, cv2.IMREAD_UNCHANGED), a), path
