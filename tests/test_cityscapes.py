"""CPU tests of the Cityscapes-3D device data path (mtt_b200.cityscapes): Pillow's NEAREST rule, the numpy restatement
(oracle/cityscapes_ref.py) against the unmodified reference's batches (tests/golden/cityscapes.pt.xz, written by
oracle/make_cityscapes_golden.py) and the live reference, the host-side invalid-id check, the collate's packing, the
raw dataset's file list, the refusals, and Swin predict() with the kernels replaced by tests/emul_ops.py."""
import os

import numpy as np
import pytest
import torch

from oracle import cityscapes_ref as R
from oracle import configs, ref_loader
from oracle import make_cityscapes_golden as G

CS_P = dict(train_db_name="Cityscapes3D", TASKS=dict(NAMES=["semseg", "depth"]), TRAIN=dict(SCALE=(1024, 2048)),
            TEST=dict(SCALE=(1024, 2048)))


def _p(dd, tasks=("semseg", "depth")):
    return dict(CS_P, dd_label_map_size=list(dd), TASKS=dict(NAMES=list(tasks)))


@pytest.fixture(scope="module")
def gold():
    return G.load()


def _by_stem(case):
    return {s["stem"]: s for s in case["samples"]}


@pytest.mark.parametrize("mode", ["F", "L"])
def test_pil_nearest_rule_exhaustive(mode):
    """The stated rule equals PIL.Image.resize(..., NEAREST) for every (n_src, n_dst) up to 64, on both axes."""
    from PIL import Image

    import mtt_b200  # noqa: F401
    from mtt_b200 import cityscapes as CS

    for ns in range(1, 65):
        ramp = np.arange(ns, dtype=np.float32 if mode == "F" else np.uint8)
        rows = Image.fromarray(np.ascontiguousarray(np.broadcast_to(ramp[:, None], (ns, 2))))
        cols = Image.fromarray(np.ascontiguousarray(np.broadcast_to(ramp[None, :], (2, ns))))
        for nd in range(1, 65):
            want_y = np.array(rows.resize((2, nd), Image.NEAREST))[:, 0].astype(np.int64)
            want_x = np.array(cols.resize((nd, 2), Image.NEAREST))[0].astype(np.int64)
            got = R.pil_nearest_index(ns, nd)
            assert np.array_equal(got, want_y) and np.array_equal(got, want_x), (mode, ns, nd)
            assert np.array_equal(CS.pil_nearest_index(ns, nd), got)
    assert R.pil_nearest_index(2, 7)[3] == 0          # floor((3 + 0.5) * 2 / 7) would be 1
    assert np.array_equal(R.pil_nearest_index(1024, 512), 2 * np.arange(512) + 1)


def test_pil_nearest_rule_at_cityscapes_sizes():
    from PIL import Image

    for ns, nd in ((1024, 512), (2048, 1024), (1024, 128), (2048, 256), (1000, 999), (999, 1000), (2047, 1023)):
        ramp = np.arange(ns, dtype=np.float32)[None, :]
        want = np.array(Image.fromarray(ramp).resize((nd, 1), Image.NEAREST))[0].astype(np.int64)
        assert np.array_equal(R.pil_nearest_index(ns, nd), want), (ns, nd)


def test_restatement_matches_golden(gold):
    for case in gold["cases"]:
        if "batch" not in case:
            continue
        samples, batch = _by_stem(case), case["batch"]
        assert batch["meta"]["img_name"] == [G_stem + "_leftImg8bit" for G_stem in case["order"]]
        for b, stem in enumerate(case["order"]):
            s = samples[stem]
            sem, dep = R.targets(s["label_ids"], s["disparity"], case["dd"])
            assert np.array_equal(sem, batch["semseg"][b]), case["name"]
            assert dep.dtype == np.float32 and np.array_equal(dep.view(np.int32), batch["depth"][b].view(np.int32))
            img = R.image(s["image"])
            assert np.array_equal(img.view(np.int32), batch["image"][b].view(np.int32)), case["name"]
            assert not R.invalid_sampled(s["label_ids"], case["dd"])
            scale = batch["meta"]["scale_factor"][b].numpy()
            assert np.array_equal(scale, [2048 / s["image"].shape[1], 1024 / s["image"].shape[0]])
            assert batch["meta"]["img_size"][b].tolist() == list(s["image"].shape[:2])
            assert batch["meta"]["dd_label_map_size"][b].tolist() == list(case["dd"])
    # the depth mask tests the RAW id 10, whatever its disparity
    case = gold["cases"][0]
    for b, stem in enumerate(case["order"]):
        s = _by_stem(case)[stem]
        ys, xs = R.sample_grid(s["label_ids"].shape, (16, 24))
        raw = s["label_ids"][ys][:, xs]
        d = s["disparity"][ys][:, xs]
        for dv in (0, 65535):
            assert ((raw == 10) & (d == dv)).any()
        assert (case["batch"]["depth"][b, 0][raw == 10] == 0).all()
        one = (raw != 10) & (d == 1)                   # disparity 1 ends at -1 like 0 (in-place steps :153, :156)
        assert one.any() and (case["batch"]["depth"][b, 0][one] == -1).all()
    names = [c["name"] for c in gold["cases"]]
    assert any("no resize" in n for n in names)
    nr = gold["cases"][names.index("no resize (dd_label_map_size 1024x2048) at 20x30")]
    assert nr["batch"]["semseg"].shape == (2, 20, 30)


def test_invalid_id_check_matches_reference(gold):
    import mtt_b200  # noqa: F401
    from mtt_b200 import cityscapes as CS

    checked = 0
    for case in gold["cases"]:
        collate = CS.make_collate(_p(case["dd"]))
        batch = [dict(case["samples"][i]) for i in range(len(case["samples"]))]
        if "raises" in case:
            assert "invalid class values" in case["raises"]
            with pytest.raises(ValueError, match="Segmentation map contained invalid class values"):
                collate(batch)
            checked += 1
        else:
            collate(batch)
        for s in case["samples"]:
            h, w = s["label_ids"].shape
            hw = CS.label_size((h, w), case["dd"])
            assert CS.invalid_sampled_ids(s["label_ids"], hw) == R.invalid_sampled(s["label_ids"], case["dd"])
    assert checked == 1
    assert any(((c["samples"][1]["label_ids"] == 40).any() and "batch" in c) for c in gold["cases"])


def test_collate_layout():
    import mtt_b200  # noqa: F401
    from mtt_b200 import cityscapes as CS

    rng = np.random.default_rng(0)
    batch = [G.make_sample(rng, "ulm", i, 9, 13) for i in range(3)]
    for s in batch:
        s["meta"] = {"img_name": s["stem"], "img_size": (9, 13), "dd_label_map_size": [4, 6],
                     "scale_factor": np.array([2048 / 13, 1024 / 9])}
    raw = CS.make_collate(_p((4, 6)))(batch)
    B, h, w = 3, 9, 13
    assert (raw["B"], raw["h"], raw["w"], raw["H"], raw["W"]) == (B, h, w, 4, 6)
    o = raw["offsets"]
    assert o[0] == 0 and all(v % 256 == 0 for v in o)
    buf = raw["buf"].numpy()
    assert buf.size == o[2] + 2 * B * h * w
    assert np.array_equal(buf[:3 * B * h * w].reshape(B, h, w, 3), np.stack([s["image"] for s in batch]))
    assert np.array_equal(buf[o[1]:o[1] + B * h * w].reshape(B, h, w), np.stack([s["label_ids"] for s in batch]))
    disp = buf[o[2]:o[2] + 2 * B * h * w].view(np.uint16).reshape(B, h, w)
    assert np.array_equal(disp, np.stack([s["disparity"] for s in batch]))
    assert raw["meta"]["img_name"] == [s["stem"] for s in batch]
    assert raw["meta"]["scale_factor"].dtype == torch.float64 and raw["meta"]["scale_factor"].shape == (3, 2)
    assert [v.tolist() for v in raw["meta"]["img_size"]] == [[9, 13]] * 3
    # semseg only: no disparity block
    raw = CS.make_collate(_p((4, 6), ("semseg",)))([{k: v for k, v in s.items() if k != "disparity"} for s in batch])
    assert len(raw["offsets"]) == 2 and raw["buf"].numel() == raw["offsets"][1] + B * h * w
    # samples of different sizes cannot be stacked
    odd = G.make_sample(rng, "ulm", 9, 9, 14)
    with pytest.raises(ValueError, match="share one size"):
        CS.make_collate(_p((4, 6)))([batch[0], odd])


def test_raw_dataset_matches_reference_file_list(gold, tmp_path):
    import mtt_b200  # noqa: F401
    from mtt_b200 import cityscapes as CS

    case = gold["cases"][0]
    root = str(tmp_path / "v1.0" / "val")       # a '.' in a directory name must not change the sample names
    G.write_tree(root, "val", case["samples"])
    ds = CS.RawCityscapes3D(_p(case["dd"]), root, split=["val"], task_list=["semseg", "depth"])
    assert len(ds) == len(case["samples"])
    samples = _by_stem(case)
    for i in range(len(ds)):
        got = ds[i]
        stem = os.path.basename(ds.files[i])[:-len("_leftImg8bit.png")]
        assert got["meta"]["img_name"] == stem + "_leftImg8bit"
        s = samples[stem]
        assert got["image"].dtype == np.uint8 and np.array_equal(got["image"], s["image"])
        assert got["label_ids"].dtype == np.uint8 and np.array_equal(got["label_ids"], s["label_ids"])
        assert got["disparity"].dtype == np.uint16 and np.array_equal(got["disparity"], s["disparity"])
        assert got["meta"]["img_size"] == s["image"].shape[:2]
    tr = gold["train"]
    root = str(tmp_path / "train")
    G.write_tree(root, "train", tr["samples"], tr["det"])
    ds = CS.RawCityscapes3D(_p(tr["dd"]), root, split="train")
    assert sorted(os.path.basename(f)[:-len("_leftImg8bit.png")] for f in ds.files) == tr["kept"]
    assert not any(n.startswith("CS3D_bad_samples") for n in os.listdir(os.getcwd()))


def test_refusals(tmp_path):
    import mtt_b200  # noqa: F401
    from mtt_b200 import augment as A
    from mtt_b200 import cityscapes as CS

    with pytest.raises(NotImplementedError, match="mmdet3d"):
        CS.RawCityscapes3D(_p((4, 6)), str(tmp_path), task_list=["semseg", "depth", "3ddet"])
    with pytest.raises(ValueError, match="semseg"):
        CS.RawCityscapes3D(_p((4, 6)), str(tmp_path), task_list=["depth"])
    with pytest.raises(NotImplementedError, match="bilinear"):
        CS.RawCityscapes3D(dict(_p((4, 6)), TEST=dict(SCALE=(512, 1024))), str(tmp_path), split=["val"])
    with pytest.raises(NotImplementedError, match="mmdet3d"):
        CS.make_collate(_p((4, 6), ("semseg", "depth", "3ddet")))
    with pytest.raises(ValueError):
        CS.DeviceTransforms(_p((4, 6), ("depth",)), device="cpu")
    with pytest.raises(NotImplementedError):
        A.make_collate(_p((4, 6)))


@pytest.mark.skipif(not ref_loader.available(), reason="reference tree not present")
def test_restatement_matches_live_reference(tmp_path):
    """Fresh random trees through the unmodified CITYSCAPES3D + collate_mil."""
    seed = int.from_bytes(os.urandom(4), "little")
    rng = np.random.default_rng(seed)
    for k in range(3):
        h, w = (int(v) for v in rng.integers(3, 70, 2))
        dd = [int(v) for v in rng.integers(2, 90, 2)]
        samples = [G.make_sample(rng, "zurich", i, h, w) for i in range(2)]
        root = str(tmp_path / f"t{k}")
        G.write_tree(root, "val", samples)
        ds, collate = G.run_reference(root, "val", dd)
        batch = collate([ds[i] for i in range(len(ds))])
        by = {s["stem"]: s for s in samples}
        for b, path in enumerate(ds.files["val"]):      # the batch follows the file list (its img_name may not)
            s = by[os.path.basename(path)[:-len("_leftImg8bit.png")]]
            sem, dep = R.targets(s["label_ids"], s["disparity"], dd)
            assert np.array_equal(sem, batch["semseg"][b].numpy()), (seed, h, w, dd)
            assert np.array_equal(dep.view(np.int32), batch["depth"][b].numpy().view(np.int32)), (seed, h, w, dd)
            assert np.array_equal(R.image(s["image"]).view(np.int32), batch["image"][b].numpy().view(np.int32)), seed


def test_meter_inputs_accept_int64_labels_only_for_confusion():
    import mtt_b200  # noqa: F401
    from mtt_b200 import ops

    pred = torch.zeros(2, 4, 6, dtype=torch.int64)
    state = torch.zeros(8, dtype=torch.int64)
    # both label forms pass the shape checks (then the CPU tensors are refused before any launch)
    for label in (torch.zeros(2, 1, 4, 6), torch.zeros(2, 4, 6, dtype=torch.int64)):
        with pytest.raises(RuntimeError, match="GPU only"):
            ops.meter_confusion_update(pred, label, 19, 255, state)
    for label in (torch.zeros(2, 1, 4, 6, dtype=torch.int64), torch.zeros(2, 4, 6), torch.zeros(2, 4, 7, dtype=torch.int64),
                  torch.zeros(2, 4, 6, dtype=torch.int32)):
        with pytest.raises(ValueError):
            ops.meter_confusion_update(pred, label, 19, 255, state)
    with pytest.raises(ValueError):
        ops.meter_depth_update(torch.zeros(2, 4, 6), torch.zeros(2, 4, 6, dtype=torch.int64), state,
                               min_depth=0.0, max_depth=80.0)


@pytest.mark.parametrize("name", ["tps_tiny", "tps_mid"])
def test_swin_predict_matches_get_output(monkeypatch, name):
    """predict() = forward + get_output (TP/utils/utils.py:27-63) fused into the final resize, with the same launch
    sequence length as the forward."""
    import emul_ops
    import mtt_b200  # noqa: F401
    from mtt_b200 import taskprompter_swin as TS
    from oracle import postproc_ref
    from oracle import taskprompter_swin_ref as SR

    emul_ops.install(monkeypatch)
    cfg = configs.taskprompter_swin(name)
    sd = SR.init_state_dict(cfg, seed=11)
    model = TS.build_from_config(cfg, nsplit=2, use_graph=False).eval()
    model.load_state_dict(sd, strict=False)
    x = torch.randn(2, 3, *cfg["img_size"], generator=torch.Generator().manual_seed(5))
    with torch.no_grad():
        ref = SR.forward(sd, cfg, x)
        got = model.plan(2, torch.device("cpu"), postproc=True).run(x, graph=False)
    for t in cfg["tasks"]:
        want = postproc_ref.get_output(ref[t], t)
        assert got[t].shape == want.shape and got[t].dtype == want.dtype, t
        if want.dtype == torch.int64:
            assert (got[t] == want).float().mean() > 0.995, t
        else:
            assert (got[t] - want).abs().max() <= 2e-3 * want.abs().max().clamp_min(1.0), t
