"""GPU: the Cityscapes-3D device data path (mtt_cityscapes_targets + preprocess_image through mtt_b200.cityscapes) bit for
bit against the unmodified reference's batches (tests/golden/cityscapes.pt.xz), the full loader path from PNG files,
the absence of host synchronisation, Swin predict() against forward + get_output, the confusion meter on int64
labels, and an end-to-end evaluation on tps_mid."""
import numpy as np
import pytest
import torch

from oracle import configs
from oracle import make_cityscapes_golden as G
from test_cityscapes import _by_stem, _p

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gold():
    return G.load()


def _device_batch(case, samples):
    from mtt_b200 import cityscapes as CS

    raw = CS.make_collate(_p(case["dd"]))(samples)
    raw["buf"] = raw["buf"].pin_memory()
    return CS.DeviceTransforms(_p(case["dd"]))(raw)


def _assert_batch_equal(got, batch, rows, name):
    torch.cuda.synchronize()
    sem, dep, img = got["semseg"].cpu().numpy(), got["depth"].cpu().numpy(), got["image"].cpu().numpy()
    for g, r in enumerate(rows):
        assert np.array_equal(sem[g], batch["semseg"][r]), name
        assert np.array_equal(dep[g].view(np.int32), batch["depth"][r].view(np.int32)), name
        assert np.array_equal(img[g].view(np.int32), batch["image"][r].view(np.int32)), name


def test_targets_and_image_match_golden_bitwise(cuda_dev, gold):
    n = 0
    for case in gold["cases"]:
        if "batch" not in case:
            continue
        samples = [_by_stem(case)[s] for s in case["order"]]
        got = _device_batch(case, samples)
        assert got["semseg"].dtype == torch.int64 and got["depth"].shape[1] == 1
        _assert_batch_equal(got, case["batch"], range(len(samples)), case["name"])
        n += 1
    assert n == 6


def test_targets_entry_point_directly(cuda_dev, gold):
    """ops.cityscapes_targets with one output at a time, and a width that is not a multiple of 4 (scalar stores)."""
    from mtt_b200 import ops

    case = gold["cases"][1]                     # 5 x 12 -> 12 x 29
    samples = [_by_stem(case)[s] for s in case["order"]]
    ids = torch.from_numpy(np.stack([s["label_ids"] for s in samples])).cuda()
    disp = torch.from_numpy(np.stack([s["disparity"].astype(np.int32) for s in samples])).to(torch.uint16).cuda()
    H, W = case["dd"]
    sem = torch.full((2, H, W), -7, dtype=torch.int64, device="cuda")
    ops.cityscapes_targets(ids, None, (H, W), semseg=sem)
    dep = torch.empty(2, 1, H, W, device="cuda")
    ops.cityscapes_targets(ids, disp, (H, W), depth=dep)
    torch.cuda.synchronize()
    assert np.array_equal(sem.cpu().numpy(), case["batch"]["semseg"])
    assert np.array_equal(dep.cpu().numpy().view(np.int32), case["batch"]["depth"].view(np.int32))
    with pytest.raises(ValueError):
        ops.cityscapes_targets(ids, None, (H, W), depth=dep)
    with pytest.raises(ValueError):
        ops.cityscapes_targets(ids, disp, (H, W), semseg=sem.view(2, 1, H, W))
    with pytest.raises(RuntimeError, match="index tables"):
        ops.cityscapes_targets(ids[:1], None, (1, 20000),
                               semseg=torch.empty(1, 1, 20000, dtype=torch.int64, device="cuda"))


def test_loader_from_png_files(cuda_dev, gold, tmp_path):
    """The golden trees rewritten as PNGs -> RawCityscapes3D -> DataLoader(pin_memory) -> DeviceTransforms."""
    from mtt_b200 import cityscapes as CS

    for k, case in enumerate(gold["cases"]):
        if "batch" not in case:
            continue
        root = str(tmp_path / f"case{k}")
        G.write_tree(root, "val", case["samples"])
        p = _p(case["dd"])
        ds = CS.RawCityscapes3D(p, root, split=["val"])
        loader = torch.utils.data.DataLoader(ds, batch_size=len(ds), collate_fn=CS.make_collate(p), pin_memory=True)
        dt = CS.DeviceTransforms(p)
        for raw in loader:
            got = dt(raw)
            names = got["meta"]["img_name"]
            rows = [case["order"].index(nm[:-len("_leftImg8bit")]) for nm in names]
            _assert_batch_equal(got, case["batch"], rows, case["name"])
            ref_meta = case["batch"]["meta"]
            assert torch.equal(got["meta"]["scale_factor"], ref_meta["scale_factor"][rows])
            assert [v.tolist() for v in got["meta"]["img_size"]] == [ref_meta["img_size"][r].tolist() for r in rows]


def test_device_transforms_do_not_synchronise(cuda_dev):
    from mtt_b200 import cityscapes as CS

    rng = np.random.default_rng(3)
    batch = [G.make_sample(rng, "ulm", i, 1024, 2048) for i in range(2)]
    p = _p((512, 1024))
    raw = CS.make_collate(p)(batch)
    raw["buf"] = raw["buf"].pin_memory()
    dt = CS.DeviceTransforms(p)
    dt(raw)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = dt(raw)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert out["image"].shape == (2, 3, 1024, 2048) and out["semseg"].shape == (2, 512, 1024)
    assert out["depth"].shape == (2, 1, 512, 1024)


def _swin(name, seed, graph):
    import mtt_b200  # noqa: F401
    from mtt_b200 import taskprompter_swin as TS
    from oracle import taskprompter_swin_ref as SR

    cfg = configs.taskprompter_swin(name)
    sd = SR.init_state_dict(cfg, seed=seed)
    m = TS.build_from_config(cfg, nsplit=2, use_graph=graph).eval()
    m.load_state_dict(sd, strict=False)
    return cfg, m.cuda(), sd


@pytest.mark.parametrize("graph", [False, True])
def test_swin_predict_matches_forward_get_output(cuda_dev, graph):
    """Tolerances of test_taskprompter_gpu.py::test_predict_fused_postprocessing: index maps bit-exact against the
    argmax of this build's own logits, float maps within 1e-4, and get_output of the oracle's logits away from near
    ties. The predict plan makes as many launches as the forward plan."""
    from mtt_b200 import ops
    from oracle import postproc_ref
    from oracle import taskprompter_swin_ref as SR

    cfg, m, sd = _swin("tps_mid", 13, graph)
    x = torch.randn(2, 3, *cfg["img_size"], generator=torch.Generator().manual_seed(6))
    with torch.no_grad():
        logits = {t: v.clone() for t, v in m(x.cuda()).items()}
        m.predict(x.cuda())                            # capture (graph) or warm-up
        n0 = ops.launch_count()
        got = {t: v.clone() for t, v in m.predict(x.cuda()).items()}   # the plan's buffers are reused below
        torch.cuda.synchronize()
        n = ops.launch_count() - n0
        ref = SR.forward(sd, cfg, x)
    fwd = m.plan(2, cuda_dev).launches_per_forward()
    assert m.plan(2, cuda_dev, postproc=True).launches_per_forward() == fwd
    if not graph:
        assert n == fwd
    for t in cfg["tasks"]:
        own = postproc_ref.get_output(logits[t], t)
        want = postproc_ref.get_output(ref[t], t)
        assert got[t].shape == want.shape and got[t].dtype == want.dtype, t
        if want.dtype == torch.int64:
            assert torch.equal(got[t], own), t
            top2 = ref[t].topk(2, dim=1).values
            safe = (top2[:, 0] - top2[:, 1]) > 1e-4 * ref[t].abs().max()
            assert (got[t].cpu() == want)[safe].all(), t
        else:
            assert (got[t] - own).abs().max() <= 1e-4 * own.abs().max().clamp_min(1.0), t
            assert (got[t].cpu() - want).abs().max() <= 2e-3 * want.abs().max().clamp_min(1.0), t


def test_confusion_meter_int64_labels_match_fp32(cuda_dev):
    from mtt_b200 import evaluate as E

    g = torch.Generator().manual_seed(4)
    labels = torch.randint(0, 21, (3, 37, 53), generator=g)
    labels[labels == 20] = 255
    labels[0, :2] = 200                                 # a value that is neither a class nor ignore
    pred = torch.randint(-1, 20, (3, 37, 53), generator=g)
    words = []
    for lab in (labels.float().unsqueeze(1), labels):
        m = E.ConfusionMeter(19, [str(i) for i in range(19)], 255)
        m.update(pred.cuda(), lab.cuda())
        m.update(pred[:1].cuda(), lab[:1].cuda())
        words.append(m.host_words())
    assert np.array_equal(words[0], words[1])
    assert words[0].sum() > 0


def test_end_to_end_tps_mid(cuda_dev, tmp_path):
    """PNG tree -> loader -> DeviceTransforms -> Swin predict() -> PerformanceMeter(['semseg', 'depth']) against
    oracle/meters_ref.py on the same predictions and labels."""
    from mtt_b200 import cityscapes as CS
    from mtt_b200 import evaluate as E
    from oracle import cityscapes_ref as R
    from oracle import meters_ref as MR

    cfg, m, _ = _swin("tps_mid", 17, graph=True)
    rng = np.random.default_rng(8)
    samples = [G.make_sample(rng, "weimar", i, *cfg["img_size"]) for i in range(4)]
    for s in samples:
        s["disparity"] = (s["disparity"] % 6000).astype(np.uint16)   # depths 0 .. 23 m (and -1 / 0)
    root = str(tmp_path / "e2e")
    G.write_tree(root, "val", samples)
    p = dict(_p(cfg["dd_label_map_size"]), ignore_index=255, TASKS=dict(NAMES=["semseg", "depth"], depth_min=0.0,
                                                                          depth_max=80.0))
    ds = CS.RawCityscapes3D(p, root, split=["val"])
    loader = torch.utils.data.DataLoader(ds, batch_size=2, collate_fn=CS.make_collate(p), pin_memory=True)
    dt = CS.DeviceTransforms(p)
    pm, rm = E.PerformanceMeter(p, ["semseg", "depth"]), MR.PerformanceMeter(p, ["semseg", "depth"])
    by = {s["stem"]: s for s in samples}
    with torch.no_grad():
        for raw in loader:
            batch = dt(raw)
            assert batch["semseg"].shape == (2, 128, 256)
            out = m.predict(batch["image"])
            pm.update(out, batch)
            labels = [R.targets(by[n[:-len("_leftImg8bit")]]["label_ids"], by[n[:-len("_leftImg8bit")]]["disparity"],
                                cfg["dd_label_map_size"]) for n in batch["meta"]["img_name"]]
            gt = {"semseg": torch.from_numpy(np.stack([lab[0] for lab in labels])),
                  "depth": torch.from_numpy(np.stack([lab[1] for lab in labels]))}
            rm.update({t: v.cpu() for t, v in out.items()}, gt)
    from test_meters import assert_scores_match

    assert_scores_match(pm.get_score(verbose=False), rm.get_score())
