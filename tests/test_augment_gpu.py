"""GPU: mtt_augment (csrc/augment.cu) against the real reference's outputs (tests/golden/augment.pt.xz) and against the numpy
restatement (oracle/augment_ref.py) at full PASCAL-Context / NYUD geometry, bit for bit."""
import os
import random

import numpy as np
import pytest
import torch

from oracle import augment_ref as R

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "augment.pt.xz")


def bits_equal(a, b):
    a, b = np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def _p(db, tasks, train_scale, test_scale=None):
    return {"train_db_name": db, "TASKS": {"NAMES": list(tasks)}, "TRAIN": {"SCALE": tuple(train_scale)},
            "TEST": {"SCALE": tuple(test_scale or train_scale)}}


def run_device(samples, tasks, size, records, train=True):
    from mtt_b200 import augment as A

    if train:
        H, W = size
    else:
        H, W = max(size[0], samples[0]["image"].shape[0]), max(size[1], samples[0]["image"].shape[1])
    buf, head = A.pack(samples, tasks, size, records)
    raw = {"buf": buf.pin_memory(), "head": head, "B": len(samples), "H": H, "W": W, "tasks": list(tasks)}
    aug = A.DeviceTransforms(_p("PASCALContext", tasks, size), train=train)
    out = aug(raw)
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in out.items()}, aug.last_chosen.cpu().tolist()


def test_golden(cuda_dev):
    from oracle import make_augment_golden as G
    g = G.load(GOLDEN)
    for name, s, rec, ref, consumed in zip(g["names"], g["samples"], g["records"], g["outputs"], g["consumed"]):
        tasks = [k for k in s if k not in ("image", "meta")]
        got, chosen = run_device([s], tasks, g["crop"], [rec])
        for k in ref:
            assert bits_equal(got[k][0], ref[k]), (name, k)
        assert chosen[0] == consumed - 1, (name, chosen, consumed)
    for s, ref in zip(g["valid_samples"], g["valid_outputs"]):
        tasks = [k for k in s if k not in ("image", "meta")]
        got, _ = run_device([s], tasks, g["valid_size"], [_identity()], train=False)
        for k in ref:
            assert bits_equal(got[k][0], ref[k]), k


def _identity():
    from mtt_b200 import augment as A
    return A._IDENTITY


def _sample(rng, h, w, tasks):
    from oracle import make_augment_golden as G
    s = G.make_sample(rng, h, w, tasks, zero_normals=True, zero_depth=True)
    # realistic label maps: large regions, so the cat_max_ratio test both passes and fails
    yy, xx = np.mgrid[0:h, 0:w]
    s["semseg"] = (((yy // 97) * 7 + (xx // 131) * 3) % 21).astype(np.float32)[..., None]
    s["semseg"][: h // 5] = 255
    return s


def _check_train(samples, tasks, size, seed):
    from mtt_b200 import augment as A
    rnd = random.Random(seed)
    records = [A.draw_params(s["image"].shape[0], s["image"].shape[1], size, rng=rnd) for s in samples]
    got, chosen = run_device(samples, tasks, size, records)
    for b, (s, rec) in enumerate(zip(samples, records)):
        ref, st = R.train_transform(s, rec, size, return_stages=True)
        assert chosen[b] == (-1 if st["chosen"] is None else st["chosen"])
        for k in ref:
            assert bits_equal(got[k][b], ref[k]), (seed, b, k)
    return records


def test_full_geometry_pascal(cuda_dev):
    rng = np.random.default_rng(0)
    tasks = ("semseg", "human_parts", "sal", "edge", "normals")
    samples = [_sample(rng, h, w, tasks) for h, w in [(375, 500), (281, 500), (500, 375), (333, 500)]]
    for seed in range(6):
        _check_train(samples, tasks, (512, 512), seed)


def test_full_geometry_nyud(cuda_dev):
    rng = np.random.default_rng(1)
    tasks = ("semseg", "depth", "normals", "edge")
    samples = [_sample(rng, 480, 640, tasks) for _ in range(2)]
    for seed in range(6):
        _check_train(samples, tasks, (448, 576), seed)


def test_photometric_every_rgb_triple(cuda_dev):
    a = np.arange(1 << 24, dtype=np.uint32)
    img = np.stack([(a >> 16) & 255, (a >> 8) & 255, a & 255], -1).astype(np.float32).reshape(4096, 4096, 3)
    s = {"image": img, "semseg": np.zeros((4096, 4096, 1), np.float32)}
    base = dict(scale=1.0, crops=None, flip=False, bright=None, f_mode=True, contrast=None, sat=None, hue=None)
    for kw in [dict(sat=0.5), dict(sat=1.4999), dict(hue=-18), dict(hue=17), dict(sat=1.21, hue=5),
               dict(bright=-12.5, contrast=1.3, sat=0.77, hue=-7, f_mode=False)]:
        rec = dict(base, **kw)
        got, _ = run_device([s], ["semseg"], (4096, 4096), [rec])
        ref = R.normalize(R.photometric(img.astype(np.uint8), rec)).transpose(2, 0, 1)
        assert bits_equal(got["image"][0], ref), kw


def test_validation_chain(cuda_dev):
    rng = np.random.default_rng(2)
    tasks = ("semseg", "human_parts", "sal", "edge", "normals")
    samples = [_sample(rng, h, w, tasks) for h, w in [(375, 500), (512, 300), (281, 512)]]
    got, _ = run_device(samples, tasks, (512, 512), [_identity()] * 3, train=False)
    for b, s in enumerate(samples):
        ref = R.valid_transform(s, (512, 512))
        for k in ref:
            assert bits_equal(got[k][b], ref[k]), (b, k)


def test_collate_to_device_does_not_synchronise(cuda_dev):
    from mtt_b200 import augment as A
    rng = np.random.default_rng(3)
    tasks = ("semseg", "depth", "normals", "edge")
    p = _p("NYUD", tasks, (448, 576))
    batch = [_sample(rng, 480, 640, tasks) for _ in range(2)]
    random.seed(0)
    raw = A.make_collate(p)(batch)
    raw["buf"] = raw["buf"].pin_memory()
    aug = A.DeviceTransforms(p)
    aug(raw)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = aug(raw)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert out["image"].shape == (2, 3, 448, 576) and out["normals"].shape == (2, 3, 448, 576)
    assert raw["meta"]["img_name"] == out["meta"]["img_name"]


def test_bad_arguments_rejected(cuda_dev):
    from mtt_b200 import augment as A
    from mtt_b200 import ops
    rng = np.random.default_rng(4)
    s = _sample(rng, 40, 50, ("semseg", "edge"))
    rec = A.draw_params(40, 50, (32, 32), rng=random.Random(0))
    buf, head = A.pack([s], ["semseg", "edge"], (32, 32), [rec])
    dev = buf.cuda()
    smp, data = dev[:head], dev[head:].view(torch.float32)
    img = torch.empty(1, 3, 32, 32, device=cuda_dev)
    lab = [torch.empty(1, 1, 32, 32, device=cuda_dev) for _ in range(2)]
    ws = torch.empty(ops.augment_workspace_bytes(1) // 4, dtype=torch.int32, device=cuda_dev)
    ok = dict(B=1, H=32, W=32, train=True, crop_hw=(32, 32), tasks=["semseg", "edge"], task_out=lab, image_out=img,
              workspace=ws)
    ops.augment(smp, data, **ok)
    bad = [dict(tasks=["edge"], task_out=lab[:1]),                       # train without semseg
           dict(tasks=["semseg", "semseg"]),                              # a task kind twice
           dict(H=30),                                                    # train output != crop
           dict(B=0),
           dict(workspace=ws[:1]),
           dict(std=(0.2, 0.0, 0.2))]
    for kw in bad:
        with pytest.raises(RuntimeError, match="mtt_augment"):
            ops.augment(smp, data, **dict(ok, **kw))
    torch.cuda.synchronize()


def test_native_loop_end_to_end(cuda_dev):
    """make_collate -> DeviceTransforms -> TrainStep.step, then PerformanceMeter over the validation chain: no host-side
    transform anywhere."""
    import math

    from mtt_b200 import augment as A
    from mtt_b200 import evaluate as E
    from mtt_b200 import losses
    from mtt_b200 import taskprompter as TP
    from mtt_b200.train import TrainStep
    from oracle import configs
    from oracle import taskprompter_ref as TPR

    cfg = configs.taskprompter("tp_tiny")
    tasks = list(cfg["tasks"])                                   # semseg, depth, normals
    hw = tuple(cfg["img_size"])
    p = dict(_p("NYUD", tasks, hw), ignore_index=255, edge_w=0.95, ignore_invalid_area_depth=True,
             loss_kwargs=dict(loss_weights={"semseg": 1.0, "depth": 1.0, "normals": 10.0}),
             TASKS=dict(NAMES=tasks, depth_min=0.0, depth_max=80.0))
    rng = np.random.default_rng(7)

    def raw(h, w):
        s = _sample(rng, h, w, ("semseg", "depth", "normals"))
        s["semseg"] = np.where(s["semseg"] == 255, 255, s["semseg"] % 5).astype(np.float32)
        return s

    train_set = [raw(int(rng.integers(56, 90)), int(rng.integers(80, 130))) for _ in range(4)]
    random.seed(0)
    loader = torch.utils.data.DataLoader(train_set, batch_size=2, collate_fn=A.make_collate(p), pin_memory=True)
    model = TP.build_from_config(dict(cfg, drop_path_rate=0.0), use_graph=False)
    model.load_state_dict(TPR.init_state_dict(cfg, seed=3), strict=True)
    step = TrainStep(model.to(cuda_dev), lr=1e-4)
    aug = A.DeviceTransforms(p)
    criterion = losses.get_criterion(p)
    for rawb in loader:
        batch = aug(rawb)
        loss = step.step(batch["image"], {t: batch[t] for t in tasks}, criterion)
        assert math.isfinite(float(loss["total"]))
    val = A.DeviceTransforms(p, train=False)
    vcollate = A.make_collate(p, train=False)
    pm = E.PerformanceMeter(p, tasks)
    model.eval()
    with torch.no_grad():
        vb = val(vcollate([raw(*hw), raw(hw[0] - 6, hw[1] - 10)]))
        pred = model.predict(vb["image"])
        pm.update(pred, {t: vb[t] for t in tasks})
    scores = pm.get_score(verbose=False)
    assert set(scores) == set(tasks)
