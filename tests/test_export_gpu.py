"""mtt_render (csrc/export.cu) and mtt_b200.export on the GPU, against the reference's files in
tests/golden/export.pt.xz and the oracle (oracle/export_ref.py)."""
import ctypes as C
import os

import cv2
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from test_export import _gold, _oracle_export, _p, _sample

pytestmark = pytest.mark.gpu


def _maps(logits, task, hw=None):
    """The oracle's get_output maps (CPU), optionally after the resize."""
    from oracle import export_ref as R
    x = logits.float()
    if hw is not None:
        x = R.resize(x, hw)
    return R.get_output(x, task)


def _render_one(dev, src, encode, crops, channels, postproc=None, table=None, out_hw=None, label=None, n_classes=None):
    from mtt_b200 import export as E, ops
    offs, total = E.pack_offsets([(c[2], c[3]) for c in crops], channels)
    out = torch.full((total,), 7, dtype=torch.uint8, device=dev)
    spec = dict(src=src.to(dev).contiguous(), postproc=postproc, encode=encode, crops=crops, offsets=offs, out=out,
                n_classes=n_classes)
    if out_hw is not None:
        spec["out_hw"] = out_hw
    if table is not None:
        spec["table"] = torch.from_numpy(np.ascontiguousarray(table)).to(dev)
    flags = None
    if label is not None:
        flags = torch.full((src.shape[0],), -1, dtype=torch.int32, device=dev)
        spec.update(label=label.to(dev).float().contiguous(), flags=flags, ignore_index=255)
    ws = torch.empty(ops.render_workspace_bytes(1, src.shape[0]) // 4, dtype=torch.int32, device=dev)
    ops.render([spec], ws)
    host = out.cpu().numpy()
    imgs = []
    for o, c in zip(offs, crops):
        a = host[o:o + c[2] * c[3] * channels]
        imgs.append(a.reshape(c[2], c[3], 3) if channels == 3 else a.reshape(c[2], c[3]))
    return imgs, (flags.cpu().numpy() if flags is not None else None)


def _vis_spec(p, task):
    from mtt_b200 import export as E
    enc, table = E.vis_encoding(p, task)
    if enc == "jet":
        table = E.jet_bgr()
    return enc, table, (3 if enc in ("palette_bgr", "normals_bgr", "jet") else 1)


def test_encode_stage_bit_exact_vis(cuda_dev):
    """Map sources (no resize, no get_output): every visualisation encoding equals the reference's files."""
    for case in _gold()["vis"]:
        p = _p(case["db"])
        B = len(case["meta"]["img_name"])
        h, w = case["meta"]["img_size"][0]
        for task, files in case["files"].items():
            m = _maps(case["logits"][task], task, (h, w))
            enc, table, ch = _vis_spec(p, task)
            n_classes = len(table) if enc == "palette_bgr" else None
            imgs, _ = _render_one(cuda_dev, m, enc, [(0, 0, h, w)] * B, ch, table=table, n_classes=n_classes)
            for jj in range(B):
                ref = files[f"{case['meta']['img_name'][jj]}_{task}.png"]
                assert np.array_equal(imgs[jj], ref), (case["name"], task, jj)


def test_encode_stage_bit_exact_export(cuda_dev):
    """Map sources on ragged crops with odd deltas: truncation, class ids with and without the Cityscapes id table,
    and the all-ignore flag, equal to the reference's files (InvPT) and the oracle (TaskPrompter's Cityscapes ids)."""
    from mtt_b200 import export as E
    for case in _gold()["export"]:
        meta = case["meta"]
        for reference in ("TaskPrompter", "InvPT"):
            for task in case["logits"]:
                p = _p(case["db"], case["save_train_class"])
                enc, table = E.export_encoding(p, task, reference)
                m = _maps(case["logits"][task], task)
                H, W = m.shape[1:3]
                crops = [E.crop_window((H, W), s) for s in meta["img_size"]]
                imgs, flags = _render_one(cuda_dev, m, enc, crops, 1, table=table, label=case["labels"][task])
                ref = _oracle_export(case, task, reference)
                gold = case["files"][reference].get(task)
                for jj, name in enumerate(meta["img_name"]):
                    f = name + ".png"
                    assert bool(flags[jj]) == (f not in ref), (case["name"], task, jj)
                    if f in ref:
                        assert np.array_equal(imgs[jj], ref[f]), (case["name"], reference, task, jj)
                        if gold is not None:
                            assert np.array_equal(imgs[jj], gold[f])


def test_jet_constant_map_and_normals_bgr(cuda_dev):
    from mtt_b200 import export as E
    from oracle import export_ref as R
    m = torch.full((2, 5, 7, 1), 3.25)
    imgs, _ = _render_one(cuda_dev, m, "jet", [(0, 0, 5, 7), (1, 2, 3, 4)], 3, table=E.jet_bgr())
    for a in imgs:
        assert np.array_equal(a, R.jet(np.full(a.shape[:2], 3.25, np.float32)))
        assert (a == E.jet_bgr()[0]).all()   # max == min: 0 / 0 = NaN, numpy's cast gives index 0
    g = torch.Generator().manual_seed(3)
    n = torch.rand((2, 6, 9, 3), generator=g) * 255
    imgs, _ = _render_one(cuda_dev, n, "normals_bgr", [(1, 1, 5, 7), (0, 0, 6, 9)], 3)
    assert np.array_equal(imgs[0], n[0, 1:6, 1:8].numpy().astype(np.uint8)[:, :, ::-1])


def _margin_masks(logits, task, hw):
    """Pixels where the fp64 result is unambiguous: top-2 logit gap > 1e-5 for class maps, distance >= 1e-3 from an
    integer for truncated channels."""
    x = F.interpolate(logits.double(), tuple(hw), mode="bilinear")
    if task in ("semseg", "human_parts"):
        top = x.topk(2, dim=1).values
        return (top[:, 0] - top[:, 1] > 1e-5).numpy()
    if task == "normals":
        v = ((F.normalize(x, dim=1) + 1) * 255 / 2).permute(0, 2, 3, 1)
        return ((v - v.floor()).clamp(1e-3, 1 - 1e-3) == (v - v.floor())).all(dim=3).numpy()
    if task == "edge":
        v = 255 / (1 + torch.exp(-x[:, 0]))
    elif task == "sal":
        v = torch.softmax(x, dim=1)[:, 1] * 255
    else:
        d = x[:, 0].clamp(min=0)
        dmin = d.flatten(1).min(1).values[:, None, None]
        dmax = d.flatten(1).max(1).values[:, None, None]
        v = (d - dmin) / (dmax - dmin).clamp(min=1e-30) * 255
    f = v - v.floor()
    return ((f >= 1e-3) & (f <= 1 - 1e-3)).numpy()


def test_full_path_against_reference(cuda_dev):
    """Logits in, resize + get_output + encode on the device, against the reference's visualisation files."""
    from mtt_b200 import export as E
    for case in _gold()["vis"]:
        p = _p(case["db"])
        B = len(case["meta"]["img_name"])
        hw = tuple(case["meta"]["img_size"][0])
        out = {t: v.float().to(cuda_dev) for t, v in case["logits"].items()}
        got = E.render(p, out, hw)
        for task, files in case["files"].items():
            g = got[task].cpu().numpy()
            ok = _margin_masks(case["logits"][task].float(), task, hw)
            for jj in range(B):
                ref = files[f"{case['meta']['img_name'][jj]}_{task}.png"]
                a = g[jj]
                if task in ("semseg", "human_parts"):
                    eq = (a == ref).all(axis=-1)
                    assert eq[ok[jj]].all(), (case["name"], task)
                    assert eq.mean() >= 0.999, (case["name"], task, eq.mean())
                elif task == "depth":
                    jet = E.jet_bgr().astype(np.int64)
                    key = lambda img: np.argmin(np.abs(img.reshape(-1, 1, 3).astype(np.int64) - jet[None]).sum(-1),
                                                axis=1).reshape(img.shape[:2])
                    ia, ir = key(a), key(ref)
                    assert (ia == ir)[ok[jj]].all() and np.abs(ia - ir).max() <= 1, (case["name"], task)
                else:
                    d = np.abs(a.astype(np.int64) - ref.astype(np.int64))
                    m = ok[jj] if d.ndim == 2 else ok[jj][..., None].repeat(3, -1)
                    assert (d[m] == 0).all() and d.max() <= 1, (case["name"], task)


def test_vis_files_and_export_pngs(cuda_dev, tmp_path):
    from mtt_b200 import export as E
    case = _gold()["vis"][0]
    p = _p(case["db"])
    out = {t: v.float().to(cuda_dev) for t, v in case["logits"].items()}
    sample = {"image": torch.zeros(2, 3, 1, 1), "meta": case["meta"]}
    hw = tuple(case["meta"]["img_size"][0])
    arrays = {t: a.cpu().numpy() for t, a in E.render(p, out, hw).items()}
    for task, files in case["files"].items():
        d = tmp_path / task
        E.vis_pred_for_one_task(p, sample, out, str(d), task)
        assert sorted(os.listdir(d)) == sorted(files)
        for jj, name in enumerate(case["meta"]["img_name"]):
            f = f"{name}_{task}.png"
            ours = arrays[task][jj]
            assert (d / f).read_bytes() == cv2.imencode(".png", ours)[1].tobytes()
            if np.array_equal(ours, files[f]):
                assert (d / f).read_bytes() == cv2.imencode(".png", files[f])[1].tobytes()
    # export through the writer from predict()-format maps: the PNGs decode to the reference's pixels
    ecase = _gold()["export"][0]
    dirs = {t: str(tmp_path / ("x_" + t)) for t in ("edge", "sal", "human_parts")}
    maps = {t: _maps(ecase["logits"][t], t).to(cuda_dev) for t in dirs}
    labels = {t: v.float().to(cuda_dev) for t, v in ecase["labels"].items()}
    with E.PredictionWriter(p, list(dirs), dirs, "InvPT", slots=2) as wr:
        wr.update(maps, labels, ecase["meta"])
    for t, d in dirs.items():
        gold = ecase["files"]["InvPT"][t]
        assert sorted(os.listdir(d)) == sorted(gold)
        for f, a in gold.items():
            assert np.array_equal(cv2.imread(os.path.join(d, f), cv2.IMREAD_UNCHANGED), a)


def test_writer_update_has_no_host_sync_and_graph_equals_eager(cuda_dev, tmp_path):
    from mtt_b200 import export as E, ops
    case = _gold()["export"][0]
    dirs = {"edge": str(tmp_path / "edge")}
    logits = {"edge": case["logits"]["edge"].float().to(cuda_dev)}
    labels = {"edge": case["labels"]["edge"].float().to(cuda_dev)}
    w = E.PredictionWriter(_p(case["db"]), ["edge"], dirs, "TaskPrompter", slots=2)
    w.update(logits, labels, case["meta"])          # first use allocates the ring
    torch.cuda.set_sync_debug_mode("error")
    try:
        for k in range(3):
            w.update(logits, labels, dict(case["meta"], img_name=[f"s{k}_{n}" for n in case["meta"]["img_name"]]))
    finally:
        torch.cuda.set_sync_debug_mode("default")
    w.close()
    assert len(os.listdir(dirs["edge"])) == 4 * 3
    # a captured graph of the two launches equals eager launches
    vcase = _gold()["vis"][1]
    src = vcase["logits"]["depth"].float().to(cuda_dev)
    hw = tuple(vcase["meta"]["img_size"][0])
    B = src.shape[0]
    offs, total = E.pack_offsets([hw] * B, 3)
    table = torch.from_numpy(E.jet_bgr()).to(cuda_dev)
    outs = [torch.zeros(total, dtype=torch.uint8, device=cuda_dev) for _ in range(2)]
    ws = torch.empty(ops.render_workspace_bytes(1, B) // 4, dtype=torch.int32, device=cuda_dev)

    def launch(o):
        ops.render([dict(src=src, postproc=4, out_hw=hw, encode="jet", table=table, crops=[(0, 0) + hw] * B,
                         offsets=offs, out=o)], ws)
    launch(outs[0])
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            launch(outs[1])
    torch.cuda.current_stream().wait_stream(s)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(outs[0], outs[1])


def test_bitwise_reproducible(cuda_dev):
    from mtt_b200 import export as E
    case = _gold()["vis"][0]
    out = {t: v.float().to(cuda_dev) for t, v in case["logits"].items()}
    hw = tuple(case["meta"]["img_size"][0])
    a = {t: v.clone() for t, v in E.render(_p(case["db"]), out, hw).items()}
    b = E.render(_p(case["db"]), out, [hw, (hw[0] - 3, hw[1] + 2)])
    c = E.render(_p(case["db"]), out, hw)
    for t in a:
        assert torch.equal(a[t], c[t])
        assert torch.equal(a[t][0], b[t][0])   # one size per image: the first image keeps the batch size


def test_argument_rejection(cuda_dev):
    from mtt_b200 import lib, ops
    dev = cuda_dev
    src = torch.randn(2, 3, 8, 9, device=dev)
    out = torch.zeros(2 * 8 * 9 * 3, dtype=torch.uint8, device=dev)
    ws = torch.empty(64, dtype=torch.int32, device=dev)
    base = dict(src=src, postproc=3, encode="normals_bgr", crops=[(0, 0, 8, 9)] * 2, offsets=[0, 216], out=out)
    ops.render([base], ws)   # valid
    bad = [
        dict(base, encode="nope"),                                        # unknown encoding (ops)
        dict(base, src=src.cpu()),                                        # device
        dict(base, src=src.half()),                                       # dtype
        dict(base, src=src.transpose(2, 3)),                              # contiguity
        dict(base, offsets=[0]),                                          # one offset for two images
    ]
    for spec in bad:
        with pytest.raises((ValueError, RuntimeError)):
            ops.render([spec], ws)
    abi = [
        dict(base, crops=[(0, 0, 9, 9)] * 2),                             # crop outside the source
        dict(base, crops=[(1, 0, 8, 9)] * 2),
        dict(base, offsets=[0, 217]),                                     # past the end of out
        dict(base, postproc=2, encode="u8", src=src[:, :1].contiguous()),  # sal needs 2 channels
        dict(base, postproc=0, encode="palette_bgr", table=torch.zeros(2, 3, dtype=torch.uint8, device=dev)),
        dict(base, postproc=1, encode="normals_bgr"),                     # a scalar map is not normals
        dict(base, postproc=4, encode="jet"),                             # JET without its table
    ]
    for spec in abi:
        with pytest.raises(RuntimeError, match="mtt_render"):
            ops.render([spec], ws)
    # the raw ABI: unknown kinds and null arguments
    L = lib.load()
    d = (lib.RenderDesc * 1)()
    crop = (C.c_int32 * 4)(0, 0, 8, 9)
    off = (C.c_int64 * 1)(0)
    d[0].src_kind, d[0].src, d[0].B, d[0].C, d[0].h, d[0].w = 7, src.data_ptr(), 1, 3, 8, 9
    d[0].out_h, d[0].out_w, d[0].postproc, d[0].encode = 8, 9, 3, lib.RENDER_NORMALS_BGR
    d[0].crop, d[0].offset, d[0].out, d[0].out_bytes = crop, off, out.data_ptr(), out.numel()
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    assert L.mtt_render(d, 1, C.c_void_p(ws.data_ptr()), s) != 0
    d[0].src_kind, d[0].encode = lib.RENDER_SRC_LOGITS, 9
    assert L.mtt_render(d, 1, C.c_void_p(ws.data_ptr()), s) != 0
    d[0].encode = lib.RENDER_NORMALS_BGR
    assert L.mtt_render(d, 1, None, s) != 0
    assert L.mtt_render(d, 0, C.c_void_p(ws.data_ptr()), s) != 0
    assert L.mtt_render(d, 1, C.c_void_p(ws.data_ptr()), s) == 0
    torch.cuda.synchronize()


def _tiny(kind, dev):
    from oracle import configs
    if kind == "tp":
        from mtt_b200 import taskprompter as M
        from oracle import taskprompter_ref as Ref
        cfg = configs.taskprompter("tp_tiny")
    else:
        from mtt_b200 import invpt as M
        from oracle import invpt_ref as Ref
        cfg = configs.invpt("ip_tiny")
    cfg = dict(cfg, tasks=list(cfg["tasks"]) + ["edge"], num_output=dict(cfg["num_output"], edge=1))
    model = M.build_from_config(cfg, nsplit=M.PARITY).eval()
    model.load_state_dict(Ref.init_state_dict(cfg, seed=4), strict=True)
    return cfg, model.to(dev)


@pytest.mark.parametrize("kind,reference", [("tp", "TaskPrompter"), ("ip", "InvPT")])
def test_end_to_end_predict_to_files(cuda_dev, tmp_path, kind, reference):
    from mtt_b200 import export as E
    from oracle import export_ref as R
    cfg, model = _tiny(kind, cuda_dev)
    H, W = cfg["img_size"]
    B = 3
    x = torch.randn(B, 3, H, W, generator=torch.Generator().manual_seed(9))
    with torch.no_grad():
        pred = {t: v.clone() for t, v in model.predict(x.to(cuda_dev)).items()}
    meta = {"img_name": [f"e{i}" for i in range(B)], "img_size": [[H - 3, W - 5], [H, W], [H - 10, W - 1]]}
    lab = torch.zeros(B, 1, H, W)
    lab[1] = 255
    p = _p("NYUD")
    dirs = {"edge": str(tmp_path / "edge"), "semseg": str(tmp_path / "semseg")}
    with E.PredictionWriter(p, ["edge", "semseg"], dirs, reference) as w:
        w.update(pred, {"edge": lab.to(cuda_dev), "semseg": lab.to(cuda_dev)}, meta)
    for t in ("edge", "semseg"):
        files = R.save_preds(p, {"meta": meta, t: lab}, {t: pred[t].cpu()}, t, reference, predicted=True)
        assert len(files) == B - 1
        assert sorted(os.listdir(dirs[t])) == sorted(files)
        for f, a in files.items():
            assert np.array_equal(cv2.imread(os.path.join(dirs[t], f), cv2.IMREAD_UNCHANGED), a), (t, f)
