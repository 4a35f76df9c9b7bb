"""-m gpu: the three-task Swin TaskPrompter (semseg, depth, 3ddet) on the device, through the CUDA-graph replay, against
the fixtures of the UNMODIFIED reference (oracle/make_golden_swin3d.py; 3ddet head = nn.Identity, so the 3ddet output is
the 4 level maps the detection head receives):

  * tps_tiny3d element by element, tps_mid3d (window 12, 0.75 scaling) on its lattice and its full 3ddet maps;
  * tps_swinB3d (cs_swinB_taskprompter.yml) at full size, 1024 x 2048, bs 1: every 2D output and every 3ddet map with the
    tolerances of test_swin_big_gpu.py (rel-L2 on the lattice < 2e-4, max-abs < 1e-3 max|ref|, full-tensor norm within
    1e-4, semseg arg-max equal at every pixel away from near ties), TaskPrompterSwin.forward and predict();
  * the gating and fea_fuse kernels at the 3ddet geometries (T = 3, f = 450 on 96x192 ... 24x48) against float64;
  * re-packing after an in-place parameter update."""
import lzma
import math
import os

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import configs
from test_swin3d import DET, GOLD, fixture, inputs, model

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]


def _check(got, ref, what, rel_l2=2e-4, max_rel=1e-3):
    g, r = got.float().cpu(), ref.float()
    assert g.shape == r.shape and torch.isfinite(g).all(), what
    e2, em = ((g - r).norm() / r.norm()).item(), ((g - r).abs().max() / r.abs().max()).item()
    assert e2 < rel_l2 and em < max_rel, (what, e2, em)


def test_tiny3d_golden_graph_replay(cuda_dev):
    from test_taskprompter_gpu import _check as check2d

    fx = fixture("tps_tiny3d")
    cfg, sd, x = inputs("tps_tiny3d")
    m = model(cfg, sd, graph=True).to(cuda_dev)
    with torch.no_grad():
        m(x.to(cuda_dev))
        got = m(x.to(cuda_dev))                  # graph replay
        torch.cuda.synchronize()
        check2d(got, fx["out"], ["semseg", "depth"], 2e-4, 1e-3)
        for il, (g, r) in enumerate(zip(got[DET], fx["out"][DET])):
            _check(g, r, ("3ddet", il))


def test_mid3d_golden_graph_replay(cuda_dev):
    from test_big_goldens_gpu import compare

    fx = fixture("tps_mid3d")
    cfg, sd, x = inputs("tps_mid3d")
    m = model(cfg, sd, graph=True).to(cuda_dev)
    with torch.no_grad():
        m(x.to(cuda_dev))
        got = m(x.to(cuda_dev))
        torch.cuda.synchronize()
        for ti, t in enumerate(("semseg", "depth")):
            compare(got[t], fx["out"][t], ti, fx["stride"])
        for il, (g, r) in enumerate(zip(got[DET], fx["out"][DET])):
            _check(g, r, ("3ddet", il))


@pytest.fixture(scope="module")
def swinB3d(cuda_dev):
    from test_big_goldens_gpu import _input

    with lzma.open(os.path.join(GOLD, "big_tps_swinB3d_b1.pt.xz"), "rb") as f:
        fx = torch.load(f, weights_only=False)
    cfg, sd, _ = inputs(fx["cfg"])
    x = _input(fx, cfg)                          # the same seeded input, its checksum checked
    m = model(cfg, sd, graph=True).to(cuda_dev)
    yield fx, cfg, m, x.to(cuda_dev)
    del m
    torch.cuda.empty_cache()


def _metrics(got, rec, ti, stride):
    """test_big_goldens_gpu.compare's measurements of one output against its lattice-sampled record, without asserting."""
    g = got.float()
    assert tuple(g.shape) == tuple(rec["shape"]) and bool(torch.isfinite(g).all())
    from test_big_goldens_gpu import lattice
    samp = []
    for b in range(g.shape[0]):
        iy, ix = lattice(b, ti, g.shape[2], g.shape[3], stride)
        samp.append(g[b][:, iy.to(g.device)][:, :, ix.to(g.device)])
    samp, ref = torch.stack(samp).cpu(), rec["samples"]
    m = {"rel_l2_lattice": ((samp - ref).norm() / ref.norm()).item(),
         "max_abs_over_max": ((samp - ref).abs().max() / rec["absmax"]).item(),
         "norm_ratio_full": g.double().norm().item() / rec["norm"]}
    if "argmax" in rec:
        agree = g.argmax(1).cpu() == rec["argmax"].long()
        safe = torch.from_numpy(np.unpackbits(rec["safe_bits"].numpy())[:agree.numel()].astype(bool)).reshape(agree.shape)
        m["argmax_mismatch_safe_pixels"] = int((~agree & safe).sum())
        m["argmax_agreement_all_pixels"] = agree.float().mean().item()
    return m


def _assert_metrics(metrics):
    """rel-L2 < 2e-4 and max-abs < 1e-3 max|ref| on the lattice; the full-tensor norm within 2e-4 (what the rel-L2 bound
    implies over the full tensor: | |g| / |r| - 1 | <= |g - r| / |r|); arg-max equal at every safe pixel, > 0.999 overall."""
    for k, m in metrics.items():
        assert m["rel_l2_lattice"] < 2e-4 and m["max_abs_over_max"] < 1e-3, (k, metrics)
        assert abs(m["norm_ratio_full"] - 1) < 2e-4, (k, metrics)
        if "argmax_mismatch_safe_pixels" in m:
            assert m["argmax_mismatch_safe_pixels"] == 0 and m["argmax_agreement_all_pixels"] > 0.999, (k, metrics)


def _det_metrics(maps, fx):
    return {f"3ddet.{il}": _metrics(g, r, 2 + il, s)
            for il, (g, r, s) in enumerate(zip(maps, fx["out"][DET], fx["det_strides"]))}


def test_swinB3d_big_golden_graph_replay(swinB3d):
    from test_big_goldens_gpu import record

    fx, cfg, m, x = swinB3d
    with torch.no_grad():
        m(x)
        got = m(x)
        torch.cuda.synchronize()
    metrics = {t: _metrics(got[t], fx["out"][t], ti, fx["stride"]) for ti, t in enumerate(("semseg", "depth"))}
    metrics.update(_det_metrics(got[DET], fx))
    record("big_tps_swinB3d_b1", {"config": fx["cfg"], "batch": fx["batch"], "mode": "parity (bf16x3), CUDA-graph replay",
                                  "reference": fx["made_by"], "tasks": metrics})
    print(metrics)
    _assert_metrics(metrics)


def test_swinB3d_backbone_forward(swinB3d):
    """TaskPrompterSwin.forward (the "backbone" plan): the 3ddet maps against the fixture, and the 2D features through
    the model's own heads and the wrapper's resize reproduce the fixture's logits."""
    fx, cfg, m, x = swinB3d
    with torch.no_grad():
        fea, info = m.backbone(x)
        assert info == {}
        metrics = _det_metrics(fea[DET], fx)
        for ti, t in enumerate(("semseg", "depth")):
            y = F.interpolate(m.heads[t](fea[t]), tuple(cfg["dd_label_map_size"]), mode="bilinear")
            metrics[t] = _metrics(y, fx["out"][t], ti, fx["stride"])
    torch.cuda.synchronize()
    print(metrics)
    _assert_metrics(metrics)


def test_swinB3d_predict(swinB3d):
    from test_big_goldens_gpu import lattice

    fx, cfg, m, x = swinB3d
    with torch.no_grad():
        m.predict(x)
        got = m.predict(x)
        torch.cuda.synchronize()
    _assert_metrics(_det_metrics(got[DET], fx))               # the head's raw output: here nn.Identity's
    rec = fx["out"]["semseg"]
    B, n, H, W = rec["shape"]
    lab = got["semseg"].cpu()
    assert lab.dtype == torch.int64 and tuple(lab.shape) == (B, H, W)
    agree = lab == rec["argmax"].long()
    safe = torch.from_numpy(np.unpackbits(rec["safe_bits"].numpy())[:agree.numel()].astype(bool)).reshape(agree.shape)
    assert int((~agree & safe).sum()) == 0 and agree.float().mean().item() > 0.999
    rec, dep = fx["out"]["depth"], got["depth"]
    assert tuple(dep.shape) == (B, H, W, 1)
    iy, ix = lattice(0, 1, H, W, fx["stride"])
    samp = dep[0, :, :, 0][iy.to(dep.device)][:, ix.to(dep.device)].cpu()
    ref = rec["samples"][0, 0].clamp_min(0)                   # get_output's depth clamp (may leave all zeros)
    assert ((samp - ref).abs().max() / rec["absmax"]).item() < 1e-3
    if ref.norm() > 0:
        assert ((samp - ref).norm() / ref.norm()).item() < 2e-4


def test_repacks_after_an_in_place_update(cuda_dev):
    """The plan follows in-place parameter updates of the backbone's 3ddet branch and of a 2D head (one re-pack, one
    re-capture); the stand-in detection head's own parameter is applied by PyTorch on every call."""
    from test_swin3d import Recorder

    cfg, sd, x = inputs("tps_tiny3d")
    m = model(cfg, sd, det_head=Recorder(), graph=True).to(cuda_dev)
    x = x.to(cuda_dev)
    with torch.no_grad():
        a = m(x)
        a = {"semseg": a["semseg"].clone(), DET: [v.clone() for v in a[DET]["maps"]]}
        m.backbone.fea_fuse[2][DET][4].bias.add_(1.0)
        m.heads["semseg"].linear_pred.bias.add_(1.0)
        m.heads[DET].scale.mul_(2.0)
        b = m(x)
        torch.cuda.synchronize()
    assert torch.allclose(b["semseg"], a["semseg"] + 1.0, atol=1e-4)
    for il in range(4):
        want = 2.0 * (a[DET][il] + 1.5 * (il == 2))          # + 1 on level 2's map, times the head's 1.5 -> 3.0 doubled
        assert torch.allclose(b[DET]["maps"][il], want, atol=1e-4, rtol=1e-5), il


# ---- the gating and fea_fuse kernels at the 3ddet geometries against float64 ---------------------------------------------------
def _levels():
    cfg = configs.taskprompter_swin("tps_swinB3d")
    E, heads = cfg["embed_dim"], cfg["heads"]
    from oracle.taskprompter_swin_ref import level_resolution
    return cfg, [(level_resolution(cfg, il), [2 * E, 4 * E, 8 * E, 8 * E][il], heads[il]) for il in range(4)]


@pytest.mark.parametrize("ns", [2, 1])
def test_gate_split_at_the_3ddet_levels_f64(cuda_dev, ns):
    """Spatial and channel gating of all 3 tasks (3ddet included) at every level of tps_swinB3d, the patch rows of the
    Swin level map (groups of P rows, no prompt rows), against float64 (2u per gated value + the split bound)."""
    import mtt_b200  # noqa: F401
    from mtt_b200 import ops
    from f64_checks import Guarded, U, check_planes, gen, randn, round_up
    from kernel_cases import ref_gates

    cfg, levels = _levels()
    T, B = len(cfg["tasks"]), 1
    for il, ((gh, gw), C, H) in enumerate(levels):
        P, rows, ldy = gh * gw, B * gh * gw, round_up(C, 8)
        N = T + P
        g = gen(60 + il)
        x = randn(g, B * P, C)
        logits = randn(g, B, H, T, N, scale=1.5)
        rc = randn(g, B, T, C, 1, 1, scale=1.5)
        pbe = round_up(ns * rows * ldy * 2, 256) // 2
        gb = Guarded((2 * T + 1, pbe), torch.bfloat16)
        flat = gb.view.reshape(-1)
        ys = ops.Split.from_planes(flat[:ns * rows * ldy].view(ns, rows, ldy), C)
        yc = ops.Split.from_planes(flat[pbe:pbe + ns * rows * ldy].view(ns, rows, ldy), C)
        gb.snapshot()
        ops.gate_split(x, P, 0, logits, rc, 0, ys, yc, B=B, T=T, N=N, H=H, Cdim=C, gh=gh, gw=gw, nh=1, nw=1,
                       ntasks=T, task_stride=2 * pbe)
        gb.unchanged_outside((slice(0, 2 * T), slice(0, ns * rows * ldy)), "gate_split")
        X = x.double().view(B, P, C)
        for t in range(T):
            gs, gc = ref_gates(logits.double(), rc.double(), B, T, H, C, gh, gw, 1, 1, t)
            for which, gate in ((0, gs), (1, gc)):
                want = (X * (1 + gate)).reshape(rows, C)
                e = 2 * U * (X.abs() * (1 + gate).abs()).reshape(rows, C)
                sp = ops.Split.from_planes(gb.view[2 * t + which, :ns * rows * ldy].view(ns, rows, ldy), C)
                check_planes(sp, want, e, f"gate_split level {il} task {t} {'Yc' if which else 'Ys'}")


@pytest.mark.parametrize("il", range(4))
def test_fea_fuse_convs_at_the_3ddet_levels_f64(cuda_dev, il):
    """fea_fuse[1..3] (3x3 conv, BatchNorm folded, GELU, split output) and fea_fuse[4] (3x3 conv, fp32 output), 450 -> 450
    channels on the level's own map, as the 3ddet branch runs them, against float64 convolutions of the operands' split
    values. Bound per output: (2 SPLIT + 2 LAM sqrt(K) u) sum |a| |w| + 2u |y| (the weight's hi + lo representation, the
    dropped lo x lo products, the fp32 accumulation over K = 9 * 450), GELU's slope (< 1.13) on top for fea_fuse[1..3]."""
    import mtt_b200  # noqa: F401
    from mtt_b200 import ops
    from f64_checks import LAM, SPLIT, U, check, check_planes, decode, gen, randn

    cfg, levels = _levels()
    (h, w), _, _ = levels[il]
    f, B = cfg["f"], 1
    K = 9 * f
    g = gen(70 + il)
    x = randn(g, B * h * w, f)
    a = ops.Split(B * h * w, f, "cuda", 2, zero=True)
    ops.split_f32(x, 2, out=a)
    av = decode(a).view(B, h, w, f).permute(0, 3, 1, 2)
    wt = randn(g, f, f, 3, 3, scale=1 / math.sqrt(K))
    bias = randn(g, f, scale=0.1)
    bn = nn.BatchNorm2d(f).to("cuda").eval()
    with torch.no_grad():
        bn.weight.uniform_(0.5, 1.5)
        bn.bias.normal_(0, 0.1)
        bn.running_mean.normal_(0, 0.1)
        bn.running_var.uniform_(0.8, 1.2)
    scale = (bn.weight.detach().double() / torch.sqrt(bn.running_var.double() + bn.eps))
    wf = wt.double() * scale[:, None, None, None]
    bf = (bias.double() - bn.running_mean.double()) * scale + bn.bias.detach().double()
    conv = lambda v, ww, bb: F.conv2d(v, ww, bb, padding=1).permute(0, 2, 3, 1).reshape(-1, f)
    rate = 2 * SPLIT + 2 * LAM * math.sqrt(K) * U
    # fea_fuse[1..3]: folded conv + GELU, split output
    w1, b1 = ops.pack_conv_weight(wt.contiguous(), bias, bn, 2)
    mid = ops.Split(B * h * w, f, "cuda", 2, zero=True)
    ops.gemm(a, w1, N=f, K=f, bias=b1, act=ops.ACT_GELU, out_split=mid, conv=(B, h, w, 3, 1))
    pre = conv(av, wf, bf)
    e = rate * conv(av.abs(), wf.abs(), bf.abs()) + 2 * U * pre.abs() + 4 * U * abs(float(bf.abs().max()))
    y = F.gelu(pre)
    check_planes(mid, y, 1.13 * e + 4 * U * y.abs() + 2 * U * pre.abs(), f"fea_fuse[1..3] level {il} {h}x{w}")
    # fea_fuse[4]: plain conv, fp32 output
    w4, b4 = ops.pack_conv_weight(wt.contiguous(), bias, None, 2)
    out = torch.full((B * h * w, f + 6), float("nan"), device="cuda")
    ops.gemm(a, w4, N=f, K=f, bias=b4, out_f32=out[:, :f], conv=(B, h, w, 3, 1))
    torch.cuda.synchronize()
    want = conv(av, wt.double(), bias.double())
    e = rate * conv(av.abs(), wt.double().abs(), bias.double().abs()) + 2 * U * want.abs()
    check(out[:, :f], want, e, f"fea_fuse[4] level {il} {h}x{w}")
    assert torch.isnan(out[:, f:]).all(), "columns past N written"
