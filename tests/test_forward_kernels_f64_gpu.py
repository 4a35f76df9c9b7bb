"""-m gpu: the forward glue kernels (csrc/prompting.cu, csrc/invpt.cu, csrc/rowwise.cu) at the geometries the benched
forwards and predict() really run -- the TaskPrompter and InvPT runs of plan_calls.RUNS: tp_cfg4, tp_cfg2, tp_cfg5 and
ip_cfg3 at bench.DEFAULT_BATCH, the reference's own model configs (tp_nyud_vitL, tp_pascal_vitB, ip_nyud_vitL) and
tp_cfg4 / ip_cfg3 at the reference's validation batch 6, and the PASCAL ones at the ragged last validation batch 5 --
against float64 references written from each operation's definition (F.interpolate, F.conv2d(groups=C), F.avg_pool2d(ceil_mode=True),
F.layer_norm, softmax, the windowed sums, exact-erf GELU), element by element.

Error model: tests/f64_checks.py. Every assert names the bound it uses.

Bilinear source coordinates are computed in fp32. Every resize ratio these plans use is a power of two, so those
coordinates and weights are exact and float64 F.interpolate is a valid reference (kernel_cases.ref_bilinear refuses a
ratio whose fp32 coordinates are inexact).

Around every output the test fills a sentinel (padding columns up to ld, guard rows before and after, the other
tasks' slices of a joint buffer, a second plane where there is one plane); after the call it must be bit-identical.

The geometry table (TABLE) is derived from oracle/configs.py and each run's batch; test_plans_call_only_tabled_shapes
runs each plan's forward and predict() once and fails when a plan calls a glue kernel at a shape the table does not
hold."""
import math

import pytest
import torch
import torch.nn.functional as F

from f64_checks import (LAM, U, Guarded, assert_planes_bit_exact, check, check_planes, decode, gen, guarded_split,
                        ops, randn, report, round_up, split_bound, sum_tol)  # noqa: F401
from kernel_cases import (E_BIL, bilinear_case, gate_case, layernorm_case, ln_bound, ln_input, postproc_case,
                          ref_bilinear, ref_gates, ref_im2col, ref_layernorm, ref_postproc, rows_of)
from plan_calls import RUNS as ALL_RUNS, IPGeom, TPGeom, bil, frozen, glue_key, recording, run_id, runs

pytestmark = [pytest.mark.timeout(1200)]      # the GPU tests are marked one by one: the CPU self-checks are not
RUNS = runs(("forward", "predict"), ("tp_", "ip_"))        # (config, batch)


def assert_pow2_ratio(src, dst):
    """The fp32 bilinear coordinates are exact only for power-of-two resize ratios: refuse any other."""
    lo, hi = min(src, dst), max(src, dst)
    r = hi // lo
    assert hi % lo == 0 and r & (r - 1) == 0, f"resize {src} -> {dst} is not a power-of-two ratio: float64 " \
                                              f"F.interpolate is no reference for the kernel's fp32 coordinates"


# ---- geometry ----------------------------------------------------------------------------------------------------------
def _geom(name, B):
    return IPGeom(name, B) if name.startswith("ip_") else TPGeom(name, B)


def _tp_table(g):
    B, T, C = g.B, g.T, g.C
    t = dict(im2col_patch=[dict(shape=(B, 3) + g.img, patch=g.patch, ld=round_up(3 * g.patch ** 2, 8))],
             broadcast_rows=[dict(T=T, C=C, B=B, group_rows=g.N, ld=C)],
             layernorm=[dict(rows=B * g.N, cols=C, ld_in=C, f32=True, split=False)],
             chan_logits=[dict(B=B, N=g.N, T=T, C=C, gh=g.gh, gw=g.gw, nh=g.nh, nw=g.nw)],
             gate_split=[dict(B=B, T=T, N=g.N, H=g.H, C=C, gh=g.gh, gw=g.gw, nh=g.nh, nw=g.nw, x_group_rows=g.N,
                              x_row_offset=T, ldx=C, ntasks=T)],
             bilinear=[bil(g.f_ld, B, g.gh, g.gw, g.f, g.h4, g.w4, "split", ld_out=g.f_ld)],
             bilinear_postproc=[], nhwc_to_nchw=[])
    if g.use_ctr:
        t["ctr_weights"] = [dict(B=B, H=g.H, T=T, N=g.N)]
        t["ctr_mix"] = [dict(T=T, M=B * g.P, Cdim=g.f_ld, ld=g.f_ld, rows_per_batch=g.P, accumulate=a)
                        for a in (False, True)]
    from mtt_b200 import ops
    for task in g.tasks:
        n = g.n_out[task]
        if task == "3ddet":                                # wrapper :34-38: the 3ddet map is not resized
            t["nhwc_to_nchw"].append(dict(ld_in=round_up(n, 4), B=B, Cd=n, H=g.h4, W=g.w4))
            continue
        t["bilinear"].append(bil(round_up(n, 4), B, g.h4, g.w4, n, *g.out_hw, "nchw"))
        t["bilinear_postproc"].append(dict(ld_in=round_up(n, 4), B=B, h=g.h4, w=g.w4, C=n, H2=g.out_hw[0],
                                           W2=g.out_hw[1], kind=ops.POSTPROC_KIND[task]))
    return t


def _ip_table(g):
    from mtt_b200 import ops
    B, T, C = g.B, g.T, g.C
    d0 = g.dims[0]
    t = dict(im2col_patch=[dict(shape=(B, 3) + g.img, patch=g.patch, ld=round_up(3 * g.patch ** 2, 8))],
             broadcast_rows=[dict(T=1, C=C, B=B, group_rows=g.N, ld=C)],
             zero_insert=[dict(B=B, h=g.gh, w=g.gw, Cdim=C, src_group=g.N, src_offset=1, ld_in=C, ld_out=C)],
             split_rows=[dict(rows=B * g.P, cols=C, in_group=g.P, src_group=g.N, src_offset=1, ld_in=C, ld_out=C)],
             layernorm_seg=[dict(rows=B * g.P, cols=C, S=1, in_group=g.P, src_group=g.N, src_offset=1, seg_stride=0,
                                 out_seg_stride=0, ld_in=C, f32=True, split=False)],
             bilinear=[bil(C, B, g.gh, g.gw, C, g.h0, g.w0, "split", ld_out=C)],
             layernorm=[], dwconv3x3_s2=[], avgpool=[], invpt_fuse_softmax=[], bilinear_sum3=[], bilinear_postproc=[])
    for task in g.tasks:                                    # inter-pred resize (transformer_net.py:36)
        n = g.n_out[task]
        t["bilinear"].append(bil(round_up(n, 4), B, g.h0, g.w0, n, *g.img, "nchw"))
    for i, s in enumerate(g.stages):
        h, w, Ci, hw = s["h"], s["w"], s["C"], s["h"] * s["w"]
        if i > 0:                                           # UpEmbed x2 of each task's slice of the previous stage
            p = g.stages[i - 1]
            phw = p["h"] * p["w"]
            t["bilinear"] += [bil(p["C"], B, p["h"], p["w"], p["C"], h, w, "split", ld_out=round_up(p["C"], 8),
                                   ibr=T * phw, ioff=k * phw) for k in range(T)]
        t["layernorm"].append(dict(rows=B * T * hw, cols=Ci, ld_in=Ci, f32=True, split=False))
        t["dwconv3x3_s2"].append(dict(B=B, T=T, h=h, w=w, Cdim=Ci, ld_in=Ci, ld_out=round_up(Ci, 8)))
        t["avgpool"].append(dict(BT=B * T, h=h, w=w, Cdim=Ci, s=s["kvs"], ld_in=Ci, ld_out=round_up(Ci, 8)))
        t["invpt_fuse_softmax"].append(dict(B=B, Lq=s["Lq"], Tk=s["Tk"], fused=i > 0, T=T, qh=h // 2, qw=w // 2,
                                            score_out=i < 2, ldp=round_up(s["Tk"], 8)))
        qhw = (h // 2) * (w // 2)                           # attention output x2 accumulated into each task's slice
        t["bilinear"] += [bil(Ci, B, h // 2, w // 2, Ci, h, w, "f32", ld_out=Ci, acc=True, ibr=T * qhw, ioff=k * qhw,
                               obr=T * hw, ooff=k * hw) for k in range(T)]
        t["layernorm_seg"].append(dict(rows=B * hw, cols=Ci, S=T, in_group=hw, src_group=T * hw, src_offset=0,
                                       seg_stride=hw, out_seg_stride=B * hw, ld_in=Ci, f32=i == 0, split=i > 0))
    s0, s1 = g.stages[0], g.stages[1]
    t["bilinear_sum3"] = [dict(B=B, Cdim=d0, H2=g.th, W2=g.tw,
                               srcs=((s0["h"], s0["w"], 0, k * B * s0["h"] * s0["w"], d0), (s1["h"], s1["w"], 0, 0, d0),
                                     (g.stages[2]["h"], g.stages[2]["w"], 0, 0, d0))) for k in range(T)]
    for task in g.tasks:
        n = g.n_out[task]
        t["bilinear"].append(bil(round_up(n, 4), B, g.th, g.tw, n, *g.img, "nchw"))
        t["bilinear_postproc"].append(dict(ld_in=round_up(n, 4), B=B, h=g.th, w=g.tw, C=n, H2=g.img[0], W2=g.img[1],
                                           kind=ops.POSTPROC_KIND[task]))
    return t


_TABLES = {}


def table(name, B):
    if (name, B) not in _TABLES:
        import mtt_b200  # noqa: F401
        g = _geom(name, B)
        _TABLES[(name, B)] = (g, _ip_table(g) if name.startswith("ip_") else _tp_table(g))
    return _TABLES[(name, B)]


def _runs_calling(fn):
    """(config, batch) parameters of the runs that call `fn`."""
    return [pytest.param(name, B, id=run_id(name, B)) for name, B in RUNS if table(name, B)[1].get(fn)]


def _cases(fn):
    """(config, batch, nsplit) parameters of the runs that call `fn` (a kernel that writes split planes)."""
    return [pytest.param(name, B, ns, id=f"{run_id(name, B)}-ns{ns}") for name, B in RUNS if table(name, B)[1].get(fn)
            for ns in (2, 1)]


RECORDED = ["im2col_patch", "broadcast_rows", "layernorm", "chan_logits", "gated_conv1x1", "ctr_weights", "ctr_mix",
            "bilinear", "bilinear_postproc", "nhwc_to_nchw", "zero_insert", "split_rows", "layernorm_seg",
            "dwconv3x3_s2", "avgpool", "invpt_fuse_softmax", "bilinear_sum3"]


@pytest.mark.gpu
def test_plans_call_only_tabled_shapes(cuda_dev):
    """Each plan at each run's batch runs one forward and, where the run list has it, one predict() (evaluation reaches
    bilinear_postproc only through predict()) with pass-through recorders around the ops glue functions: every
    (function, shape arguments) pair it calls must be in TABLE, so a plan that starts calling a kernel at a new shape
    fails here instead of leaving the table (and the kernel tests built from it) stale."""
    import bench
    from mtt_b200 import ops

    for name, B in RUNS:
        g, tab = table(name, B)
        cfg, M, _ = bench.family(name)
        torch.manual_seed(0)
        with torch.device(cuda_dev):
            model = M.build_from_config(cfg, nsplit=2, use_graph=False).eval()
        x = torch.randn(g.B, 3, *cfg["img_size"], device=cuda_dev)
        want = {(fn, frozen(d)) for fn, ds in tab.items() for d in ds}
        for mode in [m for n, b, m in ALL_RUNS if (n, b) == (name, B)]:
            with recording(ops, RECORDED, glue_key, []) as seen:
                with torch.no_grad():
                    model(x) if mode == "forward" else model.predict(x)
            torch.cuda.synchronize()
            got = {(fn, frozen(d)) for fn, d in seen}
            assert got, f"{name} b{B} {mode}: no glue call recorded"
            missing = sorted(got - want, key=str)
            assert not missing, f"{name} b{B} {mode}: the plan calls glue kernels at shapes the table does not " \
                                f"hold: {missing[:6]}"
            if mode == "predict":
                assert "bilinear_postproc" in {fn for fn, _ in got}, f"{name} b{B}: predict() made no fused " \
                                                                      f"post-processing"
            print(f"{name} b{B} {mode}: {len(got)} distinct glue calls, all in the table ({len(want)} tabled)")
        del model, x
        torch.cuda.empty_cache()


# ---- float64 references (device-agnostic: the CPU self-check runs them too) -----------------------------------------------
def ref_chan_logits(cp, x, B, T, C, gh, gw, nh, nw):
    """Rc[b,t,c,i,j] = sum over window (i, j) of cp[b,t,pix] x[b,pix,c]; x = the patch rows [B, P, C]."""
    wh, ww = gh // nh, gw // nw
    return torch.einsum("btihjw,bihjwc->btcij", cp.reshape(B, T, nh, wh, nw, ww), x.reshape(B, nh, wh, nw, ww, C))


def ref_ctr_hidden(logits, w0, b0, T):
    """hsum[b,t,o,j] = W0_t[o] . R[b,:,t,j] + b0_t[o] (the pre-GELU hidden of ctr_attn_conv)."""
    a = logits[:, :, :, :T]                                             # [B,H,T(task),T(j)]
    return torch.einsum("toh,bhtj->btoj", w0, a) + b0[None, :, :, None]


def ref_ctr_weights(logits, w0, b0, w2, b2, T):
    return torch.einsum("to,btoj->btj", w2, F.gelu(ref_ctr_hidden(logits, w0, b0, T))) + b2[None, :, None]


def ref_ctr_mix(Fm, wts, rows_per_batch):
    b = torch.arange(Fm.shape[1], device=Fm.device) // rows_per_batch
    return torch.einsum("mtj,jmc->tmc", wts[b], Fm)


def ref_dwconv(x, wgt, bias, B, T, h, w, C):
    """Per-task depthwise 3x3 stride-2 conv, padding 1: x [B*T*h*w, C] -> [B*T*(h/2)*(w/2), C] (and the same of |.|)."""
    xm = x[:, :C].reshape(B, T, h, w, C).permute(0, 1, 4, 2, 3)
    ys, ya = [], []
    for k in range(T):
        ys.append(F.conv2d(xm[:, k], wgt[k].reshape(C, 1, 3, 3), bias[k], stride=2, padding=1, groups=C))
        ya.append(F.conv2d(xm[:, k].abs(), wgt[k].abs().reshape(C, 1, 3, 3), bias[k].abs(), stride=2, padding=1, groups=C))
    f = lambda v: torch.stack(v, 1).permute(0, 1, 3, 4, 2).reshape(-1, C)
    return f(ys), f(ya)


def ref_avgpool(x, BT, h, w, C, s):
    xm = x[:, :C].reshape(BT, h, w, C).permute(0, 3, 1, 2)
    f = lambda v: F.avg_pool2d(v, s, s, 0, ceil_mode=True).permute(0, 2, 3, 1).reshape(-1, C)
    return f(xm), f(xm.abs())


def ref_fuse(raw, scale, prev, wf, bf, B, T, qh, qw):
    """InvPT's fused pre-softmax score (invpt.py:204-232): raw * scale, and with a previous stage's score the 1x1 fuse
    conv over [scale raw; bilinear x2 of prev]; (f, |.|-bound companion, up-sampled prev)."""
    s = raw * scale
    if prev is None:
        return s, s.abs(), None, None
    Tk = raw.shape[-1]
    sh, sw = qh // 2, qw // 2
    ups, upa = [], []
    for i in range(T):
        p = prev[:, :, sh * sw * i:sh * sw * (i + 1), :].permute(0, 1, 3, 2).reshape(B * 2, Tk, sh, sw)
        for v, lst in ((p, ups), (p.abs(), upa)):
            lst.append(F.interpolate(v, scale_factor=2, mode="bilinear", align_corners=False)
                       .reshape(B, 2, Tk, -1).permute(0, 1, 3, 2))
    up, upa = torch.cat(ups, dim=2), torch.cat(upa, dim=2)
    f = F.conv2d(torch.cat([s, up], dim=1), wf.reshape(2, 4, 1, 1), bf)
    fa = F.conv2d(torch.cat([s.abs(), upa], dim=1), wf.abs().reshape(2, 4, 1, 1), bf.abs())
    return f, fa, up, upa


# ---- data movement: bit-exact ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,B,ns", _cases("im2col_patch"))
@pytest.mark.gpu
def test_im2col_patch(ops, name, B, ns):
    """Patch im2col of the whole input batch: planes bit-exact against the split of F.unfold (column order c, ky, kx)."""
    g, tab = table(name, B)
    for d in tab["im2col_patch"]:
        img = randn(gen(1), *d["shape"])
        rows = d["shape"][0] * g.P
        gb, sp, reg = guarded_split(ops, ns, rows, d["ld"], ld=d["ld"])
        gb.snapshot()
        ops.im2col_patch(img, d["patch"], sp)
        gb.unchanged_outside(reg, "im2col_patch")
        assert_planes_bit_exact(sp, ref_im2col(img, d["patch"]), "im2col_patch")


@pytest.mark.parametrize("name,B", _runs_calling("broadcast_rows"))
@pytest.mark.gpu
def test_broadcast_rows_and_nhwc_to_nchw(ops, name, B):
    """Prompt / cls rows broadcast into every image's group of the joint stream (the patch rows stay as they were), and
    the 3ddet map's NHWC -> NCHW copy: bit-exact."""
    g, tab = table(name, B)
    for d in tab["broadcast_rows"]:
        src = randn(gen(2), d["T"], d["C"])
        gb = Guarded((d["B"] * d["group_rows"], d["ld"]), torch.float32)
        gb.view[:] = randn(gen(3), d["B"] * d["group_rows"], d["ld"])
        gb.snapshot()
        ops.broadcast_rows(src, gb.view, d["B"], d["group_rows"])
        rows = rows_of(d["B"], d["T"], d["group_rows"], 0, "cuda")
        gb.unchanged_outside((rows, slice(0, d["C"])), "broadcast_rows")
        assert torch.equal(gb.view[rows, :d["C"]], src.repeat(d["B"], 1)), "broadcast_rows"
    for d in tab.get("nhwc_to_nchw", []):
        x = randn(gen(4), d["B"] * d["H"] * d["W"], d["ld_in"])
        gb = Guarded((d["B"], d["Cd"], d["H"], d["W"]), torch.float32)
        gb.snapshot()
        ops.nhwc_to_nchw(x, d["ld_in"], d["B"], d["Cd"], d["H"], d["W"], gb.view)
        gb.unchanged_outside((slice(None),), "nhwc_to_nchw")
        assert torch.equal(gb.view, x[:, :d["Cd"]].reshape(d["B"], d["H"], d["W"], d["Cd"]).permute(0, 3, 1, 2))


@pytest.mark.parametrize("name,B,ns", _cases("zero_insert"))
@pytest.mark.gpu
def test_zero_insert_and_split_rows(ops, name, B, ns):
    """InvPT's scale_embed inputs from the patch rows of the joint stream (row 0 of each image is the cls token):
    zero insertion for the transposed conv and the plain row gather, planes bit-exact."""
    g, tab = table(name, B)
    for d in tab["zero_insert"]:
        B, h, w, C = d["B"], d["h"], d["w"], d["Cdim"]
        x = randn(gen(5), B * d["src_group"], d["ld_in"])
        gb, sp, reg = guarded_split(ops, ns, B * 4 * h * w, C, ld=d["ld_out"])
        gb.snapshot()
        ops.zero_insert(x, sp, B=B, h=h, w=w, Cdim=C, src_group=d["src_group"], src_offset=d["src_offset"])
        gb.unchanged_outside(reg, "zero_insert")
        src = x[rows_of(B, h * w, d["src_group"], d["src_offset"], "cuda"), :C].reshape(B, h, w, C)
        z = torch.zeros(B, 2 * h, 2 * w, C, device="cuda")
        z[:, ::2, ::2] = src
        assert_planes_bit_exact(sp, z.reshape(-1, C), "zero_insert")
    for d in tab["split_rows"]:
        x = randn(gen(6), d["rows"] // d["in_group"] * d["src_group"], d["ld_in"])
        gb, sp, reg = guarded_split(ops, ns, d["rows"], d["cols"], ld=d["ld_out"])
        gb.snapshot()
        ops.split_rows(x, sp, rows=d["rows"], cols=d["cols"], in_group=d["in_group"], src_group=d["src_group"],
                       src_offset=d["src_offset"])
        gb.unchanged_outside(reg, "split_rows")
        r = rows_of(d["rows"] // d["in_group"], d["in_group"], d["src_group"], d["src_offset"], "cuda")
        assert_planes_bit_exact(sp, x[r, :d["cols"]], "split_rows")


# ---- LayerNorm ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,B", _runs_calling("layernorm"))
@pytest.mark.gpu
def test_layernorm(ops, name, B):
    """mtt_layernorm at the plans' rows x widths: TaskPrompter's final norm (C = 1024 / 768: the register path) and
    InvPT's per-stage norm1 (C = 576 / 288 / 144, up to 81920 rows: the general path), fp32 out with ld = C."""
    g, tab = table(name, B)
    report(f"layernorm {name} b{B}", [layernorm_case(ops, d, 10 + i) for i, d in enumerate(tab["layernorm"])])


@pytest.mark.parametrize("name,B,ns", _cases("layernorm_seg"))
@pytest.mark.gpu
def test_layernorm_seg(ops, name, B, ns):
    """ViT final norm over the gathered patch rows (S = 1) and InvPT's joint-channel norm over all T tasks' slices
    (S = T segments, statistics over T * C values) with the per-task output rows; fp32 or split out as the plan has it."""
    g, tab = table(name, B)
    ratios = []
    for i, d in enumerate(tab["layernorm_seg"]):
        rows, cols, S = d["rows"], d["cols"], d["S"]
        if not d["split"] and ns == 1:
            continue
        gg = gen(20 + i)
        nphys = rows // d["in_group"] * d["src_group"]
        x = torch.zeros(nphys, d["ld_in"], device="cuda")
        base = rows_of(rows // d["in_group"], d["in_group"], d["src_group"], d["src_offset"], "cuda")
        segs = torch.stack([base + k * d["seg_stride"] for k in range(S)], 1)        # [rows, S] physical rows
        x[segs.reshape(-1), :cols] = ln_input(gg, rows, S * cols).reshape(rows * S, cols)
        gam, bet = torch.rand(S * cols, generator=gg, device="cuda") + 0.5, randn(gg, S * cols, scale=0.5)
        eps = 1e-6
        orows = (torch.arange(S, device="cuda")[None] * d["out_seg_stride"] + torch.arange(rows, device="cuda")[:, None])
        n_out = S * rows if d["out_seg_stride"] else rows
        xd = x.double()[segs.reshape(-1), :cols].reshape(rows, S * cols)
        want, e = ln_bound(xd, gam.double(), bet.double(), eps, S * math.ceil(cols / 32) + 5)
        want, e = want.reshape(rows * S, cols), e.reshape(rows * S, cols)
        o = orows.reshape(-1)
        if d["f32"]:
            gb = Guarded((n_out, cols), torch.float32)
            gb.snapshot()
            ops.layernorm_seg(x, gam, bet, eps, rows=rows, cols=cols, S=S, in_group=d["in_group"],
                              src_group=d["src_group"], src_offset=d["src_offset"], seg_stride=d["seg_stride"],
                              out_f32=gb.view, out_seg_stride=d["out_seg_stride"])
            gb.unchanged_outside((slice(None),), "layernorm_seg")
            ratios.append(check(gb.view[o], want, e, f"layernorm_seg S={S} {rows}x{cols} fp32 (LN bound)"))
        else:
            gb, sp, reg = guarded_split(ops, ns, n_out, cols)
            gb.snapshot()
            ops.layernorm_seg(x, gam, bet, eps, rows=rows, cols=cols, S=S, in_group=d["in_group"],
                              src_group=d["src_group"], src_offset=d["src_offset"], seg_stride=d["seg_stride"],
                              out_split=sp, out_seg_stride=d["out_seg_stride"])
            gb.unchanged_outside(reg, "layernorm_seg")
            v = decode(sp)[o]
            ratios.append(check(v, want, e + split_bound(ns, want.abs() + e),
                                f"layernorm_seg S={S} {rows}x{cols} split ns={ns} (LN bound + split bound)"))
    if ratios:
        report(f"layernorm_seg {name} b{B} ns={ns}", ratios)


# ---- channel-prompt logits, gating, cross-task reweighting ---------------------------------------------------------------------
@pytest.mark.parametrize("name,B,ns", _cases("chan_logits"))
@pytest.mark.gpu
def test_chan_logits(ops, name, B, ns):
    """Rc[b,t,c,window] = sum over the window's pixels of cp[b,t,pix] xn[b,T+pix,c], xn as LN1's split planes (one or
    two): 1 window of 32 x 32 (tp_cfg4), 4 x 4 windows of 7 x 9 (tp_cfg2), one 64 x 128 window whose cp slice needs
    ~111 KB of dynamic shared memory (tp_cfg5)."""
    g, tab = table(name, B)
    for d in tab["chan_logits"]:
        B, N, T, C, gh, gw, nh, nw = (d[k] for k in ("B", "N", "T", "C", "gh", "gw", "nh", "nw"))
        P = gh * gw
        gg = gen(30)
        xs = randn(gg, B * N, C)
        xn = ops.Split(B * N, C, "cuda", ns)
        ops.split_f32(xs, ns, out=xn)
        cp = randn(gg, B * T, P)
        gb = Guarded((B, T, C, nh, nw), torch.float32)
        gb.snapshot()
        ops.chan_logits(cp, xn, gb.view, B=B, N=N, T=T, Cdim=C, gh=gh, gw=gw, nh=nh, nw=nw)
        gb.unchanged_outside((slice(None),), "chan_logits")
        X = decode(xn).view(B, N, C)[:, T:]
        cpd = cp.double()
        want = ref_chan_logits(cpd, X, B, T, C, gh, gw, nh, nw)
        absum = ref_chan_logits(cpd.abs(), X.abs(), B, T, C, gh, gw, nh, nw)
        wp = (gh // nh) * (gw // nw)
        D = math.ceil(wp / 32) + 32                # serial fma over the block's pixel group, then 32 partials in order
        r = check(gb.view, want, sum_tol(D, absum), f"chan_logits {name} (sum_tol D={D})")
        report(f"chan_logits {name} b{B} ns={ns}", [r])


@pytest.mark.parametrize("name,B,ns", _cases("gate_split"))
@pytest.mark.gpu
def test_gate_split(ops, name, B, ns):
    """Spatial and channel gating of all T tasks in one launch, X = the patch rows of the joint stream (x rows offset by
    T inside groups of N), written task after task into the gated-conv workspace layout (task_stride); the slack of
    each 256-byte aligned plane set and the space after the last task stay untouched."""
    g, tab = table(name, B)
    for d in tab["gate_split"]:
        report(f"gate_split {name} b{B} ns={ns}", gate_case(ops, d, ns, f"{name} b{B}"))


@pytest.mark.parametrize("name,B", _runs_calling("ctr_mix"))
@pytest.mark.gpu
def test_ctr_weights_and_mix(ops, name, B):
    """Cross-task reweighting: w[b,t,j] = W2_t . gelu(W0_t R[b,:,t,j] + b0_t) + b2_t over H heads, then
    acc[t] (+)= sum_j w[b,t,j] F[j] over all ld columns (the header: C = ld, the padding columns carry 0 + 0 and are
    checked like the rest), accumulate off then on."""
    g, tab = table(name, B)
    d = tab["ctr_weights"][0]
    B, H, T, N = d["B"], d["H"], d["T"], d["N"]
    gg = gen(50)
    logits = randn(gg, B, H, T, N, scale=4.0)
    w0, b0 = randn(gg, T, H, H, scale=0.3), randn(gg, T, H, scale=0.3)
    w2, b2 = randn(gg, T, H, scale=0.3), randn(gg, T, scale=0.3)
    gw = Guarded((B, T, T), torch.float32)
    gw.snapshot()
    ops.ctr_weights(logits, w0, b0, w2, b2, gw.view, B=B, H=H, T=T, N=N)
    gw.unchanged_outside((slice(None),), "ctr_weights")
    L, W0, B0, W2, B2 = (v.double() for v in (logits, w0, b0, w2, b2))
    hsum = ref_ctr_hidden(L, W0, B0, T)                                       # [B,T,H(o),T(j)]
    e_h = (H + 2) * U * (torch.einsum("toh,bhtj->btoj", W0.abs(), L[:, :, :, :T].abs()) + B0.abs()[None, :, :, None])
    e_g = 1.13 * e_h + 8 * U * hsum.abs()                                     # GELU's slope < 1.13; fp32 erf-GELU
    want_w = ref_ctr_weights(L, W0, B0, W2, B2, T)
    e_w = ((H + 2) * U * (torch.einsum("to,btoj->btj", W2.abs(), F.gelu(hsum).abs()) + B2.abs()[None, :, None])
           + torch.einsum("to,btoj->btj", W2.abs(), e_g))
    ratios = [check(gw.view, want_w, e_w, f"ctr_weights {name} ((H+2)u per H-term dot, GELU 8u)")]
    wts = gw.view.clone()
    for d in tab["ctr_mix"]:
        M, ld, rpb = d["M"], d["ld"], d["rows_per_batch"]
        Fm = torch.zeros(T, M, ld, device="cuda")
        Fm[..., :g.f] = randn(gg, T, M, g.f)                                  # the plan's F: padding columns zero
        ga = Guarded((T, M, ld), torch.float32)
        acc0 = torch.zeros(T, M, ld, device="cuda")
        if d["accumulate"]:
            acc0[..., :g.f] = randn(gg, T, M, g.f)
        ga.view.copy_(acc0)
        ga.snapshot()
        ops.ctr_mix(Fm, wts, ga.view, T=T, M=M, Cdim=d["Cdim"], ld=ld, rows_per_batch=rpb, accumulate=d["accumulate"])
        ga.unchanged_outside((slice(None),), "ctr_mix")
        Wd = wts.double()
        want = ref_ctr_mix(Fm.double(), Wd, rpb) + acc0.double()
        absum = ref_ctr_mix(Fm.double().abs(), Wd.abs(), rpb) + acc0.double().abs()
        ratios.append(check(ga.view, want, (T + 1) * U * absum, f"ctr_mix {name} acc={d['accumulate']} ((T+1)u)"))
        assert (ga.view[..., g.f:] == 0).all(), "ctr_mix padding columns: sum of w x 0"
    report(f"ctr {name} b{B}", ratios)


# ---- bilinear ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,B,ns", _cases("bilinear"))
@pytest.mark.gpu
def test_bilinear(ops, name, B, ns):
    """Every bilinear resize the plan runs, in its form: NHWC split (both planes, even C, no fp32 out: the FAST form; one
    plane: the vectorised general form) for the decoder's x4 up-sampling (C = 350 / 768, two pairs per lane, a partial
    last chunk), InvPT's 32 -> 16 downsample of the final tokens and its UpEmbed x2 with in_row_offset; NHWC fp32
    accumulate with in / out row offsets (InvPT's attention output into each task's slice); NCHW to the image size."""
    g, tab = table(name, B)
    ratios = [bilinear_case(ops, d, ns, 60 + i) for i, d in enumerate(tab["bilinear"])
              if d["form"] == "split" or ns == 2]
    if ratios:
        report(f"bilinear {name} b{B} ns={ns}", ratios)


@pytest.mark.parametrize("name,B,ns", _cases("bilinear_sum3"))
@pytest.mark.gpu
def test_bilinear_sum3(ops, name, B, ns):
    """InvPT's multi-scale aggregation: the three stages' maps (16², 32², 64², the first one a task's slice of the joint
    LayerNorm output) resized to 128 x 128 and summed, written once as split planes (C = 576: 5 chunks of 128 channels,
    half the pairs of the last one idle)."""
    g, tab = table(name, B)
    ratios = []
    for i, d in enumerate(tab["bilinear_sum3"]):
        B, C, H2, W2 = d["B"], d["Cdim"], d["H2"], d["W2"]
        srcs, want, absr = [], 0, 0
        for j, (h, w, br, ro, ld) in enumerate(d["srcs"]):
            n = (B - 1) * (br or h * w) + ro + h * w
            t = randn(gen(100 + j), n, ld)
            srcs.append((t, h, w, br, ro))
            y, a = ref_bilinear(t.double(), rows_of(B, h * w, br or h * w, ro, "cuda"), B, h, w, C, H2, W2)
            want, absr = want + y, absr + a
        gb, sp, reg = guarded_split(ops, ns, B * H2 * W2, C)
        gb.snapshot()
        ops.bilinear_sum3(srcs, sp, B=B, Cdim=C, H2=H2, W2=W2)
        gb.unchanged_outside(reg, "bilinear_sum3")
        wn, an = want.permute(0, 2, 3, 1).reshape(-1, C), absr.permute(0, 2, 3, 1).reshape(-1, C)
        e = (E_BIL + 2 * U) * an                                     # each source's resize, then two more sums
        ratios.append(check_planes(sp, wn, e, f"bilinear_sum3 slice {i} (6u per source + 2u)"))
    report(f"bilinear_sum3 {name} b{B} ns={ns}", ratios)


@pytest.mark.parametrize("name,B", _runs_calling("bilinear_postproc"))
@pytest.mark.gpu
def test_bilinear_postproc(ops, name, B):
    """The final resize fused with get_output at full output size, for each task's kind: argmax over 21 / 7 / 40 / 19
    classes, 255 sigmoid, 255 softmax[1], normalised normals, clamped depth. A class must be exact wherever the float64
    top-2 margin exceeds twice the value bound, and one of the tied classes elsewhere."""
    g, tab = table(name, B)
    ratios = [postproc_case(ops, d, 120 + i) for i, d in enumerate(tab["bilinear_postproc"])]
    ratios = [r for r in ratios if r is not None]
    if ratios:
        report(f"bilinear_postproc {name} b{B}", ratios)


# ---- InvPT token reductions and cross-task attention softmax -------------------------------------------------------------------
@pytest.mark.parametrize("name,B,ns", _cases("dwconv3x3_s2"))
@pytest.mark.gpu
def test_dwconv_and_avgpool(ops, name, B, ns):
    """Per-stage Q and KV token reductions at C = 576 / 288 / 144 (256-, 256- and 128-thread blocks, ragged channel
    loops): per-task depthwise 3x3 stride-2 conv (bias + 9 fma) against F.conv2d(groups=C), and the s x s average pool
    (s = 2 / 4 / 8) against F.avg_pool2d(ceil_mode=True)."""
    g, tab = table(name, B)
    ratios = []
    for i, d in enumerate(tab["dwconv3x3_s2"]):
        B, T, h, w, C = d["B"], d["T"], d["h"], d["w"], d["Cdim"]
        gg = gen(140 + i)
        x = randn(gg, B * T * h * w, d["ld_in"])
        wgt, bias = randn(gg, T, C, 9, scale=0.3), randn(gg, T, C, scale=0.3)
        gb, sp, reg = guarded_split(ops, ns, B * T * (h // 2) * (w // 2), C, ld=d["ld_out"])
        gb.snapshot()
        ops.dwconv3x3_s2(x, wgt, bias, sp, B=B, T=T, h=h, w=w, Cdim=C)
        gb.unchanged_outside(reg, "dwconv3x3_s2")
        want, absr = ref_dwconv(x.double(), wgt.double(), bias.double(), B, T, h, w, C)
        ratios.append(check_planes(sp, want, sum_tol(10, absr), f"dwconv3x3_s2 {h}x{w} C={C} (sum_tol D=10)"))
    for i, d in enumerate(tab["avgpool"]):
        BT, h, w, C, s = d["BT"], d["h"], d["w"], d["Cdim"], d["s"]
        x = randn(gen(150 + i), BT * h * w, d["ld_in"])
        oh, ow = -(-h // s), -(-w // s)
        gb, sp, reg = guarded_split(ops, ns, BT * oh * ow, C, ld=d["ld_out"])
        gb.snapshot()
        ops.avgpool(x, sp, BT=BT, h=h, w=w, Cdim=C, s=s)
        gb.unchanged_outside(reg, "avgpool")
        want, absr = ref_avgpool(x.double(), BT, h, w, C, s)
        # a serial sum of s * s terms, then the product with 1 / count (a power of two here: exact)
        ratios.append(check_planes(sp, want, sum_tol(s * s, absr) + U * want.abs(),
                                   f"avgpool {h}x{w} s={s} C={C} (sum_tol D=s^2 + u)"))
    report(f"dwconv/avgpool {name} b{B} ns={ns}", ratios)


@pytest.mark.parametrize("name,B,ns", _cases("invpt_fuse_softmax"))
@pytest.mark.gpu
def test_invpt_fuse_softmax(ops, name, B, ns):
    """The step between InvPT's two attention GEMMs at every stage: Tk = 320 keys (10 per lane), Lq = 320 / 1280 / 5120
    queries, cross-scale fusion with the previous stage's fused score (x2 bilinear per task over the query grid) at stages
    1 and 2, the fused score written in place of the raw one (stages 0 and 1), P = softmax as split rows."""
    g, tab = table(name, B)
    ratios = []
    prev = None
    for i, d in enumerate(tab["invpt_fuse_softmax"]):
        B, Lq, Tk, T, qh, qw = d["B"], d["Lq"], d["Tk"], d["T"], d["qh"], d["qw"]
        Ci = g.stages[i]["C"]
        scale = Ci ** -0.5
        scale32 = float(torch.tensor(scale, dtype=torch.float32))          # the kernel multiplies by the fp32 scale
        gg = gen(160 + i)
        raw = randn(gg, B, 2, Lq, Tk, scale=3.0 / scale32)                  # scaled scores ~ N(0, 9)
        raw[..., ::37] += 12.0 / scale32                                     # a few strongly preferred keys
        wf, bf = randn(gg, 2, 4, scale=0.6), randn(gg, 2, scale=0.5)
        if d["fused"]:
            assert prev is not None and prev.shape[2] == T * (qh // 2) * (qw // 2)
        pv = prev if d["fused"] else None
        score = raw.clone()
        gb, sp, reg = guarded_split(ops, ns, B * 2 * Lq, Tk, ld=d["ldp"])
        gb.snapshot()
        ops.invpt_fuse_softmax(score, sp, B=B, Lq=Lq, Tk=Tk, scale=scale, prev_score=pv, T=T, qh=qh, qw=qw,
                               fuse_w=wf, fuse_b=bf, score_out=score if d["score_out"] else None)
        gb.unchanged_outside(reg, "invpt_fuse_softmax P")
        f, fa, up, upa = ref_fuse(raw.double(), scale32, None if pv is None else pv.double(), wf.double(), bf.double(),
                                  B, T, qh, qw)
        if pv is None:
            e_f = U * f.abs()
        else:   # scale (u), the x2 resize of prev (6u), the 5-term fuse (5u), each through |W|
            s_abs = (raw.double() * scale32).abs()
            wa = wf.double().abs()
            e_s, e_up = U * s_abs, E_BIL * upa
            e_f = 5 * U * fa + torch.einsum("oi,bilt->bolt", wa, torch.cat([e_s, e_up], dim=1))
        if d["score_out"]:
            ratios.append(check(score, f, e_f, f"fused score stage {i} (scale u, x2 resize 6u, fuse 5u)"))
        else:
            assert torch.equal(score, raw), "raw scores are read only without score_out"
        # softmax: a perturbation e_f moves p_i by p_i (e_f,i + max_j e_f,j); expf (2 ulp) of the rounded f - m, the row
        # sum (ceil(Tk / 32) serial + 5 shuffles), the reciprocal and the product
        m = f.amax(-1, keepdim=True)
        Pw = torch.softmax(f, -1)
        D = math.ceil(Tk / 32) + 5
        rel = (e_f + e_f.amax(-1, keepdim=True) + U * (f - m).abs() + 4 * U
               + LAM * math.sqrt(D) * U + 2 * U)
        e_P = Pw * rel + 2.0 ** -126                                         # + fp32 underflow of tiny probabilities
        ratios.append(check_planes(sp, Pw.reshape(B * 2 * Lq, Tk), e_P.reshape(B * 2 * Lq, Tk),
                                   f"softmax P stage {i} (perturbation + expf + sum_tol D={D})"))
        prev = score if d["score_out"] else None
    report(f"invpt_fuse_softmax {name} b{B} ns={ns}", ratios)


# ---- CPU self-check of the references ----------------------------------------------------------------------------------------
def test_references_against_the_torch_restatement(monkeypatch):
    """Every float64 reference builder above at a toy size against tests/emul_ops.py (the fp32 torch restatement of the
    kernels' contracts): checks the references on a machine without a GPU."""
    import emul_ops
    import mtt_b200  # noqa: F401
    from mtt_b200 import ops

    emul_ops.install(monkeypatch)
    torch.manual_seed(0)
    close = lambda a, b, what: torch.testing.assert_close(a.double(), b.double(), rtol=2e-5, atol=2e-5, msg=what)
    r = lambda *s: torch.randn(*s)
    cpu = lambda ns, rows, cols: ops.Split(rows, cols, "cpu", ns, zero=True)
    B, T, H, C, gh, gw, nh, nw = 2, 3, 2, 16, 4, 6, 2, 3
    P, N = gh * gw, T + gh * gw
    # im2col
    img = r(B, 3, 32, 48)
    sp = cpu(2, B * 6, 3 * 256)
    ops.im2col_patch(img, 16, sp)
    close(ref_im2col(img.double(), 16), sp.float(), "im2col")
    # chan logits
    xs, cp = r(B * N, C), r(B * T, P)
    xn = ops.split_f32(xs, 2)
    out = torch.zeros(B, T, C, nh, nw)
    ops.chan_logits(cp, xn, out, B=B, N=N, T=T, Cdim=C, gh=gh, gw=gw, nh=nh, nw=nw)
    X = xn.float().double().view(B, N, C)[:, T:]
    close(ref_chan_logits(cp.double(), X, B, T, C, gh, gw, nh, nw), out, "chan_logits")
    # gates
    lg, rc = r(B, H, T, N), r(B, T, C, nh, nw)
    for t in range(T):
        ys, yc = cpu(2, B * P, C), cpu(2, B * P, C)
        ops.gate_split(xs, N, T, lg, rc, t, ys, yc, B=B, T=T, N=N, H=H, Cdim=C, gh=gh, gw=gw, nh=nh, nw=nw)
        gs, gc = ref_gates(lg.double(), rc.double(), B, T, H, C, gh, gw, nh, nw, t)
        Xp = xs.double().view(B, N, C)[:, T:]
        close((Xp * (1 + gs)).reshape(-1, C), ys.float(), "gate Ys")
        close((Xp * (1 + gc)).reshape(-1, C), yc.float(), "gate Yc")
    # ctr
    w0, b0, w2, b2 = r(T, H, H), r(T, H), r(T, H), r(T)
    wts = torch.zeros(B, T, T)
    ops.ctr_weights(lg, w0, b0, w2, b2, wts, B=B, H=H, T=T, N=N)
    close(ref_ctr_weights(lg.double(), w0.double(), b0.double(), w2.double(), b2.double(), T), wts, "ctr_weights")
    Fm, acc = r(T, B * P, 8), torch.zeros(T, B * P, 8)
    ops.ctr_mix(Fm, wts, acc, T=T, M=B * P, Cdim=8, ld=8, rows_per_batch=P, accumulate=False)
    close(ref_ctr_mix(Fm.double(), wts.double(), P), acc, "ctr_mix")
    # bilinear (up and down, with row offsets) and its post-processing
    for (h, w, H2, W2) in ((4, 6, 16, 24), (8, 8, 4, 4)):
        x = r(B * 2 * h * w, C)
        o = torch.zeros(B, C, H2, W2)
        ops.bilinear(x, C, B, h, w, C, H2, W2, out_nchw=o, in_batch_rows=2 * h * w, in_row_offset=h * w)
        close(ref_bilinear(x.double(), rows_of(B, h * w, 2 * h * w, h * w, "cpu"), B, h, w, C, H2, W2)[0], o, "bilinear")
    x = r(B * 4 * 6, 8) * 3
    y = ref_bilinear(x.double(), torch.arange(B * 24), B, 4, 6, 5, 16, 24)[0]
    for kind, cc in ((0, 5), (1, 1), (2, 2), (3, 3), (4, 1)):
        shape = {0: (B, 16, 24), 3: (B, 16, 24, 3), 4: (B, 16, 24, 1)}.get(kind, (B, 16, 24))
        o = torch.zeros(shape, dtype=torch.int64 if kind == 0 else torch.float32)
        ops.bilinear_postproc(x, 8, B, 4, 6, cc, 16, 24, kind, o)
        want = ref_postproc(y[:, :cc], kind)
        if kind == 0:
            assert (want == o).double().mean() > 0.999, "postproc argmax"
        else:
            close(want, o, f"postproc kind {kind}")
    with pytest.raises(AssertionError, match="not exact"):
        ref_bilinear(x.double(), torch.arange(B * 24), B, 4, 6, 5, 12, 24)
    # sum3
    srcs = [(r(B * 4, C), 2, 2, 0, 0), (r(B * 16, C), 4, 4, 0, 0), (r(B * 64, C), 8, 8, 0, 0)]
    so = cpu(2, B * 256, C)
    ops.bilinear_sum3(srcs, so, B=B, Cdim=C, H2=16, W2=16)
    want = sum(ref_bilinear(t.double(), torch.arange(B * h * w), B, h, w, C, 16, 16)[0] for t, h, w, _, _ in srcs)
    close(want.permute(0, 2, 3, 1).reshape(-1, C), so.float(), "bilinear_sum3")
    # layernorm
    x, gam, bet = r(10, C) + 3, r(C), r(C)
    o = torch.zeros(10, C)
    ops.layernorm(x, gam, bet, 1e-6, out_f32=o)
    close(ref_layernorm(x.double(), gam.double(), bet.double(), 1e-6), o, "layernorm")
    close(ln_bound(x.double(), gam.double(), bet.double(), 1e-6, 5)[0], o, "layernorm (bound builder)")
    # dwconv / avgpool
    h, w = 6, 8
    xt, wq, bq = r(B * T * h * w, C), r(T, C, 9), r(T, C)
    q = cpu(2, B * T * (h // 2) * (w // 2), C)
    ops.dwconv3x3_s2(xt, wq, bq, q, B=B, T=T, h=h, w=w, Cdim=C)
    close(ref_dwconv(xt.double(), wq.double(), bq.double(), B, T, h, w, C)[0], q.float(), "dwconv3x3_s2")
    for s in (2, 4):
        kv = cpu(2, B * T * -(-h // s) * -(-w // s), C)
        ops.avgpool(xt, kv, BT=B * T, h=h, w=w, Cdim=C, s=s)
        close(ref_avgpool(xt.double(), B * T, h, w, C, s)[0], kv.float(), f"avgpool s={s}")
    # fuse + softmax
    qh, qw, Tk = 4, 6, 10
    Lq = T * qh * qw
    raw, pv = r(B, 2, Lq, Tk), r(B, 2, T * (qh // 2) * (qw // 2), Tk)
    wf, bf = r(2, 4), r(2)
    Pm, so = cpu(2, B * 2 * Lq, Tk), torch.zeros(B, 2, Lq, Tk)
    ops.invpt_fuse_softmax(raw, Pm, B=B, Lq=Lq, Tk=Tk, scale=0.3, prev_score=pv, T=T, qh=qh, qw=qw, fuse_w=wf,
                           fuse_b=bf, score_out=so)
    f = ref_fuse(raw.double(), 0.3, pv.double(), wf.double(), bf.double(), B, T, qh, qw)[0]
    close(f, so, "fused score")
    close(torch.softmax(f, -1).reshape(-1, Tk), Pm.float(), "softmax P")


def test_geometry_table_is_derived_for_every_benched_config():
    """The table derives for every run, holds only power-of-two resizes, and reaches the shapes the kernel tests are
    about: the 64 x 128 channel window, Tk = 320 at every ip_cfg3 stage; at the reference's own configs Tk = 252 at every
    ip_nyud_vitL stage (a ragged last lane of the softmax and a K tail of the grouped P.V GEMM), the 784-wide e and
    1024-wide f of tp_pascal_vitB with ctr over 4 x 4 channel windows at H = 12, N = 1012 tokens at 16 heads
    (tp_nyud_vitL), and M = 6 * 1029 rows at valBatch 6."""
    for name, B in RUNS:
        g, tab = table(name, B)
        assert g.B == B
        for d in tab["bilinear"] + tab.get("bilinear_postproc", []):
            assert_pow2_ratio(d["h"], d["H2"])
            assert_pow2_ratio(d["w"], d["W2"])
        for d in tab.get("bilinear_sum3", []):
            for h, w, *_ in d["srcs"]:
                assert_pow2_ratio(h, d["H2"])
                assert_pow2_ratio(w, d["W2"])
    assert {(n, B) for n, B in RUNS} >= {(n, 6) for n in ("tp_nyud_vitL", "tp_pascal_vitB", "ip_nyud_vitL", "tp_cfg4",
                                                         "ip_cfg3")} | {(n, 5) for n in ("tp_cfg4", "tp_pascal_vitB",
                                                                                          "ip_cfg3")}
    cl5 = table("tp_cfg5", 1)[1]["chan_logits"][0]
    assert cl5["gh"] * cl5["gw"] == 8192
    assert [d["Tk"] for d in table("ip_cfg3", 4)[1]["invpt_fuse_softmax"]] == [320, 320, 320]
    g, tab = table("ip_nyud_vitL", 6)
    assert [d["Tk"] for d in tab["invpt_fuse_softmax"]] == [252, 252, 252]
    assert [d["ldp"] for d in tab["invpt_fuse_softmax"]] == [256, 256, 256]
    assert [d["Lq"] for d in tab["invpt_fuse_softmax"]] == [252, 1008, 4032]
    assert [s["Tk"] % 64 for s in g.stages] == [60, 60, 60]            # P.V's K = Tk: a 60-deep last K-stage
    assert {(d["H2"], d["W2"]) for d in tab["bilinear_sum3"]} == {(112, 144)}
    g, tab = table("tp_pascal_vitB", 6)
    assert (g.e, g.e_ld, g.f, g.f_ld) == (780, 784, 1024, 1024)
    assert tab["ctr_weights"] == [dict(B=6, H=12, T=5, N=1029)]
    assert (tab["chan_logits"][0]["nh"], tab["chan_logits"][0]["nw"], tab["chan_logits"][0]["C"]) == (4, 4, 768)
    assert bil(1024, 6, 32, 32, 1024, 128, 128, "split", ld_out=1024) in tab["bilinear"]
    assert tab["layernorm"][0]["rows"] == 6 * 1029 == table("tp_cfg4", 6)[1]["layernorm"][0]["rows"]
    g, tab = table("tp_nyud_vitL", 6)
    gs = tab["gate_split"][0]
    assert (gs["N"], gs["H"], gs["C"], gs["nh"], gs["nw"], gs["gh"] // gs["nh"], gs["gw"] // gs["nw"]) == \
        (1012, 16, 1024, 4, 4, 7, 9)
    assert table("tp_pascal_vitB", 5)[1]["layernorm"][0]["rows"] == 5 * 1029
