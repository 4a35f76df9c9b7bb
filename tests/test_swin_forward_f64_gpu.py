"""The non-tensor-core kernels of the Swin TaskPrompter forward at every geometry the plans launch -- the Swin runs of
plan_calls.RUNS: tps_swinB (two tasks) and tps_swinB3d (three tasks with '3ddet', nn.Identity as its detection head) at
batch 1 in the wrapper forward ("full"), predict() ("postproc") and the backbone forward, and tps_swinB3d's predict() at
the reference's validation batch 4 -- against float64, element by element.

Geometry. SwinGeom derives, from the config alone, the stage maps (C, heads, window 12, shift 0 / 6, nW, T), the
decoder levels (maps, f) and the head and output sizes; swin_table turns it into the list of calls each mode makes
(function, shape arguments, leading dimensions). test_plans_call_exactly_the_tabled_shapes runs one eager pass of each
mode with pass-through recorders around the ops functions the plan calls (RECORDED): every recorded key must be in the
table and every table entry must be recorded, so the table goes stale in neither direction, and a speed-mode (nsplit=1)
build records the same keys. The CPU variant does the same on tps_tiny3d and tps_mid3d with tests/emul_ops.py installed.

Float64. Every table entry runs on random inputs inside NaN sentinels (pad columns, guard rows, the T prompt columns of
the logit maps, spare planes) that must come back bit-identical, in parity mode and, where the kernel writes split
planes, in speed mode. Bounds and references are those of tests/kernel_cases.py (LayerNorm, gating, bilinear,
post-processing, window attention, gather / scatter, channel attention, stride-2 convolution, channel up-projection)
under the error model of tests/f64_checks.py; data movement is bit-exact. The input downsample 1024x2048 -> 768x1536 has
a fp32 scale of 4/3 that is not exact: ref_bilinear_any interpolates at the kernel's own coordinates and bounds their
rounding. Beside the table: the stage-0 window scatter at B = 2 and conv3x3_s2_maps at B = 10, whose grid-stride loops
only run past the 4096- / 8192-block caps of their launches. Every test prints its worst err / bound."""
import collections

import pytest
import torch
import torch.nn as nn

from f64_checks import (Guarded, assert_planes_bit_exact, gen, guarded_split, ops, padded, randn,  # noqa: F401
                        report, round_up)
from kernel_cases import (E_BIL, attention_case, bilinear_case, chan_attention_case, chan_up_case, conv3x3_s2_case,
                          fp32_coords_exact, gate_case, gather_scatter_case, layernorm_case, nan_split,
                          assert_untouched, postproc_case, ref_bilinear, ref_bilinear_any, ref_im2col, rows_of)
from oracle import configs
from plan_calls import DET, RUNS, SwinGeom, bil, frozen, glue_key, recording, run_id

pytestmark = [pytest.mark.timeout(1200)]      # the GPU tests are marked one by one: the CPU checks are not
MODES = ["full", "postproc", "backbone"]
_MODES_OF = {"forward": ["full", "backbone"], "predict": ["postproc"]}
# {(config, batch): the modes its runs make}, in RUNS order
SWIN_RUNS = {}
for _n, _B, _m in RUNS:
    if _n.startswith("tps_"):
        SWIN_RUNS.setdefault((_n, _B), [])
        SWIN_RUNS[(_n, _B)] = [m for m in MODES if m in SWIN_RUNS[(_n, _B)] + _MODES_OF[_m]]
RECORDED = ["layernorm", "split_f32", "im2col_patch", "broadcast_rows", "swin_window_gather", "swin_window_attention",
            "swin_window_scatter", "transpose_split", "swin_chan_attention", "swin_merge_gather", "conv3x3_s2_maps",
            "swin_chan_up", "gated_conv1x1", "bilinear", "bilinear_postproc", "nhwc_to_nchw"]


# ---- geometry ------------------------------------------------------------------------------------------------------------
def swin_table(g, mode):
    """{function: [shape dicts]} of every recorded call one `mode` pass makes (duplicates kept out)."""
    from mtt_b200 import ops
    B, T, ce, nh = g.B, g.T, g.ce, g.nh
    t = collections.defaultdict(list)
    add = lambda fn, **d: None if d in t[fn] else t[fn].append(d)
    ln = lambda rows, cols, split=False: add("layernorm", rows=rows, cols=cols, ld_in=cols, f32=not split, split=split)
    sp32 = lambda rows, cols, ld_in: add("split_f32", rows=rows, cols=cols, ld_in=ld_in, ld_out=round_up(cols, 8))
    if g.ds != g.img:                                          # TP:676-677: every input channel as a 1-channel NCHW map
        add("bilinear", **bil(1, B * 3, *g.img, 1, *g.ds, "nchw"))
    P0 = g.stages[0]["L"]
    add("im2col_patch", shape=(B, 3) + g.ds, patch=g.patch, ld=round_up(3 * g.patch ** 2, 8))
    ln(B * P0, g.E)
    add("broadcast_rows", T=T, C=g.E, B=B, group_rows=T, ld=g.E)
    for i, s in enumerate(g.stages):
        H, W, L, C, heads, ws, nW = (s[k] for k in ("H", "W", "L", "C", "heads", "ws", "nW"))
        for j, shift in enumerate(s["shifts"]):
            last = i == len(g.stages) - 1 and j == s["depth"] - 1
            ln(B * L, C)
            ln(B * T, C)
            sp32(B * T, C, C)
            add("swin_window_gather", B=B, H=H, W=W, C=C, T=T, ws=ws, shift=shift, ldx=C, ldp=C, ld_out=round_up(C, 8))
            add("swin_window_attention", BW=B * nW, nW=nW, T=T, L=ws * ws, heads=heads, C=C,
                scale=(C // heads) ** -0.5, masked=shift > 0, ldq=round_up(3 * C, 8), ldo=round_up(C, 8))
            add("swin_window_scatter", B=B, H=H, W=W, C=C, T=T, ws=ws, shift=shift, heads=heads, last=last, ldo=C,
                ldxa=C, ldx=C, ldp=C)
            add("transpose_split", B=B, L=L, C=C, ld_in=C, ld_out=round_up(L, 8))
            add("swin_chan_attention", B=B, T=T, C=C, ce=ce, nh=nh, nw=nh, ldq=ce, ldkv=2 * ce, ldco=ce,
                ldcs=round_up(ce, 8))
        if i < len(g.stages) - 1:                              # PatchMerging (TP:430-472)
            add("swin_merge_gather", B=B, H=H, W=W, C=C, ldx=C, ldo=4 * C)
            ln(B * L // 4, 4 * C, split=True)
            add("conv3x3_s2_maps", B=B, Cin=heads * T, Cout=heads * T, H=H, W=W, in_stride=T + L, in_offset=T,
                out_stride=T + L // 4, out_offset=T)
            add("swin_chan_up", BT=B * T, C=C, Cout=2 * C, nwin=nh * nh)
            sp32(B * T, C, C)
        else:
            ln(B * L, C)                                       # the final norm (TP:709)
    for il, lv in enumerate(g.levels):                         # cal_task_feature (TP:721-774)
        h, w, C, P = lv["h"], lv["w"], lv["C"], lv["h"] * lv["w"]
        add("gate_split", B=B, T=T, N=T + P, H=lv["heads"], C=C, gh=h, gw=w, nh=nh, nw=nh, x_group_rows=P,
            x_row_offset=0, ldx=C, ntasks=T)
        if g.t2:
            add("bilinear", **bil(g.f_ld, B, h, w, g.f, 2 * h, 2 * w, "split", ld_out=g.f_ld))
            if il > 0:
                add("bilinear", **bil(g.f_ld, B, 2 * h, 2 * w, g.f, g.fh, g.fw, "f32", ld_out=g.f_ld, acc=True))
        if DET in g.tasks:
            add("nhwc_to_nchw", ld_in=g.f_ld, B=B, Cd=g.f, H=h, W=w)
    for task in g.t2:                                          # multi_scale_fuse, then the head or the NCHW features
        sp32(B * g.fh * g.fw, g.f, g.f_ld)
        n = g.n_out[task]
        if mode == "backbone":
            add("nhwc_to_nchw", ld_in=g.f_ld, B=B, Cd=g.f, H=g.fh, W=g.fw)
        elif mode == "full":
            add("bilinear", **bil(round_up(n, 4), B, g.ph, g.pw, n, *g.out_hw, "nchw"))
        else:
            add("bilinear_postproc", ld_in=round_up(n, 4), B=B, h=g.ph, w=g.pw, C=n, H2=g.out_hw[0], W2=g.out_hw[1],
                kind=ops.POSTPROC_KIND[task])
    return {fn: ds for fn, ds in t.items() if ds}


_GEOMS = {}


def geom(name, B=1):
    if (name, B) not in _GEOMS:
        _GEOMS[(name, B)] = SwinGeom(name, B)
    return _GEOMS[(name, B)]


def table(name, B=1):
    """Every call of the modes the runs of `name` at batch B make, merged."""
    out = {}
    for mode in SWIN_RUNS[(name, B)]:
        for fn, ds in swin_table(geom(name, B), mode).items():
            out.setdefault(fn, [])
            out[fn] += [d for d in ds if d not in out[fn]]
    return out


def entries(fn, split=True):
    """pytest parameters (config, batch, entry index, nsplit) of every table entry of `fn`; nsplit 1 too where the
    entry writes split planes (split: True, False, or a predicate of the entry)."""
    out = []
    for name, B in SWIN_RUNS:
        for i, d in enumerate(table(name, B).get(fn, [])):
            planes = split(d) if callable(split) else split
            for ns in ((2, 1) if planes else (2,)):
                out.append(pytest.param(name, B, i, ns, id=f"{run_id(name, B)}-{i}-ns{ns}"))
    return out


# ---- recorded keys -----------------------------------------------------------------------------------------------------------
def build(name, dev, nsplit):
    from mtt_b200 import taskprompter_swin as TS
    cfg = configs.taskprompter_swin(name)
    torch.manual_seed(0)
    with torch.device(dev):
        det = nn.Identity() if DET in cfg["tasks"] else None
        return TS.build_from_config(cfg, nsplit=nsplit, use_graph=False, det_head=det).eval()


def run_mode(model, mode, x):
    with torch.no_grad():
        if mode == "full":
            return model(x)
        if mode == "postproc":
            return model.predict(x)
        return model.backbone(x)


def recorded_keys(model, mode, x):
    """The distinct keys of one pass of `mode` (after an unrecorded pass that builds the plan and packs the weights).
    Only calls from the library's modules are recorded: an emulated composite calling another emulated function is not
    a plan call."""
    from mtt_b200 import ops
    run_mode(model, mode, x)
    with recording(ops, RECORDED, glue_key, [], library_only=True) as seen:
        run_mode(model, mode, x)
        if x.is_cuda:
            torch.cuda.synchronize()
    return {(fn, frozen(d)) for fn, d in seen}


def tabled_keys(g, mode):
    return {(fn, frozen(d)) for fn, ds in swin_table(g, mode).items() for d in ds}


def assert_same_keys(got, want, what):
    assert got, f"{what}: nothing recorded"
    extra, missing = sorted(got - want, key=str), sorted(want - got, key=str)
    assert not extra, f"{what}: the plan calls kernels at shapes the table does not hold: {extra[:4]}"
    assert not missing, f"{what}: table entries the plan did not call: {missing[:4]}"


@pytest.mark.gpu
@pytest.mark.parametrize("name,B", [pytest.param(n, B, id=run_id(n, B)) for n, B in SWIN_RUNS])
def test_plans_call_exactly_the_tabled_shapes(cuda_dev, name, B):
    """One eager pass of each mode of the run at its batch, parity build: recorded keys == table; a speed-mode build
    records the same keys in the first of them (the keys hold no plane count)."""
    import mtt_b200  # noqa: F401
    g = geom(name, B)
    x = torch.randn(g.B, 3, *g.img, device=cuda_dev)
    model = build(name, cuda_dev, 2)
    modes = SWIN_RUNS[(name, B)]
    for mode in modes:
        got = recorded_keys(model, mode, x)
        assert_same_keys(got, tabled_keys(g, mode), f"{name} b{B} {mode}")
        print(f"{name} b{B} {mode}: {len(got)} distinct calls, exactly the table's")
    par = recorded_keys(model, modes[0], x)
    del model
    torch.cuda.empty_cache()
    model = build(name, cuda_dev, 1)
    assert recorded_keys(model, modes[0], x) == par, f"{name} b{B}: the speed-mode plan calls other shapes"
    del model
    torch.cuda.empty_cache()


@pytest.mark.parametrize("name", ["tps_tiny3d", "tps_mid3d"])
def test_plans_call_exactly_the_tabled_shapes_emulated(monkeypatch, name):
    """The same check on the CPU with the kernels emulated (tests/emul_ops.py): a window clipped to the map and padded
    (tps_tiny3d), window 12 with the 0.75 input scale (tps_mid3d), 2 x 2 and 1 x 1 channel windows."""
    import emul_ops
    import mtt_b200  # noqa: F401
    from mtt_b200 import taskprompter as TP, taskprompter_swin as TS
    emul_ops.install(monkeypatch)
    monkeypatch.setattr(TP, "_check_input", lambda mod, x: None)
    monkeypatch.setattr(TS, "_check_input", lambda mod, x: None)
    g = SwinGeom(name, B=2)
    x = torch.randn(g.B, 3, *g.img)
    model = build(name, "cpu", 2)
    for mode in MODES:
        assert_same_keys(recorded_keys(model, mode, x), tabled_keys(g, mode), f"{name} {mode}")


def test_geometry_of_the_swinB_models():
    """The table reaches the shapes the kernel tests are about, at batch 1 and at tps_swinB3d's valBatch 4."""
    assert list(SWIN_RUNS) == [("tps_swinB", 1), ("tps_swinB3d", 1), ("tps_swinB3d", 4)]
    assert SWIN_RUNS[("tps_swinB", 1)] == MODES and SWIN_RUNS[("tps_swinB3d", 4)] == ["postproc"]
    for name, T in (("tps_swinB", 2), ("tps_swinB3d", 3)):
        g, tab = geom(name), table(name)
        assert g.T == T and [s["nW"] for s in g.stages] == [512, 128, 32, 8]
        assert {d["L"] for d in tab["swin_window_attention"]} == {144}
        assert {d["Cin"] for d in tab["conv3x3_s2_maps"]} == {4 * T, 8 * T, 16 * T}
        assert {"rows": 73728, "cols": 128, "ld_in": 128, "f32": True, "split": False} in tab["layernorm"]
        assert bil(1, 3, 1024, 2048, 1, 768, 1536, "nchw") in tab["bilinear"]
        assert {(d["h"], d["w"], d["H2"], d["W2"]) for d in tab["bilinear_postproc"]} == {(384, 768, 512, 1024)}
    assert len(table("tps_swinB3d")["nhwc_to_nchw"]) == 3 + 1          # 3 distinct level maps (two share 24x48) + fea
    assert not fp32_coords_exact(1024, 768) and fp32_coords_exact(384, 512)
    tab = table("tps_swinB3d", 4)
    assert {(d["BW"], d["nW"]) for d in tab["swin_window_attention"]} == {(4 * 512, 512), (4 * 128, 128), (4 * 32, 32),
                                                                          (4 * 8, 8)}
    assert {"rows": 4 * 73728, "cols": 128, "ld_in": 128, "f32": True, "split": False} in tab["layernorm"]
    assert {(d["B"], d["H2"], d["W2"]) for d in tab["bilinear_postproc"]} == {(4, 512, 1024)}
    assert bil(1, 12, 1024, 2048, 1, 768, 1536, "nchw") in tab["bilinear"]
    assert len(tab["nhwc_to_nchw"]) == 3                                  # predict(): the 3ddet level maps, no fea


# ---- float64: window attention, gather / scatter, channel attention, merging ------------------------------------------------
def _stage_of(g, C):
    return next(s for s in g.stages if s["C"] == C)


@pytest.mark.gpu
@pytest.mark.parametrize("name,B,i,ns", entries("swin_window_attention"))
def test_window_attention(ops, cuda_dev, name, B, i, ns):
    """Window attention at each stage x shift of the table (N = T + 144: 146 or 147 rows), all T raw-logit rows."""
    d = table(name, B)["swin_window_attention"][i]
    s = _stage_of(geom(name, B), d["C"])
    shift = 6 if d["masked"] else 0
    r = attention_case(ops, cuda_dev, B=d["BW"] // d["nW"], nWy=s["H"] // s["ws"], nWx=s["W"] // s["ws"],
                           ws=s["ws"], shift=shift, T=d["T"], heads=d["heads"], dh=d["C"] // d["heads"],
                           seed=100 * i + d["T"], ns=ns)
    report(f"window attention {name} b{B} C={d['C']} shift={shift} ns={ns} (out, raw logits)", r)
    torch.cuda.empty_cache()


def _gather_scatter(ops, dev, d, ns, B=None):
    r = gather_scatter_case(ops, dev, B=B or d["B"], H=d["H"], W=d["W"], C=d["C"], T=d["T"], heads=d["heads"],
                                ws=d["ws"], shift=d["shift"], ns=ns, lasts=(d["last"],))
    torch.cuda.empty_cache()
    return r


@pytest.mark.gpu
@pytest.mark.parametrize("name,B,i,ns", entries("swin_window_scatter"))
def test_window_gather_and_scatter(ops, cuda_dev, name, B, i, ns):
    """Gather (split planes, bit-exact) and scatter (xa, x += xa and the [B, heads, T, T + L] logits map bit-exact,
    the prompt mean within its bound) at each stage x shift x last of the table."""
    d = table(name, B)["swin_window_scatter"][i]
    report(f"window scatter {name} b{B} C={d['C']} shift={d['shift']} last={d['last']} (prompt mean)",
           [_gather_scatter(ops, cuda_dev, d, ns)])


@pytest.mark.gpu
@pytest.mark.parametrize("T", [2, 3])
def test_window_scatter_grid_stride(ops, cuda_dev, T):
    """Stage 0 of Swin-B at B = 2: 2 * 4 * T * 147456 logits (1 179 648 / 1 769 472) > 4096 blocks of 256, so the
    logits kernel's grid-stride loop runs (predict() and the evaluation loader run at B > 1)."""
    d = next(d for d in table("tps_swinB3d" if T == 3 else "tps_swinB")["swin_window_scatter"] if d["C"] == 128)
    assert 2 * d["heads"] * T * d["H"] * d["W"] > 4096 * 256
    report(f"window scatter B=2 T={T} stage 0", [_gather_scatter(ops, cuda_dev, dict(d, last=False), 2, B=2)])


@pytest.mark.gpu
@pytest.mark.parametrize("name,B,i,ns", entries("transpose_split"))
def test_transpose_split(ops, cuda_dev, name, B, i, ns):
    """[B, L, C] -> split [B*C, L] per stage (L = 73728 ... 1152), NaN pad columns read past C would show: bit-exact."""
    d = table(name, B)["transpose_split"][i]
    B, L, C = d["B"], d["L"], d["C"]
    x = padded(B * L, C, cuda_dev)
    x.copy_(randn(gen(200 + i), B * L, C))
    out = nan_split(B * C, L, cuda_dev, ns=ns)
    ops.transpose_split(x, out, B=B, L=L, Cdim=C)
    torch.cuda.synchronize()
    assert_planes_bit_exact(out, x.reshape(B, L, C).transpose(1, 2).reshape(B * C, L), "transpose_split")
    assert_untouched(out, B * C, L)


@pytest.mark.gpu
@pytest.mark.parametrize("name,B,i,ns", entries("swin_chan_attention"))
def test_chan_attention(ops, cuda_dev, name, B, i, ns):
    """Channel attention of the T prompts over the C channels of each stage (C = 128 ... 1024, one 16 x 16 window)."""
    d = table(name, B)["swin_chan_attention"][i]
    r = chan_attention_case(ops, cuda_dev, B=d["B"], T=d["T"], C=d["C"], nh=d["nh"], ns=ns)
    report(f"chan attention {name} b{B} T={d['T']} C={d['C']} ns={ns} (raw_chan, chan_out)", r)


@pytest.mark.gpu
@pytest.mark.parametrize("name,B,i,ns", entries("swin_merge_gather", split=False))
def test_merge_gather(ops, cuda_dev, name, B, i, ns):
    """2 x 2 merge (0,0), (1,0), (0,1), (1,1) at each merging stage: bit-exact, pad columns untouched."""
    d = table(name, B)["swin_merge_gather"][i]
    B, H, W, C = d["B"], d["H"], d["W"], d["C"]
    x = padded(B * H * W, C, cuda_dev)
    x.copy_(randn(gen(300 + i), B * H * W, C))
    gb = Guarded((B * H * W // 4, d["ldo"] + 4), torch.float32)
    gb.snapshot()
    ops.swin_merge_gather(x, gb.view[:, :d["ldo"]], B=B, H=H, W=W, Cdim=C)
    gb.unchanged_outside((slice(None), slice(0, 4 * C)), "merge_gather")
    m = x.reshape(B, H, W, C)
    want = torch.cat([m[:, 0::2, 0::2], m[:, 1::2, 0::2], m[:, 0::2, 1::2], m[:, 1::2, 1::2]], -1)
    assert torch.equal(gb.view[:, :4 * C], want.reshape(-1, 4 * C))


@pytest.mark.gpu
@pytest.mark.parametrize("name,B,i,ns", entries("conv3x3_s2_maps", split=False))
def test_conv3x3_s2_maps(ops, cuda_dev, name, B, i, ns):
    """spa_attn_ds at each merge: Cin = Cout = heads * T (8 / 16 / 32 at T = 2, 12 / 24 / 48 at T = 3)."""
    d = table(name, B)["conv3x3_s2_maps"][i]
    T = d["in_offset"]
    r = conv3x3_s2_case(ops, cuda_dev, B=d["B"], T=T, H=d["H"], W=d["W"], Cin=d["Cin"], seed=400 + i)
    report(f"conv3x3_s2 {name} b{B} Cin={d['Cin']}", [r])


@pytest.mark.gpu
def test_conv3x3_s2_maps_grid_stride(ops, cuda_dev):
    """Stage 0 at B = 10, Cin = 12: 10 * 12 * 96 * 192 = 2 211 840 outputs > 8192 blocks of 256: the loop runs."""
    d = table("tps_swinB3d")["conv3x3_s2_maps"][0]
    assert d["Cin"] == 12 and 10 * 12 * (d["H"] // 2) * (d["W"] // 2) > 8192 * 256
    report("conv3x3_s2 B=10 Cin=12", [conv3x3_s2_case(ops, cuda_dev, B=10, T=3, H=d["H"], W=d["W"], Cin=12,
                                                          seed=499)])


@pytest.mark.gpu
@pytest.mark.parametrize("name,B,i,ns", entries("swin_chan_up", split=False))
def test_chan_up(ops, cuda_dev, name, B, i, ns):
    """process_chan_attn C -> 2C at each merge, B * T rows."""
    d = table(name, B)["swin_chan_up"][i]
    r = chan_up_case(ops, cuda_dev, BT=d["BT"], C=d["C"], nwin=d["nwin"], seed=500 + i)
    report(f"chan_up {name} b{B} BT={d['BT']} C={d['C']}", [r])


# ---- float64: stem, LayerNorm, splits, gating, resampling, layout -----------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name,B,i,ns", entries("im2col_patch"))
def test_im2col_patch(ops, name, B, i, ns):
    """Patch 4 on the 768 x 1536 downsampled input: planes bit-exact against the split of F.unfold."""
    d = table(name, B)["im2col_patch"][i]
    img = randn(gen(600), *d["shape"])
    rows = d["shape"][0] * (d["shape"][2] // d["patch"]) * (d["shape"][3] // d["patch"])
    gb, sp, reg = guarded_split(ops, ns, rows, d["ld"], ld=d["ld"])
    gb.snapshot()
    ops.im2col_patch(img, d["patch"], sp)
    gb.unchanged_outside(reg, "im2col_patch")
    assert_planes_bit_exact(sp, ref_im2col(img, d["patch"]), "im2col_patch")


@pytest.mark.gpu
@pytest.mark.parametrize("name,B,i,ns", entries("broadcast_rows", split=False))
def test_broadcast_rows(ops, name, B, i, ns):
    """The T task prompts into each image's prompt rows: bit-exact, nothing else written."""
    d = table(name, B)["broadcast_rows"][i]
    src = randn(gen(610), d["T"], d["C"])
    gb = Guarded((d["B"] * d["group_rows"], d["ld"]), torch.float32)
    gb.snapshot()
    ops.broadcast_rows(src, gb.view, d["B"], d["group_rows"])
    rows = rows_of(d["B"], d["T"], d["group_rows"], 0, "cuda")
    gb.unchanged_outside((rows, slice(0, d["C"])), "broadcast_rows")
    assert torch.equal(gb.view[rows, :d["C"]], src.repeat(d["B"], 1))


@pytest.mark.gpu
@pytest.mark.parametrize("name,B,i,ns", entries("split_f32"))
def test_split_f32(ops, name, B, i, ns):
    """The prompt rows and the level sum as planes: bit-exact, input pad columns (NaN) not read."""
    d = table(name, B)["split_f32"][i]
    x = torch.full((d["rows"], d["ld_in"]), float("nan"), device="cuda")[:, :d["cols"]]
    x.copy_(randn(gen(620 + i), d["rows"], d["cols"]))
    gb, sp, reg = guarded_split(ops, ns, d["rows"], d["cols"], ld=d["ld_out"])
    gb.snapshot()
    ops.split_f32(x, ns, out=sp)
    gb.unchanged_outside(reg, "split_f32")
    assert_planes_bit_exact(sp, x, "split_f32")


@pytest.mark.gpu
@pytest.mark.parametrize("name,B,i,ns", entries("layernorm", split=lambda d: d["split"]))
def test_layernorm(ops, name, B, i, ns):
    """Every LayerNorm: the stage norms over 73 728 x 128 ... 288 x 1024 rows, the prompt rows, the merge norm into
    split planes (4C = 512 ... 4096 columns), the final norm."""
    d = table(name, B)["layernorm"][i]
    report(f"layernorm {name} b{B} {d['rows']}x{d['cols']} split={d['split']} ns={ns}",
           [layernorm_case(ops, d, 700 + i, ns)])


@pytest.mark.gpu
@pytest.mark.parametrize("name,B,i,ns", entries("gate_split"))
def test_gate(ops, name, B, i, ns):
    """The gating stage of gated_conv1x1 at each decoder level: all T tasks in one launch, x = the level map (group
    P, offset 0), prompt logits [B, heads, T, T + P], channel logits of the 2C up-projection."""
    d = table(name, B)["gate_split"][i]
    report(f"gate {name} b{B} level C={d['C']} {d['gh']}x{d['gw']} ns={ns}", gate_case(ops, d, ns, f"{name} b{B}", seed=800 + i))


@pytest.mark.gpu
@pytest.mark.parametrize("name,B,i,ns", entries("bilinear", split=lambda d: d["form"] == "split"))
def test_bilinear(ops, name, B, i, ns):
    """The input downsample 1024x2048 -> 768x1536 (fp32 scale 4/3, inexact: ref_bilinear_any), the level x2
    up-samplings into split planes (f = 450, ld 456), the level sums into the 192 x 384 accumulator, the head resize
    384x768 -> 512x1024 (scale 0.75, exact)."""
    d = table(name, B)["bilinear"][i]
    report(f"bilinear {name} b{B} {d['h']}x{d['w']}->{d['H2']}x{d['W2']} {d['form']} ns={ns}",
           [bilinear_case(ops, d, ns, 900 + i)])
    torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("name,B,i,ns", entries("bilinear_postproc", split=False))
def test_bilinear_postproc(ops, name, B, i, ns):
    """predict()'s final resize fused with get_output: semseg argmax over 19 classes exact where the float64 top-2
    margin exceeds twice the logit bound, depth (kind 4) within the logit bound."""
    d = table(name, B)["bilinear_postproc"][i]
    r = postproc_case(ops, d, 950 + i)
    if r is not None:
        report(f"bilinear_postproc {name} b{B} kind {d['kind']}", [r])


@pytest.mark.gpu
@pytest.mark.parametrize("name,B,i,ns", entries("nhwc_to_nchw", split=False))
def test_nhwc_to_nchw(ops, name, B, i, ns):
    """The 3ddet level maps and the backbone features (f = 450 of ld 456) to NCHW: bit-exact."""
    d = table(name, B)["nhwc_to_nchw"][i]
    x = torch.full((d["B"] * d["H"] * d["W"], d["ld_in"]), float("nan"), device="cuda")
    x[:, :d["Cd"]] = randn(gen(980 + i), d["B"] * d["H"] * d["W"], d["Cd"])
    gb = Guarded((d["B"], d["Cd"], d["H"], d["W"]), torch.float32)
    gb.snapshot()
    ops.nhwc_to_nchw(x, d["ld_in"], d["B"], d["Cd"], d["H"], d["W"], gb.view)
    gb.unchanged_outside((slice(None),), "nhwc_to_nchw")
    assert torch.equal(gb.view, x[:, :d["Cd"]].reshape(d["B"], d["H"], d["W"], d["Cd"]).permute(0, 3, 1, 2))


# ---- CPU self-check of the any-ratio bilinear reference -------------------------------------------------------------------------
def _kernel_bilinear_cpu(x, B, h, w, C, H2, W2, fma, coord=None):
    """The kernel's arithmetic on the host in fp32 (bilin_coord with or without a fused multiply-add, then
    hy (hx p00 + lx p01) + ly (hx p10 + lx p11)), NCHW."""
    def axis(n, n2):
        sc = torch.tensor(n, dtype=torch.float32) / torch.tensor(n2, dtype=torch.float32)
        d = torch.arange(n2, dtype=torch.float32) + 0.5
        if coord is not None:
            s = coord(sc, d)
        elif fma:
            s = (sc.double() * d.double() - 0.5).float()                # one rounding
        else:
            s = sc * d - 0.5                                            # two
        s = s.clamp(min=0)
        i0 = s.long().clamp(max=n - 1)
        return i0, (i0 + 1).clamp(max=n - 1), s - i0.float()
    y0, y1, ly = axis(h, H2)
    x0, x1, lx = axis(w, W2)
    img = x[:, :C].reshape(B, h, w, C).permute(0, 3, 1, 2)
    hy, hx = (1 - ly)[:, None], 1 - lx
    r0, r1 = img[:, :, y0], img[:, :, y1]
    return hy * (hx * r0[..., x0] + lx * r0[..., x1]) + ly[:, None] * (hx * r1[..., x0] + lx * r1[..., x1])


def test_bilinear_any_ratio_reference():
    """ref_bilinear_any at toy non-power-of-two sizes: the host model of the kernel (both coordinate roundings) and
    tests/emul_ops.bilinear lie within E_BIL of the |.| resize + the coordinate term; where the coordinates are exact
    it equals float64 F.interpolate; a kernel that drops the half-pixel offset on one axis falls outside."""
    import emul_ops
    import mtt_b200  # noqa: F401
    from mtt_b200 import ops
    torch.manual_seed(0)
    B, C = 2, 3
    for (h, w, H2, W2) in ((12, 16, 9, 12), (7, 11, 10, 13), (30, 40, 23, 31), (9, 12, 12, 16)):
        x = torch.randn(B * h * w, C) * 3
        rows = torch.arange(B * h * w)
        y, a, ec = ref_bilinear_any(x.double(), rows, B, h, w, C, H2, W2)
        bound = E_BIL * a + ec
        for fma in (False, True):
            got = _kernel_bilinear_cpu(x, B, h, w, C, H2, W2, fma).double()
            assert bool(((got - y).abs() <= bound).all()), (h, w, H2, W2, fma, float(((got - y).abs() / bound).max()))
        with pytest.MonkeyPatch.context() as mp:
            emul_ops.install(mp)
            o = torch.zeros(B, C, H2, W2)
            ops.bilinear(x, C, B, h, w, C, H2, W2, out_nchw=o)
        assert bool(((o.double() - y).abs() <= bound).all()), (h, w, H2, W2, "emul_ops")
        if fp32_coords_exact(h, H2) and fp32_coords_exact(w, W2):
            y2, a2 = ref_bilinear(x.double(), rows, B, h, w, C, H2, W2)
            torch.testing.assert_close(y, y2, rtol=1e-13, atol=1e-13)
        bad = _kernel_bilinear_cpu(x, B, h, w, C, H2, W2, False, coord=lambda sc, d: sc * (d - 0.5)).double()
        assert bool(((bad - y).abs() > bound).any()), (h, w, H2, W2, "a shifted coordinate is not caught")
