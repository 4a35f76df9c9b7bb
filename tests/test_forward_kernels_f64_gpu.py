"""-m gpu: the forward glue kernels (csrc/prompting.cu, csrc/invpt.cu, csrc/rowwise.cu) at the geometries the benched
forwards really run -- tp_cfg4, tp_cfg2, tp_cfg5 and ip_cfg3 at bench.DEFAULT_BATCH -- against float64 references
written from each operation's definition (F.interpolate, F.conv2d(groups=C), F.avg_pool2d(ceil_mode=True),
F.layer_norm, softmax, the windowed sums, exact-erf GELU), element by element.

Error model: the one of test_train_kernels_f64_gpu.py (u per fp32 operation, LAM sqrt(D) u sum|a_i| for a reduction of
depth D counted from the kernel's launch geometry, SPLIT |x| + SPLIT_ABS for a value stored as hi + lo bf16 planes).
A value stored as the hi plane alone (speed mode, nsplit = 1: the lo pointer is NULL) carries HI |x| + HI_ABS. Pure data
movement is bit-exact. Every assert names the bound it uses.

Bilinear source coordinates are computed in fp32. Every resize ratio these plans use is a power of two, so those
coordinates and weights are exact and float64 F.interpolate is a valid reference (ref_bilinear refuses a ratio whose
fp32 coordinates are inexact). ref_bilinear_any, for the Swin plans' 4/3 input downsample, interpolates at the
kernel's own coordinates and bounds their fp32 rounding.

Around every output the test fills a NaN sentinel (padding columns up to ld, guard rows before and after, the other
tasks' slices of a joint buffer, a second plane where there is one plane); after the call it must be bit-identical.

The geometry table (TABLE) is derived from oracle/configs.py and bench.DEFAULT_BATCH; test_plans_call_only_tabled_shapes
runs each benched plan once and fails when a plan calls a glue kernel at a shape the table does not hold."""
import inspect
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import configs
from test_train_kernels_f64_gpu import LAM, SPLIT, SPLIT_ABS, U, check, sum_tol

pytestmark = [pytest.mark.timeout(1200)]      # the GPU tests are marked one by one: the CPU self-checks are not
HI = 2.0 ** -8            # relative precision of the hi bf16 plane alone: bf16 unit roundoff (8-bit significand)
HI_ABS = 2.0 ** -133      # ... and its absolute floor: the bf16 subnormal spacing
E_BIL = 6 * U             # one bilinear value: 4 products and 3 sums, each term rounded at most 4 times (plus slack)
BENCHED = ["tp_cfg4", "tp_cfg2", "tp_cfg5", "ip_cfg3"]
F32_SENT = 0x7FC0BEEF     # NaN sentinels: a kernel that leaves an output element unwritten leaves a NaN behind
BF16_SENT = 0x7FB5
I64_SENT = -0x5A5A5A5A5A5A5A5B


def round_up(x, m):
    return (x + m - 1) // m * m


def assert_pow2_ratio(src, dst):
    """The fp32 bilinear coordinates are exact only for power-of-two resize ratios: refuse any other."""
    lo, hi = min(src, dst), max(src, dst)
    r = hi // lo
    assert hi % lo == 0 and r & (r - 1) == 0, f"resize {src} -> {dst} is not a power-of-two ratio: float64 " \
                                              f"F.interpolate is no reference for the kernel's fp32 coordinates"


# ---- geometry ----------------------------------------------------------------------------------------------------------
class TPGeom:
    """A benched TaskPrompter (ViT) forward at its bench batch."""

    def __init__(self, name):
        import bench

        cfg = configs.taskprompter(name)
        self.name, self.cfg = name, cfg
        self.B = bench.DEFAULT_BATCH[name]
        self.tasks, self.T = list(cfg["tasks"]), len(cfg["tasks"])
        self.img = tuple(cfg["img_size"])
        self.patch = cfg["patch"]
        self.gh, self.gw = self.img[0] // self.patch, self.img[1] // self.patch
        self.P = self.gh * self.gw
        self.N = self.T + self.P
        self.C, self.H = cfg["C"], cfg["heads"]
        self.nh = self.nw = int(round(math.sqrt(cfg["chan_nheads"])))
        self.f = cfg["f"]
        self.f_ld = round_up(self.f, 8)
        self.use_ctr = cfg["use_ctr"]
        self.h4, self.w4 = 4 * self.gh, 4 * self.gw      # ConvHead: predictions at 4x the token grid
        self.out_hw = tuple(cfg.get("dd_label_map_size", self.img))
        self.n_out = dict(cfg["num_output"])


class IPGeom:
    """The benched InvPT forward at its bench batch (invpt.py _Plan)."""

    def __init__(self, name):
        import bench

        cfg = configs.invpt(name)
        self.name, self.cfg = name, cfg
        self.B = bench.DEFAULT_BATCH[name]
        self.tasks, self.T = list(cfg["tasks"]), len(cfg["tasks"])
        self.img = tuple(cfg["img_size"])
        self.patch = cfg["patch"]
        self.gh, self.gw = self.img[0] // self.patch, self.img[1] // self.patch
        self.P = self.gh * self.gw
        self.N = 1 + self.P
        self.C = cfg["C"]
        self.E = cfg["embed_dim"]
        d0 = cfg["embed_dim"] + cfg["pred_const"]
        self.dims = [d0, d0 // 2, d0 // 4]
        self.h0, self.w0 = self.gh // cfg["down"], self.gw // cfg["down"]
        self.th, self.tw = 8 * self.h0, 8 * self.w0
        self.n_out = dict(cfg["num_output"])
        self.stages = []
        for i in range(3):
            h, w, kvs = self.h0 * 2 ** i, self.w0 * 2 ** i, 2 ** (i + 1)
            kh, kw = -(-h // kvs), -(-w // kvs)
            self.stages.append(dict(h=h, w=w, C=self.dims[i], kvs=kvs, Lq=self.T * (h // 2) * (w // 2),
                                    Tk=self.T * kh * kw))


def _geom(name):
    return IPGeom(name) if name.startswith("ip_") else TPGeom(name)


def _bil(ld_in, B, h, w, C, H2, W2, form, ld_out=0, acc=False, ibr=0, ioff=0, obr=0, ooff=0):
    return dict(ld_in=ld_in, B=B, h=h, w=w, C=C, H2=H2, W2=W2, form=form, ld_out=ld_out, acc=acc, ibr=ibr, ioff=ioff,
                obr=obr, ooff=ooff)


def _tp_table(g):
    B, T, C = g.B, g.T, g.C
    t = dict(im2col_patch=[dict(shape=(B, 3) + g.img, patch=g.patch, ld=round_up(3 * g.patch ** 2, 8))],
             broadcast_rows=[dict(T=T, C=C, B=B, group_rows=g.N, ld=C)],
             layernorm=[dict(rows=B * g.N, cols=C, ld_in=C, f32=True, split=False)],
             chan_logits=[dict(B=B, N=g.N, T=T, C=C, gh=g.gh, gw=g.gw, nh=g.nh, nw=g.nw)],
             gate_split=[dict(B=B, T=T, N=g.N, H=g.H, C=C, gh=g.gh, gw=g.gw, nh=g.nh, nw=g.nw, x_group_rows=g.N,
                              x_row_offset=T, ldx=C, ntasks=T)],
             bilinear=[_bil(g.f_ld, B, g.gh, g.gw, g.f, g.h4, g.w4, "split", ld_out=g.f_ld)],
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
        t["bilinear"].append(_bil(round_up(n, 4), B, g.h4, g.w4, n, *g.out_hw, "nchw"))
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
             bilinear=[_bil(C, B, g.gh, g.gw, C, g.h0, g.w0, "split", ld_out=C)],
             layernorm=[], dwconv3x3_s2=[], avgpool=[], invpt_fuse_softmax=[], bilinear_sum3=[], bilinear_postproc=[])
    for task in g.tasks:                                    # inter-pred resize (transformer_net.py:36)
        n = g.n_out[task]
        t["bilinear"].append(_bil(round_up(n, 4), B, g.h0, g.w0, n, *g.img, "nchw"))
    for i, s in enumerate(g.stages):
        h, w, Ci, hw = s["h"], s["w"], s["C"], s["h"] * s["w"]
        if i > 0:                                           # UpEmbed x2 of each task's slice of the previous stage
            p = g.stages[i - 1]
            phw = p["h"] * p["w"]
            t["bilinear"] += [_bil(p["C"], B, p["h"], p["w"], p["C"], h, w, "split", ld_out=round_up(p["C"], 8),
                                   ibr=T * phw, ioff=k * phw) for k in range(T)]
        t["layernorm"].append(dict(rows=B * T * hw, cols=Ci, ld_in=Ci, f32=True, split=False))
        t["dwconv3x3_s2"].append(dict(B=B, T=T, h=h, w=w, Cdim=Ci, ld_in=Ci, ld_out=round_up(Ci, 8)))
        t["avgpool"].append(dict(BT=B * T, h=h, w=w, Cdim=Ci, s=s["kvs"], ld_in=Ci, ld_out=round_up(Ci, 8)))
        t["invpt_fuse_softmax"].append(dict(B=B, Lq=s["Lq"], Tk=s["Tk"], fused=i > 0, T=T, qh=h // 2, qw=w // 2,
                                            score_out=i < 2, ldp=round_up(s["Tk"], 8)))
        qhw = (h // 2) * (w // 2)                           # attention output x2 accumulated into each task's slice
        t["bilinear"] += [_bil(Ci, B, h // 2, w // 2, Ci, h, w, "f32", ld_out=Ci, acc=True, ibr=T * qhw, ioff=k * qhw,
                               obr=T * hw, ooff=k * hw) for k in range(T)]
        t["layernorm_seg"].append(dict(rows=B * hw, cols=Ci, S=T, in_group=hw, src_group=T * hw, src_offset=0,
                                       seg_stride=hw, out_seg_stride=B * hw, ld_in=Ci, f32=i == 0, split=i > 0))
    s0, s1 = g.stages[0], g.stages[1]
    t["bilinear_sum3"] = [dict(B=B, Cdim=d0, H2=g.th, W2=g.tw,
                               srcs=((s0["h"], s0["w"], 0, k * B * s0["h"] * s0["w"], d0), (s1["h"], s1["w"], 0, 0, d0),
                                     (g.stages[2]["h"], g.stages[2]["w"], 0, 0, d0))) for k in range(T)]
    for task in g.tasks:
        n = g.n_out[task]
        t["bilinear"].append(_bil(round_up(n, 4), B, g.th, g.tw, n, *g.img, "nchw"))
        t["bilinear_postproc"].append(dict(ld_in=round_up(n, 4), B=B, h=g.th, w=g.tw, C=n, H2=g.img[0], W2=g.img[1],
                                           kind=ops.POSTPROC_KIND[task]))
    return t


_TABLES = {}


def table(name):
    if name not in _TABLES:
        import mtt_b200  # noqa: F401
        g = _geom(name)
        _TABLES[name] = (g, _ip_table(g) if name.startswith("ip_") else _tp_table(g))
    return _TABLES[name]


def _cases(fn):
    """(config, nsplit) parameters of the configs whose benched forward calls `fn` (a kernel that writes split planes)."""
    out = []
    for name in BENCHED:
        if table(name)[1].get(fn):
            out += [pytest.param(name, ns, id=f"{name}-ns{ns}") for ns in (2, 1)]
    return out


# ---- what a recorded ops call looks like in the table ----------------------------------------------------------------------
def _key_of_call(fn, a):
    """The table entry of one ops.<fn> call, a = its bound arguments (defaults applied)."""
    if fn == "im2col_patch":
        return "im2col_patch", dict(shape=tuple(a["img"].shape), patch=a["patch"], ld=a["out"].ld)
    if fn == "broadcast_rows":
        T, Cc = a["src"].shape
        return fn, dict(T=T, C=Cc, B=a["B"], group_rows=a["group_rows"], ld=a["dst"].stride(0))
    if fn == "layernorm":
        return fn, dict(rows=a["x"].shape[0], cols=a["x"].shape[1], ld_in=a["x"].stride(0),
                        f32=a["out_f32"] is not None, split=a["out_split"] is not None)
    if fn == "chan_logits":
        return fn, dict(B=a["B"], N=a["N"], T=a["T"], C=a["Cdim"], gh=a["gh"], gw=a["gw"], nh=a["nh"], nw=a["nw"])
    if fn == "gated_conv1x1":                               # its gating launch is mtt_gate_split over all its tasks
        return "gate_split", dict(B=a["B"], T=a["T"], N=a["N"], H=a["H"], C=a["Cdim"], gh=a["gh"], gw=a["gw"],
                                  nh=a["nh"], nw=a["nw"], x_group_rows=a["x_group_rows"],
                                  x_row_offset=a["x_row_offset"], ldx=a["x"].stride(-2), ntasks=len(a["tasks"]))
    if fn == "ctr_weights":
        return fn, dict(B=a["B"], H=a["H"], T=a["T"], N=a["N"])
    if fn == "ctr_mix":
        return fn, dict(T=a["T"], M=a["M"], Cdim=a["Cdim"], ld=a["ld"], rows_per_batch=a["rows_per_batch"],
                        accumulate=bool(a["accumulate"]))
    if fn == "bilinear":
        form = "nchw" if a["out_nchw"] is not None else ("split" if a["out_split"] is not None else "f32")
        ld_out = {"nchw": 0, "split": a["out_split"].ld if a["out_split"] is not None else 0,
                  "f32": a["out_f32"].stride(-2) if a["out_f32"] is not None else 0}[form]
        return fn, _bil(a["ld_in"], a["B"], a["h"], a["w"], a["Cdim"], a["H2"], a["W2"], form, ld_out=ld_out,
                        acc=bool(a["accumulate"]), ibr=a["in_batch_rows"], ioff=a["in_row_offset"],
                        obr=a["out_batch_rows"], ooff=a["out_row_offset"])
    if fn == "bilinear_postproc":
        return fn, dict(ld_in=a["ld_in"], B=a["B"], h=a["h"], w=a["w"], C=a["Cdim"], H2=a["H2"], W2=a["W2"],
                        kind=a["kind"])
    if fn == "nhwc_to_nchw":
        return fn, dict(ld_in=a["ld_in"], B=a["B"], Cd=a["Cd"], H=a["H"], W=a["W"])
    if fn == "zero_insert":
        return fn, dict(B=a["B"], h=a["h"], w=a["w"], Cdim=a["Cdim"], src_group=a["src_group"],
                        src_offset=a["src_offset"], ld_in=a["x"].stride(-2), ld_out=a["out"].ld)
    if fn == "split_rows":
        return fn, dict(rows=a["rows"], cols=a["cols"], in_group=a["in_group"], src_group=a["src_group"],
                        src_offset=a["src_offset"], ld_in=a["x"].stride(-2), ld_out=a["out"].ld)
    if fn == "layernorm_seg":
        return fn, dict(rows=a["rows"], cols=a["cols"], S=a["S"], in_group=a["in_group"], src_group=a["src_group"],
                        src_offset=a["src_offset"], seg_stride=a["seg_stride"], out_seg_stride=a["out_seg_stride"],
                        ld_in=a["x"].stride(-2), f32=a["out_f32"] is not None, split=a["out_split"] is not None)
    if fn == "dwconv3x3_s2":
        return fn, dict(B=a["B"], T=a["T"], h=a["h"], w=a["w"], Cdim=a["Cdim"], ld_in=a["x"].stride(-2),
                        ld_out=a["out"].ld)
    if fn == "avgpool":
        return fn, dict(BT=a["BT"], h=a["h"], w=a["w"], Cdim=a["Cdim"], s=a["s"], ld_in=a["x"].stride(-2),
                        ld_out=a["out"].ld)
    if fn == "invpt_fuse_softmax":
        so = a["score_out"]
        assert so is None or so.data_ptr() == a["raw"].data_ptr(), "score_out is written in place of raw"
        return fn, dict(B=a["B"], Lq=a["Lq"], Tk=a["Tk"], fused=a["prev_score"] is not None, T=a["T"], qh=a["qh"],
                        qw=a["qw"], score_out=so is not None, ldp=a["P"].ld)
    if fn == "bilinear_sum3":
        return fn, dict(B=a["B"], Cdim=a["Cdim"], H2=a["H2"], W2=a["W2"],
                        srcs=tuple((h, w, br, ro, t.stride(-2)) for t, h, w, br, ro in a["srcs"]))
    raise KeyError(fn)


RECORDED = ["im2col_patch", "broadcast_rows", "layernorm", "chan_logits", "gated_conv1x1", "ctr_weights", "ctr_mix",
            "bilinear", "bilinear_postproc", "nhwc_to_nchw", "zero_insert", "split_rows", "layernorm_seg",
            "dwconv3x3_s2", "avgpool", "invpt_fuse_softmax", "bilinear_sum3"]


def _frozen(d):
    return tuple(sorted(d.items()))


@pytest.mark.gpu
def test_plans_call_only_tabled_shapes(cuda_dev, monkeypatch):
    """Each benched plan at its bench batch runs one forward with pass-through recorders around the ops glue functions:
    every (function, shape arguments) pair it calls must be in TABLE, so a plan that starts calling a kernel at a new
    shape fails here instead of leaving the table (and the kernel tests built from it) stale."""
    import bench
    from mtt_b200 import ops

    seen = []
    for fn in RECORDED:
        orig = getattr(ops, fn)
        sig = inspect.signature(orig)

        def rec(*a, _fn=fn, _orig=orig, _sig=sig, **k):
            ba = _sig.bind(*a, **k)
            ba.apply_defaults()
            seen.append(_key_of_call(_fn, ba.arguments))
            return _orig(*a, **k)
        monkeypatch.setattr(ops, fn, rec)
    for name in BENCHED:
        g, tab = table(name)
        cfg, M, _ = bench.family(name)
        seen.clear()
        torch.manual_seed(0)
        with torch.device(cuda_dev):
            model = M.build_from_config(cfg, nsplit=2, use_graph=False).eval()
        with torch.no_grad():
            model(torch.randn(g.B, 3, *cfg["img_size"], device=cuda_dev))
        torch.cuda.synchronize()
        del model
        torch.cuda.empty_cache()
        want = {(fn, _frozen(d)) for fn, ds in tab.items() for d in ds}
        got = {(fn, _frozen(d)) for fn, d in seen}
        assert got, f"{name}: no glue call recorded"
        missing = sorted(got - want, key=str)
        assert not missing, f"{name}: the plan calls glue kernels at shapes the table does not hold: {missing[:6]}"
        print(f"{name}: {len(got)} distinct glue calls, all in the table ({len(want)} tabled)")


# ---- float64 references (device-agnostic: the CPU self-check runs them too) -----------------------------------------------
def rows_of(B, n, batch_rows, offset, device):
    """Physical rows of image b's n logical rows: b * batch_rows + offset + i."""
    return (torch.arange(B, device=device)[:, None] * batch_rows + offset + torch.arange(n, device=device)[None]).reshape(-1)


def fp32_scale(n, n2):
    """The kernels' resize scale: fp32(n) / fp32(n2), correctly rounded (computed on the host)."""
    return float(torch.tensor(n, dtype=torch.float32) / torch.tensor(n2, dtype=torch.float32))


def fp32_coords_exact(n, n2):
    """True when the fp32 scale equals n / n2 and every source coordinate scale (d + 0.5) - 0.5, d < n2, is exact in
    fp32 (power-of-two ratios, but also 384 -> 512): then float64 F.interpolate computes the kernel's coordinates."""
    sc = fp32_scale(n, n2)
    if sc != n / n2:
        return False
    p = sc * (torch.arange(n2, dtype=torch.float64) + 0.5)
    return bool(torch.equal(p.float().double(), p) and torch.equal((p - 0.5).float().double(), p - 0.5))


def ref_bilinear(x, rows, B, h, w, C, H2, W2):
    """NHWC rows `rows` of x (float64) resized to H2 x W2, align_corners=False: (y, the same resize of |x|), NCHW.
    Only where the fp32 coordinates are exact (ref_bilinear_any covers the other ratios)."""
    assert fp32_coords_exact(h, H2) and fp32_coords_exact(w, W2), \
        f"resize {h}x{w} -> {H2}x{W2}: the fp32 coordinates are not exact, so float64 F.interpolate is no reference " \
        f"for the kernel's; use ref_bilinear_any"
    img = x[rows, :C].reshape(B, h, w, C).permute(0, 3, 1, 2)
    it = lambda v: F.interpolate(v, size=(H2, W2), mode="bilinear", align_corners=False)
    return it(img), it(img.abs())


def _bil_axis(n, n2, device):
    """bilin_coord (postproc.cuh) along one axis in float64 from the kernel's fp32 scale: (i0, i1, l1, e_s). e_s is one
    ulp of the coordinate s = scale (d + 0.5) - 0.5: the fp32 rounding of the product and of the subtraction (or of the
    one fused multiply-add) is at most 2^-24 (|s| + 0.5) + 2^-24 |s| <= 2^-23 (|s| + 1); the clamp at 0 does not add."""
    s = fp32_scale(n, n2) * (torch.arange(n2, dtype=torch.float64, device=device) + 0.5) - 0.5
    e_s = 2.0 ** -23 * (s.abs() + 1)
    s = s.clamp(min=0)
    i0 = s.floor().long().clamp(max=n - 1)
    return i0, (i0 + 1).clamp(max=n - 1), s - i0, e_s


def _nbr_max(G, ry, rx):
    """max of G [B, C, h, w] over the rows ry x columns rx (lists of [H2] / [W2] index tensors, clamped): [B, C, H2, W2]."""
    h, w = G.shape[-2:]
    m = torch.stack([G[:, :, r.clamp(0, h - 1)] for r in ry]).amax(0)
    return torch.stack([m[..., c.clamp(0, w - 1)] for c in rx]).amax(0)


def ref_bilinear_any(x, rows, B, h, w, C, H2, W2):
    """ref_bilinear at any ratio: the interpolation in float64 at the coordinates the kernel derives from its fp32
    scale, (y, |.| resize, e_coord), NCHW. The kernel rounds each coordinate in fp32 (at most e_s off, _bil_axis); the
    resize is continuous and piecewise linear in each coordinate, so a coordinate off by e moves the value by at most
    e times the largest difference of neighbouring source values it can see: rows i0 - 1 .. i0 + 2 (the shifted
    coordinate may cross into the next cell) by columns j0 - 1 .. j0 + 2. e_coord is that term for both axes; the
    kernel's arithmetic on its own weights is E_BIL of the |.| resize, as with exact coordinates."""
    img = x[rows, :C].reshape(B, h, w, C).permute(0, 3, 1, 2)
    y0, y1, ly, ey = _bil_axis(h, H2, x.device)
    x0, x1, lx, ex = _bil_axis(w, W2, x.device)

    def it(v):
        r0, r1 = v[:, :, y0], v[:, :, y1]
        top = r0[..., x0] * (1 - lx) + r0[..., x1] * lx
        bot = r1[..., x0] * (1 - lx) + r1[..., x1] * lx
        return top * (1 - ly)[:, None] + bot * ly[:, None]

    gy = F.pad((img[:, :, 1:] - img[:, :, :-1]).abs(), (0, 0, 0, 1))
    gx = F.pad((img[..., 1:] - img[..., :-1]).abs(), (0, 1))
    dy = _nbr_max(gy, [y0 - 1, y0, y0 + 1], [x0 - 1, x0, x0 + 1, x0 + 2])
    dx = _nbr_max(gx, [y0 - 1, y0, y0 + 1, y0 + 2], [x0 - 1, x0, x0 + 1])
    return it(img), it(img.abs()), ey[:, None] * dy + ex[None, :] * dx


def ref_bilinear_kernel(x, rows, B, h, w, C, H2, W2):
    """(y, |.| resize, coordinate term): float64 F.interpolate with a zero coordinate term where the fp32 coordinates
    are exact, ref_bilinear_any elsewhere."""
    if fp32_coords_exact(h, H2) and fp32_coords_exact(w, W2):
        y, a = ref_bilinear(x, rows, B, h, w, C, H2, W2)
        return y, a, torch.zeros_like(y)
    return ref_bilinear_any(x, rows, B, h, w, C, H2, W2)


def ref_im2col(img, patch):
    B, Cin = img.shape[:2]
    return F.unfold(img, patch, stride=patch).transpose(1, 2).reshape(-1, Cin * patch * patch)


def ref_chan_logits(cp, x, B, T, C, gh, gw, nh, nw):
    """Rc[b,t,c,i,j] = sum over window (i, j) of cp[b,t,pix] x[b,pix,c]; x = the patch rows [B, P, C]."""
    wh, ww = gh // nh, gw // nw
    return torch.einsum("btihjw,bihjwc->btcij", cp.reshape(B, T, nh, wh, nw, ww), x.reshape(B, nh, wh, nw, ww, C))


def ref_gates(logits, rc, B, T, H, C, gh, gw, nh, nw, task):
    """(g_s, g_c) [B, P, C] of one task: the prompt's spatial logit of the pixel for the channel's head, and the task's
    channel logit of the pixel's window."""
    P = gh * gw
    gs = logits[:, :, task, T:].permute(0, 2, 1).repeat_interleave(C // H, dim=2)
    gc = rc[:, task].reshape(B, C, nh, 1, nw, 1).expand(B, C, nh, gh // nh, nw, gw // nw).reshape(B, C, P)
    return gs, gc.permute(0, 2, 1)


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


def ref_layernorm(x, gamma, beta, eps):
    return F.layer_norm(x, (x.shape[1],), gamma, beta, eps)


def ref_postproc(y, kind):
    """get_output (TP/utils/utils.py:27-63) of NCHW logits y: kind 0 argmax, 1 255 sigmoid, 2 255 softmax[1],
    3 (normalize + 1) 255 / 2 as [B,H,W,3], 4 clamp(min 0) as [B,H,W,1]."""
    if kind == 0:
        return y.argmax(1)
    if kind == 1:
        return 255 * torch.sigmoid(y[:, 0])
    if kind == 2:
        return 255 * torch.softmax(y[:, :2], 1)[:, 1]
    if kind == 3:
        return ((F.normalize(y[:, :3], dim=1) + 1) * 255 / 2).permute(0, 2, 3, 1)
    return y[:, :1].clamp(min=0).permute(0, 2, 3, 1)


# ---- sentinels --------------------------------------------------------------------------------------------------------------
_INT = {torch.float32: torch.int32, torch.bfloat16: torch.int16, torch.int64: torch.int64}
_SENT = {torch.float32: F32_SENT, torch.bfloat16: BF16_SENT, torch.int64: I64_SENT}


class Guarded:
    """A flat buffer filled with the sentinel of its dtype; `view` is the kernel's output inside it, `g` elements from
    either end. unchanged_outside(region) asserts every element outside `region` (index into `view`, or a bool mask of
    the flat buffer) still holds what it held before the call."""

    def __init__(self, shape, dtype, g=4096):
        n = math.prod(shape)
        self.flat = torch.empty(n + 2 * g, dtype=dtype, device="cuda")
        self.flat.view(_INT[dtype]).fill_(_SENT[dtype])
        self.g, self.n = g, n
        self.view = self.flat[g:g + n].view(shape)

    def snapshot(self):
        self.before = self.flat.clone()

    def unchanged_outside(self, region, what):
        torch.cuda.synchronize()
        written = torch.zeros(self.flat.shape, dtype=torch.bool, device="cuda")
        if isinstance(region, torch.Tensor) and region.dtype == torch.bool and region.shape == self.flat.shape:
            written = region
        else:
            written[self.g:self.g + self.n].view(self.view.shape)[region] = True
        it = _INT[self.flat.dtype]
        same = self.flat.view(it)[~written] == self.before.view(it)[~written]
        assert bool(same.all()), f"{what}: {int((~same).sum())} elements outside the output changed"


def guarded_split(ops, ns, rows, cols, ld=None, g=16):
    """A Split [rows, cols] of ns planes inside a 2-plane bf16 buffer with g sentinel rows around each plane, padding
    columns up to ld and (ns = 1) a whole sentinel second plane. Returns (Guarded, Split, region of the planes)."""
    ld = round_up(cols, 8) if ld is None else ld
    gb = Guarded((2, rows + 2 * g, ld), torch.bfloat16, g=64)
    sp = ops.Split.from_planes(gb.view[:ns, g:g + rows], cols)
    return gb, sp, (slice(0, ns), slice(g, g + rows), slice(0, cols))


def planes_value(sp):
    """float64 value the planes hold (hi + lo, or hi alone)."""
    v = sp.buf[0, :, :sp.cols].double()
    if sp.nsplit == 2:
        v = v + sp.buf[1, :, :sp.cols].double()
    return v


def split_bound(ns, mag):
    """What storing a value of magnitude mag as planes adds: SPLIT |x| + SPLIT_ABS (hi + lo) or HI |x| + HI_ABS (hi)."""
    return SPLIT * mag + SPLIT_ABS if ns == 2 else HI * mag + HI_ABS


def check_planes(sp, ref, e, what):
    """|planes - ref| <= e (the fp32 computation's bound) + the split bound of the stored value."""
    return check(planes_value(sp), ref, e + split_bound(sp.nsplit, ref.abs() + e), f"{what} (nsplit={sp.nsplit})")


def split_bits(x, ns):
    """The planes the kernels write for fp32 x: hi = bf16(x) (round to nearest even), lo = bf16(x - hi)."""
    hi = x.bfloat16()
    return (hi,) if ns == 1 else (hi, (x - hi.float()).bfloat16())


def assert_planes_bit_exact(sp, x, what):
    for i, p in enumerate(split_bits(x, sp.nsplit)):
        assert torch.equal(sp.buf[i, :, :sp.cols].view(torch.int16), p.view(torch.int16)), f"{what}: plane {i} differs"


def report(name, ratios):
    print(f"{name}: worst error / bound = {max(ratios):.3f}")


def gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def randn(g, *shape, scale=1.0):
    return torch.randn(*shape, generator=g, device="cuda") * scale


@pytest.fixture(scope="module")
def ops(cuda_dev):
    import mtt_b200  # noqa: F401
    from mtt_b200 import ops as o
    return o


# ---- data movement: bit-exact ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,ns", _cases("im2col_patch"))
@pytest.mark.gpu
def test_im2col_patch(ops, name, ns):
    """Patch im2col of the whole input batch: planes bit-exact against the split of F.unfold (column order c, ky, kx)."""
    g, tab = table(name)
    for d in tab["im2col_patch"]:
        img = randn(gen(1), *d["shape"])
        rows = d["shape"][0] * g.P
        gb, sp, reg = guarded_split(ops, ns, rows, d["ld"], ld=d["ld"])
        gb.snapshot()
        ops.im2col_patch(img, d["patch"], sp)
        gb.unchanged_outside(reg, "im2col_patch")
        assert_planes_bit_exact(sp, ref_im2col(img, d["patch"]), "im2col_patch")


@pytest.mark.parametrize("name", BENCHED)
@pytest.mark.gpu
def test_broadcast_rows_and_nhwc_to_nchw(ops, name):
    """Prompt / cls rows broadcast into every image's group of the joint stream (the patch rows stay as they were), and
    the 3ddet map's NHWC -> NCHW copy: bit-exact."""
    g, tab = table(name)
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


@pytest.mark.parametrize("name,ns", _cases("zero_insert"))
@pytest.mark.gpu
def test_zero_insert_and_split_rows(ops, name, ns):
    """InvPT's scale_embed inputs from the patch rows of the joint stream (row 0 of each image is the cls token):
    zero insertion for the transposed conv and the plain row gather, planes bit-exact."""
    g, tab = table(name)
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
def _ln_input(g, rows, cols):
    """Rows of std 0.5 around a per-row offset: a quarter at 25 (50 x their std: the two-pass variance's cancellation)."""
    x = randn(g, rows, cols, scale=0.5)
    off = torch.zeros(rows, 1, device="cuda")
    off[::4] = 25.0
    off[1::4] = -3.0
    return x + off


def _ln_bound(xd, gam, bet, eps, D):
    """Elementwise bound of LayerNorm in fp32 (test_train_kernels_f64_gpu's model): mean and the centred sum of squares
    are reductions of depth D, rstd = 1 / sqrt(var + eps) adds 3u, y = (x - mean) rstd gamma + beta 4u."""
    n = xd.shape[1]
    mean, var = xd.mean(1, keepdim=True), xd.var(1, unbiased=False, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + eps)
    xh = (xd - mean) * rstd
    e_mean = sum_tol(D, xd.abs().sum(1, keepdim=True)) / n + U * mean.abs()
    e_var = sum_tol(D, ((xd - mean) ** 2).sum(1, keepdim=True)) / n + 3 * U * var + e_mean ** 2
    e_rr = 0.5 * e_var / (var + eps) + 3 * U
    e_xh = e_mean * rstd + xh.abs() * (e_rr + 2 * U)
    y = xh * gam + bet
    return y, gam.abs() * e_xh + 4 * U * ((xh * gam).abs() + y.abs())


@pytest.mark.parametrize("name", [n for n in BENCHED if table(n)[1].get("layernorm")])
@pytest.mark.gpu
def test_layernorm(ops, name):
    """mtt_layernorm at the plans' rows x widths: TaskPrompter's final norm (C = 1024 / 768: the register path) and
    InvPT's per-stage norm1 (C = 576 / 288 / 144, up to 81920 rows: the general path), fp32 out with ld = C."""
    g, tab = table(name)
    report(f"layernorm {name}", [layernorm_case(ops, d, 10 + i) for i, d in enumerate(tab["layernorm"])])


def layernorm_case(ops, d, seed, ns=2):
    """One mtt_layernorm call of a table (rows x cols, input ld): fp32 out (ld = ld_in) or split out (ns planes)."""
    rows, cols = d["rows"], d["cols"]
    gg = gen(seed)
    x = torch.full((rows, d["ld_in"]), float("nan"), device="cuda")[:, :cols]      # NaN input pad columns
    x.copy_(_ln_input(gg, rows, cols))
    gam, bet = torch.rand(cols, generator=gg, device="cuda") + 0.5, randn(gg, cols, scale=0.5)
    eps = 1e-6
    fast = cols % 128 == 0 and cols <= 1024
    D = (cols // 128 + 7) if fast else (math.ceil(cols / 32) + 5)   # per-lane serial chain + 5 shuffle levels
    want, e = _ln_bound(x.double(), gam.double(), bet.double(), eps, D)
    assert torch.allclose(want, ref_layernorm(x.double(), gam.double(), bet.double(), eps), rtol=1e-12, atol=1e-12)
    if d.get("split"):
        gb, sp, reg = guarded_split(ops, ns, rows, cols)
        gb.snapshot()
        ops.layernorm(x, gam, bet, eps, out_split=sp)
        gb.unchanged_outside(reg, "layernorm split")
        return check_planes(sp, want, e, f"layernorm {rows}x{cols} split (LN bound, D={D})")
    gb = Guarded((rows, d["ld_in"]), torch.float32)
    gb.snapshot()
    ops.layernorm(x, gam, bet, eps, out_f32=gb.view)
    gb.unchanged_outside((slice(None), slice(0, cols)), "layernorm")
    return check(gb.view[:, :cols], want, e, f"layernorm {rows}x{cols} (LN bound, D={D})")


@pytest.mark.parametrize("name,ns", _cases("layernorm_seg"))
@pytest.mark.gpu
def test_layernorm_seg(ops, name, ns):
    """ViT final norm over the gathered patch rows (S = 1) and InvPT's joint-channel norm over all T tasks' slices
    (S = T segments, statistics over T * C values) with the per-task output rows; fp32 or split out as the plan has it."""
    g, tab = table(name)
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
        x[segs.reshape(-1), :cols] = _ln_input(gg, rows, S * cols).reshape(rows * S, cols)
        gam, bet = torch.rand(S * cols, generator=gg, device="cuda") + 0.5, randn(gg, S * cols, scale=0.5)
        eps = 1e-6
        orows = (torch.arange(S, device="cuda")[None] * d["out_seg_stride"] + torch.arange(rows, device="cuda")[:, None])
        n_out = S * rows if d["out_seg_stride"] else rows
        xd = x.double()[segs.reshape(-1), :cols].reshape(rows, S * cols)
        want, e = _ln_bound(xd, gam.double(), bet.double(), eps, S * math.ceil(cols / 32) + 5)
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
            v = planes_value(sp)[o]
            ratios.append(check(v, want, e + split_bound(ns, want.abs() + e),
                                f"layernorm_seg S={S} {rows}x{cols} split ns={ns} (LN bound + split bound)"))
    if ratios:
        report(f"layernorm_seg {name} ns={ns}", ratios)


# ---- channel-prompt logits, gating, cross-task reweighting ---------------------------------------------------------------------
@pytest.mark.parametrize("name,ns", _cases("chan_logits"))
@pytest.mark.gpu
def test_chan_logits(ops, name, ns):
    """Rc[b,t,c,window] = sum over the window's pixels of cp[b,t,pix] xn[b,T+pix,c], xn as LN1's split planes (one or
    two): 1 window of 32 x 32 (tp_cfg4), 4 x 4 windows of 7 x 9 (tp_cfg2), one 64 x 128 window whose cp slice needs
    ~111 KB of dynamic shared memory (tp_cfg5)."""
    g, tab = table(name)
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
        X = planes_value(xn).view(B, N, C)[:, T:]
        cpd = cp.double()
        want = ref_chan_logits(cpd, X, B, T, C, gh, gw, nh, nw)
        absum = ref_chan_logits(cpd.abs(), X.abs(), B, T, C, gh, gw, nh, nw)
        wp = (gh // nh) * (gw // nw)
        D = math.ceil(wp / 32) + 32                # serial fma over the block's pixel group, then 32 partials in order
        r = check(gb.view, want, sum_tol(D, absum), f"chan_logits {name} (sum_tol D={D})")
        report(f"chan_logits {name} ns={ns}", [r])


@pytest.mark.parametrize("name,ns", _cases("gate_split"))
@pytest.mark.gpu
def test_gate_split(ops, name, ns):
    """Spatial and channel gating of all T tasks in one launch, X = the patch rows of the joint stream (x rows offset by
    T inside groups of N), written task after task into the gated-conv workspace layout (task_stride); the slack of
    each 256-byte aligned plane set and the space after the last task stay untouched."""
    g, tab = table(name)
    for d in tab["gate_split"]:
        report(f"gate_split {name} ns={ns}", gate_case(ops, d, ns, name))


def gate_case(ops, d, ns, name, seed=40):
    """One gating launch of a table entry (the gating stage of gated_conv1x1: all its tasks, x rows of image b at
    b * x_group_rows + x_row_offset); err / bound ratios per task and gate."""
    B, T, N, H, C, gh, gw, nh, nw = (d[k] for k in ("B", "T", "N", "H", "C", "gh", "gw", "nh", "nw"))
    xg, xo = d["x_group_rows"], d["x_row_offset"]
    P, rows, ldy = gh * gw, B * gh * gw, round_up(C, 8)
    gg = gen(seed)
    x = randn(gg, B * xg, d["ldx"])
    logits = randn(gg, B, H, T, N, scale=1.5)
    rc = randn(gg, B, T, C, nh, nw, scale=1.5)
    pbe = round_up(ns * rows * ldy * 2, 256) // 2        # elements of one task's ys (or yc) plane set
    gb = Guarded((2 * T + 1, pbe), torch.bfloat16)        # one spare plane set after the last task
    flat = gb.view.reshape(-1)
    ys = ops.Split.from_planes(flat[:ns * rows * ldy].view(ns, rows, ldy), C)
    yc = ops.Split.from_planes(flat[pbe:pbe + ns * rows * ldy].view(ns, rows, ldy), C)
    gb.snapshot()
    ops.gate_split(x, xg, xo, logits, rc, 0, ys, yc, B=B, T=T, N=N, H=H, Cdim=C, gh=gh, gw=gw, nh=nh, nw=nw,
                   ntasks=d["ntasks"], task_stride=2 * pbe)
    gb.unchanged_outside((slice(0, 2 * T), slice(0, ns * rows * ldy)), "gate_split")
    X = x.double()[rows_of(B, P, xg, xo, "cuda"), :C].view(B, P, C)
    ratios = []
    for t in range(T):
        gs, gc = ref_gates(logits.double(), rc.double(), B, T, H, C, gh, gw, nh, nw, t)
        for which, gate in ((0, gs), (1, gc)):
            want = (X * (1 + gate)).reshape(rows, C)
            e = 2 * U * (X.abs() * (1 + gate).abs()).reshape(rows, C)      # fl(1 + g), then the product
            k = 2 * t + which
            sp = ops.Split.from_planes(gb.view[k, :ns * rows * ldy].view(ns, rows, ldy), C)
            ratios.append(check_planes(sp, want, e, f"gate_split {name} task {t} {'Yc' if which else 'Ys'} (2u)"))
    return ratios


@pytest.mark.parametrize("name", [n for n in BENCHED if table(n)[1].get("ctr_mix")])
@pytest.mark.gpu
def test_ctr_weights_and_mix(ops, name):
    """Cross-task reweighting: w[b,t,j] = W2_t . gelu(W0_t R[b,:,t,j] + b0_t) + b2_t over H heads, then
    acc[t] (+)= sum_j w[b,t,j] F[j] over all ld columns (the header: C = ld, the padding columns carry 0 + 0 and are
    checked like the rest), accumulate off then on."""
    g, tab = table(name)
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
    report(f"ctr {name}", ratios)


# ---- bilinear ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,ns", _cases("bilinear"))
@pytest.mark.gpu
def test_bilinear(ops, name, ns):
    """Every bilinear resize the plan runs, in its form: NHWC split (both planes, even C, no fp32 out: the FAST form; one
    plane: the vectorised general form) for the decoder's x4 up-sampling (C = 350 / 768, two pairs per lane, a partial
    last chunk), InvPT's 32 -> 16 downsample of the final tokens and its UpEmbed x2 with in_row_offset; NHWC fp32
    accumulate with in / out row offsets (InvPT's attention output into each task's slice); NCHW to the image size."""
    g, tab = table(name)
    ratios = [bilinear_case(ops, d, ns, 60 + i) for i, d in enumerate(tab["bilinear"])
              if d["form"] == "split" or ns == 2]
    if ratios:
        report(f"bilinear {name} ns={ns}", ratios)


def bilinear_case(ops, d, ns, seed):
    """One bilinear call of a table (_bil fields) in its output form, inside sentinels; its err / bound ratio. The
    bound is E_BIL of the |.| resize plus, at a ratio whose fp32 coordinates are inexact, ref_bilinear_any's coordinate
    term."""
    B, h, w, C, H2, W2 = d["B"], d["h"], d["w"], d["C"], d["H2"], d["W2"]
    ibr = d["ibr"] or h * w
    nin = (B - 1) * ibr + d["ioff"] + h * w
    x = randn(gen(seed), nin, d["ld_in"])
    rin = rows_of(B, h * w, ibr, d["ioff"], "cuda")
    want, absr, ec = ref_bilinear_kernel(x.double(), rin, B, h, w, C, H2, W2)
    what = f"bilinear {h}x{w}->{H2}x{W2} C={C} {d['form']} ioff={d['ioff']} ooff={d['ooff']}"
    kw = dict(in_batch_rows=d["ibr"], in_row_offset=d["ioff"], out_batch_rows=d["obr"], out_row_offset=d["ooff"])
    if d["form"] == "nchw":
        gb = Guarded((B, C, H2, W2), torch.float32)
        gb.snapshot()
        ops.bilinear(x, d["ld_in"], B, h, w, C, H2, W2, out_nchw=gb.view, **kw)
        gb.unchanged_outside((slice(None),), what)
        return check(gb.view, want, E_BIL * absr + ec, f"{what} (6u of the |.| resize + coordinate term)")
    obr = d["obr"] or H2 * W2
    nout = (B - 1) * obr + d["ooff"] + H2 * W2
    rout = rows_of(B, H2 * W2, obr, d["ooff"], "cuda")
    wn = want.permute(0, 2, 3, 1).reshape(-1, C)
    an = (E_BIL * absr + ec).permute(0, 2, 3, 1).reshape(-1, C)
    if d["form"] == "f32":
        gb = Guarded((nout, d["ld_out"]), torch.float32)
        base = randn(gen(seed + 30), nout, d["ld_out"])
        gb.view.copy_(base)
        gb.snapshot()
        ops.bilinear(x, d["ld_in"], B, h, w, C, H2, W2, out_f32=gb.view, accumulate=d["acc"], **kw)
        gb.unchanged_outside((rout, slice(0, C)), what)
        old = base.double()[rout, :C] if d["acc"] else 0
        ref = wn + old
        return check(gb.view[rout, :C], ref, an + U * ref.abs(), f"{what} (6u + u of the sum)")
    gb, sp, reg = guarded_split(ops, ns, nout, C, ld=d["ld_out"])
    gb.snapshot()
    ops.bilinear(x, d["ld_in"], B, h, w, C, H2, W2, out_split=sp, **kw)
    region = torch.zeros(gb.view.shape, dtype=torch.bool, device="cuda")
    region[:ns, 16 + rout, :C] = True
    gb.unchanged_outside(region, what)
    return check(planes_value(sp)[rout], wn, an + split_bound(ns, wn.abs() + an), f"{what} ns={ns} (6u + split bound)")


@pytest.mark.parametrize("name,ns", _cases("bilinear_sum3"))
@pytest.mark.gpu
def test_bilinear_sum3(ops, name, ns):
    """InvPT's multi-scale aggregation: the three stages' maps (16², 32², 64², the first one a task's slice of the joint
    LayerNorm output) resized to 128 x 128 and summed, written once as split planes (C = 576: 5 chunks of 128 channels,
    half the pairs of the last one idle)."""
    g, tab = table(name)
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
    report(f"bilinear_sum3 {name} ns={ns}", ratios)


@pytest.mark.parametrize("name", [n for n in BENCHED if table(n)[1].get("bilinear_postproc")])
@pytest.mark.gpu
def test_bilinear_postproc(ops, name):
    """The final resize fused with get_output at full output size, for each task's kind: argmax over 21 / 7 / 40 / 19
    classes, 255 sigmoid, 255 softmax[1], normalised normals, clamped depth. A class must be exact wherever the float64
    top-2 margin exceeds twice the value bound, and one of the tied classes elsewhere."""
    g, tab = table(name)
    ratios = [postproc_case(ops, d, 120 + i) for i, d in enumerate(tab["bilinear_postproc"])]
    ratios = [r for r in ratios if r is not None]
    if ratios:
        report(f"bilinear_postproc {name}", ratios)


def postproc_case(ops, d, seed):
    """One bilinear_postproc call of a table; its err / bound ratio (None for the argmax, which is checked exactly
    where the top-2 margin is clear)."""
    B, h, w, C, H2, W2, kind = (d[k] for k in ("B", "h", "w", "C", "H2", "W2", "kind"))
    x = randn(gen(seed), B * h * w, d["ld_in"], scale=3.0)
    y, ya, ec = ref_bilinear_kernel(x.double(), torch.arange(B * h * w, device="cuda"), B, h, w, C, H2, W2)
    ev = E_BIL * ya + ec                                         # bound of each resized logit
    shape = {0: (B, H2, W2), 3: (B, H2, W2, 3), 4: (B, H2, W2, 1)}.get(kind, (B, H2, W2))
    gb = Guarded(shape, torch.int64 if kind == 0 else torch.float32)
    gb.snapshot()
    ops.bilinear_postproc(x, d["ld_in"], B, h, w, C, H2, W2, kind, gb.view)
    gb.unchanged_outside((slice(None),), f"bilinear_postproc kind {kind}")
    what = f"bilinear_postproc {h}x{w}->{H2}x{W2} kind {kind} C={C}"
    got = gb.view
    if kind == 0:
        top2 = y.topk(2, dim=1)
        margin = top2.values[:, 0] - top2.values[:, 1]
        emax = ev.amax(1)
        clear = margin > 2 * emax
        assert torch.equal(got[clear], top2.indices[:, 0][clear]), f"{what}: class off where the top-2 margin is clear"
        picked = y.gather(1, got.clamp(0, C - 1)[:, None])[:, 0]
        assert ((got >= 0) & (got < C)).all() and (picked >= top2.values[:, 0] - 2 * emax).all(), \
            f"{what}: class outside the tied set"
        print(f"{what}: {int((~clear).sum())} of {clear.numel()} pixels within the tie margin")
        return None
    want = ref_postproc(y, kind)
    if kind == 1:        # sigmoid' <= 1/4; expf, 1 +, reciprocal and * 255: 6u
        e = 255 * 0.25 * ev[:, 0] + 6 * U * want.abs()
    elif kind == 2:      # d softmax[1] / d x_c <= 1/4 each; two expf, a sum, a division, * 255: 8u
        e = 255 * 0.25 * (ev[:, 0] + ev[:, 1]) + 8 * U * want.abs()
    elif kind == 3:      # d (x / |x|) moves by at most 2 |e| / |x|; sqrt, divisions, + 1, * 255 / 2: 8u of 255
        n = y[:, :3].norm(dim=1, keepdim=True).clamp_min(1e-12)
        e = (255 / 2 * 2 * ev[:, :3].norm(dim=1, keepdim=True) / n + 8 * U * 255).permute(0, 2, 3, 1).expand_as(want)
    else:                # clamp is exact
        e = ev[:, :1].permute(0, 2, 3, 1)
    return check(got, want, e, f"{what} (logit bound through the post-processing)")


# ---- InvPT token reductions and cross-task attention softmax -------------------------------------------------------------------
@pytest.mark.parametrize("name,ns", _cases("dwconv3x3_s2"))
@pytest.mark.gpu
def test_dwconv_and_avgpool(ops, name, ns):
    """Per-stage Q and KV token reductions at C = 576 / 288 / 144 (256-, 256- and 128-thread blocks, ragged channel
    loops): per-task depthwise 3x3 stride-2 conv (bias + 9 fma) against F.conv2d(groups=C), and the s x s average pool
    (s = 2 / 4 / 8) against F.avg_pool2d(ceil_mode=True)."""
    g, tab = table(name)
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
    report(f"dwconv/avgpool {name} ns={ns}", ratios)


@pytest.mark.parametrize("name,ns", _cases("invpt_fuse_softmax"))
@pytest.mark.gpu
def test_invpt_fuse_softmax(ops, name, ns):
    """The step between InvPT's two attention GEMMs at every stage: Tk = 320 keys (10 per lane), Lq = 320 / 1280 / 5120
    queries, cross-scale fusion with the previous stage's fused score (x2 bilinear per task over the query grid) at stages
    1 and 2, the fused score written in place of the raw one (stages 0 and 1), P = softmax as split rows."""
    g, tab = table(name)
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
    report(f"invpt_fuse_softmax {name} ns={ns}", ratios)


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
    close(_ln_bound(x.double(), gam.double(), bet.double(), 1e-6, 5)[0], o, "layernorm (bound builder)")
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
    """The table derives for every benched config, holds only power-of-two resizes, and reaches the shapes the kernel
    tests are about (the 64 x 128 channel window, Tk = 320 at every InvPT stage)."""
    for name in BENCHED:
        g, tab = table(name)
        for d in tab["bilinear"]:
            assert_pow2_ratio(d["h"], d["H2"])
            assert_pow2_ratio(d["w"], d["W2"])
        for d in tab.get("bilinear_postproc", []):
            assert_pow2_ratio(d["h"], d["H2"])
            assert_pow2_ratio(d["w"], d["W2"])
    assert table("tp_cfg5")[1]["chan_logits"][0]["gh"] * table("tp_cfg5")[1]["chan_logits"][0]["gw"] == 8192
    assert [d["Tk"] for d in table("ip_cfg3")[1]["invpt_fuse_softmax"]] == [320, 320, 320]
