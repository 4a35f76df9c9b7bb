"""What the plans launch: the runs the float64 suites cover (RUNS), their geometries, the key of each recorded ops
call, and the recorder.

A plan test runs a forward with pass-through recorders around some ops functions (recording) and turns each call into a
hashable key, so the calls can be compared with a table derived from the config (glue_key) or replayed on fresh buffers
(test_tensor_core_f64_gpu.call_key)."""
import contextlib
import inspect
import math
import sys

import pytest

from f64_checks import round_up
from oracle import configs


def frozen(d):
    return tuple(sorted(d.items()))


# ---- the runs -------------------------------------------------------------------------------------------------------------
def bench_batch(name):
    import bench
    return bench.DEFAULT_BATCH[name]


BENCHED = ["tp_cfg4", "tp_cfg2", "tp_cfg5", "ip_cfg3", "tps_swinB"]
VAL_BATCH = 6            # valBatch of every ViT yml of the reference (TP/configs/**, IP/configs/**)
LAST_PASCAL_BATCH = 5    # the ragged last validation batch of PASCAL-Context: 5105 images = 850 x 6 + 5
TR_BATCH = 2             # trBatch of the same ymls
SWIN_VAL_BATCH = 4       # valBatch of cs_swinB_taskprompter.yml


def _runs():
    """(config, batch, mode) of every run the float64 suites cover. mode: "forward" (model(x); for a Swin model also
    model.backbone(x)), "predict" (model.predict(x)) or "train" (one TrainStep forward and reverse pass). The bench
    configs at the bench batch; the reference's own model configs (and those of tp_cfg4 = pascal_vitLp16_taskprompter,
    ip_cfg3 = InvPT pascal_vitLp16, tps_swinB3d = cs_swinB_taskprompter) at its validation and training batches: the
    batch sets every GEMM's row count, its tile count and stream-K split, and the trip counts of the glue kernels."""
    runs = []
    for name in BENCHED:
        # a ViT TaskPrompter with the '3ddet' task has no predict(): get_output is not defined for '3ddet' (plans.py)
        vit_det = name.startswith("tp_") and "3ddet" in configs.taskprompter(name)["tasks"]
        modes = ("forward",) if vit_det else ("forward", "predict")
        runs += [(name, bench_batch(name), m) for m in modes]
    runs += [("tps_swinB3d", 1, m) for m in ("forward", "predict")]
    runs += [(name, 4, "train") for name in ("tp_cfg4", "tp_cfg2")]
    for name in ("tp_nyud_vitL", "tp_pascal_vitB", "ip_nyud_vitL", "tp_cfg4", "ip_cfg3"):
        runs += [(name, VAL_BATCH, m) for m in ("forward", "predict")]
    for name in ("tp_cfg4", "tp_pascal_vitB", "ip_cfg3"):
        runs += [(name, LAST_PASCAL_BATCH, m) for m in ("forward", "predict")]
    runs.append(("tps_swinB3d", SWIN_VAL_BATCH, "predict"))
    runs += [(name, TR_BATCH, "train") for name in ("tp_cfg4", "tp_pascal_vitB", "tp_nyud_vitL")]
    assert len(set(runs)) == len(runs)
    return runs


RUNS = _runs()
# the batch each config was first tested at: its runs there keep the config name alone as their test id
_FIRST_BATCH = {"tp_cfg4": 4, "tp_cfg2": 4, "tp_cfg5": 1, "ip_cfg3": 4, "tps_swinB": 1, "tps_swinB3d": 1}


def run_id(name, B):
    """The test id of a run: the config and the batch (tp_pascal_vitB-b6); the config alone at its first batch."""
    return name if _FIRST_BATCH.get(name) == B else f"{name}-b{B}"


def runs(modes, family=None):
    """The distinct (config, batch) of the runs in `modes`, in RUNS order; family: the config name prefix ("tp_", "ip_",
    "tps_") or a tuple of them."""
    out = []
    for name, B, m in RUNS:
        if m in modes and (family is None or name.startswith(family)) and (name, B) not in out:
            out.append((name, B))
    return out


# ---- geometry ------------------------------------------------------------------------------------------------------------
class TPGeom:
    """A TaskPrompter (ViT) forward or training step at batch B (default: the bench batch, bench.DEFAULT_BATCH)."""

    def __init__(self, name, B=None):
        cfg = configs.taskprompter(name)
        self.name, self.cfg = name, cfg
        self.B = bench_batch(name) if B is None else B
        self.tasks, self.T = list(cfg["tasks"]), len(cfg["tasks"])
        self.img = tuple(cfg["img_size"])
        self.patch = cfg["patch"]
        self.gh, self.gw = self.img[0] // self.patch, self.img[1] // self.patch
        self.P = self.gh * self.gw
        self.N = self.T + self.P
        self.C, self.H = cfg["C"], cfg["heads"]
        self.dh = self.C // self.H
        self.nh = self.nw = int(round(math.sqrt(cfg["chan_nheads"])))
        self.e, self.f = cfg["e"], cfg["f"]
        self.e_ld, self.f_ld = round_up(self.e, 8), round_up(self.f, 8)
        self.use_ctr = cfg["use_ctr"]
        self.h4, self.w4 = 4 * self.gh, 4 * self.gw      # ConvHead: predictions at 4x the token grid
        self.M4 = self.B * self.h4 * self.w4             # rows of the heads' mt_proj.1 BatchNorm
        self.Mp = self.B * self.P                        # rows of the decoder's fea_fuse.*.2 BatchNorm (token grid)
        self.out_hw = tuple(cfg.get("dd_label_map_size", self.img))
        self.n_out = dict(cfg["num_output"])


class IPGeom:
    """An InvPT forward at batch B (default: the bench batch) (invpt.py _Plan)."""

    def __init__(self, name, B=None):
        cfg = configs.invpt(name)
        self.name, self.cfg = name, cfg
        self.B = bench_batch(name) if B is None else B
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


DET = "3ddet"
STRIDES = (8, 16, 32, 32)           # Swin decoder level il at 1 / STRIDES[il] of the full image (before img_ds_ratio)


class SwinGeom:
    """One Swin TaskPrompter forward at batch B, from its config: stages, decoder levels, head and output sizes."""

    def __init__(self, name, B=1):
        cfg = configs.taskprompter_swin(name)
        self.name, self.cfg, self.B = name, cfg, B
        self.tasks = list(cfg["tasks"])
        self.T = len(self.tasks)
        self.t2 = [t for t in self.tasks if t != DET]
        self.img = tuple(cfg["img_size"])
        r = cfg["img_ds_ratio"]
        self.ds = tuple(int(s * r) for s in self.img)
        self.patch, E = cfg["patch"], cfg["embed_dim"]
        self.E = E
        gh, gw = self.ds[0] // self.patch, self.ds[1] // self.patch
        self.ce, self.nh = cfg["chan_embed_dim"], int(round(math.sqrt(cfg["chan_nheads"])))
        self.stages = []
        for i, (depth, heads) in enumerate(zip(cfg["depths"], cfg["heads"])):
            H, W = gh >> i, gw >> i
            ws, shift = cfg["window"], cfg["window"] // 2
            if min(H, W) <= ws:                               # the window clipped to the map, no shift
                ws, shift = min(H, W), 0
            Hp, Wp = -(-H // ws) * ws, -(-W // ws) * ws
            self.stages.append(dict(H=H, W=W, L=H * W, C=E << i, heads=heads, ws=ws, nW=(Hp // ws) * (Wp // ws),
                                    shifts=[0 if j % 2 == 0 else shift for j in range(depth)], depth=depth))
        self.f, self.Lv = cfg["f"], cfg["level_embed_dim"]
        self.f_ld = round_up(self.f, 8)
        chans = [2 * E, 4 * E, 8 * E, 8 * E]
        self.levels = [dict(h=int(self.img[0] // s * r), w=int(self.img[1] // s * r), C=chans[il],
                            heads=self.stages[il]["heads"]) for il, s in enumerate(STRIDES)]
        self.fh, self.fw = 2 * self.levels[0]["h"], 2 * self.levels[0]["w"]
        k = 2 if cfg.get("head", "conv") == "deconv" else 1
        self.ph, self.pw = k * self.fh, k * self.fw            # the head's prediction map
        self.out_hw = tuple(cfg.get("dd_label_map_size", self.img))
        self.n_out = dict(cfg["num_output"])


# ---- the key of a glue call ------------------------------------------------------------------------------------------------
def bil(ld_in, B, h, w, C, H2, W2, form, ld_out=0, acc=False, ibr=0, ioff=0, obr=0, ooff=0):
    """The table entry of one bilinear call."""
    return dict(ld_in=ld_in, B=B, h=h, w=w, C=C, H2=H2, W2=W2, form=form, ld_out=ld_out, acc=acc, ibr=ibr, ioff=ioff,
                obr=obr, ooff=ooff)


def glue_key(fn, a):
    """The table entry (function, shape arguments) of one ops.<fn> call, a = its bound arguments (defaults applied)."""
    if fn == "im2col_patch":
        return fn, dict(shape=tuple(a["img"].shape), patch=a["patch"], ld=a["out"].ld)
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
        return fn, bil(a["ld_in"], a["B"], a["h"], a["w"], a["Cdim"], a["H2"], a["W2"], form, ld_out=ld_out,
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
    if fn == "split_f32":
        x, o = a["x"], a["out"]
        assert a["cols_pad"] in (None, x.shape[1])
        return fn, dict(rows=x.shape[0], cols=x.shape[1], ld_in=x.stride(0), ld_out=o.ld)
    if fn in ("swin_window_gather", "swin_window_scatter"):
        d = dict(B=a["B"], H=a["H"], W=a["W"], C=a["Cdim"], T=a["T"], ws=a["ws"], shift=a["shift"])
        if fn == "swin_window_gather":
            return fn, dict(d, ldx=a["xn"].stride(0), ldp=a["pn"].stride(0), ld_out=a["out"].ld)
        return fn, dict(d, heads=a["heads"], last=bool(a["last"]), ldo=a["o32"].stride(0), ldxa=a["xa"].stride(0),
                        ldx=a["x"].stride(0), ldp=a["p"].stride(0))
    if fn == "swin_window_attention":
        return fn, dict(BW=a["BW"], nW=a["nW"], T=a["T"], L=a["L"], heads=a["heads"], C=a["out"].cols,
                        scale=a["scale"], masked=a["maskT"] is not None, ldq=a["qkv"].ld, ldo=a["out"].ld)
    if fn == "transpose_split":
        return fn, dict(B=a["B"], L=a["L"], C=a["Cdim"], ld_in=a["x"].stride(0), ld_out=a["out"].ld)
    if fn == "swin_chan_attention":
        return fn, dict(B=a["B"], T=a["T"], C=a["Cdim"], ce=a["ce"], nh=a["nh"], nw=a["nw"], ldq=a["q"].stride(0),
                        ldkv=a["kv"].stride(0), ldco=a["co32"].stride(0), ldcs=a["cos"].ld)
    if fn == "swin_merge_gather":
        return fn, dict(B=a["B"], H=a["H"], W=a["W"], C=a["Cdim"], ldx=a["x"].stride(0), ldo=a["out"].stride(0))
    if fn == "conv3x3_s2_maps":
        return fn, dict(B=a["B"], Cin=a["Cin"], Cout=a["w"].shape[0], H=a["H"], W=a["W"], in_stride=a["in_stride"],
                        in_offset=a["in_offset"], out_stride=a["out_stride"], out_offset=a["out_offset"])
    if fn == "swin_chan_up":
        return fn, dict(BT=a["BT"], C=a["Cdim"], Cout=a["w"].shape[0], nwin=a["nwin"])
    raise KeyError(fn)


# ---- the recorder ----------------------------------------------------------------------------------------------------------
@contextlib.contextmanager
def recording(ops, fns, key, seen, library_only=False, outermost_only=False):
    """Pass-through recorders around ops.<fns>: each call appends key(fn, bound arguments with defaults) to `seen`.
    library_only: only calls made from the library's own modules (an emulated composite calling another emulated
    function is not a plan call). outermost_only: calls made from inside a recorded call belong to the outer call."""
    depth = [0]
    mp = pytest.MonkeyPatch()
    for fn in fns:
        orig = getattr(ops, fn)
        sig = inspect.signature(orig)

        def rec(*a, _fn=fn, _orig=orig, _sig=sig, **k):
            if (depth[0] == 0 or not outermost_only) and \
                    (not library_only or sys._getframe(1).f_globals.get("__name__", "").startswith("mtt_b200")):
                ba = _sig.bind(*a, **k)
                ba.apply_defaults()
                seen.append(key(_fn, ba.arguments))
            depth[0] += 1
            try:
                return _orig(*a, **k)
            finally:
                depth[0] -= 1
        mp.setattr(ops, fn, rec)
    try:
        yield seen
    finally:
        mp.undo()
