"""CPU: the three-task Swin TaskPrompter (semseg, depth, 3ddet -- the reference's Cityscapes-3D model). The '3ddet' task
is an ordinary task in the backbone (prompt row, gating, fea_fuse at each level) whose level maps skip the bilinear x2 and
the multi-scale fusion and go to the detection head as a list of 4 maps (TP taskprompter_swin.py:709-710, :741, :764).

  * the oracle's 3ddet branch against the fixtures of the UNMODIFIED reference (oracle/make_golden_swin3d.py) and, where
    the reference tree is present, against a live reference model;
  * the launch plan (kernels emulated by tests/emul_ops.py) against the oracle: wrapper forward, TaskPrompterSwin.forward,
    predict(), and random geometries that include '3ddet';
  * accelerate() on a live three-task reference wrapper with a stand-in detection head;
  * names and shapes of the state dict against the reference's, and the error behaviour."""
import os
import random

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import configs, ref_loader
from oracle import taskprompter_swin_ref as R
from oracle.make_golden import big_input, sd_checksum
from oracle.make_golden_swin3d import JOBS, state_dict

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
DET = "3ddet"


def fixture(name):
    return torch.load(os.path.join(GOLD, f"{name}.pt"), weights_only=False)


def oracle_forward(sd, cfg, x):
    """The reference wrapper with nn.Identity as the 3ddet head: 2D logits at the output size, '3ddet' the 4 level maps."""
    feats = R.backbone_forward(sd, cfg, x)
    size = tuple(cfg["dd_label_map_size"]) if "dd_label_map_size" in cfg else x.shape[-2:]
    head = R.deconv_head if cfg.get("head", "conv") == "deconv" else R.conv_head
    return {t: feats[t] if t == DET else F.interpolate(head(sd, t, feats[t]), size, mode="bilinear") for t in cfg["tasks"]}


def model(cfg, sd, det_head=None, graph=False):
    import mtt_b200  # noqa: F401
    from mtt_b200 import taskprompter_swin as TS

    m = TS.build_from_config(cfg, nsplit=2, use_graph=graph, det_head=det_head or nn.Identity()).eval()
    missing, unexpected = m.load_state_dict(sd, strict=False)     # index / mask buffers are derived, not stored;
    assert not unexpected and all("relative_position_index" in k or "attn_mask" in k or k.startswith("heads.3ddet.")
                                  for k in missing), (missing, unexpected)   # a stand-in head keeps its own parameters
    return m


def inputs(name):
    """(cfg, oracle state dict, input) of a fixture, the weights checked against its checksum."""
    seed, batch = JOBS[name]
    cfg = configs.taskprompter_swin(name)
    sd = state_dict(cfg, seed)
    return cfg, sd, big_input(cfg, seed, batch)


def rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


def assert_maps(got, want, what, tol=2e-4):
    assert len(got) == len(want) == 4, what
    for il, (g, w) in enumerate(zip(got, want)):
        assert tuple(g.shape) == tuple(w.shape), (what, il)
        assert rel(g, w) < tol, (what, il, rel(g, w))


def lattice_values(y, rec, ti, stride):
    from test_big_goldens_gpu import lattice
    samp = []
    for b in range(y.shape[0]):
        iy, ix = lattice(b, ti, y.shape[2], y.shape[3], stride)
        samp.append(y[b][:, iy][:, :, ix])
    return torch.stack(samp)


# ---- the oracle against the reference ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["tps_tiny3d", "tps_mid3d"])
def test_oracle_3ddet_branch_matches_the_reference_fixture(name):
    fx = fixture(name)
    cfg, sd, x = inputs(name)
    assert sd_checksum(sd) == fx["sd_sha256"]
    if "x" in fx:
        assert torch.equal(x, fx["x"])
    with torch.no_grad():
        out = oracle_forward(sd, cfg, x)
    ref_det = fx["out"][DET]
    assert len(out[DET]) == 4
    for il, (g, r) in enumerate(zip(out[DET], ref_det)):
        h, w = R.level_resolution(cfg, il)
        assert tuple(r.shape) == (x.shape[0], cfg["f"], h, w)          # each level at its own resolution, f channels
        assert tuple(g.shape) == tuple(r.shape)
        assert (g - r).abs().max() <= 5e-6 * r.abs().max().clamp_min(1.0), (name, il)
    for ti, t in enumerate(t for t in cfg["tasks"] if t != DET):
        r = fx["out"][t]
        if isinstance(r, dict):                                            # lattice-sampled (tps_mid3d)
            g = lattice_values(out[t], r, ti, fx["stride"])
            assert tuple(out[t].shape) == tuple(r["shape"])
            assert (g - r["samples"]).abs().max() <= 5e-6 * max(r["absmax"], 1.0), (name, t)
            assert abs(float(out[t].double().norm()) / r["norm"] - 1) < 1e-5
        else:
            assert (out[t] - r).abs().max() <= 5e-6 * r.abs().max().clamp_min(1.0), (name, t)


@pytest.mark.skipif(not ref_loader.available(), reason="reference tree not present")
def test_oracle_3ddet_branch_matches_a_live_reference():
    """The reference's own initialisation, BatchNorm statistics perturbed: the oracle on its state dict reproduces its
    forward, the 3ddet maps included."""
    from oracle.make_golden_swin3d import reference_model

    cfg = configs.taskprompter_swin("tps_tiny3d")
    torch.manual_seed(3)
    ref = reference_model(cfg)
    for m in ref.modules():
        if isinstance(m, nn.BatchNorm2d):
            m.running_mean.normal_(0, 0.1)
            m.running_var.uniform_(0.8, 1.2)
    x = torch.randn(2, 3, *cfg["img_size"])
    with torch.no_grad():
        want = ref(x)
        got = oracle_forward(ref.state_dict(), cfg, x)
    for t in cfg["tasks"]:
        pairs = zip(got[t], want[t]) if t == DET else [(got[t], want[t])]
        for g, w in pairs:
            assert g.shape == w.shape
            assert (g - w).abs().max() <= 5e-6 * w.abs().max().clamp_min(1.0), t


# ---- the launch plan (kernels emulated) against the oracle ------------------------------------------------------------------
@pytest.fixture
def emulated(monkeypatch):
    import mtt_b200  # noqa: F401
    from mtt_b200 import taskprompter as TP, taskprompter_swin as TS
    import emul_ops

    emul_ops.install(monkeypatch)
    monkeypatch.setattr(TP, "_check_input", lambda mod, x: None)
    monkeypatch.setattr(TS, "_check_input", lambda mod, x: None)


@pytest.mark.parametrize("name", ["tps_tiny3d", "tps_mid3d"])
def test_plan_matches_oracle_emulated(emulated, name):
    """Wrapper forward, TaskPrompterSwin.forward and predict() of the three-task model against the oracle."""
    cfg, sd, x = inputs(name)
    m = model(cfg, sd)
    with torch.no_grad():
        want = oracle_forward(sd, cfg, x)
        feats = R.backbone_forward(sd, cfg, x)
        got = m(x)
        assert list(got) == cfg["tasks"]
        for t in cfg["tasks"]:
            if t == DET:
                assert_maps(got[t], want[t], (name, "forward"))
            else:
                assert got[t].shape == want[t].shape and rel(got[t], want[t]) < 2e-4, (name, t)
        # TaskPrompterSwin.forward: (task_fea, info), the reference's contract
        fea, info = m.backbone(x)
        assert info == {} and list(fea) == cfg["tasks"]
        for t in cfg["tasks"]:
            if t == DET:
                assert_maps(fea[t], feats[t], (name, "backbone"))
            else:
                h0, w0 = R.level_resolution(cfg, 0)
                assert tuple(fea[t].shape) == (x.shape[0], cfg["f"], 2 * h0, 2 * w0)
                assert rel(fea[t], feats[t]) < 2e-4, (name, "backbone", t)
        # predict(): the 2D tasks' get_output maps, '3ddet' the head's raw output
        pred = m.predict(x)
        assert_maps(pred[DET], want[DET], (name, "predict"))
        lab, dep = pred["semseg"], pred["depth"]
        H, W = want["semseg"].shape[-2:]
        assert lab.dtype == torch.int64 and tuple(lab.shape) == (x.shape[0], H, W)
        r = want["semseg"]
        top2 = r.topk(2, dim=1).values
        safe = (top2[:, 0] - top2[:, 1]) > 1e-4 * r.abs().max()
        assert torch.equal(lab[safe], r.argmax(1)[safe])
        assert tuple(dep.shape) == (x.shape[0], H, W, 1)
        assert rel(dep[..., 0], want["depth"][:, 0].clamp_min(0)) < 2e-4


class Recorder(nn.Module):
    """A stand-in detection head with a parameter of its own: records what it receives, returns a fresh object."""

    def __init__(self):
        super().__init__()
        self.scale = nn.Parameter(torch.tensor(1.5))
        self.seen = []

    def forward(self, maps):
        self.seen.append([tuple(m.shape) for m in maps])
        self.last = {"maps": [m * self.scale for m in maps]}
        return self.last


@pytest.mark.skipif(not ref_loader.available(), reason="reference tree not present")
def test_accelerate_live_three_task_reference(emulated):
    """accelerate() on the unmodified reference wrapper (own initialisation, BatchNorm statistics perturbed) with a
    stand-in 3ddet head: the strict load works and the names equal the fixture's, the head is the reference's module
    itself, it receives the 4 level maps in level order with the reference's shapes, and out['3ddet'] is its output."""
    import mtt_b200  # noqa: F401
    from mtt_b200 import taskprompter_swin as TS

    cfg = configs.taskprompter_swin("tps_tiny3d")
    torch.manual_seed(9)
    ref = ref_loader.build_taskprompter_swin(cfg)
    ref.heads[DET] = Recorder()
    for m in ref.modules():
        if isinstance(m, nn.BatchNorm2d):
            m.running_mean.normal_(0, 0.1)
            m.running_var.uniform_(0.8, 1.2)
    ref.eval()
    mine = TS.accelerate(ref, use_graph=False)
    assert mine.heads[DET] is ref.heads[DET]
    keys = {k: tuple(v.shape) for k, v in mine.state_dict().items() if not k.startswith("heads.3ddet.")}
    assert keys == dict(fixture("tps_tiny3d")["keys"])
    x = torch.randn(2, 3, *cfg["img_size"])
    with torch.no_grad():
        want = ref(x)
        want_maps = [m.clone() for m in want[DET]["maps"]]
        got = mine(x)
    rec = ref.heads[DET]
    assert got[DET] is rec.last
    shapes = [(2, cfg["f"], *R.level_resolution(cfg, il)) for il in range(4)]
    assert rec.seen == [shapes, shapes]                         # the reference's call, then ours: same maps, same order
    assert_maps(got[DET]["maps"], want_maps, "accelerate")
    for t in ("semseg", "depth"):
        assert got[t].shape == want[t].shape and rel(got[t], want[t]) < 2e-4, t


@pytest.mark.skipif(not ref_loader.available(), reason="reference tree not present")
def test_accelerate_live_two_task_reference(emulated):
    import mtt_b200  # noqa: F401
    from mtt_b200 import taskprompter_swin as TS

    cfg = configs.taskprompter_swin("tps_tiny")
    torch.manual_seed(10)
    ref = ref_loader.build_taskprompter_swin(cfg).eval()
    mine = TS.accelerate(ref, use_graph=False)
    x = torch.randn(1, 3, *cfg["img_size"])
    with torch.no_grad():
        want, got = ref(x), mine(x)
    for t in cfg["tasks"]:
        assert got[t].shape == want[t].shape and rel(got[t], want[t]) < 2e-4, t


# ---- random geometries with '3ddet' -------------------------------------------------------------------------------------------
def draw_swin3d(seed):
    from test_random_configs import draw_swin

    cfg, B = draw_swin(seed)
    rng = random.Random(4000 + seed)
    tasks = list(cfg["tasks"])[:2]
    tasks.insert(rng.randint(0, len(tasks)), DET)
    cfg.update(tasks=tasks, num_output={**{t: cfg["num_output"][t] for t in tasks if t != DET}, DET: 1},
               name=f"random_swin3d{seed}")
    return cfg, B


@pytest.mark.parametrize("seed", range(6))
def test_plan_and_oracle_on_random_geometries_with_3ddet(emulated, seed):
    cfg, B = draw_swin3d(seed)
    sd = {k: v for k, v in R.init_state_dict(cfg, seed=seed).items() if not k.startswith("heads.3ddet.")}
    torch.manual_seed(seed)
    x = torch.randn(B, 3, *cfg["img_size"])
    m = model(cfg, sd)
    with torch.no_grad():
        want = oracle_forward(sd, cfg, x)
        got = m(x)
    for t in cfg["tasks"]:
        if t == DET:
            assert_maps(got[t], want[t], cfg)
        else:
            assert got[t].shape == want[t].shape and rel(got[t], want[t]) < 2e-4, (cfg, t)
    if ref_loader.available():
        from oracle.make_golden_swin3d import reference_model
        torch.manual_seed(seed)
        ref = reference_model(cfg)
        with torch.no_grad():
            r2, o2 = ref(x), oracle_forward(ref.state_dict(), cfg, x)
        for t in cfg["tasks"]:
            for g, w in (zip(o2[t], r2[t]) if t == DET else [(o2[t], r2[t])]):
                assert (g - w).abs().max() <= 5e-6 * w.abs().max().clamp_min(1.0), (cfg, t)


# ---- names, shapes and errors -------------------------------------------------------------------------------------------------
def test_state_dict_matches_the_reference_names_at_swinB():
    """tps_swinB3d (the yml) built here has the reference's parameter and buffer names and shapes, with no
    multi_scale_fuse.3ddet: a checkpoint of the reference's three-task model loads with strict=True."""
    import mtt_b200  # noqa: F401
    from mtt_b200 import taskprompter_swin as TS
    import lzma

    with lzma.open(os.path.join(GOLD, "big_tps_swinB3d_b1.pt.xz"), "rb") as f:
        keys = dict(torch.load(f, weights_only=False)["keys"])
    m = TS.build_from_config(configs.taskprompter_swin("tps_swinB3d"), det_head=nn.Identity())
    mine = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert mine == keys
    assert not any(k.startswith("backbone.multi_scale_fuse.3ddet") for k in mine)
    assert mine["backbone.task_prompts"] == (3, 128)


def test_three_task_swin_needs_a_detection_head():
    import mtt_b200  # noqa: F401
    from mtt_b200 import taskprompter_swin as TS
    from mtt_b200.taskprompter import TaskPrompterWrapper

    cfg = configs.taskprompter_swin("tps_tiny3d")
    with pytest.raises(ValueError, match="'3ddet' task needs det_head="):
        TS.build_from_config(cfg)
    m = TS.build_from_config(cfg, det_head=nn.Identity())
    heads = nn.ModuleDict({t: m.heads[t] for t in ("semseg", "depth")})
    with pytest.raises(ValueError, match="needs a detection head module"):
        TaskPrompterWrapper(m.backbone.p, m.backbone, heads)
    with pytest.raises(NotImplementedError, match="absolute position embedding"):
        TS.TaskPrompterSwin(m.backbone.p, img_size=(64, 128), embed_dim=16, depths=(2, 2, 2, 2), num_heads=(1, 2, 4, 8),
                            window_size=6, ape=True)


def test_vit_wrapper_still_refuses_a_foreign_3ddet_head():
    """The ViT path is unchanged: its '3ddet' task runs a ConvHead stand-in on the device, any other head is refused."""
    import mtt_b200  # noqa: F401
    from mtt_b200 import taskprompter as TP

    cfg = dict(configs.taskprompter("tp_tiny"), tasks=["semseg", DET], num_output={"semseg": 5, DET: 4})
    m = TP.build_from_config(cfg)
    heads = nn.ModuleDict({"semseg": m.heads["semseg"], DET: nn.Identity()})
    with pytest.raises(NotImplementedError, match="unsupported head Identity"):
        TP.TaskPrompterWrapper(m.backbone.p, m.backbone, heads)
