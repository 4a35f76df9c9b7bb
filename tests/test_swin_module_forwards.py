"""The Swin TaskPrompter's sub-module forwards: SwinTransformerBlock.forward(x, task_prompts),
PatchMerging.forward(x, task_prompts, attn_weight) and BasicLayer.forward(x, task_prompts), with the reference's
signatures, layouts and return values (TP taskprompter_swin.py:310-405, :430-477, :527-537), on the plan's launch code.

CPU:
  * the oracle's block() and patch_merging() against the goldens of the unmodified reference's modules
    (oracle/make_golden_swin_modules.py, tests/golden/swin_modules.pt.xz), tps_tiny3d and Swin-B width;
  * every module forward of tps_tiny3d, kernels emulated (tests/emul_ops.py and, for the
    layout kernel the forwards add, tests/emul_swin_modules.py), against the same goldens: shifted and
    padded, unshifted, clamped windows, chan_nheads = 4, the '3ddet' prompt, the model's last block;
  * BasicLayer is its blocks, then its PatchMerging; WindowAttention.forward and train mode raise;
  * the plan launches exactly what it launched before the forwards shared its code (tests/swin_plan_launches.py).
GPU (-m gpu): the same forwards through the C ABI against the goldens (tps_tiny3d in full, Swin-B width on the lattice);
the four BasicLayers and the final norm chained at Swin-B reproduce what TaskPrompterSwin.forward's plan computes; the
new layout kernel mtt_swin_logit_maps bit-exact at the production geometries."""
import lzma

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import configs
from oracle import taskprompter_swin_ref as R
from oracle.make_golden import sd_checksum
from oracle.make_golden_swin3d import state_dict
from oracle.make_golden_swin_modules import JOBS, PATH, sample, stage_geometry, stage_inputs

TOL = 2e-4          # rel-L2 of the module forwards (as tests/test_module_forwards.py)
_GOLD = {}


def golden(name):
    if not _GOLD:
        with lzma.open(PATH, "rb") as f:
            _GOLD.update(torch.load(f, weights_only=False))
    return _GOLD[name]


def rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30))


def check(got, want, what, tol=TOL):
    """got: a module output; want: the golden (a tensor, or the lattice record of a large map)."""
    got = got.detach().float().cpu()
    if isinstance(want, dict):
        assert tuple(got.shape) == tuple(want["shape"]), what
        e = rel(sample(got, want["hw"], want["stride"]), want["samples"])
        n = abs(float(got.double().norm()) / want["norm"] - 1)
        assert e < tol and n < tol, (what, e, n)
        return max(e, n)
    assert tuple(got.shape) == tuple(want.shape), (what, tuple(got.shape), tuple(want.shape))
    e = rel(got, want)
    assert e < tol, (what, e)
    return e


def check_outputs(out, want, what, tol=TOL):
    """out = (x, prompts, [raw_spa, raw_chan])."""
    x, p, (spa, chan) = out
    return max(check(x, want["x"], (what, "x"), tol), check(p, want["prompts"], (what, "prompts"), tol),
               check(spa, want["raw_spa"], (what, "raw_spa"), tol), check(chan, want["raw_chan"], (what, "raw_chan"), tol))


def model(name, device="cpu"):
    import mtt_b200  # noqa: F401
    from mtt_b200 import taskprompter_swin as TS

    seed, _, _ = JOBS[name]
    cfg = configs.taskprompter_swin(name)
    sd = state_dict(cfg, seed)
    assert sd_checksum(sd) == golden(name)["sd_sha256"]
    m = TS.build_from_config(cfg, nsplit=2, use_graph=False, det_head=nn.Identity()).eval()
    missing, unexpected = m.load_state_dict(sd, strict=False)
    assert not unexpected and all("relative_position_index" in k or "attn_mask" in k for k in missing)
    return cfg, sd, m.to(device)


def run_stage(layer, cfg, name, i, device):
    """{"block{j}" | "merge" | "layer": (x, prompts, [raw_spa, raw_chan])} of the module forwards of stage i."""
    seed, B, _ = JOBS[name]
    x, p, spa, chan = (t.to(device) for t in stage_inputs(cfg, seed, B, i))
    out = {}
    with torch.no_grad():
        for j, blk in enumerate(layer.blocks):
            xo, attn, po = blk(x, p)
            out[f"block{j}"] = (xo, po, attn)
        if layer.downsample is not None:
            out["merge"] = layer.downsample(x, p, [spa, chan])
        xo, attn, po = layer(x, p)
        out["layer"] = (xo, po, attn)
    return out


# ---- the oracle against the reference's modules ---------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(JOBS))
def test_oracle_block_and_patch_merging_match_the_reference_modules(name):
    """oracle block() / patch_merging() on the goldens' inputs reproduce the reference's SwinTransformerBlock,
    PatchMerging and BasicLayer (<= 1e-5 rel-L2: fp32 on the CPU, different operation order)."""
    seed, B, stages = JOBS[name]
    cfg = configs.taskprompter_swin(name)
    sd = state_dict(cfg, seed)
    gold = golden(name)
    assert sd_checksum(sd) == gold["sd_sha256"]
    n_stage = len(cfg["depths"])
    for i in stages:
        dim, res, ws, shifts = R.stage_geometry(cfg, i)
        heads = cfg["heads"][i]
        x, p, spa, chan = stage_inputs(cfg, seed, B, i)
        want = gold["stages"][i]
        pre = f"backbone.layers.{i}."
        with torch.no_grad():
            xl, pl, al = x, p, None
            for j, shift in enumerate(shifts):
                last = i == n_stage - 1 and j == len(shifts) - 1
                xo, po, so, co = R.block(sd, f"{pre}blocks.{j}.", cfg, x, p, dim, res, ws, shift, heads, last)
                check_outputs((xo, po, [so, co]), want[f"block{j}"], (name, i, j), tol=1e-5)
                xl, pl, so, co = R.block(sd, f"{pre}blocks.{j}.", cfg, xl, pl, dim, res, ws, shift, heads, last)
                al = [so, co]
            if i < n_stage - 1:
                xo, po, so, co = R.patch_merging(sd, f"{pre}downsample.", x, p, spa, chan, res)
                check_outputs((xo, po, [so, co]), want["merge"], (name, i, "merge"), tol=1e-5)
                xl, pl, so, co = R.patch_merging(sd, f"{pre}downsample.", xl, pl, al[0], al[1], res)
                al = [so, co]
            check_outputs((xl, pl, al), want["layer"], (name, i, "layer"), tol=1e-5)


# ---- the module forwards, kernels emulated ------------------------------------------------------------------------------
@pytest.fixture
def emulated(monkeypatch):
    import mtt_b200  # noqa: F401
    from mtt_b200 import taskprompter_swin as TS
    import emul_swin_modules

    emul_swin_modules.install(monkeypatch)
    monkeypatch.setattr(TS, "_check_input", lambda mod, x: None)


def test_module_forwards_match_the_reference_emulated(emulated):
    """Every block, PatchMerging and BasicLayer of tps_tiny3d (batch 2) against the reference's modules."""
    name = "tps_tiny3d"
    cfg, _, m = model(name)
    gold = golden(name)
    for i in JOBS[name][2]:
        got = run_stage(m.backbone.layers[i], cfg, name, i, "cpu")
        assert sorted(got) == sorted(gold["stages"][i])
        for k, out in got.items():
            check_outputs(out, gold["stages"][i][k], (name, i, k))


def test_basic_layer_is_its_blocks_then_its_merge(emulated):
    """BasicLayer.forward = the blocks' forwards in turn, then PatchMerging.forward on the last block's attn_weight
    (the reference's loop, TP:527-537): the same values, the maps and prompts handed over through the reference's
    layouts in one case and the plan's in the other."""
    name = "tps_tiny3d"
    cfg, _, m = model(name)
    seed, B, _ = JOBS[name]
    for i, layer in enumerate(m.backbone.layers):
        x, p, _, _ = stage_inputs(cfg, seed, B, i)
        with torch.no_grad():
            want = layer(x, p)
            xc, pc = x, p
            for blk in layer.blocks:
                xc, attn, pc = blk(xc, pc)
            if layer.downsample is not None:
                xc, pc, attn = layer.downsample(xc, pc, attn)
        got = (xc, attn, pc)
        for g, w in ((got[0], want[0]), (got[2], want[2]), (got[1][0], want[1][0]), (got[1][1], want[1][1])):
            assert g.shape == w.shape and torch.equal(g, w), i


def test_outputs_are_fresh_and_inputs_untouched(emulated):
    name = "tps_tiny3d"
    cfg, _, m = model(name)
    seed, B, _ = JOBS[name]
    x, p, spa, chan = stage_inputs(cfg, seed, B, 0)
    keep = [t.clone() for t in (x, p, spa, chan)]
    blk, dsm = m.backbone.layers[0].blocks[1], m.backbone.layers[0].downsample
    with torch.no_grad():
        a = blk(x, p)
        b = blk(x, p)
        dsm(x, p, [spa, chan])
    for t, k in zip((x, p, spa, chan), keep):
        assert torch.equal(t, k)
    for u, v in ((a[0], b[0]), (a[2], b[2]), (a[1][0], b[1][0]), (a[1][1], b[1][1])):
        assert torch.equal(u, v) and u.data_ptr() != v.data_ptr()


def test_window_attention_forward_and_train_mode_raise():
    import mtt_b200  # noqa: F401
    from mtt_b200 import taskprompter_swin as TS

    cfg = configs.taskprompter_swin("tps_tiny3d")
    m = TS.build_from_config(cfg, det_head=nn.Identity())
    layer = m.backbone.layers[0]
    with pytest.raises(NotImplementedError, match="full .* pre-softmax map"):
        layer.blocks[0].attn(torch.zeros(2, 36, 16), torch.zeros(1, 3, 16))
    x, p, spa, chan = stage_inputs(cfg, 31, 2, 0)
    for mod, args in ((layer.blocks[0], (x, p)), (layer.downsample, (x, p, [spa, chan])), (layer, (x, p))):
        mod.train()
        with pytest.raises(NotImplementedError, match="eval-only"):
            mod(*args)


def test_bad_shapes_raise(emulated):
    name = "tps_tiny3d"
    cfg, _, m = model(name)
    layer = m.backbone.layers[0]
    x, p, spa, chan = stage_inputs(cfg, 31, 2, 0)
    with pytest.raises(ValueError, match="expected x"):
        layer.blocks[0](x[:, 1:], p)
    with pytest.raises(ValueError, match="expected attn_weight"):
        layer.downsample(x, p, [spa[:, :, :, 1:], chan])


def test_plan_launches_are_unchanged():
    """The plan of every mode of tps_tiny, tps_tiny3d and tps_swinB3d launches the same entry points, in the same order,
    with the same arguments and the same buffer aliasing as before its block and merge launches became the functions
    the sub-module forwards call."""
    import json

    import mtt_b200  # noqa: F401
    import swin_plan_launches as SPL

    want = SPL.load()
    got = json.loads(json.dumps(SPL.record_all()))
    assert sorted(got) == sorted(want)
    for k in want:
        assert len(got[k]) == len(want[k]), k
        for n, (g, w) in enumerate(zip(got[k], want[k])):
            assert g == w, (k, n, g[0], w[0])


# ---- on the H100 ------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(JOBS))
def test_module_forwards_match_the_reference_gpu(name):
    """Through the C ABI: every module forward of the golden's stages against the reference's modules, rel-L2 < 2e-4 on
    x, task_prompts, raw_spa_attn and raw_chan_attn (Swin-B width: on the lattice, and the exact norms)."""
    cfg, _, m = model(name, "cuda")
    gold = golden(name)
    worst = 0.0
    for i in JOBS[name][2]:
        got = run_stage(m.backbone.layers[i], cfg, name, i, "cuda")
        torch.cuda.synchronize()
        assert sorted(got) == sorted(gold["stages"][i])
        for k, out in got.items():
            worst = max(worst, check_outputs(out, gold["stages"][i][k], (name, i, k)))
    print(f"{name}: worst rel-L2 {worst:.2e}")


@pytest.mark.gpu
def test_basic_layers_chained_reproduce_the_plan_at_swinB_gpu(monkeypatch):
    """tps_swinB3d, batch 1: TaskPrompterSwin.forward (the plan) on an image, recording the input of every stage; the
    four BasicLayer forwards chained from the stage-0 input, and the final norm, reproduce every stage's input (the
    merged map and prompts), the down-sampled maps and channel logits handed to decoder levels 0-2, the last stage's
    maps, and the normed map of level 3: everything the plan's task features are computed from."""
    import mtt_b200  # noqa: F401
    from mtt_b200 import taskprompter_swin as TS

    cfg, sd, m = model("tps_swinB3d", "cuda")
    bb = m.backbone
    seen = {}
    orig = TS._launch_swin_block

    def snap(s, w, shift, spa=None):
        seen.setdefault(id(s), (s.x.clone(), s.p.clone()))
        orig(s, w, shift, spa)
    monkeypatch.setattr(TS, "_launch_swin_block", snap)
    img = torch.randn(1, 3, *cfg["img_size"], generator=torch.Generator().manual_seed(5)).cuda()
    with torch.no_grad():
        bb(img)
    monkeypatch.setattr(TS, "_launch_swin_block", orig)
    pl = next(iter(bb._mtt_plans.values()))
    ins = [seen[id(s)] for s in pl.st]
    B, T = 1, len(cfg["tasks"])
    x = ins[0][0].view(B, -1, pl.st[0].C)
    p = ins[0][1].view(B, T, -1)
    worst = 0.0
    with torch.no_grad():
        for i, layer in enumerate(bb.layers):
            x, attn, p = layer(x, p)
            s = pl.st[i]
            if layer.downsample is not None:
                n = pl.st[i + 1]
                pairs = [(x, ins[i + 1][0].view(x.shape)), (p, ins[i + 1][1].view(p.shape)),
                         (attn[0], s.logits_ds[..., T:].reshape(attn[0].shape)), (attn[1], s.rc_up)]
                assert n.C == x.shape[-1]
            else:
                pairs = [(x, s.x.view(x.shape)), (attn[0], s.logits[..., T:].reshape(attn[0].shape)),
                         (attn[1], s.rc)]
            for k, (g, w) in enumerate(pairs):
                e = rel(g, w)
                worst = max(worst, e)
                assert e < TOL, (i, k, e)
        xfin = F.layer_norm(x.double(), (x.shape[-1],), bb.norm.weight.double(), bb.norm.bias.double(), bb.norm.eps)
        e = rel(xfin.view(pl.xfin.shape), pl.xfin)
        assert e < TOL, e
    print(f"tps_swinB3d: chained BasicLayers vs the plan, worst rel-L2 {max(worst, e):.2e}")


@pytest.mark.gpu
@pytest.mark.parametrize("stage", [0, 3])
def test_logit_maps_kernel_exact_at_swinB_gpu(stage):
    """mtt_swin_logit_maps both ways at the Swin-B stage geometries of the reference's validation batch 4 (stage 0:
    4 heads x 3 tasks of 192 x 384; stage 3: 32 heads of 24 x 48): bit-exact against the indexing it restates, and the
    first T columns of the logits (NaN sentinels) untouched."""
    import mtt_b200  # noqa: F401
    from mtt_b200 import ops

    cfg = configs.taskprompter_swin("tps_swinB3d")
    _, (H, W), heads, T, _ = stage_geometry(cfg, stage)
    B = 4
    g = torch.Generator().manual_seed(stage)
    logits = torch.randn(B, heads, T, T + H * W, generator=g).cuda()
    logits[..., :T] = float("nan")
    maps = torch.full((B, heads, T, H, W), float("nan"), device="cuda")
    ops.swin_logit_maps(logits, maps, T=T, to_maps=True)
    assert torch.equal(maps, logits[..., T:].reshape(maps.shape))
    back = torch.full_like(logits, float("nan"))
    src = torch.randn(B, heads, T, H, W, generator=g).cuda()
    ops.swin_logit_maps(back, src, T=T, to_maps=False)
    torch.cuda.synchronize()
    assert torch.equal(back[..., T:], src.reshape(B, heads, T, H * W))
    assert torch.isnan(back[..., :T]).all()
