"""Generates the golden vectors of the Swin TaskPrompter's sub-module forwards by running the UNMODIFIED reference's own
SwinTransformerBlock, PatchMerging and BasicLayer (TP/models/transformers/taskprompter_swin.py:310-405, :430-477,
:527-537) on seeded inputs. TEST INFRASTRUCTURE.

The modules are those of the reference wrapper of oracle/make_golden_swin3d.py (same configs, seeds and weights), called
one by one on the inputs of stage_inputs(): x [B, H*W, C], task_prompts [B, T, C] and, for PatchMerging, attn_weight =
[raw_spa_attn [B, heads, T, H, W], raw_chan_attn [B, T, C, nh, nw]] drawn from a generator seeded per (config, stage).

    tps_tiny3d  batch 2, every stage: a shifted padded block (stage 0, 16 x 32 in 6 x 6 windows), unshifted blocks, the
                clamped windows of stages 2 and 3, chan_nheads = 4, the model's last block, every PatchMerging and every
                BasicLayer; every output in full
    tps_swinB3d batch 1 (the reference's Cityscapes-3D model at Swin-B width): stages 0 (192 x 384, C = 128) and 3
                (24 x 48, C = 1024, the last block): both blocks, the PatchMerging of stage 0, both BasicLayers; maps of
                more than 4096 values as their values on a lattice (sample()) with the exact norm

into tests/golden/swin_modules.pt.xz:
    {config: {"seed", "batch", "sd_sha256", "stages": {i: {"block{j}" | "merge" | "layer": {"x", "prompts",
     "raw_spa", "raw_chan": tensor or lattice record}}}}}

    python -m oracle.make_golden_swin_modules
"""
import lzma
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import configs, ref_loader  # noqa: E402
from oracle.make_golden import GOLD, sd_checksum  # noqa: E402

PATH = os.path.join(GOLD, "swin_modules.pt.xz")
JOBS = {"tps_tiny3d": (31, 2, (0, 1, 2, 3)), "tps_swinB3d": (47, 1, (0, 3))}    # config -> (seed, batch, stages)
FULL_MAX = 4096                    # maps with more values than this are stored as lattice samples


def stage_geometry(cfg, i):
    """(C, (H, W), heads, T, nh) of stage i."""
    from oracle import taskprompter_swin_ref as R
    dim, res, _, _ = R.stage_geometry(cfg, i)
    return dim, res, cfg["heads"][i], len(cfg["tasks"]), int(round(cfg["chan_nheads"] ** 0.5))


def stage_inputs(cfg, seed, B, i):
    """x [B, H*W, C], task_prompts [B, T, C], raw_spa [B, heads, T, H, W], raw_chan [B, T, C, nh, nw] of stage i."""
    C, (H, W), heads, T, nh = stage_geometry(cfg, i)
    g = torch.Generator().manual_seed(1000 * seed + i)
    x = torch.randn(B, H * W, C, generator=g)
    prompts = 1 + torch.randn(B, T, C, generator=g)                   # the task prompts are drawn around 1 (TP:571)
    raw_spa = 2 * torch.randn(B, heads, T, H, W, generator=g)
    raw_chan = 2 * torch.randn(B, T, C, nh, nh, generator=g)
    return x, prompts, raw_spa, raw_chan


def _maps(y, hw):
    """A module output as maps [B, n, H, W]: tokens [B, H*W, C] -> [B, C, H, W]; [B, heads, T, H, W] -> [B, heads*T, H, W]."""
    if y.dim() == 3:
        return y.transpose(1, 2).reshape(y.shape[0], y.shape[2], *hw)
    return y.reshape(y.shape[0], -1, *y.shape[-2:])


def sample(y, hw, stride):
    """The values of y's maps at rows / columns stride // 2 + k * stride."""
    m = _maps(y, hw)
    o = stride // 2
    return m[:, :, o::stride, o::stride].contiguous()


def record(y, hw):
    if y.numel() <= FULL_MAX:
        return y.clone()
    stride = 16 if hw[0] * hw[1] >= 16384 else 8
    return {"shape": tuple(y.shape), "hw": tuple(hw), "stride": stride, "samples": sample(y, hw, stride),
            "norm": float(y.double().norm())}


def outputs(x, prompts, attn, hw):
    return {"x": record(x, hw), "prompts": record(prompts, hw), "raw_spa": record(attn[0], hw),
            "raw_chan": record(attn[1], hw)}


def make(name):
    from oracle.make_golden_swin3d import reference_model, state_dict
    seed, B, stages = JOBS[name]
    cfg = configs.taskprompter_swin(name)
    sd = state_dict(cfg, seed)
    ref = reference_model(cfg, sd).backbone
    fx = {"seed": seed, "batch": B, "sd_sha256": sd_checksum(sd), "torch": torch.__version__, "stages": {},
          "made_by": "oracle/make_golden_swin_modules.py: the unmodified reference's SwinTransformerBlock, PatchMerging "
                     "and BasicLayer (eval, fp32, CPU)"}
    for i in stages:
        layer = ref.layers[i]
        x, p, spa, chan = stage_inputs(cfg, seed, B, i)
        _, (H, W), _, _, _ = stage_geometry(cfg, i)
        st = {}
        with torch.no_grad():
            for j, blk in enumerate(layer.blocks):
                xo, attn, po = blk(x.clone(), p.clone())
                st[f"block{j}"] = outputs(xo, po, attn, (H, W))
            if layer.downsample is not None:
                xo, po, attn = layer.downsample(x.clone(), p.clone(), [spa.clone(), chan.clone()])
                st["merge"] = outputs(xo, po, attn, (H // 2, W // 2))
            xo, attn, po = layer(x.clone(), p.clone())
            hw = (H, W) if layer.downsample is None else (H // 2, W // 2)
            st["layer"] = outputs(xo, po, attn, hw)
        fx["stages"][i] = st
    return fx


def main():
    if not ref_loader.available():
        raise SystemExit("reference not found (set MTT_REFERENCE or mount /root/reference)")
    out = {}
    for name in JOBS:
        t0 = time.time()
        out[name] = make(name)
        print(f"{name}: {time.time() - t0:.0f} s", flush=True)
    with lzma.open(PATH, "wb", preset=9 | lzma.PRESET_EXTREME) as f:
        torch.save(out, f)
    print(f"wrote {PATH} ({os.path.getsize(PATH) / 1024:.0f} KiB)")


if __name__ == "__main__":
    main()
