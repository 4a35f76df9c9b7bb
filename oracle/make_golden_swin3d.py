"""Generates the golden vectors of the three-task Swin TaskPrompter (semseg, depth, 3ddet: the reference's Cityscapes-3D
model, TP/configs/cityscapes3d/cs_swinB_taskprompter.yml) by running the UNMODIFIED reference. TEST INFRASTRUCTURE.

The reference's TaskPrompterWrapper and its 2D heads run as they are; the 3ddet head (FCOS3DHead, mmdet3d) is replaced by
nn.Identity, so out['3ddet'] is exactly what FCOS3D receives: the list of the 4 level maps [B, f, h_l, w_l]
(TP taskprompter_swin.py:709-710, taskprompter_wrapper.py:37-38). Weights: oracle.taskprompter_swin_ref.init_state_dict
without the oracle's dense stand-in parameters for '3ddet' (heads.3ddet.*), loaded into the reference.

    tests/golden/tps_tiny3d.pt              tiny, batch 2, every output in full
    tests/golden/tps_mid3d.pt               window 12 / 0.75 scaling, batch 1: the 2D outputs on a stride-8 lattice
                                            (oracle.make_golden.compress_output), the 3ddet maps in full
    tests/golden/big_tps_swinB3d_b1.pt.xz   the yml at 1024 x 2048, batch 1: everything lattice-sampled with exact norms

Each fixture also carries `keys`: the reference wrapper's state-dict names and shapes (3ddet head excluded).

    python -m oracle.make_golden_swin3d [tps_tiny3d tps_mid3d tps_swinB3d]
"""
import hashlib
import lzma
import os
import sys
import time

import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import configs, ref_loader  # noqa: E402
from oracle.make_golden import GOLD, big_input, compress_output, ref_keys, sd_checksum  # noqa: E402

JOBS = {"tps_tiny3d": (31, 2), "tps_mid3d": (32, 1), "tps_swinB3d": (47, 1)}   # config -> (seed, batch)
SWINB_STRIDE = 16                  # 2D outputs at 512 x 1024, as big_tps_swinB_b1
DET_STRIDES = (16, 16, 8, 8)       # 3ddet level maps 96x192 / 48x96 / 24x48 / 24x48 (450 channels each)


def state_dict(cfg, seed):
    """The oracle's deterministic weights without its dense stand-in head for '3ddet'."""
    from oracle import taskprompter_swin_ref as R
    return {k: v for k, v in R.init_state_dict(cfg, seed=seed).items() if not k.startswith("heads.3ddet.")}


def reference_model(cfg, sd=None):
    """The unmodified reference wrapper with nn.Identity as the 3ddet head (optionally with weights sd loaded)."""
    model = ref_loader.build_taskprompter_swin(cfg)
    model.heads["3ddet"] = nn.Identity()
    if sd is not None:
        missing, unexpected = model.load_state_dict(sd, strict=False)   # index / mask buffers are derived, not stored
        assert not unexpected and all("relative_position_index" in k or "attn_mask" in k for k in missing), \
            (missing, unexpected)
    return model.eval()


def make(name):
    seed, batch = JOBS[name]
    cfg = configs.taskprompter_swin(name)
    sd = state_dict(cfg, seed)
    model = reference_model(cfg, sd)
    x = big_input(cfg, seed, batch)
    with torch.no_grad():
        y = model(x)
    det = [m.clone() for m in y["3ddet"]]
    fx = {"family": "taskprompter_swin", "cfg": name, "seed": seed, "batch": batch, "keys": ref_keys(model),
          "x_sha256": hashlib.sha256(x.numpy().tobytes()).hexdigest(), "sd_sha256": sd_checksum(sd),
          "torch": torch.__version__,
          "made_by": "oracle/make_golden_swin3d.py: unmodified reference Swin TaskPrompter (eval, fp32, CPU), "
                     "3ddet head = nn.Identity"}
    tasks2d = [t for t in cfg["tasks"] if t != "3ddet"]
    if name == "tps_tiny3d":
        fx.update(x=x, out={**{t: y[t].clone() for t in tasks2d}, "3ddet": det})
    elif name == "tps_mid3d":
        fx.update(stride=8, out={**{t: compress_output(y[t], ti, stride=8) for ti, t in enumerate(tasks2d)}, "3ddet": det})
    else:
        fx.update(stride=SWINB_STRIDE, det_strides=DET_STRIDES,
                  out={**{t: compress_output(y[t], ti, stride=SWINB_STRIDE) for ti, t in enumerate(tasks2d)},
                       "3ddet": [compress_output(m, 2 + il, with_argmax=False, stride=s)
                                 for il, (m, s) in enumerate(zip(det, DET_STRIDES))]})
    return fx


def main(only=None):
    if not ref_loader.available():
        raise SystemExit("reference not found (set MTT_REFERENCE or mount /root/reference)")
    for name in JOBS:
        if only and name not in only:
            continue
        t0 = time.time()
        fx = make(name)
        if name == "tps_swinB3d":
            path = os.path.join(GOLD, f"big_{name}_b{fx['batch']}.pt.xz")
            with lzma.open(path, "wb", preset=9 | lzma.PRESET_EXTREME) as f:
                torch.save(fx, f)
        else:
            path = os.path.join(GOLD, f"{name}.pt")
            torch.save(fx, path)
        print(f"wrote {path} ({os.path.getsize(path) / 1024:.0f} KiB, {time.time() - t0:.0f} s)", flush=True)


if __name__ == "__main__":
    main(set(sys.argv[1:]) or None)
