"""-m gpu: the BASELINE.json configurations at FULL size and at the batch the bench times, through the same
CUDA-graph replay the bench uses, against golden vectors made here by the UNMODIFIED reference
(oracle/make_golden.py `big`; tests/golden/big_*.pt). No oracle run on the GPU box, no environment gate.

  big_tp_cfg5_d4_b1   TaskPrompter 1024x2048, N = 8195 tokens (65 query tiles, ragged last key block), 4 blocks
  big_tp_cfg5_b1      the same geometry, all 24 blocks (BASELINE.json configs[4])
  big_tp_cfg4_b4      the bench configuration: ViT-L PASCAL 512x512, 24 blocks, bs 4, graph replay
  big_tp_cfg2_b4      ViT-B NYUD 448x576 bs 4 (configs[1])
  big_ip_cfg3_b4      InvPT ViT-L PASCAL 512x512 bs 4 (configs[2])
  big_tps_swinB_b1    Swin-B TaskPrompter Cityscapes-3D 1024x2048 bs 1, stride-16 lattice, .pt.xz (tests/test_swin_big_gpu.py:
                      forward and predict())

A fixture holds every output value on a stride-8 pixel lattice (offset varies per image and task), the exact
norm and max of the full tensors, and for multi-class tasks the full-resolution arg-max map plus the mask of
pixels whose reference top-2 margin exceeds 1e-4 * max|logit| (bit-packed).

Tolerances (north_star: 1e-3 relative fp32, arg-max exact): rel-L2 on the lattice < 2e-4, max-abs on the lattice
< 1e-3 * max|ref|, |norm(got) / norm(ref) - 1| < 1e-4 on the FULL tensor, arg-max equal at every safe pixel of the
FULL map and > 0.999 agreement overall. Every measured number is appended to test_records/parity.json.
"""
import hashlib
import json
import os

import pytest
import torch

from oracle import configs
from oracle import invpt_ref as IPR
from oracle import taskprompter_ref as TPR

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
RECORD = os.path.join(ROOT, "test_records", "parity.json")


def lattice(b, ti, H, W, stride):
    oy, ox = (3 * b + 5 * ti + 1) % stride, (5 * b + 3 * ti + 2) % stride
    return torch.arange(oy, H, stride), torch.arange(ox, W, stride)


def record(case, metrics):
    os.makedirs(os.path.dirname(RECORD), exist_ok=True)
    data = {}
    if os.path.exists(RECORD):
        try:
            with open(RECORD) as f:
                data = json.load(f)
        except Exception:
            data = {}
    data[case] = metrics
    with open(RECORD, "w") as f:
        json.dump(data, f, indent=1, sort_keys=True)


def compare(got, rec, ti, stride, rel_l2=2e-4, max_rel=1e-3):
    """got: CUDA tensor [B,n,H,W]; rec: fixture record. Returns the metrics dict (asserts the tolerances)."""
    assert tuple(got.shape) == tuple(rec["shape"])
    assert torch.isfinite(got).all()
    B, n, H, W = got.shape
    g = got.float()
    samp = []
    for b in range(B):
        iy, ix = lattice(b, ti, H, W, stride)
        samp.append(g[b][:, iy.to(g.device)][:, :, ix.to(g.device)])
    samp = torch.stack(samp).cpu()
    ref = rec["samples"]
    m = {"rel_l2_lattice": ((samp - ref).norm() / ref.norm()).item(),
         "max_abs_over_max": ((samp - ref).abs().max() / rec["absmax"]).item(),
         "norm_ratio_full": g.double().norm().item() / rec["norm"],
         "lattice_points": int(ref.numel()), "full_elements": int(g.numel())}
    if "argmax" in rec:
        am = g.argmax(1).cpu()
        agree = am == rec["argmax"].long()
        import numpy as np
        safe = torch.from_numpy(np.unpackbits(rec["safe_bits"].numpy())[:agree.numel()].astype(bool)).reshape(agree.shape)
        m["argmax_agreement_all_pixels"] = agree.float().mean().item()
        m["argmax_pixels"] = int(agree.numel())
        m["margin_masked_pixels"] = int((~safe).sum())
        m["argmax_mismatch_safe_pixels"] = int((~agree & safe).sum())
        m["argmax_mismatch_masked_pixels"] = int((~agree & ~safe).sum())
    assert m["rel_l2_lattice"] < rel_l2, m
    assert m["max_abs_over_max"] < max_rel, m
    assert abs(m["norm_ratio_full"] - 1) < 1e-4, m
    if "argmax" in rec:
        assert m["argmax_mismatch_safe_pixels"] == 0, m
        assert m["argmax_agreement_all_pixels"] > 0.999, m
    return m


def _input(fx, cfg):
    g = torch.Generator().manual_seed(fx["seed"] + 1000)
    x = torch.randn(fx["batch"], 3, *cfg["img_size"], generator=g)
    assert hashlib.sha256(x.numpy().tobytes()).hexdigest() == fx["x_sha256"], "input regeneration differs"
    return x


BIG = ["big_tp_cfg5_d4_b1", "big_tp_cfg4_b4", "big_tp_cfg2_b4", "big_ip_cfg3_b4", "big_tp_cfg5_b1"]


@pytest.mark.parametrize("name", BIG)
def test_big_golden_graph_replay(cuda_dev, name):
    path = os.path.join(GOLD, name + ".pt")
    assert os.path.exists(path), f"{path} missing: python -m oracle.make_golden big"
    fx = torch.load(path, weights_only=False)
    import mtt_b200  # noqa: F401
    if fx["family"] == "taskprompter":
        from mtt_b200 import taskprompter as M
        cfg = configs.taskprompter(fx["cfg"])
        sd = TPR.init_state_dict(cfg, seed=fx["seed"])
    else:
        from mtt_b200 import invpt as M
        cfg = configs.invpt(fx["cfg"])
        sd = IPR.init_state_dict(cfg, seed=fx["seed"])
    x = _input(fx, cfg)
    model = M.build_from_config(cfg, nsplit=2, use_graph=True).eval()
    model.load_state_dict(sd, strict=True)
    model = model.cuda()
    with torch.no_grad():
        model(x.cuda())            # capture
        got = model(x.cuda())      # pure graph replay: what bench.py times
    torch.cuda.synchronize()
    metrics = {}
    for ti, t in enumerate(cfg["tasks"]):
        metrics[t] = compare(got[t], fx["out"][t], ti, fx["stride"])
    if fx.get("inter_preds"):
        for ti, t in enumerate(cfg["tasks"]):
            metrics["inter_preds." + t] = compare(got["inter_preds"][t], fx["inter_preds"][t], ti, fx["stride"])
    record(name, {"config": fx["cfg"], "batch": fx["batch"], "mode": "parity (bf16x3), CUDA-graph replay",
                  "reference": fx["made_by"], "tasks": metrics})
    del model
    torch.cuda.empty_cache()
