"""-m gpu: the Swin-B TaskPrompter (tps_swinB, the Cityscapes-3D model bench.py times) at FULL size, 1024x2048, bs 1,
through the CUDA-graph replay the bench uses, against the golden vectors of the UNMODIFIED reference
(tests/golden/big_tps_swinB_b1.pt.xz, `python -m oracle.make_golden big tps_swinB`). The fixture samples the outputs on
a stride-16 lattice (at stride 8 the 19 channels at 512x1024 are 620 KB of fp32 that does not compress) and keeps the
full-tensor norms and the full-resolution arg-max map. The fixture's weights come from
oracle.taskprompter_swin_ref.init_state_dict: relative-position bias tables at std 0.5 and non-trivial BatchNorm
statistics, so a mis-indexed bias or shift-mask entry moves the output.

Two cases:
  forward    the wrapper forward (logits at dd_label_map_size 512x1024) with the tolerances of test_big_goldens_gpu.py:
             rel-L2 on the lattice < 2e-4, max-abs < 1e-3 * max|ref|, full-tensor norm ratio within 1e-4, arg-max exact
             at every safe pixel and > 0.999 overall. Metrics go to test_records/parity.json.
  predict()  the reference's get_output fused into the final resize, what the Cityscapes-3D meters read: the semseg label
             map equals the fixture's arg-max at every safe pixel; depth post-processing is max(x, 0), so the depth map
             is checked on the lattice against the clamped fixture samples with the same tolerances.
"""
import lzma
import os

import numpy as np
import pytest
import torch

from oracle import configs
from oracle import taskprompter_swin_ref as R

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
NAME = "big_tps_swinB_b1"


@pytest.fixture(scope="module")
def swinB(cuda_dev):
    """(fixture, cfg, model on the GPU with the fixture's weights, input on the GPU)."""
    from test_big_goldens_gpu import _input

    path = os.path.join(GOLD, NAME + ".pt.xz")
    assert os.path.exists(path), f"{path} missing: python -m oracle.make_golden big tps_swinB"
    with lzma.open(path, "rb") as f:
        fx = torch.load(f, weights_only=False)
    import mtt_b200  # noqa: F401
    from mtt_b200 import taskprompter_swin as TS

    cfg = configs.taskprompter_swin(fx["cfg"])
    sd = R.init_state_dict(cfg, seed=fx["seed"])
    x = _input(fx, cfg)
    model = TS.build_from_config(cfg, nsplit=2, use_graph=True).eval()
    missing, unexpected = model.load_state_dict(sd, strict=False)     # index / mask buffers are derived, not stored
    assert not unexpected and all("relative_position_index" in k or "attn_mask" in k for k in missing)
    yield fx, cfg, model.to(cuda_dev), x.to(cuda_dev)
    del model
    torch.cuda.empty_cache()


def test_swinB_big_golden_graph_replay(swinB):
    from test_big_goldens_gpu import compare, record

    fx, cfg, model, x = swinB
    with torch.no_grad():
        model(x)                 # capture
        got = model(x)           # pure graph replay: what bench.py times
    torch.cuda.synchronize()
    metrics = {t: compare(got[t], fx["out"][t], ti, fx["stride"]) for ti, t in enumerate(cfg["tasks"])}
    record(NAME, {"config": fx["cfg"], "batch": fx["batch"], "mode": "parity (bf16x3), CUDA-graph replay",
                  "reference": fx["made_by"], "tasks": metrics})


def test_swinB_big_golden_predict(swinB):
    from test_big_goldens_gpu import lattice

    fx, cfg, model, x = swinB
    with torch.no_grad():
        model.predict(x)         # capture
        got = model.predict(x)   # graph replay
    torch.cuda.synchronize()
    rec = fx["out"]["semseg"]
    B, n, H, W = rec["shape"]
    lab = got["semseg"].cpu()
    assert lab.dtype == torch.int64 and tuple(lab.shape) == (B, H, W)
    agree = lab == rec["argmax"].long()
    safe = torch.from_numpy(np.unpackbits(rec["safe_bits"].numpy())[:agree.numel()].astype(bool)).reshape(agree.shape)
    assert int((~agree & safe).sum()) == 0, int((~agree & safe).sum())
    assert agree.float().mean().item() > 0.999
    ti, rec = cfg["tasks"].index("depth"), fx["out"]["depth"]
    dep = got["depth"]
    assert tuple(dep.shape) == (B, H, W, 1) and torch.isfinite(dep).all()
    samp = []
    for b in range(B):
        iy, ix = lattice(b, ti, H, W, fx["stride"])
        samp.append(dep[b, :, :, 0][iy.to(dep.device)][:, ix.to(dep.device)].cpu())
    samp, ref = torch.stack(samp), rec["samples"][:, 0].clamp_min(0)     # get_output's depth clamp
    assert ((samp - ref).norm() / ref.norm()).item() < 2e-4
    assert ((samp - ref).abs().max() / rec["absmax"]).item() < 1e-3
