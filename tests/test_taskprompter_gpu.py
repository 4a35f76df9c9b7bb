"""-m gpu: the fused CUDA TaskPrompter forward (through the C ABI) against the oracle restatement and the
golden vectors of the unmodified reference.

Tolerances (written here, per north_star: 1e-3 relative fp32; argmax exact):
  parity mode (nsplit=2): rel-L2 per task < 2e-4 and max-abs error < 1e-3 * max|ref|;
  argmax over classes must agree everywhere except pixels whose reference top-2 margin is below
  1e-4 * max|logit| (near ties flip under ANY change of fp32 summation order).
  speed mode (nsplit=1, plain bf16): rel-L2 < 6e-2, reported, not a parity claim.
"""
import os

import pytest
import torch

from model_checks import check_parity as _check
from oracle import configs
from oracle import taskprompter_ref as TPR

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _build(cfg, sd, nsplit, graph):
    import mtt_b200  # noqa: F401
    from mtt_b200 import taskprompter as TP

    m = TP.build_from_config(cfg, nsplit=nsplit, use_graph=graph).eval()
    m.load_state_dict(sd, strict=True)
    return m.cuda()


@pytest.mark.parametrize("name", ["tp_tiny", "tp_tiny1", "tp_tiny_de"])
def test_golden_parity(cuda_dev, name):
    fx = torch.load(os.path.join(GOLD, f"{name}.pt"), weights_only=False)
    cfg = configs.taskprompter(fx["cfg"])
    sd = TPR.init_state_dict(cfg, seed=fx["seed"])
    m = _build(cfg, sd, 2, False)
    with torch.no_grad():
        got = m(fx["x"].cuda())
    torch.cuda.synchronize()
    _check(got, fx["out"], cfg["tasks"], 2e-4, 1e-3)


@pytest.mark.parametrize("name", ["tp_tiny"])
def test_graph_replay_equals_eager_launch(cuda_dev, name):
    cfg = configs.taskprompter(name)
    sd = TPR.init_state_dict(cfg, seed=9)
    x = torch.randn(2, 3, *cfg["img_size"], device=cuda_dev)
    a = {k: v.clone() for k, v in _build(cfg, sd, 2, False)(x).items()}
    m = _build(cfg, sd, 2, True)
    m(x)
    b = m(x)   # second call = pure replay
    torch.cuda.synchronize()
    for t in cfg["tasks"]:
        assert torch.equal(a[t], b[t])


def test_speed_mode_error_reported(cuda_dev):
    cfg = configs.taskprompter("tp_tiny")
    sd = TPR.init_state_dict(cfg, seed=3)
    torch.manual_seed(5)
    x = torch.randn(2, 3, *cfg["img_size"])
    with torch.no_grad():
        ref = TPR.forward(sd, cfg, x)
        got = _build(cfg, sd, 1, False)(x.cuda())
    torch.cuda.synchronize()
    _check(got, ref, cfg["tasks"], 6e-2, 2e-1, check_argmax=False)


@pytest.mark.parametrize("name,batch", [("tp_cfg4_d4", 2), ("tp_cfg4", 1), ("tp_cfg2", 1), ("tp_long", 1)])
def test_full_width_parity(cuda_dev, name, batch):
    """Full-width parity against the CPU oracle on the same seeded weights and input: ViT-L cfg4 geometry
    (C=1024, 16 heads, N=1029, e=300, f=350, CTR) as a 4-block slice at bs 2 and the full 24-block model
    at bs 1; cfg2 (ViT-B, 448x576, 4x4 channel windows of 7x9, e=f=768, no CTR); and `tp_long` (256x2048, N = 2050,
    2x2 channel windows). The cfg5 geometry (N = 8195) and the bench batch sizes are covered against golden vectors of
    the unmodified reference in test_big_goldens_gpu.py."""
    cfg = configs.taskprompter(name)
    sd = TPR.init_state_dict(cfg, seed=21)
    torch.manual_seed(22)
    x = torch.randn(batch, 3, *cfg["img_size"])
    with torch.no_grad():
        ref = TPR.forward(sd, cfg, x)
    m = _build(cfg, sd, 2, True)
    with torch.no_grad():
        got = m(x.cuda())
    torch.cuda.synchronize()
    _check(got, ref, cfg["tasks"], 2e-4, 1e-3)


def test_predict_fused_postprocessing(cuda_dev):
    """predict(): bilinear-to-image fused with get_output (TP/utils/utils.py:27-63). Index maps must be
    bit-exact against the argmax of this build's own logits (same arithmetic), float maps within 1e-4, and
    agree with get_output(oracle logits) away from near ties."""
    from oracle import postproc_ref

    for name in ("tp_tiny", "tp_tiny1"):
        cfg = configs.taskprompter(name)
        sd = TPR.init_state_dict(cfg, seed=13)
        torch.manual_seed(14)
        x = torch.randn(2, 3, *cfg["img_size"])
        m = _build(cfg, sd, 2, False)
        with torch.no_grad():
            logits = {k: v.clone() for k, v in m(x.cuda()).items()}
            pred = m.predict(x.cuda())
            ref = TPR.forward(sd, cfg, x)
        torch.cuda.synchronize()
        for t in cfg["tasks"]:
            own = postproc_ref.get_output(logits[t], t)
            want = postproc_ref.get_output(ref[t], t)
            assert pred[t].shape == want.shape and pred[t].dtype == want.dtype
            if want.dtype == torch.int64:
                assert torch.equal(pred[t], own), t
                top2 = ref[t].topk(2, dim=1).values
                safe = (top2[:, 0] - top2[:, 1]) > 1e-4 * ref[t].abs().max()
                assert (pred[t].cpu() == want)[safe].all(), t
            else:
                assert (pred[t] - own).abs().max() <= 1e-4 * own.abs().max().clamp_min(1.0), t
                assert (pred[t].cpu() - want).abs().max() <= 2e-3 * want.abs().max().clamp_min(1.0), t
