"""-m gpu: the fused CUDA InvPT forward (ViT backbone + inverted-pyramid decoder) against the golden
vectors of the unmodified reference and the CPU oracle restatement. Tolerances as in
test_taskprompter_gpu.py (parity mode: rel-L2 < 2e-4, max-abs < 1e-3 of max|ref|, argmax exact away
from near ties)."""
import os

import pytest
import torch

from model_checks import check_parity as _check
from oracle import configs
from oracle import invpt_ref as IPR

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _build(cfg, sd, nsplit, graph):
    import mtt_b200  # noqa: F401
    from mtt_b200 import invpt as IP

    m = IP.build_from_config(cfg, nsplit=nsplit, use_graph=graph).eval()
    m.load_state_dict(sd, strict=True)
    return m.cuda()


@pytest.mark.parametrize("name", ["ip_tiny", "ip_cfg1"])
def test_golden_parity(cuda_dev, name):
    fx = torch.load(os.path.join(GOLD, f"{name}.pt"), weights_only=False)
    cfg = configs.invpt(fx["cfg"])
    sd = IPR.init_state_dict(cfg, seed=fx["seed"])
    m = _build(cfg, sd, 2, False)
    with torch.no_grad():
        got = m(fx["x"].cuda())
    torch.cuda.synchronize()
    _check(got, fx["out"], cfg["tasks"], 2e-4, 1e-3)
    if fx["inter_preds"] is not None:
        _check(got["inter_preds"], fx["inter_preds"], cfg["tasks"], 2e-4, 1e-3)


def test_graph_replay_equals_eager_launch(cuda_dev):
    cfg = configs.invpt("ip_tiny")
    sd = IPR.init_state_dict(cfg, seed=9)
    x = torch.randn(2, 3, *cfg["img_size"], device=cuda_dev)
    a = _build(cfg, sd, 2, False)(x)
    a = {k: a[k].clone() for k in cfg["tasks"]}
    m = _build(cfg, sd, 2, True)
    m(x)
    b = m(x)
    torch.cuda.synchronize()
    for t in cfg["tasks"]:
        assert torch.equal(a[t], b[t])


def test_full_width_parity(cuda_dev):
    """InvPT ViT-L PASCAL-Context (BASELINE.json configs[2]) at bs 1 against the CPU oracle."""
    cfg = configs.invpt("ip_cfg3")
    sd = IPR.init_state_dict(cfg, seed=31)
    torch.manual_seed(32)
    x = torch.randn(1, 3, *cfg["img_size"])
    with torch.no_grad():
        ref = IPR.forward(sd, cfg, x)
    m = _build(cfg, sd, 2, True)
    with torch.no_grad():
        got = m(x.cuda())
    torch.cuda.synchronize()
    _check(got, ref, cfg["tasks"], 2e-4, 1e-3)
    _check(got["inter_preds"], ref["inter_preds"], cfg["tasks"], 2e-4, 1e-3)
