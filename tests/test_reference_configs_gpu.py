"""-m gpu: the reference's own model configs that the bench does not run -- TaskPrompter nyud_vitLp16_taskprompter
(tp_nyud_vitL), pascal_vitBp16_taskprompter (tp_pascal_vitB) and InvPT nyud_vitLp16 (ip_nyud_vitL) -- as whole models on
the device: the forward at full depth through the CUDA-graph replay against the oracle restatement in float64 on the
device with the same seeded weights, predict() at the reference's validation batch 6, and the reverse pass of a 4-block
slice of tp_pascal_vitB, the first whole reverse pass with cross-task reweighting over several channel windows.

Tolerances as in test_taskprompter_gpu.py (parity mode: rel-L2 per task < 2e-4, max-abs < 1e-3 max|ref|, arg-max
equal away from near ties); the reverse pass uses the bound and floor of
test_train_kernels_f64_gpu.py::test_training_step_reverse_pass_tp_cfg2_d4 (tests/model_checks.py)."""
import pytest
import torch

from model_checks import check_parity, reverse_pass_errors
from oracle import configs, postproc_ref

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
NEW = ["tp_nyud_vitL", "tp_pascal_vitB", "ip_nyud_vitL"]


def _model(name, seed, graph):
    """(cfg, state dict, device model with that state) of a TaskPrompter or InvPT config."""
    import mtt_b200  # noqa: F401
    from mtt_b200 import invpt as IP, taskprompter as TP
    from oracle import invpt_ref as IPR, taskprompter_ref as TPR

    ip = name.startswith("ip_")
    cfg = (configs.invpt if ip else configs.taskprompter)(name)
    sd = (IPR if ip else TPR).init_state_dict(cfg, seed=seed)
    m = (IP if ip else TP).build_from_config(cfg, nsplit=2, use_graph=graph).eval()
    m.load_state_dict(sd, strict=True)
    return cfg, sd, m.cuda()


@pytest.mark.parametrize("name", NEW)
def test_forward_parity_f64(cuda_dev, name):
    """Full depth, batch 2, the second call of a graph-captured plan (a pure replay) against the float64 oracle."""
    from oracle import invpt_ref as IPR, taskprompter_ref as TPR

    cfg, sd, m = _model(name, seed=51, graph=True)
    g = torch.Generator().manual_seed(52)
    x = torch.randn(2, 3, *cfg["img_size"], generator=g).to(cuda_dev)
    with torch.no_grad():
        m(x)
        got = m(x)
        got = {k: ({t: v.clone() for t, v in o.items()} if isinstance(o, dict) else o.clone()) for k, o in got.items()}
    torch.cuda.synchronize()
    del m
    torch.cuda.empty_cache()
    sdd = {k: (v.to(cuda_dev).double() if v.is_floating_point() else v.to(cuda_dev)) for k, v in sd.items()}
    with torch.no_grad():
        ref = (IPR if name.startswith("ip_") else TPR).forward(sdd, cfg, x.double())
    errs = check_parity(got, ref, cfg["tasks"], 2e-4, 1e-3)
    if name.startswith("ip_"):
        inter = check_parity(got["inter_preds"], ref["inter_preds"], cfg["tasks"], 2e-4, 1e-3)
        errs.update({f"inter_preds.{t}": v for t, v in inter.items()})
    for t, (e2, em) in errs.items():
        print(f"{name} b2 {t}: rel-L2 {e2:.2e} (< 2e-4), max-abs / max|ref| {em:.2e} (< 1e-3)")


@pytest.mark.parametrize("name", NEW)
def test_predict_at_the_validation_batch(cuda_dev, name):
    """predict() at valBatch 6: index maps bit-exact against the arg-max of the same build's logits (the same
    arithmetic), float maps within 1e-4 of get_output of them."""
    cfg, _, m = _model(name, seed=53, graph=True)
    g = torch.Generator().manual_seed(54)
    x = torch.randn(6, 3, *cfg["img_size"], generator=g).to(cuda_dev)
    with torch.no_grad():
        out = m(x)
        logits = {t: out[t].clone() for t in cfg["tasks"]}
        pred = m.predict(x)
    torch.cuda.synchronize()
    for t in cfg["tasks"]:
        own = postproc_ref.get_output(logits[t], t)
        assert pred[t].shape == own.shape and pred[t].dtype == own.dtype, t
        if own.dtype == torch.int64:
            assert torch.equal(pred[t], own), f"{name} {t}: {int((pred[t] != own).sum())} class indices differ"
            print(f"{name} b6 {t}: class map bit-exact")
        else:
            err = float((pred[t] - own).abs().max() / own.abs().max().clamp_min(1.0))
            assert err <= 1e-4, f"{name} {t}: {err:.2e}"
            print(f"{name} b6 {t}: max-abs / max {err:.2e} (<= 1e-4)")


def test_training_step_reverse_pass_tp_pascal_vitB_d4(cuda_dev):
    """tp_pascal_vitB_d4 (ViT-B width, 512 x 512, the 5 PASCAL tasks, ctr with 12 heads over 4 x 4 channel windows,
    e = 780, f = 1024), batch 2: every parameter gradient of TrainStep.backward against float64 autograd of the
    train-mode restatement, fed the same d loss / d prediction."""
    fwd, bad, n = reverse_pass_errors("tp_pascal_vitB_d4", cuda_dev, seed=41, B=2)
    for t, err in fwd.items():
        assert err < 2e-4, f"train-mode forward {t}: rel-L2 {err:.3e}"
    print(f"tp_pascal_vitB_d4 b2: train-mode forward rel-L2 max {max(fwd.values()):.2e}; {n} parameter gradients, "
          f"{len(bad)} off")
    assert not bad, f"{len(bad)} of {n} parameter gradients off: {bad[:8]}"
