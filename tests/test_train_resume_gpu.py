"""-m gpu: eval forwards after native training steps use the trained weights, and checkpoint / resume of the native loop
(TrainStep.state_dict / load_state_dict) through libmtt_sm90.so; the comparisons are those of tests/test_train_resume.py."""
import pytest
import torch

from test_train_resume import (as_torch_1_10, batches, build, criterion, native_checkpoint, native_steps,
                               next_step_mismatches, resume_mismatches, setup, torch_checkpoint)

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]


def _eval_calls(model, x):
    """model(x), model.predict(x), the backbone's and every head's own forward (outputs cloned: the wrapper writes into
    its plan's static buffers)."""
    with torch.no_grad():
        out = {f"forward.{t}": v.clone() for t, v in model(x).items()}
        out.update({f"predict.{t}": v.clone() for t, v in model.predict(x).items()})
        fea = model.backbone(x)[0]
        out.update({f"backbone.{t}": v for t, v in fea.items()})
        out.update({f"heads.{t}": model.heads[t](fea[t]) for t in model.tasks})
    return out


def _fresh_copy(cfg, model, device):
    fresh, _ = build(cfg, {k: v.clone() for k, v in model.state_dict().items()}, device)
    return fresh


@pytest.mark.parametrize("use_graph", [False, True])
def test_eval_forwards_use_the_trained_weights(cuda_dev, use_graph):
    """Plans and packed weights exist before training; after two native steps every eval forward is bit-identical to
    the same call on a fresh model holding the trained state_dict (same kernels, same packing)."""
    cfg, sd = setup()
    model, ts = build(cfg, sd, cuda_dev, use_graph=use_graph)
    model.use_graph = True
    x = batches(cfg, 1, cuda_dev, seed=3)[0][0]
    model.eval()
    _eval_calls(model, x)
    model.train()
    native_steps(ts, criterion(cfg, cuda_dev), batches(cfg, 2, cuda_dev))
    model.eval()
    got = _eval_calls(model, x)
    fresh = _fresh_copy(cfg, model, cuda_dev).eval()
    fresh.use_graph = True
    want = _eval_calls(fresh, x)
    stale = [k for k in want if not torch.equal(got[k], want[k])]
    assert not stale, f"eval forwards on older weights: {stale}"


def test_eval_forward_after_steps_full_width(cuda_dev):
    """tp_cfg4_d4 (ViT-L width, 512 x 512, 5 PASCAL tasks): model(x) after two native steps, BatchNorm folding of the
    trained running statistics at full width."""
    cfg, sd = setup("tp_cfg4_d4")
    model, ts = build(cfg, sd, cuda_dev)
    x = batches(cfg, 1, cuda_dev, seed=3)[0][0]
    with torch.no_grad():
        model.eval()(x)
    native_steps(ts, criterion(cfg, cuda_dev), batches(cfg, 2, cuda_dev))
    with torch.no_grad():
        got = {t: v.clone() for t, v in model.eval()(x).items()}
        want = _fresh_copy(cfg, model, cuda_dev).eval()(x)
    stale = [t for t in want if not torch.equal(got[t], want[t])]
    assert not stale, f"model(x) on older weights: {stale}"


@pytest.mark.parametrize("use_graph", [False, True])
def test_resume_equals_uninterrupted_run(cuda_dev, tmp_path, use_graph):
    assert resume_mismatches(cuda_dev, use_graph, tmp_path) == []
    # without the optimizer state (zero moments, step 1) the same comparison fails
    assert resume_mismatches(cuda_dev, use_graph, tmp_path, load_optimizer=False) != []


@pytest.mark.parametrize("source", ["native", "torch", "torch_1_10"])
def test_interchange_with_torch_adam(cuda_dev, tmp_path, source):
    """(native) a native checkpoint's 'optimizer' loads into torch.optim.Adam; (torch) TrainStep loads what
    torch.optim.Adam wrote after torch-facing steps; (torch_1_10) the same with int step counts. Then one native and one
    torch-facing step on the same batch make the same parameter updates."""
    ck = native_checkpoint(cuda_dev) if source == "native" else torch_checkpoint(cuda_dev)
    if source == "torch_1_10":
        ck["optimizer"] = as_torch_1_10(ck["optimizer"])
    assert next_step_mismatches(ck, cuda_dev, tmp_path) == []
