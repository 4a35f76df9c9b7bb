"""Whole-model comparisons shared by the model-level GPU tests: the output parity check against a reference forward,
and the reverse pass of a TaskPrompter training step against float64 autograd of the train-mode restatement."""
import math

import torch

from oracle import configs

GRAD_REL_L2 = 2e-3       # per parameter gradient, relative to max(|ref|, GRAD_FLOOR x the norm of all gradients)
GRAD_FLOOR = 1e-4


def check_parity(got, ref, tasks, rel_l2, max_rel, check_argmax=True):
    """Per task: finite, rel-L2 < rel_l2, max-abs error < max_rel * max|ref|, and (with check_argmax, for maps of more
    than one channel) the arg-max over channels equal wherever the reference's top-2 margin exceeds 1e-4 max|ref| (near
    ties flip under any change of fp32 summation order) and on more than 99.9 % of the pixels. Returns {task: (rel-L2,
    max-abs / max|ref|)}."""
    errs = {}
    for t in tasks:
        g, r = got[t].float().cpu(), ref[t].float().cpu()
        assert g.shape == r.shape, (t, g.shape, r.shape)
        assert torch.isfinite(g).all(), t
        e2 = ((g - r).norm() / r.norm()).item()
        em = ((g - r).abs().max() / r.abs().max()).item()
        errs[t] = (e2, em)
        assert e2 < rel_l2, f"{t}: rel-L2 {e2:.3e}"
        assert em < max_rel, f"{t}: max-abs/max {em:.3e}"
        if check_argmax and r.shape[1] > 1:
            top2 = r.topk(2, dim=1).values
            margin = top2[:, 0] - top2[:, 1]
            safe = margin > 1e-4 * r.abs().max()
            agree = g.argmax(1) == r.argmax(1)
            assert agree[safe].all(), f"{t}: argmax differs at {(~agree & safe).sum().item()} safe pixels"
            assert agree.float().mean().item() > 0.999, f"{t}: argmax agreement {agree.float().mean().item():.5f}"
    return errs


def reverse_pass_errors(name, dev, seed, B):
    """The TaskPrompter config `name` at batch B with seeded weights, train mode: the same d loss / d prediction through
    TrainStep.backward and through float64 autograd of the train-mode restatement (oracle/taskprompter_ref.py, DropPath
    draws from a CPU generator in the reference's call order). Returns ({task: rel-L2 of the train-mode forward},
    [(parameter, error) of every gradient whose error is not below GRAD_REL_L2, worst first], number of parameters); a
    gradient's error is its L2 distance from float64 over max(its norm, GRAD_FLOOR x the norm of all gradients).

    Why 2e-3: split-bf16 GEMMs carry 2^-17 relative per operand; chained through the blocks and the decoder the
    gradients of the 4-block slices stay within 2e-3 rel-L2, and the floor admits parameters whose gradient is zero up
    to noise."""
    import mtt_b200  # noqa: F401
    from mtt_b200 import losses
    from mtt_b200 import taskprompter as TP
    from mtt_b200.train import TrainStep
    from oracle import taskprompter_ref as TPR
    from oracle.make_golden import train_inputs

    cfg = configs.taskprompter(name)
    sd = TPR.init_state_dict(cfg, seed=seed)
    model = TP.build_from_config(cfg, use_graph=False)
    model.load_state_dict(sd, strict=True)
    model.to(dev)
    ts = TrainStep(model)
    n_act = sum(1 for r in torch.linspace(0, 0.15, cfg["depth"]) if float(r) > 0)
    gcpu = torch.Generator().manual_seed(seed + 900)
    masks = [torch.rand(B, 1, 1, generator=gcpu) for _ in range(4 * n_act)]
    x, labels = train_inputs(cfg, seed, B)
    ts.zero_grad()
    with torch.no_grad():
        out = ts.forward(x.to(dev), drop_rand=masks)
    p = dict(TASKS=dict(NAMES=list(cfg["tasks"])), edge_w=0.95, ignore_index=255, ignore_invalid_area_depth=True,
             loss_kwargs=dict(loss_weights={t: 1.0 for t in cfg["tasks"]}))
    leaves = {t: out[t].detach().requires_grad_(True) for t in cfg["tasks"]}
    loss = losses.get_criterion(p)(leaves, {t: v.to(dev) for t, v in labels.items()}, tasks=cfg["tasks"])
    grads = dict(zip(cfg["tasks"], torch.autograd.grad(loss["total"], [leaves[t] for t in cfg["tasks"]])))
    with torch.no_grad():
        ts.backward(grads)
    torch.cuda.synchronize()
    # float64 autograd of the train-mode restatement with the same draws and the same d loss / d prediction
    sdd = {k: (v.to(dev).double() if v.is_floating_point() else v.to(dev)) for k, v in sd.items()}
    params = {k: v.requires_grad_(True) for k, v in sdd.items() if v.is_floating_point() and "running_" not in k}
    with TPR.train_mode(0.15, rand=[m.to(dev).double() for m in masks]):
        ref_out = TPR.forward(sdd, cfg, x.to(dev).double())
    fwd = {t: ((out[t].double() - ref_out[t].detach()).norm() / ref_out[t].detach().norm()).item() for t in cfg["tasks"]}
    torch.autograd.backward([ref_out[t] for t in cfg["tasks"]], [grads[t].double() for t in cfg["tasks"]])
    og = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in params.items()}
    total = math.sqrt(sum(float((g ** 2).sum()) for g in og.values()))
    floor = GRAD_FLOOR * total
    bad = []
    for k, ref in og.items():
        err = (ts.G_(k).double() - ref).norm().item() / max(ref.norm().item(), floor)
        if not err < GRAD_REL_L2:
            bad.append((k, err))
    return fwd, sorted(bad, key=lambda kv: -kv[1]), len(og)
