"""Checkpoint and resume of the native training loop (TrainStep.state_dict / load_state_dict, the Adam state in
torch.optim.Adam's format): a resumed run continues the uninterrupted one, the state interchanges with torch.optim.Adam in
both directions (torch 1.10's int step counts included), and malformed state is refused.

CPU: the kernels emulated through tests/emul_ops.py. tests/test_train_resume_gpu.py (-m gpu) runs the same comparisons
through libmtt_sm90.so and checks that eval forwards after native steps use the trained weights. DropPath is 0 wherever
two runs are compared."""
import pytest
import torch

from oracle import configs, loss_ref
from oracle import taskprompter_ref as TPR

LR = 1e-4
WEIGHTS = {"semseg": 1.0, "human_parts": 2.0, "sal": 5.0, "edge": 50.0, "normals": 10.0, "depth": 1.0}


def relerr(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).abs().max() / b.abs().max().clamp_min(1e-30)).item()


def setup(name="tp_tiny1", seed=5):
    cfg = configs.taskprompter(name)
    cfg["drop_path_rate"] = 0.0
    return cfg, TPR.init_state_dict(cfg, seed=seed)


def build(cfg, sd, device, use_graph=False, lr=LR):
    """A fresh model holding `sd` and its TrainStep."""
    import mtt_b200  # noqa: F401
    from mtt_b200 import taskprompter as TP
    from mtt_b200.train import TrainStep

    model = TP.build_from_config(cfg, use_graph=False)
    model.load_state_dict(sd, strict=True)
    model.to(device)
    return model, TrainStep(model, lr=lr, use_graph=use_graph)


def batches(cfg, n, device, B=2, seed=9):
    from oracle.make_golden import synthetic_labels

    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(n):
        x = torch.randn(B, 3, *cfg["img_size"], generator=g)
        y = synthetic_labels(cfg["tasks"], cfg["num_output"], B, *cfg["img_size"], g)
        out.append((x.to(device), {t: v.to(device) for t, v in y.items()}))
    return out


def criterion(cfg, device):
    """The library's loss kernels on the GPU; their torch restatement (oracle/loss_ref.py) under emulation."""
    w = {t: WEIGHTS[t] for t in cfg["tasks"]}
    if device.type == "cuda":
        from mtt_b200 import losses

        return losses.get_criterion(dict(TASKS=dict(NAMES=list(cfg["tasks"])), edge_w=0.95, ignore_index=255,
                                         ignore_invalid_area_depth=True, loss_kwargs=dict(loss_weights=w)))
    return lambda out, y, tasks=None: loss_ref.multi_task_loss(out, y, tasks, w)


def native_steps(ts, crit, bs):
    with torch.no_grad():
        return [float(ts.step(x, y, crit)["total"]) for x, y in bs]


def torch_step(ts, opt, crit, x, y):
    """One step of the reference loop on the torch-facing front end (train_utils.py:36-50)."""
    out = ts.apply(x)
    loss = crit(out, y, tasks=ts.tasks)
    loss["total"].backward()
    torch.nn.utils.clip_grad_norm_(ts.model.parameters(), 10.0)
    opt.step()
    return float(loss["total"].detach())


def save_load(ckpt, path):
    torch.save(ckpt, path)
    return torch.load(path, weights_only=False)


def resume_mismatches(device, use_graph, tmp_path, load_optimizer=True):
    """Run A: 5 native steps. Run B: 3 steps, checkpoint to a file, a fresh model + TrainStep load it (the optimizer
    state only when `load_optimizer`), 2 more steps on the same batches. Returns what differs from run A (empty = the
    resumed run continues A): losses of steps 4 and 5 (1e-4 relative), Adam moments and gradients (1e-3 relative to the
    largest element), parameters (as test_train_gpu.py::test_graph_replay_equals_eager_steps compares running
    statistics: a bias in front of a BatchNorm has a zero gradient up to atomics-order noise, which Adam turns into
    +-lr steps)."""
    cfg, sd = setup()
    crit = criterion(cfg, device)
    bs = batches(cfg, 5, device)
    model_a, ts_a = build(cfg, sd, device)
    loss_a = native_steps(ts_a, crit, bs)
    model_b, ts_b = build(cfg, sd, device)
    native_steps(ts_b, crit, bs[:3])
    ck = save_load({"model": model_b.state_dict(), "optimizer": ts_b.state_dict()}, tmp_path / "ckpt.pt")
    del model_b, ts_b
    model_c, ts_c = build(cfg, setup(seed=6)[1], device, use_graph=use_graph)     # other weights: all must come from ck
    model_c.load_state_dict(ck["model"])
    if load_optimizer:
        ts_c.load_state_dict(ck["optimizer"])
    loss_c = native_steps(ts_c, crit, bs[3:])
    if device.type == "cuda":
        torch.cuda.synchronize()
    bad = [f"loss of step {i + 4}: {a} vs {c}" for i, (a, c) in enumerate(zip(loss_a[3:], loss_c))
           if abs(a - c) > 1e-4 * max(1.0, abs(a))]
    for what, a, c in (("exp_avg", ts_a.m, ts_c.m), ("exp_avg_sq", ts_a.v, ts_c.v), ("gradients", ts_a.grads.flat,
                                                                                      ts_c.grads.flat)):
        if not relerr(c, a) < 1e-3:
            bad.append(f"{what}: relative error {relerr(c, a):.2e}")
    sa, sc = model_a.state_dict(), model_c.state_dict()
    bad += [k for k in sa if sa[k].is_floating_point() and not torch.allclose(sa[k], sc[k], rtol=2e-3, atol=5e-3)]
    if ts_c.step_no != ts_a.step_no:
        bad.append(f"step count {ts_c.step_no} vs {ts_a.step_no}")
    return bad


def next_step_mismatches(ck, device, tmp_path):
    """From the checkpoint `ck` = {'model', 'optimizer'} one native step (TrainStep.load_state_dict) and one torch-facing
    step (torch.optim.Adam.load_state_dict) on the same batch. Returns the parameters whose updates differ by the rule
    of test_train_gpu.py::_run_step (more than 2 % of elements off by more than 1e-3 relative + 2e-7); parameters whose
    gradient is below 1e-4 of the total norm are skipped (zero up to rounding: Adam's step is then noise)."""
    cfg, _ = setup()
    crit = criterion(cfg, device)
    x, y = batches(cfg, 1, device, seed=11)[0]
    ck = save_load(ck, tmp_path / "next.pt")
    model_n, ts_n = build(cfg, ck["model"], device, lr=1.0)          # the hyper-parameters must come from ck
    ts_n.load_state_dict(ck["optimizer"])
    model_t, ts_t = build(cfg, ck["model"], device)
    opt = torch.optim.Adam(model_t.parameters())
    opt.load_state_dict(ck["optimizer"])
    before = {k: v.clone() for k, v in model_n.named_parameters()}
    native_steps(ts_n, crit, [(x, y)])
    torch_step(ts_t, opt, crit, x, y)
    total = float(ts_n.grads.flat.norm())
    bad = []
    for (k, got), (_, ref) in zip(model_n.named_parameters(), model_t.named_parameters()):
        if float(ts_n.G_(k).norm()) < 1e-4 * total:
            continue
        step_got, step_ref = (got - before[k]).detach().cpu(), (ref - before[k]).detach().cpu()
        close = (step_got - step_ref).abs() <= 1e-3 * step_ref.abs() + 2e-7
        if not close.float().mean() > 0.98:
            bad.append((k, close.float().mean().item()))
    return bad


def native_checkpoint(device, n=2):
    cfg, sd = setup()
    model, ts = build(cfg, sd, device)
    native_steps(ts, criterion(cfg, device), batches(cfg, n, device))
    return {"model": model.state_dict(), "optimizer": ts.state_dict()}


def torch_checkpoint(device, n=2):
    """n torch-facing steps with torch.optim.Adam: the checkpoint the reference's loop writes (train_utils.py:128)."""
    cfg, sd = setup()
    model, ts = build(cfg, sd, device)
    opt = torch.optim.Adam(model.parameters(), lr=LR, weight_decay=1e-6)
    crit = criterion(cfg, device)
    for x, y in batches(cfg, n, device):
        torch_step(ts, opt, crit, x, y)
    return {"model": model.state_dict(), "optimizer": opt.state_dict()}


def as_torch_1_10(osd):
    """What torch 1.10's Adam writes: 'step' as a Python int and no group keys newer than amsgrad."""
    g = {k: osd["param_groups"][0][k] for k in ("lr", "betas", "eps", "weight_decay", "amsgrad", "params")}
    state = {i: dict(s, step=int(s["step"])) for i, s in osd["state"].items()}
    return {"state": state, "param_groups": [g]}


# ---- CPU (kernels emulated) ------------------------------------------------------------------------------------------
@pytest.fixture
def emulated(monkeypatch):
    import mtt_b200  # noqa: F401
    import emul_ops

    emul_ops.install(monkeypatch)
    return torch.device("cpu")


def test_state_dict_is_torch_adams(emulated):
    cfg, sd = setup()
    model, ts = build(cfg, sd, emulated)
    opt = torch.optim.Adam(model.parameters(), lr=LR, weight_decay=1e-6)
    assert ts.state_dict() == opt.state_dict()                        # fresh: no state, same group
    crit = criterion(cfg, emulated)
    bs = batches(cfg, 3, emulated)
    native_steps(ts, crit, bs[:2])
    got = ts.state_dict()
    names = [n for n, _ in model.named_parameters()]
    assert got["param_groups"] == opt.state_dict()["param_groups"]
    assert sorted(got["state"]) == list(range(len(names)))
    for i, n in enumerate(names):
        s = got["state"][i]
        assert set(s) == {"step", "exp_avg", "exp_avg_sq"}
        assert s["step"].dtype == torch.get_default_dtype() and s["step"].dim() == 0 and float(s["step"]) == 2
        assert torch.equal(s["exp_avg"], ts._moment(ts.m, n)) and torch.equal(s["exp_avg_sq"], ts._moment(ts.v, n))
    # copies: a kept dict does not move under later steps
    keep = {i: s["exp_avg"].clone() for i, s in got["state"].items()}
    native_steps(ts, crit, bs[2:])
    assert all(torch.equal(got["state"][i]["exp_avg"], keep[i]) for i in keep)
    assert float(ts.state_dict()["state"][0]["step"]) == 3


def test_load_state_dict_round_trip_and_fresh_optimizer(emulated):
    cfg, sd = setup()
    model, ts = build(cfg, sd, emulated)
    native_steps(ts, criterion(cfg, emulated), batches(cfg, 2, emulated))
    osd = ts.state_dict()
    m_ptr, v_ptr = ts.m.data_ptr(), ts.v.data_ptr()
    _, ts2 = build(cfg, sd, emulated, lr=1.0)
    ts2.load_state_dict(osd)
    assert ts2.step_no == 2 and ts2.hyper == ts.hyper
    assert torch.equal(ts2.m, ts.m) and torch.equal(ts2.v, ts.v)
    ts.load_state_dict(torch.optim.Adam(model.parameters(), lr=3e-4).state_dict())    # empty state = step 0
    assert (ts.m.data_ptr(), ts.v.data_ptr()) == (m_ptr, v_ptr)                        # in place
    assert ts.step_no == 0 and ts.hyper["lr"] == 3e-4 and not ts.m.any() and not ts.v.any()
    ts.load_state_dict(as_torch_1_10(osd))                                             # int steps, older group keys
    assert ts.step_no == 2 and ts.hyper == ts2.hyper
    assert torch.equal(ts.m, ts2.m) and torch.equal(ts.v, ts2.v)


def test_resume_equals_uninterrupted_run(emulated, tmp_path):
    assert resume_mismatches(emulated, False, tmp_path) == []
    assert resume_mismatches(emulated, False, tmp_path, load_optimizer=False) != []


@pytest.mark.parametrize("source", ["native", "torch", "torch_1_10"])
def test_interchange_with_torch_adam(emulated, tmp_path, source):
    ck = native_checkpoint(emulated) if source == "native" else torch_checkpoint(emulated)
    if source == "torch_1_10":
        ck["optimizer"] = as_torch_1_10(ck["optimizer"])
    assert next_step_mismatches(ck, emulated, tmp_path) == []


def _refusal_cases(osd):
    import copy

    def edit(fn):
        d = copy.deepcopy(osd)
        fn(d)
        return d
    g = lambda d: d["param_groups"][0]
    return {
        "parameters in the group": edit(lambda d: g(d)["params"].pop()),
        "has shape": edit(lambda d: d["state"][3].update(exp_avg=torch.zeros(7))),
        "param groups": edit(lambda d: d["param_groups"].append(dict(g(d), params=[]))),
        "'amsgrad' is set": edit(lambda d: g(d).update(amsgrad=True)),
        "'maximize' is set": edit(lambda d: g(d).update(maximize=True)),
        "differ between parameters": edit(lambda d: d["state"][5].update(step=torch.tensor(7.0))),
        "state for": edit(lambda d: d["state"].pop(4)),
    }


def test_load_state_dict_refuses_what_it_cannot_continue(emulated):
    cfg, sd = setup()
    model, ts = build(cfg, sd, emulated)
    native_steps(ts, criterion(cfg, emulated), batches(cfg, 1, emulated))
    osd = ts.state_dict()
    m, v = ts.m.clone(), ts.v.clone()
    for reason, bad in _refusal_cases(osd).items():
        with pytest.raises(ValueError, match=reason):
            ts.load_state_dict(bad)
        assert torch.equal(ts.m, m) and torch.equal(ts.v, v) and ts.step_no == 1, reason     # nothing half loaded
