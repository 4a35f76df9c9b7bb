"""GPU: the device evaluation meters (csrc/metrics.cu through mtt_b200.evaluate) against the unmodified reference
meters' results in tests/golden/meters.pt and against oracle/meters_ref.py on predict() outputs."""
import pytest
import torch

from test_meters import PROJECTS, _gold, _params, assert_counters_match, assert_scores_match

pytestmark = pytest.mark.gpu


def _cuda(d, dev):
    return {k: v.to(dev) for k, v in d.items()}


def device_counters(pm):
    """The device state in the reference meters' attribute names (one device-to-host copy)."""
    from mtt_b200 import evaluate as E

    host = pm.state.cpu().numpy()
    out, off = {}, 0
    for t in pm.tasks:
        m = pm.meters[t]
        w = host[off:off + m.words()]
        off += m.words()
        if isinstance(m, E.ConfusionMeter):
            tp, fp, fn = m.counts(w)
            out[t] = {"tp": list(tp), "fp": list(fp), "fn": list(fn)}
        elif isinstance(m, E.SaliencyMeter):
            out[t] = dict(zip(("true_positives", "predicted_positives", "actual_positives"), m.counts(w)))
        elif isinstance(m, E.NormalsMeter):
            out[t] = dict(zip(("sum_deg_diff", "total"), m.counts(w)))
        elif isinstance(m, E.DepthMeter):
            out[t] = dict(zip(("n_valid", "total_rmses", "total_log_rmses", "abs_rel", "sq_rel"), m.counts(w)))
        elif isinstance(m, E.EdgeMeter):
            out[t] = dict(zip(("loss", "n"), m.counts(w)))
    return out


@pytest.mark.parametrize("project", PROJECTS)
def test_fixture_counters_and_scores(cuda_dev, project):
    from mtt_b200 import evaluate as E

    for sc in _gold()["scenarios"]:
        ref = sc["ref"][project]
        pm = E.PerformanceMeter(_params(sc["database"]), sc["tasks"], reference=project)
        for pred, gt in sc["updates"]:
            pm.update(_cuda(pred, cuda_dev), _cuda(gt, cuda_dev))
        assert_counters_match(device_counters(pm), ref["counters"])
        assert_scores_match(pm.get_score(verbose=False), ref["scores"])
        pm.reset()                                                     # reset, then the same again
        for pred, gt in sc["updates"]:
            pm.update(_cuda(pred, cuda_dev), _cuda(gt, cuda_dev))
        assert_scores_match(pm.get_score(verbose=False), ref["scores"])


def test_inputs_are_not_modified_and_results_reproducible(cuda_dev):
    from mtt_b200 import evaluate as E

    sc = [s for s in _gold()["scenarios"] if "depth" in s["tasks"]][0]
    ups = [(_cuda(p, cuda_dev), _cuda(g, cuda_dev)) for p, g in sc["updates"]]
    before = [({k: v.clone() for k, v in p.items()}, {k: v.clone() for k, v in g.items()}) for p, g in ups]
    states = []
    for _ in range(2):
        pm = E.PerformanceMeter(_params(sc["database"]), sc["tasks"])
        for p, g in ups:
            pm.update(p, g)
        states.append(pm.state.clone())
    assert torch.equal(states[0], states[1])                          # bitwise, float sums included
    for (p, g), (p0, g0) in zip(ups, before):
        for k in p:
            assert torch.equal(p[k], p0[k]) and torch.equal(g[k], g0[k])


def test_single_task_meter(cuda_dev):
    from mtt_b200 import evaluate as E

    sc = _gold()["scenarios"][0]
    ref = sc["ref"]["InvPT"]
    for t in sc["tasks"]:
        m = E.get_single_task_meter(_params(sc["database"]), sc["database"], t, reference="InvPT")
        for pred, gt in sc["updates"]:
            m.update(pred[t].to(cuda_dev), gt[t].to(cuda_dev))
        assert_scores_match({t: m.get_score(verbose=False)}, {t: ref["scores"][t]})


def test_update_in_cuda_graph_matches_eager(cuda_dev):
    from mtt_b200 import evaluate as E

    for sc in _gold()["scenarios"]:
        ups = [(_cuda(p, cuda_dev), _cuda(g, cuda_dev)) for p, g in sc["updates"]]
        eager = E.PerformanceMeter(_params(sc["database"]), sc["tasks"])
        for _ in range(2):
            for p, g in ups:
                eager.update(p, g)
        pm = E.PerformanceMeter(_params(sc["database"]), sc["tasks"])
        pm.update(*ups[0])                                             # allocates the state outside the capture
        pm.reset()
        graph = torch.cuda.CUDAGraph()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            with torch.cuda.graph(graph, stream=s):
                for p, g in ups:
                    pm.update(p, g)
        torch.cuda.current_stream().wait_stream(s)
        graph.replay()
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(pm.state, eager.state), sc["name"]


def test_update_does_not_synchronise(cuda_dev):
    from mtt_b200 import evaluate as E

    sc = _gold()["scenarios"][0]
    ups = [(_cuda(p, cuda_dev), _cuda(g, cuda_dev)) for p, g in sc["updates"]]
    pm = E.PerformanceMeter(_params(sc["database"]), sc["tasks"])
    pm.update(*ups[0])
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for p, g in ups:
            pm.update(p, g)
        pm.reset()
        pm.update(*ups[1])
    finally:
        torch.cuda.set_sync_debug_mode("default")


def _predict(name, B, seed, dev):
    import mtt_b200  # noqa: F401
    from mtt_b200 import taskprompter as TP
    from oracle import configs
    from oracle import taskprompter_ref as TPR

    cfg = configs.taskprompter(name)
    model = TP.build_from_config(cfg, nsplit=TP.PARITY).eval()
    model.load_state_dict(TPR.init_state_dict(cfg, seed=seed), strict=True)
    model = model.to(dev)
    x = torch.randn(B, 3, *cfg["img_size"], generator=torch.Generator().manual_seed(seed + 1))
    with torch.no_grad():
        out = model.predict(x.to(dev))
    return cfg, {t: v.clone() for t, v in out.items()}


@pytest.mark.parametrize("name,database,ncls,projects", [
    ("tp_cfg4_d4", "PASCALContext", {"semseg": 21, "human_parts": 7}, ("TaskPrompter",)),
    ("tp_tiny", "NYUD", {"semseg": 40}, PROJECTS),
])
def test_end_to_end_on_predict(cuda_dev, name, database, ncls, projects):
    from mtt_b200 import evaluate as E
    from oracle import meters_ref as R

    g = torch.Generator().manual_seed(5)
    preds, labels = [], []
    for B, seed in ((2, 11), (1, 12)):
        cfg, out = _predict(name, B, seed, cuda_dev)
        _, gt = R.synthetic_batch(cfg["tasks"], ncls, B, *cfg["img_size"], g)
        preds.append(out)
        labels.append(_cuda(gt, cuda_dev))
    for project in projects:
        pm = E.PerformanceMeter(_params(database), cfg["tasks"], reference=project)
        rm = R.PerformanceMeter(_params(database), cfg["tasks"], reference=project)
        for out, gt in zip(preds, labels):
            pm.update(out, gt)
            rm.update({t: v.cpu() for t, v in out.items()}, {t: v.cpu() for t, v in gt.items()})
        got, ref = pm.get_score(verbose=False), rm.get_score()
        assert_scores_match(got, ref)
        c = device_counters(pm)
        for t in cfg["tasks"]:
            if t in ("semseg", "human_parts"):
                assert c[t] == {k: [int(x) for x in v] for k, v in rm.counters()[t].items()}, t
