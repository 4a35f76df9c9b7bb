"""CPU: the device meters' host side (mtt_b200.evaluate) and the meters oracle (oracle/meters_ref.py) against the
unmodified reference meters of both projects (tests/golden/meters.pt, and the reference itself where importable)."""
import math
import os

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "meters.pt")
PROJECTS = ("TaskPrompter", "InvPT")


def _gold():
    """The fixture, with its inputs restored to predict()'s dtypes (int64 class maps, fp32 maps)."""
    from oracle import meters_ref as R

    gold = torch.load(GOLD, weights_only=False)
    for sc in gold["scenarios"]:
        sc["updates"] = R.unpack_updates(sc["updates"])
    return gold


def _params(database):
    return dict(train_db_name=database, ignore_index=255, edge_w=0.95, TASKS=dict(depth_min=0.0, depth_max=80.0))


def _close(a, b, rel=1e-5):
    a, b = float(a), float(b)
    return a == b or abs(a - b) <= rel * max(abs(a), abs(b))


def assert_counters_match(got, ref, tol=1e-5):
    """Integer counters equal, float sums within tol relative."""
    assert set(got) == set(ref)
    for t in ref:
        assert set(got[t]) == set(ref[t]), t
        for k, v in ref[t].items():
            g = got[t][k]
            if isinstance(v, torch.Tensor) or isinstance(v, list):
                assert [int(x) for x in np.asarray(g, dtype=np.float64)] == [int(x) for x in np.asarray(v, dtype=np.float64)], (t, k)
            elif k in ("total", "n", "n_valid"):
                assert int(g) == int(v), (t, k, g, v)
            else:
                assert _close(g, v, tol), (t, k, g, v)


def assert_scores_match(got, ref, tol=1e-5):
    assert set(got) == set(ref)
    for t in ref:
        assert set(got[t]) == set(ref[t]), (t, set(got[t]), set(ref[t]))
        for k in ref[t]:
            assert _close(got[t][k], ref[t][k], tol), (t, k, got[t][k], ref[t][k])


def encode_words(meter, c):
    """State words (csrc/metrics.cu layout) that hold the reference counters c of one task."""
    from mtt_b200 import evaluate as E

    w = np.zeros(meter.words(), dtype=np.int64)
    f64 = lambda i, x: w[i:i + 1].view(np.float64).__setitem__(0, x)
    if isinstance(meter, E.ConfusionMeter):
        n = meter.n_classes
        M = w[:(n + 1) ** 2].reshape(n + 1, n + 1)
        for i in range(n):
            M[i, i], M[n, i], M[i, n] = c["tp"][i], c["fp"][i], c["fn"][i]
    elif isinstance(meter, E.SaliencyMeter):
        T = meter.n
        for j, k in enumerate(("true_positives", "predicted_positives", "actual_positives")):
            w[j * T:(j + 1) * T] = np.asarray(c[k], dtype=np.float64).astype(np.int64)
    elif isinstance(meter, E.NormalsMeter):
        f64(0, c["sum_deg_diff"])
        w[1] = c["total"]
    elif isinstance(meter, E.DepthMeter):
        w[0] = int(c["n_valid"])
        for i, k in enumerate(("total_rmses", "total_log_rmses", "abs_rel", "sq_rel")):
            f64(1 + i, c[k])
    elif isinstance(meter, E.EdgeMeter):
        f64(0, c["loss"])
        w[1] = c["n"]
    return w


@pytest.mark.parametrize("project", PROJECTS)
def test_get_score_formulas_on_fixture_counters(project):
    import mtt_b200  # noqa: F401
    from mtt_b200 import evaluate as E

    for sc in _gold()["scenarios"]:
        ref = sc["ref"][project]
        pm = E.PerformanceMeter(_params(sc["database"]), sc["tasks"], reference=project)
        got = {t: pm.meters[t].score(encode_words(pm.meters[t], ref["counters"][t]), verbose=False) for t in sc["tasks"]}
        assert_scores_match(got, ref["scores"], tol=1e-12)


@pytest.mark.parametrize("project", PROJECTS)
def test_oracle_against_fixture(project):
    from oracle import meters_ref as R

    for sc in _gold()["scenarios"]:
        m = R.PerformanceMeter(_params(sc["database"]), sc["tasks"], reference=project)
        for pred, gt in sc["updates"]:
            m.update(pred, gt)
        assert_counters_match(m.counters(), sc["ref"][project]["counters"])
        assert_scores_match(m.get_score(), sc["ref"][project]["scores"])


def test_fixture_covers_the_edge_cases():
    for sc in _gold()["scenarios"]:
        Bs = [u[1][sc["tasks"][0]].shape[0] for u in sc["updates"]]
        assert 1 in Bs and 3 in Bs and len(Bs) >= 3
        assert any(u[1][sc["tasks"][0]].shape[-1] % 2 == 1 for u in sc["updates"])
        for t in sc["tasks"]:
            gts = [u[1][t] for u in sc["updates"]]
            assert any(bool((g == 255).any()) for g in gts), t
            assert any(bool((g.flatten(1) == 255).all(dim=1).any()) for g in gts), t    # an all-ignore image
        if "depth" in sc["tasks"]:
            assert any(bool((u[1]["depth"] == 0.0).any() and (u[1]["depth"] == 80.0).any()) for u in sc["updates"])
        if "normals" in sc["tasks"]:
            assert any(bool((u[0]["normals"] == 127.5).all(dim=-1).any()) for u in sc["updates"])
        if "semseg" in sc["tasks"]:
            assert any(bool(((u[1]["semseg"] != 255) & (u[1]["semseg"] >= 21)).any()) for u in sc["updates"])


@pytest.mark.parametrize("project", PROJECTS)
def test_oracle_against_reference_fresh_batches(project):
    from oracle import ref_loader

    if not ref_loader.available():
        pytest.skip("reference tree not available")
    from oracle import make_meters_golden as MG
    from oracle import meters_ref as R

    g = torch.Generator().manual_seed(99)
    for name, database, tasks, ncls, shapes in MG.SCENARIOS:
        updates = [R.synthetic_batch(tasks, ncls, B, H + 2, W + 4, g, all_ignore=ai) for B, H, W, ai in shapes]
        rc, rs = MG.run_reference(project, database, tasks, updates)
        m = R.PerformanceMeter(_params(database), tasks, reference=project)
        for pred, gt in updates:
            m.update(pred, gt)
        assert_counters_match(m.counters(), rc)
        assert_scores_match(m.get_score(), rs)


def test_constructor_errors():
    import mtt_b200  # noqa: F401
    from mtt_b200 import evaluate as E

    with pytest.raises(NotImplementedError):
        E.PerformanceMeter(_params("KITTI"), ["semseg"])
    with pytest.raises(NotImplementedError):
        E.PerformanceMeter(_params("PASCALContext"), ["3ddet"])
    with pytest.raises(NotImplementedError):
        E.PerformanceMeter(_params("NYUD"), ["human_parts"])
    with pytest.raises(NotImplementedError):
        E.PerformanceMeter(_params("Cityscapes3D"), ["semseg"], reference="InvPT")
    assert E.PerformanceMeter(_params("Cityscapes3D"), ["semseg"]).meters["semseg"].n_classes == 19
    with pytest.raises(ValueError):
        E.PerformanceMeter(_params("NYUD"), ["semseg"], reference="MTI-Net")
    m = E.PerformanceMeter(_params("NYUD"), ["semseg", "depth"], reference="InvPT")
    assert m.meters["semseg"].n_classes == 40 and m.meters["depth"].ignore_index == 255


def test_library_refuses_bad_kinds_and_sizes():
    import mtt_b200  # noqa: F401
    from mtt_b200 import ops

    assert ops.meter_state_bytes(ops.METER_CONFUSION, 40) == 41 * 41 * 8
    assert ops.meter_state_bytes(ops.METER_SALIENCY, 19) == 3 * 19 * 8
    with pytest.raises(ValueError, match="capacity|bad size"):
        ops.meter_state_bytes(ops.METER_CONFUSION, 65)
    with pytest.raises(ValueError, match="unknown kind"):
        ops.meter_state_bytes(7, 1)
    with pytest.raises(ValueError):
        ops.meter_state_bytes(ops.METER_SALIENCY, 33)


def test_shape_and_dtype_mismatch_raise_before_any_launch():
    import mtt_b200  # noqa: F401
    from mtt_b200 import ops

    st = torch.zeros(41 * 41, dtype=torch.int64)
    lab = torch.zeros(2, 1, 5, 7)
    with pytest.raises(ValueError, match="prediction"):
        ops.meter_confusion_update(torch.zeros(2, 5, 6, dtype=torch.int64), lab, 40, 255, st)
    with pytest.raises(ValueError, match="prediction"):
        ops.meter_confusion_update(torch.zeros(2, 5, 7), lab, 40, 255, st)           # fp32 class map
    with pytest.raises(ValueError, match="label"):
        ops.meter_normals_update(torch.zeros(2, 5, 7, 3), lab, 255, st)              # normals need 3 label channels
    with pytest.raises(ValueError, match="label"):
        ops.meter_edge_update(torch.zeros(2, 5, 7), lab.double(), 0.95, 255, st)
    with pytest.raises(ValueError, match="prediction"):
        ops.meter_depth_update(torch.zeros(2, 5, 7, 3), lab, st, min_depth=0.0, max_depth=80.0)


def test_update_refuses_cpu_tensors():
    import mtt_b200  # noqa: F401
    from mtt_b200 import evaluate as E
    from oracle import meters_ref as R

    pred, gt = R.synthetic_batch(["semseg", "depth"], {"semseg": 40}, 1, 4, 5, torch.Generator().manual_seed(0))
    m = E.PerformanceMeter(_params("NYUD"), ["semseg", "depth"])
    with pytest.raises(RuntimeError, match="GPU only"):
        m.update(pred, gt)
    assert m.state is None


def test_score_of_empty_meter_follows_the_reference_guards():
    """No update: IoU 0 by the max(..., 1e-8) guard, maxF 0 by NaN -> 0, as the reference's fresh meters give."""
    import mtt_b200  # noqa: F401
    from mtt_b200 import evaluate as E

    m = E.PerformanceMeter(_params("PASCALContext"), ["semseg", "human_parts", "sal"])
    s = m.get_score(verbose=False)
    assert s["semseg"]["mIoU"] == 0.0 and s["human_parts"]["mIoU"] == 0.0 and s["sal"]["maxF"] == 0.0
    assert not math.isnan(s["sal"]["maxF"])
