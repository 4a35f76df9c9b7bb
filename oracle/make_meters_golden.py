"""Generates tests/golden/meters.pt by running the UNMODIFIED reference evaluation meters of both projects
(TaskPrompter/evaluation, InvPT/evaluation, imported through oracle/shim and oracle/ref_loader) on seeded synthetic
batches. TEST INFRASTRUCTURE.

evaluate_utils.py imports imageio, which the build container does not have, so the meter classes are imported one
module at a time (evaluation.eval_semseg, ...) and assembled as evaluate_utils.py:35-66 does. The inputs are stored
in meters_ref.pack_updates()'s compact form (int8 class maps, fp16 float maps), which holds the drawn values exactly.

    python -m oracle.make_meters_golden
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import meters_ref, ref_loader  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden", "meters.pt")

# (name, database, tasks, n_classes, updates as (B, H, W, all-ignore images))
SCENARIOS = [
    ("pascal", "PASCALContext", ["semseg", "human_parts", "sal", "normals", "edge"], {"semseg": 21, "human_parts": 7},
     [(3, 21, 27, (1,)), (1, 37, 53, ()), (2, 17, 23, ())]),
    ("nyud", "NYUD", ["semseg", "normals", "depth"], {"semseg": 40},
     [(3, 21, 27, (2,)), (1, 37, 53, ()), (2, 17, 23, ())]),
]
P = dict(ignore_index=255, edge_w=0.95, TASKS=dict(depth_min=0.0, depth_max=80.0))     # TP utils/config.py:48-49


def reference_meters(project, database, tasks):
    """The reference's own meter classes, constructed as its get_single_task_meter does (evaluate_utils.py:35-66)."""
    ref_loader._activate(project)
    import importlib
    m = {}
    for t in tasks:
        if t == "semseg":
            m[t] = importlib.import_module("evaluation.eval_semseg").SemsegMeter(database, ignore_idx=P["ignore_index"])
        elif t == "human_parts":
            m[t] = importlib.import_module("evaluation.eval_human_parts").HumanPartsMeter(
                database, ignore_idx=P["ignore_index"])
        elif t == "normals":
            m[t] = importlib.import_module("evaluation.eval_normals").NormalsMeter(ignore_index=P["ignore_index"])
        elif t == "sal":
            m[t] = importlib.import_module("evaluation.eval_sal").SaliencyMeter(
                ignore_index=P["ignore_index"], threshold_step=0.05, beta_squared=0.3)
        elif t == "depth":
            D = importlib.import_module("evaluation.eval_depth").DepthMeter
            m[t] = (D(max_depth=P["TASKS"]["depth_max"], min_depth=P["TASKS"]["depth_min"]) if project == "TaskPrompter"
                    else D(ignore_index=P["ignore_index"]))
        elif t == "edge":
            m[t] = importlib.import_module("evaluation.eval_edge").EdgeMeter(pos_weight=P["edge_w"],
                                                                              ignore_index=P["ignore_index"])
    return m


def counters(t, m):
    """A reference meter's accumulated statistics, under its own attribute names."""
    if t in ("semseg", "human_parts"):
        return {"tp": list(m.tp), "fp": list(m.fp), "fn": list(m.fn)}
    if t == "sal":
        return {"true_positives": m.true_positives.clone(), "predicted_positives": m.predicted_positives.clone(),
                "actual_positives": m.actual_positives.clone()}
    if t == "normals":
        return {"sum_deg_diff": m.sum_deg_diff, "total": m.total}
    if t == "depth":
        return {k: getattr(m, k) for k in ("n_valid", "total_rmses", "total_log_rmses", "abs_rel", "sq_rel")}
    if t == "edge":
        return {"loss": m.loss, "n": m.n}
    raise ValueError(t)


def run_reference(project, database, tasks, updates):
    meters = reference_meters(project, database, tasks)
    for pred, gt in updates:
        for t in tasks:
            p, y = pred[t].clone(), gt[t].clone()          # TP eval_depth.py:41-42 writes into its inputs
            if t == "edge" and p.shape[0] == 1:
                p = p[0]                                   # eval_edge.py:24 indexes [B,H,W] with a squeezed [H,W] mask
            meters[t].update(p, y)
    return ({t: counters(t, meters[t]) for t in tasks}, {t: meters[t].get_score(verbose=False) for t in tasks})


def main():
    g = torch.Generator().manual_seed(20261016)
    out = {"params": P, "scenarios": [], "torch": torch.__version__,
           "made_by": "oracle/make_meters_golden.py from the unmodified reference meters of both projects (CPU)"}
    for name, database, tasks, ncls, shapes in SCENARIOS:
        updates = [meters_ref.synthetic_batch(tasks, ncls, B, H, W, g, all_ignore=ai) for B, H, W, ai in shapes]
        sc = {"name": name, "database": database, "tasks": tasks, "updates": meters_ref.pack_updates(updates), "ref": {}}
        for project in ("TaskPrompter", "InvPT"):
            c, s = run_reference(project, database, tasks, updates)
            sc["ref"][project] = {"counters": c, "scores": s}
        out["scenarios"].append(sc)
    torch.save(out, GOLD)
    print("wrote", GOLD, os.path.getsize(GOLD), "bytes")


if __name__ == "__main__":
    main()
