"""Prediction export and visualisation throughput.

A test_phase-shaped loop (TP/utils/test_utils.py:29-45) on the TaskPrompter cfg4 model (ViT-L/16, 512 x 512, five
PASCAL tasks; parity mode): predict() + the device meters + the edge save of every batch, over N batches of synthetic
images, edge labels and meta (original sizes up to 375 x 500, padded to 512), timed with host clocks around work that
ends after every file is written (files go to a temporary directory):
  1. reference-style save: oracle/export_ref.py's save_preds on the CUDA tensors (label.unique() twice, crop, .cpu()
     per image) and cv2.imwrite, on the loop's thread;
  2. mtt_b200.export.PredictionWriter (two launches per batch, no host sync, PNGs written by a thread pool);
  3. as 2 without writing files (render and copy only).
Then the inference visualisation (TP/inference.py:118-164) for one 375 x 500 image and the five tasks: forward, then
vis_pred_for_one_task per task, reference-style (oracle vis_preds + cv2.imwrite) against mtt_b200.export's. Prints one
JSON line per way with the card's name, power limit and clock read in the same run.

    python scripts/export_throughput.py --batches 20 --warmup 3 [--batch 4] [--vis-reps 20]
"""
import argparse
import json
import os
import sys
import tempfile
import time

import cv2
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import mtt_b200  # noqa: E402,F401
from eval_throughput import P, card  # noqa: E402
from mtt_b200 import evaluate as E  # noqa: E402
from mtt_b200 import export as X  # noqa: E402
from mtt_b200 import taskprompter as TP  # noqa: E402
from oracle import configs  # noqa: E402
from oracle import export_ref as R  # noqa: E402
from oracle import taskprompter_ref as TPR  # noqa: E402

SIZES = [(375, 500), (500, 375), (333, 500), (512, 384)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="tp_cfg4")
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--batches", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--vis-reps", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("export_throughput.py measures on the GPU; no CUDA device found (nothing measured)")
    dev = torch.device("cuda:0")
    cfg = configs.taskprompter(args.config)
    tasks = list(cfg["tasks"])
    model = TP.build_from_config(cfg, nsplit=TP.PARITY, use_graph=True).eval()
    model.load_state_dict(TPR.init_state_dict(cfg, seed=0), strict=True)
    model = model.to(dev)
    H, W = cfg["img_size"]
    g = torch.Generator().manual_seed(0)
    x = torch.randn(args.batch, 3, H, W, generator=g).to(dev)
    gt = {"semseg": torch.randint(0, 21, (args.batch, 1, H, W), generator=g).float(),
          "human_parts": torch.randint(0, 7, (args.batch, 1, H, W), generator=g).float(),
          "sal": (torch.rand(args.batch, 1, H, W, generator=g) < 0.3).float(),
          "normals": torch.nn.functional.normalize(torch.randn(args.batch, 3, H, W, generator=g), dim=1),
          "edge": (torch.rand(args.batch, 1, H, W, generator=g) < 0.1).float()}
    gt = {t: v.to(dev) for t, v in gt.items()}
    p = dict(P, semseg_save_train_class=True)
    info = dict(card(), config=args.config, batch=args.batch, batches=args.batches, mode="parity")

    def meta(i):
        return {"img_name": [f"b{i:04d}_{j}" for j in range(args.batch)],
                "img_size": [SIZES[(i + j) % len(SIZES)] for j in range(args.batch)]}

    def reference_save(out, i, d):
        sample = {"meta": meta(i), "edge": gt["edge"]}
        for f, a in R.save_preds(p, sample, out, "edge", predicted=True).items():
            cv2.imwrite(os.path.join(d, f), a)

    def loop(n, way, d):
        meter = E.PerformanceMeter(P, tasks)
        writer = None
        if way != "reference":
            writer = X.PredictionWriter(p, ["edge"], {"edge": d}, slots=3,
                                        imwrite=(lambda path, a: None) if way == "no-write" else None)
        for i in range(n):
            with torch.no_grad():
                out = model.predict(x)
            meter.update(out, gt)
            if writer is None:
                reference_save(out, i, d)
            else:
                writer.update(out, gt, meta(i))
        meter.get_score(verbose=False)
        if writer is not None:
            writer.close()
        torch.cuda.synchronize()

    for way in ("reference", "writer", "no-write"):
        with tempfile.TemporaryDirectory() as d:
            loop(args.warmup, way, d)
            t0 = time.perf_counter()
            loop(args.batches, way, d)
            dt = time.perf_counter() - t0
        print(json.dumps(dict(info, way=f"predict+meters+edge_save:{way}", seconds=round(dt, 4),
                              images_per_s=round(args.batches * args.batch / dt, 3))), flush=True)

    # inference visualisation: batch 1, an original size of 375 x 500, the five PASCAL tasks
    x1 = x[:1].contiguous()
    sample = {"image": x1, "meta": {"img_name": ["vis"], "img_size": [(375, 500)]}}
    pv = dict(p)

    def vis(way, d):
        with torch.no_grad():
            out = model(x1)
        for t in tasks:
            if way == "reference":
                for f, a in R.vis_preds(pv, sample, out, t).items():
                    cv2.imwrite(os.path.join(d, f), a)
            else:
                X.vis_pred_for_one_task(pv, sample, out, d, t)
        torch.cuda.synchronize()

    for way in ("reference", "device"):
        with tempfile.TemporaryDirectory() as d:
            for _ in range(3):
                vis(way, d)
            t0 = time.perf_counter()
            for _ in range(args.vis_reps):
                vis(way, d)
            dt = time.perf_counter() - t0
        print(json.dumps(dict(info, batch=1, way=f"inference_vis:{way}", ms_per_image=round(dt / args.vis_reps * 1e3, 3))),
              flush=True)
    # encode only: the render of the five tasks at 375 x 500 from the logits, CUDA events
    with torch.no_grad():
        out = model(x1)
    for _ in range(3):
        X.render(pv, out, (375, 500))
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.vis_reps):
        X.render(pv, out, (375, 500))
    e1.record()
    torch.cuda.synchronize()
    print(json.dumps(dict(info, batch=1, way="render_5_tasks_375x500", ms=round(e0.elapsed_time(e1) / args.vis_reps, 4))),
          flush=True)


if __name__ == "__main__":
    main()
