"""Validation-loop throughput: predict() alone, predict() + reference-style meters, predict() + the device meters.

A test_phase-shaped loop (TP/utils/test_utils.py:29-45) over N batches of synthetic images and PASCAL labels on the
TaskPrompter cfg4 model (ViT-L/16, 512 x 512, five PASCAL tasks; parity mode), timed three ways with host clocks
around work that ends in a device synchronise:
  1. predict() alone;
  2. predict() + oracle/meters_ref.py's PerformanceMeter on the CUDA tensors: the reference's per-class and
     per-threshold loops with the same host reads (.item(), .cpu(), boolean indexing);
  3. predict() + mtt_b200.evaluate.PerformanceMeter (one kernel per task per batch, no sync until get_score()).
get_score() is inside the timed region of ways 2 and 3. Prints one JSON line per way, plus the card's name and power
limit read in the same run, and the largest relative difference between the two meters' scores.

    python scripts/eval_throughput.py --batches 20 --warmup 3 [--config tp_cfg4] [--batch 4]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import mtt_b200  # noqa: E402,F401
from mtt_b200 import evaluate as E  # noqa: E402
from mtt_b200 import taskprompter as TP  # noqa: E402
from oracle import configs, meters_ref  # noqa: E402
from oracle import taskprompter_ref as TPR  # noqa: E402

P = dict(train_db_name="PASCALContext", ignore_index=255, edge_w=0.95, TASKS=dict(depth_min=0.0, depth_max=80.0))
NCLS = {"semseg": 21, "human_parts": 7}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, plim, clk = (s.strip() for s in q.split(","))
        return {"gpu": name, "power_limit": plim, "max_sm_clock": clk}
    except Exception as e:                                      # noqa: BLE001
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": f"not read ({e})", "max_sm_clock": None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="tp_cfg4")
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--batches", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--distinct", type=int, default=4, help="distinct image / label batches, cycled")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("eval_throughput.py measures on the GPU; no CUDA device found (nothing measured)")
    dev = torch.device("cuda:0")
    cfg = configs.taskprompter(args.config)
    tasks = list(cfg["tasks"])
    model = TP.build_from_config(cfg, nsplit=TP.PARITY, use_graph=True).eval()
    model.load_state_dict(TPR.init_state_dict(cfg, seed=0), strict=True)
    model = model.to(dev)
    g = torch.Generator().manual_seed(0)
    xs, gts = [], []
    for _ in range(args.distinct):
        xs.append(torch.randn(args.batch, 3, *cfg["img_size"], generator=g).to(dev))
        gts.append({t: v.to(dev) for t, v in meters_ref.synthetic_batch(tasks, NCLS, args.batch, *cfg["img_size"], g)[1].items()})

    def loop(n, meter):
        if meter is not None:
            meter.reset()
        for i in range(n):
            with torch.no_grad():
                out = model.predict(xs[i % args.distinct])
            if meter is not None:
                meter.update(out, gts[i % args.distinct])
        score = meter.get_score(verbose=False) if meter is not None else None
        torch.cuda.synchronize()
        return score

    ways = [("predict", lambda: None), ("predict+reference_meters", lambda: meters_ref.PerformanceMeter(P, tasks)),
            ("predict+device_meters", lambda: E.PerformanceMeter(P, tasks))]
    info = dict(card(), config=args.config, batch=args.batch, batches=args.batches, mode="parity")
    scores = {}
    for name, make in ways:
        meter = make()
        loop(args.warmup, meter)
        t0 = time.perf_counter()
        scores[name] = loop(args.batches, meter)
        dt = time.perf_counter() - t0
        print(json.dumps(dict(info, way=name, seconds=round(dt, 4), images_per_s=round(args.batches * args.batch / dt, 3))),
              flush=True)
    a, b = scores["predict+reference_meters"], scores["predict+device_meters"]
    worst = max(abs(float(a[t][k]) - float(b[t][k])) / max(abs(float(a[t][k])), 1e-12) for t in a for k in a[t])
    print(json.dumps({"score_max_rel_diff": worst, "device_scores": {t: {k: float(v) for k, v in d.items()} for t, d in b.items()}}))


if __name__ == "__main__":
    main()
