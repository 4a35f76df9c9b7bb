"""Images per second of the Swin TaskPrompter's fused forward at batch 1, 1024 x 2048: tps_swinB (semseg + depth) and
tps_swinB3d (the reference's Cityscapes-3D model: semseg + depth + 3ddet), CUDA-graph replay. The 3ddet head (FCOS3D)
is excluded: the tps_swinB3d model here carries nn.Identity as its detection head, so the figure is everything up to the
head's input (the 4 level maps). Random weights; the input is fixed.

Each model is warmed up (capture + replays), then timed with CUDA events over --iters replays, --repeats times; the
median and the spread are printed with the card's name and power limit, read in the same run.

    python scripts/swin_throughput.py [--iters 20] [--repeats 5] [--warmup 3]

Prints one JSON line."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.nn as nn  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def measure(name, iters, repeats, warmup):
    import mtt_b200  # noqa: F401
    from mtt_b200 import configs
    from mtt_b200 import taskprompter_swin as TS

    cfg = configs.taskprompter_swin(name)
    torch.manual_seed(0)
    det = nn.Identity() if "3ddet" in cfg["tasks"] else None
    with torch.device("cuda"):
        model = TS.build_from_config(cfg, use_graph=True, det_head=det).eval()
    x = torch.randn(1, 3, *cfg["img_size"], device="cuda")
    with torch.no_grad():
        for _ in range(warmup):
            model(x)
        torch.cuda.synchronize()
        ms = []
        for _ in range(repeats):
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            for _ in range(iters):
                model(x)
            t1.record()
            torch.cuda.synchronize()
            ms.append(t0.elapsed_time(t1) / iters)
    del model
    torch.cuda.empty_cache()
    med = statistics.median(ms)
    return {"ms_per_image_median": round(med, 3), "ms_per_image_min": round(min(ms), 3),
            "ms_per_image_max": round(max(ms), 3), "images_per_s": round(1e3 / med, 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("swin_throughput: no CUDA device")
    res = {name: measure(name, args.iters, args.repeats, args.warmup) for name in ("tps_swinB", "tps_swinB3d")}
    print(json.dumps({"batch": 1, "image": [1024, 2048], "mode": "parity (bf16x3), CUDA-graph replay",
                      "3ddet_head": "excluded (nn.Identity)", "iters": args.iters, "repeats": args.repeats,
                      "results": res, "card": card()}))


if __name__ == "__main__":
    main()
