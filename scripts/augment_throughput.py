"""Device time per batch of the train transform chain (mtt_augment: select + image + labels kernels, plus the one H2D
copy of the packed batch), next to the CPU time per sample of the same chain as the numpy restatement computes it.

    python scripts/augment_throughput.py [--db PASCALContext|NYUD] [--batch 4] [--iters 50]

Prints one JSON line; quote it with the card and power limit it reports."""
import argparse
import json
import os
import random
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

GEOMETRY = {"PASCALContext": (("semseg", "human_parts", "sal", "edge", "normals"), (512, 512),
                              [(375, 500), (281, 500), (500, 375), (333, 500)]),
            "NYUD": (("semseg", "depth", "normals", "edge"), (448, 576), [(480, 640)] * 4)}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--db", default="PASCALContext", choices=sorted(GEOMETRY))
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--cpu-samples", type=int, default=4)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("augment_throughput: no CUDA device")
    import mtt_b200  # noqa: F401
    from mtt_b200 import augment as A
    from oracle import augment_ref as R
    from oracle import make_augment_golden as G

    tasks, size, shapes = GEOMETRY[args.db]
    p = {"train_db_name": args.db, "TASKS": {"NAMES": list(tasks)}, "TRAIN": {"SCALE": size}, "TEST": {"SCALE": size}}
    rng = np.random.default_rng(0)
    samples = [G.make_sample(rng, *shapes[i % len(shapes)], tasks) for i in range(args.batch)]
    collate = A.make_collate(p)
    random.seed(0)
    raws = [collate(samples) for _ in range(4)]
    for r in raws:
        r["buf"] = r["buf"].pin_memory()
    aug = A.DeviceTransforms(p)
    for r in raws:
        aug(r)
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for i in range(args.iters):
        aug(raws[i % len(raws)])
    t1.record()
    torch.cuda.synchronize()
    dev_ms = t0.elapsed_time(t1) / args.iters
    in_bytes = raws[0]["buf"].numel()
    out_bytes = 4 * args.batch * size[0] * size[1] * (3 + sum(3 if t == "normals" else 1 for t in tasks))

    cpu = []
    for i in range(args.cpu_samples):
        s, rec = samples[i % len(samples)], raws[0]["records"][i % len(samples)]
        t = time.perf_counter()
        R.train_transform(s, rec, size)
        cpu.append((time.perf_counter() - t) * 1e3)
    print(json.dumps({"db": args.db, "batch": args.batch, "crop": size, "device_ms_per_batch": round(dev_ms, 4),
                      "h2d_plus_output_bytes": in_bytes + out_bytes,
                      "cpu_restatement_ms_per_sample": round(float(np.median(cpu)), 2),
                      "card": card()}))


if __name__ == "__main__":
    main()
