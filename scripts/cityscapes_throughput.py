"""Device time per batch of the Cityscapes-3D data path (one H2D copy of the packed raw batch, the preprocess_image
launch and the mtt_cityscapes_targets launch), next to the CPU time per sample of the reference's per-sample work
(float image, encode_segmap's 35 passes, disparity conversion, two PIL NEAREST resizes, the validity check,
normalisation) as oracle/cityscapes_ref.reference_sample_work restates it, and the device time of the targets launch
alone.

    python scripts/cityscapes_throughput.py [--batch 4] [--iters 50]

Prints one JSON line; quote it with the card and power limit it reports."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

SRC, DST = (1024, 2048), (512, 1024)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def _time(fn, iters):
    fn()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for i in range(iters):
        fn()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--cpu-samples", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("cityscapes_throughput: no CUDA device")
    import mtt_b200  # noqa: F401
    from mtt_b200 import cityscapes as CS
    from mtt_b200 import ops
    from oracle import cityscapes_ref as R
    from oracle import make_cityscapes_golden as G

    p = {"TASKS": {"NAMES": ["semseg", "depth"]}, "dd_label_map_size": list(DST)}
    rng = np.random.default_rng(0)
    samples = [G.make_sample(rng, "bench", i, *SRC) for i in range(args.batch)]
    raws = [CS.make_collate(p)(samples) for _ in range(2)]
    for r in raws:
        r["buf"] = r["buf"].pin_memory()
    dt = CS.DeviceTransforms(p)
    k = [0]

    def step():
        k[0] += 1
        dt(raws[k[0] % len(raws)])

    dev_ms = _time(step, args.iters)
    B, n = args.batch, args.batch * SRC[0] * SRC[1]
    dev = raws[0]["buf"].cuda()
    o = raws[0]["offsets"]
    ids = dev[o[1]:o[1] + n].view(B, *SRC)
    disp = dev[o[2]:o[2] + 2 * n].view(torch.uint16).view(B, *SRC)
    sem = torch.empty(B, *DST, dtype=torch.int64, device="cuda")
    dep = torch.empty(B, 1, *DST, device="cuda")
    targets_us = 1e3 * _time(lambda: ops.cityscapes_targets(ids, disp, DST, semseg=sem, depth=dep), args.iters)
    cpu = []
    for i in range(args.cpu_samples):
        s = samples[i % len(samples)]
        t = time.perf_counter()
        R.reference_sample_work(s["image"], s["label_ids"], s["disparity"], DST)
        cpu.append((time.perf_counter() - t) * 1e3)
    print(json.dumps({"batch": B, "src": SRC, "labels": DST, "device_ms_per_batch": round(dev_ms, 4),
                      "h2d_bytes": raws[0]["buf"].numel(), "targets_kernel_us": round(targets_us, 2),
                      "targets_algorithmic_bytes": B * DST[0] * DST[1] * 15,
                      "cpu_reference_ms_per_sample": round(float(np.median(cpu)), 2), "card": card()}))


if __name__ == "__main__":
    main()
