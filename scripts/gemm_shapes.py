"""Per-shape time of the wgmma GEMM / implicit-GEMM conv kernels in one TaskPrompter forward (default: tp_cfg4, bs 4,
parity mode), split into MMA + fold, operand delivery and epilogue.

The shapes are the exact descriptors the forward passes (seeded random-init weights and input): the forward is
enqueued eagerly on one stream behind a device-side blocker, the library records CUDA events around every mtt_gemm /
mtt_gemm_grouped launch (mtt_profile_begin / mtt_profile_end), and the launches are grouped by (M, N, K) -- a grouped
launch reports M summed over its problems, a 3x3 convolution K x 9. Enough forwards run that every shape is timed over
at least --min-launches launches after --warmup forwards. One torch.profiler pass over a single forward names the
kernel instantiation (tile width, grouped or not) and grid of every launch.

Run four times, each in its own process because the library reads MTT_GEMM_DEBUG once:
  full           the kernel as shipped;
  no_loads       MTT_GEMM_DEBUG=1: the producer issues no TMA loads (the consumers compute on stale shared memory);
  no_epilogue    MTT_GEMM_DEBUG=2: no epilogue after the mainloop (no bias / residual reads, no stores);
  no_stores      MTT_GEMM_DEBUG=4: the whole epilogue except its global stores.
Only the timings of the debug runs are used, never their outputs. full - no_loads approximates the operand delivery
cost, full - no_epilogue the epilogue cost, and full - no_stores the part of it that is store drain; what no_loads
leaves is MMA + fold (+ epilogue).

Prints one JSON line per (run, shape), then one summary line per run. Needs a GPU; reads the card's name, power limit
and SM clock with nvidia-smi in the same call.
"""
import argparse
import json
import math
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PEAK_BF16_TFLOPS = 989.0  # H100 SXM data sheet, dense bf16 (700 W card): a ceiling, not a measured rate
RUNS = (("full", None), ("no_loads", "1"), ("no_epilogue", "2"), ("no_stores", "4"))


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, check=True)
    return dict(zip(q.split(","), (s.strip() for s in r.stdout.strip().split(","))))


def _kernels_of_one_forward(plan, x):
    """[(kernel name, grid CTAs)] of the GEMM-family launches of one eager forward, in launch order."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        plan._launch(x)
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            ev = json.load(f)["traceEvents"]
    ks = sorted((e for e in ev if e.get("cat") == "kernel" and "gemm_tc" in e.get("name", "")), key=lambda e: e["ts"])
    return [(e["name"], int(math.prod(e.get("args", {}).get("grid", [0])))) for e in ks]


def _tile_of(kernel_name):
    """(tile width, label) from 'void mtt::gemm_tc_kernel<2, 256, false>(...)' / 'mtt::gemm_tc_grouped_kernel<2, 128>'."""
    args = kernel_name.split("<", 1)[1].split(">", 1)[0].replace(" ", "").split(",")
    bn = int(args[1])
    if "grouped" in kernel_name:
        return bn, f"128x{bn} grouped"
    return bn, f"128x{bn}" + (" stream-K" if len(args) > 2 and args[2] == "true" else "")


def worker(args):
    import torch

    sys.path.insert(0, ROOT)
    import mtt_b200  # noqa: F401
    from mtt_b200 import configs, ops
    from mtt_b200 import taskprompter as TP

    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    cfg = configs.taskprompter(args.config)
    torch.manual_seed(0)
    with torch.device(dev):
        model = TP.build_from_config(cfg, nsplit=TP.PARITY, use_graph=True).eval()
    H, W = cfg["img_size"]
    x = torch.randn(args.batch, 3, H, W, generator=torch.Generator().manual_seed(1)).to(dev)
    plan = model.plan(args.batch, dev)
    plan.serial = True
    recs = []
    with torch.no_grad():
        model(x)
        for _ in range(args.warmup):
            plan._launch(x)
        torch.cuda.synchronize()
        kernels = _kernels_of_one_forward(plan, x)
        fwd = 0
        while True:
            torch.cuda._sleep(int(60e6))  # the host enqueues the whole forward before the first kernel runs
            ops.profile_begin()
            plan._launch(x)
            prof = [r for r in ops.profile_end() if r[0] == 0]
            if len(prof) != len(kernels):
                raise RuntimeError(f"{len(prof)} profiled GEMM launches vs {len(kernels)} GEMM kernels in the trace")
            recs += [(k, r) for k, r in zip(kernels, prof)]
            fwd += 1
            per_shape = {}
            for _, (_, M, N, K, _, _) in recs:
                per_shape[(M, N, K)] = per_shape.get((M, N, K), 0) + 1
            if min(per_shape.values()) >= args.min_launches:
                break
    shapes = {}
    for (kname, grid), (_, M, N, K, ms, fl) in recs:
        s = shapes.setdefault((M, N, K), {"ms": [], "flops": fl, "kernel": kname, "grid": grid})
        s["ms"].append(ms)
    out = []
    for (M, N, K), s in shapes.items():
        ms = sorted(s["ms"])
        med = ms[len(ms) // 2]
        per_fwd = len(ms) // fwd
        bn, tile = _tile_of(s["kernel"])
        tiles = math.ceil(M / 128) * math.ceil(N / bn)  # conv: 128-pixel patches of a 128-wide image = M / 128 too
        alg = s["flops"] / (med * 1e-3) / 1e12
        out.append({
            "M": M, "N": N, "K": K, "part": "backbone" if min(N, K) >= 1024 else "decoder/head",
            "launches_per_forward": per_fwd, "timed_launches": len(ms), "ms_median": med, "ms_min": ms[0],
            "ms_per_forward": med * per_fwd, "alg_tflops": alg, "issued_tflops": 3 * alg,
            "issued_frac_of_989": 3 * alg / PEAK_BF16_TFLOPS, "tile": tile, "ctas": s["grid"],
            "waves": tiles / s["grid"] if s["grid"] else None,
        })
    out.sort(key=lambda r: -r["ms_per_forward"])
    print(json.dumps({"forwards": fwd, "shapes": out}))


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--config", default="tp_cfg4")
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--warmup", type=int, default=3, help="untimed forwards first")
    ap.add_argument("--min-launches", type=int, default=50, help="timed launches per shape, at least")
    ap.add_argument("--worker", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.worker:
        return worker(args)
    gpu = gpu_info()
    totals = {}
    for run, dbg in RUNS:
        env = dict(os.environ)
        env.pop("MTT_GEMM_DEBUG", None)
        if dbg:
            env["MTT_GEMM_DEBUG"] = dbg
        cmd = [sys.executable, os.path.abspath(__file__), "--worker", "--config", args.config, "--batch",
               str(args.batch), "--warmup", str(args.warmup), "--min-launches", str(args.min_launches)]
        r = subprocess.run(cmd, env=env, capture_output=True, text=True, cwd=ROOT)
        if r.returncode != 0:
            sys.stderr.write(r.stderr)
            raise SystemExit(f"{run}: worker failed ({r.returncode})")
        res = json.loads(r.stdout.strip().splitlines()[-1])
        for s in res["shapes"]:
            print(json.dumps({"run": run, "MTT_GEMM_DEBUG": dbg, **s}))
        totals[run] = {"gemm_ms_per_forward": sum(s["ms_per_forward"] for s in res["shapes"]),
                       "backbone_ms_per_forward": sum(s["ms_per_forward"] for s in res["shapes"]
                                                      if s["part"] == "backbone"),
                       "forwards_timed": res["forwards"]}
    for run, t in totals.items():
        print(json.dumps({"summary": run, **t, "config": args.config, "batch": args.batch, "gpu": gpu}))


if __name__ == "__main__":
    main()
