"""Time mtt_attention alone at the attention shapes of the bench workloads (default: tp_cfg4, tp_cfg2, ip_cfg3 and
tp_cfg5 at their bench batch sizes, parity and speed mode).

The shapes are taken from the forward itself: one eager forward of each workload (seeded random-init weights and
input) runs with ops.attention wrapped, which records every (B, N, H, T, prompt logits, plane counts) it is called
with. Each distinct shape is then launched on seeded random operands of unit variance: --warmup launches, then
--launches launches between two CUDA events. Prints one JSON line per (workload, mode, shape) with microseconds per
launch, algorithmic TFLOP/s (4 B H N^2 64: QK^T and PV) and issued TFLOP/s (x3 in parity mode, which runs hi*hi,
hi*lo and lo*hi), then one line with the card's name, power limit and SM clock read in the same call.

--dump DIR saves every launch's outputs (hi / lo planes, prompt logits) to DIR/attention_outputs.pt, so that two
builds of the library (--lib) can be compared bit for bit on the same inputs. Needs a GPU.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKLOADS = {"tp_cfg4": 4, "tp_cfg2": 4, "ip_cfg3": 4, "tp_cfg5": 1}  # bench.py's batch size per workload


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, check=True)
    return dict(zip(q.split(","), (s.strip() for s in r.stdout.strip().split(","))))


def shapes_of_forward(name, batch, nsplit, dev):
    """The distinct attention launches of one eager forward, in first-call order."""
    import torch
    from mtt_b200 import configs, ops

    if name.startswith("ip_"):
        from mtt_b200 import invpt as M
        cfg = configs.invpt(name)
    else:
        from mtt_b200 import taskprompter as M
        cfg = configs.taskprompter(name)
    torch.manual_seed(0)
    with torch.device(dev):
        model = M.build_from_config(cfg, nsplit=nsplit, use_graph=False).eval()
    x = torch.randn(batch, 3, *cfg["img_size"], generator=torch.Generator().manual_seed(1)).to(dev)
    seen = []
    real = ops.attention

    def record(qkv, out, *, B, N, H, scale, prompt_logits=None, T=0):
        key = (B, N, H, T if prompt_logits is not None else 0, qkv.nsplit, out.nsplit)
        if key not in seen:
            seen.append(key)
        return real(qkv, out, B=B, N=N, H=H, scale=scale, prompt_logits=prompt_logits, T=T)

    ops.attention = record
    try:
        with torch.no_grad():
            model(x)
        torch.cuda.synchronize()
    finally:
        ops.attention = real
    del model
    torch.cuda.empty_cache()
    return seen


def time_shape(key, args, dev, seed):
    import torch
    from mtt_b200 import ops

    B, N, H, T, qs, os_ = key
    C = 64 * H
    g = torch.Generator(device=dev).manual_seed(seed)
    x = torch.randn(B * N, 3 * C, device=dev, generator=g)
    qkv = ops.Split(B * N, 3 * C, dev, nsplit=qs)
    qkv.buf[0] = x.to(torch.bfloat16)
    if qs == 2:
        qkv.buf[1] = (x - qkv.buf[0].float()).to(torch.bfloat16)
    out = ops.Split(B * N, C, dev, nsplit=os_, zero=True)
    logits = torch.zeros(B, H, T, N, device=dev) if T else None

    def launch():
        ops.attention(qkv, out, B=B, N=N, H=H, scale=64 ** -0.5, prompt_logits=logits, T=T)

    for _ in range(args.warmup):
        launch()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(args.launches):
        launch()
    e.record()
    torch.cuda.synchronize()
    us = s.elapsed_time(e) * 1e3 / args.launches
    launch()  # the outputs of one launch on these inputs
    torch.cuda.synchronize()
    outs = {"hi": out.buf[0].cpu()}
    if os_ == 2:
        outs["lo"] = out.buf[1].cpu()
    if logits is not None:
        outs["prompt_logits"] = logits.cpu()
    return us, outs


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--workloads", nargs="+", default=list(WORKLOADS), choices=list(WORKLOADS))
    ap.add_argument("--modes", nargs="+", default=["parity", "speed"], choices=["parity", "speed"])
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--lib", default=None, help="path of the libmtt_sm90.so to load instead of the tree's")
    ap.add_argument("--dump", metavar="DIR", default=None)
    args = ap.parse_args()

    import torch

    sys.path.insert(0, ROOT)
    import mtt_b200  # noqa: F401
    from mtt_b200 import lib

    if args.lib:
        lib.LIB_PATH = os.path.abspath(args.lib)
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    dumped = {}
    for name in args.workloads:
        for mode in args.modes:
            nsplit = 2 if mode == "parity" else 1
            for i, key in enumerate(shapes_of_forward(name, WORKLOADS[name], nsplit, dev)):
                B, N, H, T, qs, os_ = key
                us, outs = time_shape(key, args, dev, seed=1000 + i)
                alg = 4.0 * B * H * N * N * 64 / (us * 1e-6) / 1e12
                issued = alg * (3 if min(qs, os_) == 2 else 1)
                print(json.dumps({"workload": name, "mode": mode, "B": B, "N": N, "H": H, "T": T,
                                  "qkv_planes": qs, "out_planes": os_, "us_per_launch": round(us, 2),
                                  "alg_tflops": round(alg, 1), "issued_tflops": round(issued, 1)}), flush=True)
                for k, v in outs.items():
                    dumped[f"{name}/{mode}/{B}x{N}x{H}x{T}/{k}"] = v
    print(json.dumps({"gpu": gpu_info(), "lib": lib.LIB_PATH}), flush=True)
    if args.dump:
        os.makedirs(args.dump, exist_ok=True)
        torch.save(dumped, os.path.join(args.dump, "attention_outputs.pt"))


if __name__ == "__main__":
    main()
