"""The launch sequence of the Swin TaskPrompter plan, recorded on the CPU without running a kernel.

The plan is built with the kernels emulated (tests/emul_ops.py: its packed weights and workspace are real tensors),
then every ops function is replaced by a recorder that only notes its call: the entry point and its bound arguments,
with each tensor / Split written as (buffer, shape, strides) and the buffer numbered in order of first use, so the
record pins which buffers alias which, not where they live. Recording needs no GPU and no forward, so it covers Swin-B.

tests/golden/swin_plan_launches.json.xz holds the record of every mode of tps_tiny, tps_tiny3d and tps_swinB3d made
before the sub-module forwards shared the plan's block and merge launch code; test_swin_module_forwards checks that the
plan still launches exactly that.

    python tests/swin_plan_launches.py      # rewrites the fixture from the current plan code
"""
import inspect
import json
import lzma
import os
import sys

import pytest
import torch
import torch.nn as nn

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURE = os.path.join(HERE, "golden", "swin_plan_launches.json.xz")
CASES = [("tps_tiny", 2), ("tps_tiny3d", 2), ("tps_swinB3d", 1)]
MODES = ("full", "postproc", "backbone")


def _canon(v, ids):
    from mtt_b200 import ops
    if isinstance(v, ops.Split):
        return ["S", ids.setdefault(v.buf.data_ptr(), len(ids)), v.rows, v.cols, v.ld, v.nsplit]
    if isinstance(v, torch.Tensor):
        return ["T", ids.setdefault(v.data_ptr(), len(ids)), list(v.shape), list(v.stride()), str(v.dtype)]
    if isinstance(v, dict):
        return {k: _canon(x, ids) for k, x in sorted(v.items())}
    if isinstance(v, (list, tuple)):
        return [_canon(x, ids) for x in v]
    if callable(v):
        raise TypeError(f"a callable argument cannot be recorded: {v!r}")
    return v


def record(mp, name, B, mode):
    """[[entry point, {argument: value}], ...] of one eager launch of the plan of config `name` in `mode`."""
    import emul_ops
    from mtt_b200 import ops, taskprompter_swin as TS
    from oracle import configs

    emul_ops.install(mp)
    cfg = configs.taskprompter_swin(name)
    torch.manual_seed(0)
    m = TS.build_from_config(cfg, nsplit=2, use_graph=False, det_head=nn.Identity()).eval()
    heads = None if mode == "backbone" else m.heads
    pl = TS._SwinPlan(m.backbone, heads, cfg["tasks"], m.target_size if mode != "backbone" else None, B, "cpu", 2,
                      mode=mode)
    img = torch.zeros(B, 3, *pl.img)
    calls, ids = [], {}
    names = [n for n, f in vars(ops).items() if inspect.isfunction(f) and not n.startswith("_")]
    with pytest.MonkeyPatch.context() as rec:
        for n in names:
            sig = inspect.signature(getattr(ops, n))

            def fn(*a, _n=n, _sig=sig, **k):
                ba = _sig.bind(*a, **k)
                ba.apply_defaults()
                calls.append([_n, _canon(dict(ba.arguments), ids)])
            rec.setattr(ops, n, fn)
        pl._launch(img)
    return calls


def record_all():
    out = {}
    for name, B in CASES:
        for mode in MODES:
            with pytest.MonkeyPatch.context() as mp:
                out[f"{name}/b{B}/{mode}"] = record(mp, name, B, mode)
    return out


def load():
    with lzma.open(FIXTURE, "rt") as f:
        return json.load(f)


if __name__ == "__main__":
    sys.path.insert(0, HERE)
    sys.path.insert(0, os.path.dirname(HERE))
    import mtt_b200  # noqa: F401
    rec_ = record_all()
    with lzma.open(FIXTURE, "wt", preset=9) as f:
        json.dump(rec_, f, separators=(",", ":"))
    print(f"wrote {FIXTURE}: " + ", ".join(f"{k} {len(v)} calls" for k, v in rec_.items()))
