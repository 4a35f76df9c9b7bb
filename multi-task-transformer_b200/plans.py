"""What the launch plans of the three model families (taskprompter.py, invpt.py, taskprompter_swin.py) share.

A plan is one forward for one (batch size, device, nsplit, mode): packed weights resolved from per-module caches, a fixed
workspace and one launch sequence, replayed as ONE CUDA graph. `Plan` owns that lifecycle (device check, streams,
re-packing after an in-place parameter update, graph capture and replay); a family's plan class adds only its geometry,
workspace and launch sequence. Packed weights (split-bf16, BatchNorm folded, tap-major convs) are cached per module,
device, precision mode and parameter version, so every plan and sub-module forward over the same module shares one copy.
The packers of the layers more than one family has live here too.
"""
import contextlib
from types import SimpleNamespace

import torch

from . import ops

MAX_PLANS = 4         # cached plans (workspace + CUDA graph) per module, least recently used is dropped


# --------------------------------------------------------------------------------------------
# per-module caches and the device context
# --------------------------------------------------------------------------------------------
def _version(mod):
    return sum(int(q._version) for q in mod.parameters()) + sum(int(b._version) for b in mod.buffers())


def _cached(mod, key, build, versioned=True):
    """build() once per (module, key, parameter version); lives in the module's __dict__ (not a parameter / buffer)."""
    store = mod.__dict__.setdefault("_mtt_cache", {})
    ver = _version(mod) if versioned else 0
    hit = store.get(key)
    if hit is None or hit[0] != ver:
        with _dev_ctx(key[1]):
            hit = (ver, build())
        store[key] = hit
    return hit[1]


def _dev_ctx(device):
    """torch.cuda.device(device) for CUDA devices (the C side works on the CURRENT device: streams, kernel attributes,
    SM count), a no-op otherwise (CPU emulation in the tests)."""
    device = torch.device(device)
    return torch.cuda.device(device) if device.type == "cuda" else contextlib.nullcontext()


def _f32(t, device):
    return t.detach().to(device=device, dtype=torch.float32).contiguous()


def _check_input(mod, x):
    if mod.training:
        raise NotImplementedError("mtt_b200: the fused forward is eval-only; call .eval() (backward kernels: "
                                  "SURVEY.md section 8f N1)")
    if not x.is_cuda:
        raise RuntimeError("mtt_b200 has no CPU path: input must be a CUDA tensor on an sm_90a (H100) device")
    ops.device_check()


class _Streams:
    """Fork / join of side streams off the current stream (captured into the same CUDA graph)."""

    def __init__(self, dev, n):
        self.dev, self.n, self.side, self.serial = dev, max(n, 1), None, False

    def fork(self, n):
        if self.dev.type != "cuda" or self.serial:   # serial: one stream (per-kernel timing)
            return None, [None] * n
        if self.side is None:
            self.side = [torch.cuda.Stream(device=self.dev) for _ in range(self.n)]
        main = torch.cuda.current_stream()
        for st in self.side[:n]:
            st.wait_stream(main)
        return main, self.side[:n]

    def join(self, main, n):
        if main is not None:
            for st in self.side[:n]:
                main.wait_stream(st)

    def par(self, fns):
        """Run the callables concurrently, one per side stream."""
        main, side = self.fork(len(fns))
        for st, fn in zip(side, fns):
            if st is None:
                fn()
            else:
                with torch.cuda.stream(st):
                    fn()
        self.join(main, len(fns))


def _plan_for(mod, key, build):
    """LRU cache of plans on `mod` (a plan = workspace + CUDA graph for one batch size; weights are shared)."""
    plans = mod.__dict__.setdefault("_mtt_plans", {})
    pl = plans.pop(key, None)
    if pl is None:
        pl = build()
    plans[key] = pl                      # most recently used last
    while len(plans) > MAX_PLANS:
        plans.pop(next(iter(plans)))
    return pl


# --------------------------------------------------------------------------------------------
# the plan lifecycle
# --------------------------------------------------------------------------------------------
class Plan:
    """Base of the launch plans. A subclass builds its workspace under `_dev_ctx(self.dev)` after calling `_repack()`,
    sets `img` (and `in_chans` when it is not 3) when it takes an image, and supplies `_pack()` (resolves the packed
    weights from the per-module caches), `_launch(img)` (enqueues the forward on the current stream) and, when it
    returns more than `self.out`, `_result()`."""

    in_chans = 3

    def __init__(self, modules, B, device, nsplit, n_streams):
        """modules: the nn.Modules whose parameters the packed weights follow (None entries are skipped)."""
        ops.device_check()
        self.tracked = [m for m in modules if m is not None]
        self.B, self.dev, self.ns = B, torch.device(device), nsplit
        self.streams = _Streams(self.dev, n_streams)
        self.graph = None
        self.static_in = None

    def _repack(self):
        """(Re)resolve the packed weights from the per-module caches (cheap when nothing changed)."""
        self._pack()
        self.version = self._param_version()

    def _param_version(self):
        return sum(_version(m) for m in self.tracked)

    def _result(self):
        return dict(self.out)

    @property
    def serial(self):
        return self.streams.serial

    @serial.setter
    def serial(self, v):
        self.streams.serial = bool(v)

    def run(self, x, graph=True):
        """x [B, in_chans, *img] fp32 -> the outputs (the plan's static buffers). Launches eagerly when `graph` is False;
        otherwise copies x into a static input, captures the forward into a CUDA graph on the first call (after one
        warm-up launch outside capture) and replays it. A plan that takes no image (x None) launches eagerly on inputs
        loaded into its buffers beforehand."""
        if x is not None and (tuple(x.shape[1:]) != (self.in_chans, *self.img) or x.dtype != torch.float32):
            raise ValueError(f"expected fp32 input [B,{self.in_chans},{self.img[0]},{self.img[1]}], got "
                             f"{tuple(x.shape)} {x.dtype}")
        with _dev_ctx(self.dev):
            if self._param_version() != self.version:   # parameters changed in place: re-pack (same shapes), re-capture
                self._repack()
                self.graph = None
            if x is None or not graph:
                self._launch(None if x is None else x.contiguous())
                return self._result()
            if self.static_in is None:
                self.static_in = torch.empty_like(x, memory_format=torch.contiguous_format)
            self.static_in.copy_(x, non_blocking=True)
            if self.graph is None:
                self._launch(self.static_in)  # warm-up outside capture (sets kernel attributes, loads modules)
                torch.cuda.synchronize()
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    self._launch(self.static_in)
                self.graph = g
            self.graph.replay()
            return self._result()

    def launches_per_forward(self):
        with _dev_ctx(self.dev):
            n0 = ops.launch_count()
            self._launch(self.static_in if self.static_in is not None else
                         torch.zeros(self.B, self.in_chans, *self.img, device=self.dev))
            return ops.launch_count() - n0


def _predict_outputs(tasks, B, hw, device):
    """Output buffers of predict() at hw = (H, W): {task: int64 [B,H,W] class map | fp32 map}, by the task's
    get_output post-processing (ops.POSTPROC_KIND)."""
    oh, ow = hw
    shapes = {0: (B, oh, ow), 1: (B, oh, ow), 2: (B, oh, ow), 3: (B, oh, ow, 3), 4: (B, oh, ow, 1)}
    out = {}
    for t in tasks:
        if t not in ops.POSTPROC_KIND:
            raise ValueError(f"no get_output post-processing defined for task {t!r}")
        kind = ops.POSTPROC_KIND[t]
        out[t] = torch.zeros(shapes[kind], device=device, dtype=torch.int64 if kind == 0 else torch.float32)
    return out


# --------------------------------------------------------------------------------------------
# packers of the layers the families share
# --------------------------------------------------------------------------------------------
def _lin(mod, device, ns):
    """Linear or 1x1 Conv2d -> (packed weight [N, K], fp32 bias or None)."""
    w = ops.pack_weight(_f32(mod.weight, device).reshape(mod.weight.shape[0], -1), ns)
    b = _f32(mod.bias, device) if mod.bias is not None else None
    return w, b


def _pack_stem(bb, device, ns):
    """Patch embedding, the rows the backbone adds to the token stream (position embedding without the cls slot, cls
    token + its position, task prompts: whichever it has), the patch-embedding norm of Swin and the final norm; cached
    on the backbone."""
    def build():
        f = lambda t: _f32(t, device)
        pe = bb.patch_embed
        W = SimpleNamespace()
        W.pe_w, W.pe_b = _lin(pe.proj, device, ns)
        if hasattr(pe, "norm"):                                                    # Swin: patch_norm=True
            W.pnw, W.pnb, W.pneps = f(pe.norm.weight), f(pe.norm.bias), pe.norm.eps
        if hasattr(bb, "pos_embed"):
            W.pos = f(bb.pos_embed)[0, 1:].contiguous()                            # [P, C] (cls slot skipped)
        if hasattr(bb, "cls_token"):
            W.cls = (f(bb.cls_token)[0] + f(bb.pos_embed)[0, :1]).contiguous()    # IP vit.py:334-339, row 0
        if hasattr(bb, "task_prompts"):
            W.prompts = f(bb.task_prompts)
        W.nw, W.nb, W.neps = f(bb.norm.weight), f(bb.norm.bias), bb.norm.eps
        return W
    return _cached(bb, ("stem", device, ns), build)


def _pack_vit_block(blk, device, ns):
    """LayerNorms, qkv, proj, fc1 and fc2 of a ViT block (TaskPrompter `Block`, InvPT `VitBlock`), cached on the block.
    A TaskPrompter block's attention adds token_trans / token_trans1 (TP taskprompter.py:219, :250)."""
    def build():
        f = lambda t: _f32(t, device)
        a = blk.attn
        w = SimpleNamespace()
        w.n1w, w.n1b, w.n2w, w.n2b = f(blk.norm1.weight), f(blk.norm1.bias), f(blk.norm2.weight), f(blk.norm2.bias)
        w.eps = blk.norm1.eps
        w.qkv, w.qkv_b = _lin(a.qkv, device, ns)
        if w.qkv_b is None:                                   # qkv_bias=False: a zero bias for mtt_ln_qkv
            w.qkv_b = torch.zeros(a.qkv.out_features, device=device)
        w.proj, w.proj_b = _lin(a.proj, device, ns)
        w.fc1, w.fc1_b = _lin(blk.mlp.fc1, device, ns)
        w.fc2, w.fc2_b = _lin(blk.mlp.fc2, device, ns)
        if hasattr(a, "token_trans"):
            w.tt, w.tt_b = _lin(a.token_trans, device, ns)
            w.tt1, w.tt1_b = _lin(a.token_trans1, device, ns)
        return w
    return _cached(blk, ("pack", device, ns), build)
