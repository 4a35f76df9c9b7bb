"""TaskPrompter (ViT) with the reference's nn.Module boundaries and a fused sm_90a forward.

Module classes, constructor signatures and parameter names mirror the reference so that its
checkpoints (`backbone.blocks.{i}.attn.qkv.weight`, `backbone.fea_fuse.{il}.{task}.1.weight`,
`heads.{task}.mt_proj.0.weight`, ...) load unchanged:

  Attention / Block / TaskPrompter / ConvHead   TaskPrompter/models/transformers/taskprompter.py:168-487,688-698
  TaskPrompterWrapper                           TaskPrompter/models/taskprompter_wrapper.py:9-40

The modules OWN parameters and expose the reference's forward signatures; all arithmetic runs in
libmtt_sm90.so through `ops`:

  TaskPrompterWrapper.forward(x)      -> {task: [B,n_out,H,W]}      the fused path: one `_Plan` (plans.Plan: packed
                                                                    weights + fixed workspace) replayed as ONE CUDA graph
  TaskPrompter.forward(x)             -> (task_fea {task: [B,f,4h,4w]}, {})      taskprompter.py:392-422
  Block.forward(x, task_prompts)      -> (x, (prompt_logits, raw_chan), task_prompts)   :270-279
  ConvHead / DEConvHead.forward(x)    -> [B,n_out,h,w] / [B,n_out,2h,2w]          :697, :712-715

The sub-module forwards run the SAME kernels eagerly on small private workspaces (NCHW tensors in and out like the
reference); they exist so that code written against the reference's module boundaries keeps working, the wrapper
forward is the one to time. The plan lifecycle and the per-module weight caches that every plan and sub-module forward
shares are in plans.py.

Changes to the reference's internal contract: `Block` returns `(prompt_logits [B,H,T,N], raw_chan [B,T,C,nh,nw])`
in place of the full [B,H,N,N] attention maps (only those parts are ever consumed, SURVEY.md H4; the logits are
None unless `Block.emit_logits` is set, which TaskPrompter does for the blocks that need them), and dead code
(`chan_x`, taskprompter.py:241-245) is not executed. Forward is eval-mode only (DropPath identity, BatchNorm running
statistics); training raises.
"""
import math
from types import SimpleNamespace

import torch
import torch.nn as nn

from . import ops
from .plans import (Plan, _cached, _check_input, _dev_ctx, _f32, _lin, _pack_stem, _pack_vit_block, _plan_for,
                    _predict_outputs, _Streams)

PARITY, SPEED = 2, 1  # nsplit: 3-MMA split-bf16 (fp32-grade) vs plain bf16


# --------------------------------------------------------------------------------------------
# parameter containers (names = reference state_dict keys) with the reference's forward signatures
# --------------------------------------------------------------------------------------------
class Mlp(nn.Module):
    """timm.models.layers.Mlp parameters (fc1, fc2)."""

    def __init__(self, in_features, hidden_features):
        super().__init__()
        self.fc1 = nn.Linear(in_features, hidden_features)
        self.fc2 = nn.Linear(hidden_features, in_features)


class Attention(nn.Module):
    """taskprompter.py:168-193."""

    def __init__(self, chan_nheads, resolution, dim, num_heads=8, qkv_bias=False):
        super().__init__()
        self.num_heads = num_heads
        self.dim = dim
        self.resolution = resolution
        self.pixel_no = int(resolution[0] * resolution[1])
        self.chan_nheads = chan_nheads
        self.scale = (dim // num_heads) ** -0.5
        self.qkv = nn.Linear(dim, dim * 3, bias=qkv_bias)
        self.proj = nn.Linear(dim, dim)
        self.token_trans = nn.Linear(dim, self.pixel_no)
        self.token_trans1 = nn.Linear(self.pixel_no, dim)


class _BlockSpace:
    """Activations of the joint [prompts; patches] stream for one batch size (shared by all blocks of a plan)."""

    def __init__(self, B, T, gh, gw, C, H, hidden, chan_nheads, device, ns, streams=None):
        self.B, self.T, self.gh, self.gw, self.C, self.H, self.ns, self.dev = B, T, gh, gw, C, H, ns, device
        self.P = P = gh * gw
        self.N = N = T + P
        self.nh = self.nw = int(round(math.sqrt(chan_nheads)))
        S = lambda r, c, **kw: ops.Split(r, c, device, ns, **kw)
        z = lambda *s: torch.zeros(*s, device=device, dtype=torch.float32)
        self.xs = z(B * N, C)
        self.qkv = S(B * N, 3 * C)
        self.ao = S(B * N, C)
        self.logits = z(B, H, T, N)
        self.cp = z(B * T, P)
        self.cps = S(B * T, P)
        self.rc = z(B, T, C, self.nh, self.nw)
        # workspaces of the two LayerNorm-fronted operators; LN1's output is read back by the channel-prompt path
        self.ws_qkv = ops.workspace(ops.workspace_bytes(ops.OP_LN_QKV, rows=B * N, Cdim=C, nsplit=ns), device)
        self.ws_mlp = ops.workspace(ops.workspace_bytes(ops.OP_LN_MLP_RESIDUAL, rows=B * N, Cdim=C, hidden=hidden,
                                                        nsplit=ns), device)
        self.xn = ops.ws_split_view(self.ws_qkv, 0, B * N, C, ns)
        self.streams = streams if streams is not None else _Streams(device, max(T, 1))


def _launch_block(sp, w, want_logits):
    """One Block on the joint stream sp.xs (taskprompter.py:270-279, Attention :195-254)."""
    B, N, T = sp.B, sp.N, sp.T
    ops.ln_qkv(sp.xs, w.n1w, w.n1b, w.eps, w.qkv, w.qkv_b, sp.qkv, sp.ws_qkv)                 # :272, :199, :201
    # the channel-prompt path (token_trans -> raw channel logits -> token_trans1) needs only LN1's output and the
    # prompt rows of xs: it runs on a side stream next to the attention kernel and joins before proj
    main, side = sp.streams.fork(1)
    if side[0] is None:
        _launch_chan_path(sp, w, want_logits)
    else:
        with torch.cuda.stream(side[0]):
            _launch_chan_path(sp, w, want_logits)
    ops.attention(sp.qkv, sp.ao, B=B, N=N, H=sp.H, scale=64 ** -0.5,
                  prompt_logits=sp.logits if want_logits else None, T=T)                      # :204-210
    sp.streams.join(main, 1)
    ops.proj_residual(sp.ao, w.proj, w.proj_b, sp.xs)                                          # :212, :273, :276
    ops.ln_mlp_residual(sp.xs, w.n2w, w.n2b, w.eps, w.fc1, w.fc1_b, w.fc2, w.fc2_b, sp.ws_mlp)  # :274, :277


def prompt_row_chunks(B, T):
    """(b0, nb): images [b0, b0 + nb) per GEMM launch over prompt rows: their T prompt rows each form one gathered
    128-row A tile."""
    bstep = max(1, 128 // T)
    for b0 in range(0, B, bstep):
        yield b0, min(bstep, B - b0)


def _launch_chan_path(sp, w, want_logits):
    B, N, T, C = sp.B, sp.N, sp.T, sp.C
    for b0, nb in prompt_row_chunks(B, T):
        ops.gemm(sp.xn, w.tt, M=nb * T, bias=w.tt_b, a_gather=(T, N), a_row_offset=b0 * N,
                 out_f32=sp.cp, out_split=sp.cps, regroup=(nb * T, nb * T, b0 * T))           # :219 token_trans
    if want_logits:
        ops.chan_logits(sp.cp, sp.xn, sp.rc, B=B, N=N, T=T, Cdim=C, gh=sp.gh, gw=sp.gw,
                        nh=sp.nh, nw=sp.nw)                                                   # :236-246
    for b0, nb in prompt_row_chunks(B, T):
        ops.gemm(sp.cps, w.tt1, M=nb * T, bias=w.tt1_b, a_row_offset=b0 * T, residual=sp.xs,
                 out_f32=sp.xs, regroup=(T, N, b0 * N))                                       # :250 token_trans1


class Block(nn.Module):
    """taskprompter.py:257-279. forward(x [B,P,C], task_prompts [B,T,C]) -> (x, attn_weight, task_prompts) with
    attn_weight = (prompt_logits [B,H,T,N] | None, raw_chan [B,T,C,nh,nw] | None): the parts of the reference's
    attention maps that cal_task_feature consumes, produced when `emit_logits` is set."""

    def __init__(self, chan_nheads, resolution, dim, num_heads, mlp_ratio=4., qkv_bias=False):
        super().__init__()
        self.norm1 = nn.LayerNorm(dim, eps=1e-6)
        self.attn = Attention(chan_nheads, resolution, dim, num_heads=num_heads, qkv_bias=qkv_bias)
        self.norm2 = nn.LayerNorm(dim, eps=1e-6)
        self.mlp = Mlp(dim, int(dim * mlp_ratio))
        self.nsplit = PARITY
        self.emit_logits = True

    def forward(self, x, task_prompts):
        _check_input(self, x)
        B, P, C = x.shape
        T = task_prompts.shape[1]
        a = self.attn
        if P != a.pixel_no or C != a.dim or C // a.num_heads != 64:
            raise ValueError(f"Block: expected x [B,{a.pixel_no},{a.dim}] with head dim 64, got {tuple(x.shape)}")
        dev, ns = x.device, self.nsplit
        with _dev_ctx(dev):
            w = _pack_vit_block(self, dev, ns)
            sp = _cached(self, ("space", dev, ns, B, T), lambda: _BlockSpace(
                B, T, a.resolution[0], a.resolution[1], C, a.num_heads, self.mlp.fc1.out_features, a.chan_nheads, dev,
                ns), versioned=False)
            xs = sp.xs.view(B, sp.N, C)
            xs[:, :T].copy_(task_prompts)                                                     # :199 prompts first
            xs[:, T:].copy_(x)
            _launch_block(sp, w, self.emit_logits)
            attn_weight = (sp.logits.clone(), sp.rc.clone()) if self.emit_logits else (None, None)
            return xs[:, T:].clone(), attn_weight, xs[:, :T].clone()


class PatchEmbed(nn.Module):
    """timm PatchEmbed parameters (proj = Conv2d k = s = patch)."""

    def __init__(self, img_size, patch_size, in_chans, embed_dim):
        super().__init__()
        self.img_size = tuple(img_size)
        self.patch_size = (patch_size, patch_size)
        self.grid_size = (img_size[0] // patch_size, img_size[1] // patch_size)
        self.num_patches = self.grid_size[0] * self.grid_size[1]
        self.proj = nn.Conv2d(in_chans, embed_dim, kernel_size=patch_size, stride=patch_size)


def _trunc_normal_(t, mean=0., std=1., a=-2., b=2.):
    with torch.no_grad():
        return nn.init.trunc_normal_(t, mean=mean, std=std, a=a, b=b)


class TaskPrompter(nn.Module):
    """taskprompter.py:281-422 (same constructor arguments; `p` needs TASKS.NAMES, prompt_len, chan_nheads, use_ctr,
    embed_dim, final_embed_dim). forward(x [B,3,H,W]) -> (task_fea {task: [B,f,4h,4w]}, info {})."""

    def __init__(self, p, select_list, img_size=(224, 224), patch_size=16, in_chans=3, embed_dim=768, depth=12,
                 num_heads=12, chan_nheads=1, mlp_ratio=4., qkv_bias=True, drop_rate=0., attn_drop_rate=0.,
                 drop_path_rate=0., **_unused):
        super().__init__()
        if isinstance(img_size, int):
            img_size = (img_size, img_size)
        self.p = p
        self.embed_dim = self.num_features = embed_dim
        self.num_heads = num_heads
        self.depth = depth
        self.drop_path_rate = float(drop_path_rate)     # stochastic depth acts in the training step only (train.py)
        self.patch_size = patch_size
        self.in_chans = in_chans
        self.patch_embed = PatchEmbed(img_size, patch_size, in_chans, embed_dim)
        num_patches = self.patch_embed.num_patches
        self.pos_embed = nn.Parameter(torch.zeros(1, num_patches + 1, embed_dim))
        self.resolution = [img_size[0] // patch_size, img_size[1] // patch_size]
        self.blocks = nn.Sequential(*[
            Block(chan_nheads, self.resolution, embed_dim, num_heads, mlp_ratio, qkv_bias) for _ in range(depth)])
        self.norm = nn.LayerNorm(embed_dim, eps=1e-6)
        self.select_list = list(select_list)
        self.num_layers = 4
        assert len(self.select_list) == self.num_layers - 1
        tasks = list(p.TASKS.NAMES)
        self.pixel_no = num_patches
        self.prompt_len = p.prompt_len
        assert self.prompt_len == 1, "prompt_len != 1 is unsupported (as in the reference's channel branch)"
        self.prompts_len = len(tasks) * p.prompt_len
        self.task_prompts = nn.Parameter(torch.ones(self.prompts_len, embed_dim))
        self.chan_nheads = chan_nheads
        nh = int(round(math.sqrt(chan_nheads)))
        if nh * nh != chan_nheads or self.resolution[0] % nh or self.resolution[1] % nh:
            # taskprompter.py:233 takes nh = nw = int(sqrt(chan_nheads)) windows per axis and rearranges the token grid
            # "(nh h nw w)" (:236): the reference's configurations use 1, 4 and 16, and an indivisible grid fails there too
            raise ValueError(f"TaskPrompter: chan_nheads={chan_nheads} must be a perfect square whose root divides the "
                             f"token grid {self.resolution[0]} x {self.resolution[1]}")
        e, f = p.embed_dim, p.final_embed_dim
        prompt_dim = num_heads * p.prompt_len
        self.fea_fuse = nn.ModuleList()
        if p.use_ctr:
            self.ctr_attn_conv = nn.ModuleList()
        self.fea_decode_spa = nn.ModuleList()
        self.fea_decode_chan = nn.ModuleList()
        for _ in range(self.num_layers):
            self.fea_fuse.append(nn.ModuleDict())
            if p.use_ctr:
                self.ctr_attn_conv.append(nn.ModuleDict())
            self.fea_decode_spa.append(nn.ModuleDict())
            self.fea_decode_chan.append(nn.ModuleDict())
            for t in tasks:
                self.fea_fuse[-1][t] = nn.Sequential(nn.Conv2d(e * 2, f, 1), nn.Conv2d(f, f, 3, padding=1),
                                                     nn.BatchNorm2d(f), nn.GELU(), nn.Conv2d(f, f, 1))
                if p.use_ctr:
                    self.ctr_attn_conv[-1][t] = nn.Sequential(nn.Conv2d(prompt_dim, prompt_dim, 1), nn.GELU(),
                                                              nn.Conv2d(prompt_dim, 1, 1))
                self.fea_decode_spa[-1][t] = nn.Sequential(nn.Conv2d(embed_dim, e, 1))
                self.fea_decode_chan[-1][t] = nn.Sequential(nn.Conv2d(embed_dim, e, 1))
        self.nsplit = PARITY
        self.use_graph = False
        self._init_weights()

    def _init_weights(self):
        # taskprompter.py:343-344,373,378,496-522
        _trunc_normal_(self.task_prompts, mean=1., std=1.)
        _trunc_normal_(self.pos_embed, std=.02)
        for m in self.modules():
            if isinstance(m, nn.Linear):
                _trunc_normal_(m.weight, std=.02)
                if m.bias is not None:
                    nn.init.zeros_(m.bias)
            elif isinstance(m, (nn.LayerNorm, nn.BatchNorm2d)):
                nn.init.zeros_(m.bias)
                nn.init.ones_(m.weight)

    def forward(self, x):
        """taskprompter.py:392-422: {task: [B, final_embed_dim, 4h, 4w]} (summed over the 4 levels, bilinear x4) and the
        (empty) info dict. Outputs are fresh tensors."""
        _check_input(self, x)
        pl = _plan_for(self, (x.shape[0], x.device, self.nsplit, "backbone"), lambda: _Plan(
            self, None, list(self.p.TASKS.NAMES), None, x.shape[0], x.device, self.nsplit, mode="backbone"))
        out = pl.run(x, graph=self.use_graph)
        return {t: v.clone() for t, v in out.items()}, {}


def _pack_head(hd, device, ns):
    """ConvHead (taskprompter.py:688-698) / DEConvHead (:700-715) operands, BatchNorm folded."""
    def build():
        f = lambda t: _f32(t, device)
        hw = SimpleNamespace()
        hw.deconv = isinstance(hd.mt_proj[0], nn.ConvTranspose2d)
        if hw.deconv:
            # ConvTranspose2d(k2, s2, p0): out[2y+dy, 2x+dx] = W[:, :, dy, dx]^T . in[y, x] -- four dense GEMMs, one per
            # output phase (dy, dx), each scattering its rows into the 2x map (mtt_gemm out_row_stride); eval
            # BatchNorm folds into every phase alike
            wt = f(hd.mt_proj[0].weight)                                              # [Cin, Cout, 2, 2]
            hw.mid = wt.shape[1]
            hw.dc = []
            for dy in range(2):
                for dx in range(2):
                    wp, bp = ops.pack_conv_weight(wt[:, :, dy, dx].contiguous().reshape(wt.shape[0], hw.mid, 1, 1),
                                                  hd.mt_proj[0].bias, hd.mt_proj[1], ns, transposed=True)
                    hw.dc.append((dy, dx, wp, bp))
            hw.mt, hw.mt_b = ops.pack_conv_weight(f(hd.mt_proj[3].weight), hd.mt_proj[3].bias, hd.mt_proj[4], ns)
        else:
            hw.mid = hd.mt_proj[0].weight.shape[0]
            hw.mt, hw.mt_b = ops.pack_conv_weight(f(hd.mt_proj[0].weight), hd.mt_proj[0].bias, hd.mt_proj[1], ns)
        hw.cin = hd.mt_proj[0].weight.shape[0] if hw.deconv else hd.mt_proj[0].weight.shape[1]
        hw.lp, hw.lp_b = _lin(hd.linear_pred, device, ns)
        hw.n_out = hd.linear_pred.weight.shape[0]
        return hw
    return _cached(hd, ("pack", device, ns), build)


class _HeadSpace:
    """Input / hidden / prediction maps of one head for B images of h x w (NHWC)."""

    def __init__(self, hw, B, h, w, device, ns):
        S = lambda r, c, **kw: ops.Split(r, c, device, ns, **kw)
        k = 2 if hw.deconv else 1
        self.B, self.h, self.w, self.ph, self.pw = B, h, w, k * h, k * w
        rows = B * self.ph * self.pw
        self.up = S(B * h * w, hw.cin, zero=True)
        self.hdc = S(rows, hw.mid, zero=True) if hw.deconv else None
        self.hmid = S(rows, hw.mid, zero=True)
        self.pred = torch.zeros(rows, ops.round_up(hw.n_out, 4), device=device, dtype=torch.float32)


def _launch_head(hs, hw):
    """hs.up (NHWC split head input) -> hs.pred (NHWC fp32 logits at the head's resolution)."""
    B = hs.B
    if hw.deconv:                                                                             # DEConvHead :700-715
        for dy, dx, wp, bp in hw.dc:                                                          # mt_proj[0..2]
            ops.gemm(hs.up, wp, N=hw.mid, K=hw.cin, bias=bp, act=ops.ACT_GELU, out_split=hs.hdc,
                     regroup=(hs.w, 4 * hs.w, 2 * hs.w * dy + dx, 2))
        ops.conv3x3_bn_act(hs.hdc, hw.mt, hw.mt_b, hw.mid, hw.mid, ops.ACT_GELU, B=B, H=hs.ph, W=hs.pw, mid=hs.hmid,
                           w_head=hw.lp, b_head=hw.lp_b, n_out=hw.n_out, out_f32=hs.pred)     # mt_proj[3..5], linear_pred
    else:                                                                                     # ConvHead :688-698
        ops.conv3x3_bn_act(hs.up, hw.mt, hw.mt_b, hw.cin, hw.mid, ops.ACT_GELU, B=B, H=hs.ph, W=hs.pw, mid=hs.hmid,
                           w_head=hw.lp, b_head=hw.lp_b, n_out=hw.n_out, out_f32=hs.pred)


class _HeadForward:
    """forward(x [B,Cin,h,w] NCHW fp32) -> [B,n_out,h',w'] NCHW, like the reference heads."""

    nsplit = PARITY

    def forward(self, x):
        _check_input(self, x)
        B, Cin, h, w = x.shape
        dev, ns = x.device, self.nsplit
        with _dev_ctx(dev):
            hw = _pack_head(self, dev, ns)
            if Cin != hw.cin:
                raise ValueError(f"{type(self).__name__}: expected {hw.cin} input channels, got {Cin}")
            hs = _cached(self, ("space", dev, ns, B, h, w), lambda: _HeadSpace(hw, B, h, w, dev, ns), versioned=False)
            ops.nchw_to_nhwc_split(x.contiguous(), hs.up)
            _launch_head(hs, hw)
            out = torch.empty(B, hw.n_out, hs.ph, hs.pw, device=dev, dtype=torch.float32)
            ops.nhwc_to_nchw(hs.pred, hs.pred.stride(0), B, hw.n_out, hs.ph, hs.pw, out)
            return out


class ConvHead(_HeadForward, nn.Module):
    """taskprompter.py:688-698."""

    def __init__(self, in_channels, num_classes):
        super().__init__()
        self.mt_proj = nn.Sequential(nn.Conv2d(in_channels, in_channels, 3, padding=1),
                                     nn.BatchNorm2d(in_channels), nn.GELU())
        _trunc_normal_(self.mt_proj[0].weight, std=0.02)
        self.linear_pred = nn.Conv2d(in_channels, num_classes, kernel_size=1)


class DEConvHead(_HeadForward, nn.Module):
    """taskprompter.py:700-715 (`head: deconv`, utils/common_config.py:68-70): ConvTranspose2d(k2,s2) + BN + GELU,
    3x3 conv + BN + GELU, 1x1 conv -- predicts at twice the resolution of its input."""

    def __init__(self, in_channels, num_classes):
        super().__init__()
        h2 = in_channels // 2
        self.mt_proj = nn.Sequential(nn.ConvTranspose2d(in_channels, h2, 2, stride=2, padding=0),
                                     nn.BatchNorm2d(h2), nn.GELU(),
                                     nn.Conv2d(h2, h2, 3, padding=1), nn.BatchNorm2d(h2), nn.GELU())
        self.linear_pred = nn.Conv2d(h2, num_classes, kernel_size=1)
        _trunc_normal_(self.mt_proj[0].weight, std=0.02)
        _trunc_normal_(self.mt_proj[3].weight, std=0.02)
        _trunc_normal_(self.linear_pred.weight, std=0.02)


class TaskPrompterWrapper(nn.Module):
    """models/taskprompter_wrapper.py:9-40: backbone -> per-task head -> bilinear resize to the input size (or
    p.dd_label_map_size; the '3ddet' task is NOT resized, :34-38). forward(x [B,3,H,W]) -> {task: [B,n_out,H,W]}
    fp32, written into the plan's static buffers (clone to keep results across calls).

    With a TaskPrompterSwin backbone, heads['3ddet'] may be any nn.Module (in practice the reference's FCOS3DHead): it
    runs in PyTorch on the 4 level maps the fused forward leaves in static buffers, on the same stream, and its output
    is out['3ddet'] as the head returns it (the hybrid head, INTEGRATION.md section 1)."""

    def __init__(self, p, backbone, heads, nsplit=PARITY, use_graph=True):
        super().__init__()
        self.tasks = list(p.TASKS.NAMES)
        self.backbone = backbone
        self.heads = heads
        keys = p.keys() if hasattr(p, "keys") else vars(p).keys()
        self.target_size = tuple(p.dd_label_map_size) if "dd_label_map_size" in keys else None
        self.nsplit = nsplit
        self.use_graph = use_graph
        swin = self._swin()
        for t in self.tasks:
            if swin and t == "3ddet":
                if t not in heads or not isinstance(heads[t], nn.Module):
                    raise ValueError("mtt_b200 TaskPrompterSwin: the '3ddet' task needs a detection head module in "
                                     "heads['3ddet'] (the reference's FCOS3DHead, or any module taking the 4 level maps)")
                continue
            if not isinstance(heads[t], (ConvHead, DEConvHead)):
                raise NotImplementedError(f"mtt_b200: unsupported head {type(heads[t]).__name__} for task {t!r} (the "
                                          "FCOS3D detection head of the reference needs mmdet3d: SURVEY.md 8f N4)")

    def _swin(self):
        return type(self.backbone).__name__ == "TaskPrompterSwin"

    def plan(self, batch, device, postproc=False):
        mode = "postproc" if postproc else "full"
        P = _Plan
        if self._swin():                                              # the Swin family has its own launch plan
            from .taskprompter_swin import _SwinPlan as P
        return _plan_for(self, (int(batch), torch.device(device), int(self.nsplit), mode), lambda: P(
            self.backbone, self.heads, self.tasks, self.target_size, batch, torch.device(device), self.nsplit, mode=mode))

    def _run(self, x, postproc):
        out = self.plan(x.shape[0], x.device, postproc=postproc).run(x, graph=self.use_graph)
        if self._swin() and "3ddet" in out:          # wrapper :37-38: the detection head on the level maps, not resized
            with _dev_ctx(x.device):
                out["3ddet"] = self.heads["3ddet"](out["3ddet"])
        return out

    def forward(self, x):
        _check_input(self, x)
        return self._run(x, postproc=False)

    def predict(self, x):
        """forward + the reference's `get_output` post-processing (TaskPrompter/utils/utils.py:27-63) fused
        into the final resize: {task: int64 [B,H,W] class map | fp32 map} without materialising the
        full-resolution logits (semseg / human_parts argmax, edge 255*sigmoid, sal 255*softmax[1], normals
        (normalize+1)*255/2, depth clamp). With a Swin backbone, '3ddet' holds the detection head's RAW output: the
        reference's get_output('3ddet') decodes boxes with p.detmodel (mmdet3d), which this library does not have."""
        _check_input(self, x)
        return self._run(x, postproc=True)


# --------------------------------------------------------------------------------------------
# the fused forward
# --------------------------------------------------------------------------------------------
def _pack_fuse(bb, il, t, device, ns):
    """fea_decode_spa / fea_decode_chan / fea_fuse of task t at level il (:352-366), for both backbones: fea_fuse[0]'s K
    laid out like the zero-padded `cat` buffer, fea_fuse[1] folded with its eval BatchNorm."""
    f = lambda x: _f32(x, device)
    tw = SimpleNamespace()
    tw.spa, tw.spa_b = _lin(bb.fea_decode_spa[il][t][0], device, ns)
    tw.chan, tw.chan_b = _lin(bb.fea_decode_chan[il][t][0], device, ns)
    fu = bb.fea_fuse[il][t]
    ff, e = fu[0].weight.shape[0], fu[0].weight.shape[1] // 2
    e_pad = ops.round_up(e, 8)
    w0 = f(fu[0].weight).reshape(ff, 2 * e)
    w0p = torch.zeros(ff, 2 * e_pad, device=device)
    w0p[:, :e] = w0[:, :e]
    w0p[:, e_pad:e_pad + e] = w0[:, e:]
    tw.f0, tw.f0_b = ops.pack_weight(w0p, ns), f(fu[0].bias)
    tw.f1, tw.f1_b = ops.pack_conv_weight(f(fu[1].weight), fu[1].bias, fu[2], ns)
    if fu[4].kernel_size == (1, 1):
        tw.f4, tw.f4_b = _lin(fu[4], device, ns)
    else:                                                                 # 3x3 in TaskPrompterSwin (TP swin :630)
        tw.f4, tw.f4_b = ops.pack_conv_weight(f(fu[4].weight), fu[4].bias, None, ns)
    return tw


def _pack_levels(bb, tasks, device, ns):
    """fea_decode_spa / fea_decode_chan / fea_fuse / ctr_attn_conv operands of all 4 levels (:352-366)."""
    def build():
        f = lambda t: _f32(t, device)
        H = bb.num_heads
        levels = []
        for il in range(4):
            lv = SimpleNamespace(tasks=[_pack_fuse(bb, il, t, device, ns) for t in tasks])
            if bb.p.use_ctr:
                cc = [bb.ctr_attn_conv[il][t] for t in tasks]
                lv.c0 = torch.stack([f(c[0].weight).reshape(H, H) for c in cc]).contiguous()
                lv.c0b = torch.stack([f(c[0].bias) for c in cc]).contiguous()
                lv.c2 = torch.stack([f(c[2].weight).reshape(H) for c in cc]).contiguous()
                lv.c2b = torch.stack([f(c[2].bias).reshape(()) for c in cc]).contiguous()
            levels.append(lv)
        return levels
    return _cached(bb, ("levels", device, ns, tuple(tasks)), build)


class _Plan(Plan):
    """Geometry, workspace and launch sequence of one TaskPrompter (ViT) forward. mode: "full" = wrapper forward
    (logits at the output size), "postproc" = predict(), "backbone" = TaskPrompter.forward alone (task features,
    NCHW)."""

    def __init__(self, bb, heads, tasks, target, B, device, nsplit, mode="full"):
        super().__init__((bb, heads), B, device, nsplit, len(tasks))
        device = self.dev
        self.mode = mode
        self.postproc = mode == "postproc"
        p = bb.p
        self.bb, self.heads = bb, heads
        self.tasks = list(tasks)
        self.T = T = len(self.tasks)
        self.C = C = bb.embed_dim
        self.H = bb.num_heads
        if C // self.H != 64 or C % self.H:
            raise ValueError(f"TaskPrompter: embed_dim / num_heads = {C} / {self.H} must be 64 (mtt_attention is built for "
                             "head dim 64: ViT-B 768 / 12, ViT-L 1024 / 16)")
        self.gh, self.gw = bb.resolution
        self.P = P = self.gh * self.gw
        self.N = N = T + P
        self.patch = bb.patch_size
        self.img = (self.gh * self.patch, self.gw * self.patch)
        self.depth = bb.depth
        self.select = list(bb.select_list)
        self.e, self.f = p.embed_dim, p.final_embed_dim
        self.e_pad = ops.round_up(self.e, 8)
        self.f_ld = ops.round_up(self.f, 8)
        self.use_ctr = bool(p.use_ctr)
        self.target = target
        ns = nsplit
        e_pad, f = self.e_pad, self.f
        with _dev_ctx(device):
            self._repack()
            # ---- workspace ------------------------------------------------------------------------------
            S = lambda r, c, **kw: ops.Split(r, c, device, ns, **kw)
            z = lambda *s: torch.zeros(*s, device=device, dtype=torch.float32)
            self.cols = S(B * P, self.patch * self.patch * bb.in_chans)
            self.sp = _BlockSpace(B, T, self.gh, self.gw, C, self.H, bb.blocks[0].mlp.fc1.out_features, bb.chan_nheads,
                                  device, ns, streams=self.streams)
            self.nh, self.nw = self.sp.nh, self.sp.nw
            self.xs, self.logits, self.rc = self.sp.xs, self.sp.logits, self.sp.rc
            self.xfin = z(B * N, C)
            # one set of decoder scratch buffers per task: the T tasks' identically shaped convolutions of a level run
            # as grouped launches
            self.ws_gate = ops.workspace(ops.workspace_bytes(ops.OP_GATED_CONV1X1, rows=B * P, Cdim=C, nsplit=ns, T=T),
                                         device)
            self.cat = [S(B * P, 2 * e_pad, zero=True) for _ in range(T)]
            self.f1 = [S(B * P, f, zero=True) for _ in range(T)]
            self.f2 = [S(B * P, f, zero=True) for _ in range(T)]
            self.acc = z(T, B * P, self.f_ld)
            if self.use_ctr:
                self.F = z(T, B * P, self.f_ld)
                self.ctrw = z(B, T, T)
            gh4, gw4 = 4 * self.gh, 4 * self.gw
            oh, ow = self.target if self.target is not None else self.img
            self.out_hw = (oh, ow)
            if mode == "backbone":
                self.hs = None
                self.out = {t: z(B, f, gh4, gw4) for t in self.tasks}
                return
            self.hs = [_HeadSpace(hw, B, gh4, gw4, device, ns) for hw in self.Wh]
            if self.postproc:
                self.out = _predict_outputs(self.tasks, B, (oh, ow), device)
            else:                                                  # wrapper :34-38: '3ddet' is not resized
                self.out = {t: z(B, hw.n_out, hs.ph, hs.pw) if t == "3ddet" else z(B, hw.n_out, oh, ow)
                            for t, hw, hs in zip(self.tasks, self.Wh, self.hs)}

    def _pack(self):
        bb, dev, ns = self.bb, self.dev, self.ns
        self.Ws = _pack_stem(bb, dev, ns)
        self.Wb = [_pack_vit_block(blk, dev, ns) for blk in bb.blocks]
        self.Wl = _pack_levels(bb, self.tasks, dev, ns)
        self.Wh = [_pack_head(self.heads[t], dev, ns) for t in self.tasks] if self.heads is not None else None

    # -- launch sequence ------------------------------------------------------------------------
    def _level(self, il, x_src):
        """cal_task_feature (:424-487) on X = x_src rows [b*N + T + pix]; accumulates into self.acc. The T tasks'
        identically shaped convolutions run as grouped launches (T x 96 tiles instead of T single-wave launches)."""
        B, N, T, C, P = self.B, self.N, self.T, self.C, self.P
        lv = self.Wl[il]
        first = il == 0
        ops.gated_conv1x1(x_src, N, T, self.logits, self.rc,
                          [(tw.spa, tw.spa_b, tw.chan, tw.chan_b, self.cat[ti]) for ti, tw in enumerate(lv.tasks)],
                          self.e, self.e_pad, self.ws_gate, B=B, T=T, N=N, H=self.H, Cdim=C, gh=self.gh, gw=self.gw,
                          nh=self.nh, nw=self.nw)                                            # :436-447, :452-468, :471
        ops.gemm_grouped([(self.cat[ti], tw.f0, dict(bias=tw.f0_b, out_split=self.f1[ti], N=self.f))
                          for ti, tw in enumerate(lv.tasks)])                                # fea_fuse[0]
        ops.gemm_grouped([(self.f1[ti], tw.f1, dict(N=self.f, K=self.f, bias=tw.f1_b, act=ops.ACT_GELU,
                                                    out_split=self.f2[ti], conv=(B, self.gh, self.gw, 3, 1)))
                          for ti, tw in enumerate(lv.tasks)])                                # fea_fuse[1..3]
        if self.use_ctr:
            ops.gemm_grouped([(self.f2[ti], tw.f4, dict(bias=tw.f4_b, out_f32=self.F[ti][:, :self.f], N=self.f))
                              for ti, tw in enumerate(lv.tasks)])                            # fea_fuse[4]
            ops.ctr_weights(self.logits, lv.c0, lv.c0b, lv.c2, lv.c2b, self.ctrw, B=B, H=self.H, T=T, N=N)
            ops.ctr_mix(self.F, self.ctrw, self.acc, T=T, M=B * P, Cdim=self.f_ld, ld=self.f_ld,
                        rows_per_batch=P, accumulate=not first)                              # :481-485,:411
        else:
            ops.gemm_grouped([(self.f2[ti], tw.f4, dict(bias=tw.f4_b, out_f32=self.acc[ti][:, :self.f], N=self.f,
                                                        residual=None if first else self.acc[ti][:, :self.f]))
                              for ti, tw in enumerate(lv.tasks)])                            # fea_fuse[4] + level sum :411

    def _head_chain(self, ti, t, hw, hs):
        B = self.B
        oh, ow = self.out_hw
        ops.bilinear(self.acc[ti], self.f_ld, B, self.gh, self.gw, self.f, hs.h, hs.w, out_split=hs.up)      # :420
        _launch_head(hs, hw)
        if t == "3ddet":
            ops.nhwc_to_nchw(hs.pred, hs.pred.stride(0), B, hw.n_out, hs.ph, hs.pw, self.out[t])            # wrapper :38
        elif self.postproc:
            ops.bilinear_postproc(hs.pred, hs.pred.stride(0), B, hs.ph, hs.pw, hw.n_out, oh, ow,
                                  ops.POSTPROC_KIND[t], self.out[t])                         # wrapper :35 + utils.py:27-63
        else:
            ops.bilinear(hs.pred, hs.pred.stride(0), B, hs.ph, hs.pw, hw.n_out, oh, ow, out_nchw=self.out[t])  # :35

    def _launch(self, img):
        B, N, T, P = self.B, self.N, self.T, self.P
        W = self.Ws
        ops.im2col_patch(img, self.patch, self.cols)
        ops.gemm(self.cols, W.pe_w, bias=W.pe_b, residual=W.pos, res_row_mod=P, out_f32=self.xs,
                 regroup=(P, N, T))                                                          # :393-394
        ops.broadcast_rows(W.prompts, self.xs, B, N)                                         # :397
        for idx, w in enumerate(self.Wb):
            sel = (idx + 1) in self.select
            _launch_block(self.sp, w, sel or idx == self.depth - 1)
            if sel:
                il = sum(1 for s in self.select if idx >= s - 1) - 1                         # :408
                self._level(il, self.xs)
        ops.layernorm(self.xs, W.nw, W.nb, W.neps, out_f32=self.xfin)                        # :413
        self._level(3, self.xfin)                                                            # :416-417
        if self.mode == "backbone":
            gh4, gw4 = 4 * self.gh, 4 * self.gw
            self.streams.par([lambda ti=ti, t=t: ops.bilinear(self.acc[ti], self.f_ld, B, self.gh, self.gw, self.f, gh4,
                                                              gw4, out_nchw=self.out[t])
                              for ti, t in enumerate(self.tasks)])                           # :419-420
            return
        self.streams.par([lambda ti=ti, t=t, hw=hw, hs=hs: self._head_chain(ti, t, hw, hs)
                          for ti, (t, hw, hs) in enumerate(zip(self.tasks, self.Wh, self.hs))])


# --------------------------------------------------------------------------------------------
# factories mirroring the reference (taskprompter.py:671-685, utils/common_config.py:17-90)
# --------------------------------------------------------------------------------------------
def taskprompter_vit_large_patch16_384(pretrained=False, **kwargs):
    kw = dict(select_list=range(6, 24, 6), patch_size=16, embed_dim=1024, depth=24, num_heads=16,
              chan_nheads=kwargs['p'].chan_nheads)
    kw.update(kwargs)
    return TaskPrompter(**kw)


def taskprompter_vit_base_patch16_384(pretrained=False, **kwargs):
    kw = dict(select_list=range(3, 12, 3), patch_size=16, embed_dim=768, depth=12, num_heads=12,
              chan_nheads=kwargs['p'].chan_nheads)
    kw.update(kwargs)
    return TaskPrompter(**kw)


def build_from_config(cfg, nsplit=PARITY, use_graph=True):
    """cfg: dict as in oracle/configs.py (tasks, num_output, img_size, patch, C, depth, heads, select,
    e, f, chan_nheads, use_ctr)."""
    p = SimpleNamespace(TASKS=SimpleNamespace(NAMES=list(cfg["tasks"]), NUM_OUTPUT=dict(cfg["num_output"])),
                        prompt_len=1, chan_nheads=cfg["chan_nheads"], use_ctr=cfg["use_ctr"],
                        embed_dim=cfg["e"], final_embed_dim=cfg["f"])
    if "dd_label_map_size" in cfg:
        p.dd_label_map_size = tuple(cfg["dd_label_map_size"])
    bb = TaskPrompter(p, cfg["select"], img_size=tuple(cfg["img_size"]), patch_size=cfg["patch"],
                      embed_dim=cfg["C"], depth=cfg["depth"], num_heads=cfg["heads"],
                      chan_nheads=cfg["chan_nheads"], drop_path_rate=cfg.get("drop_path_rate", 0.15))   # common_config.py:22
    head_cls = DEConvHead if cfg.get("head", "conv") == "deconv" else ConvHead       # utils/common_config.py:64-70
    heads = nn.ModuleDict({t: head_cls(cfg["f"], cfg["num_output"][t]) for t in cfg["tasks"]})
    return TaskPrompterWrapper(p, bb, heads, nsplit=nsplit, use_graph=use_graph)


def _mirror_head(t, hd):
    """This library's ConvHead (:688-698) or DEConvHead (:700-715) shaped like the reference head hd, told apart by the
    first layer (parameters are loaded afterwards)."""
    if not hasattr(hd, "mt_proj") or not hasattr(hd, "linear_pred"):
        raise NotImplementedError(f"mtt_b200.accelerate: unsupported head {type(hd).__name__} for task {t!r} "
                                  "(FCOS3DHead / '3ddet' needs mmdet3d: SURVEY.md 8f N4)")
    if isinstance(hd.mt_proj[0], nn.ConvTranspose2d):
        return DEConvHead(hd.mt_proj[0].weight.shape[0], hd.linear_pred.weight.shape[0])
    return ConvHead(hd.linear_pred.weight.shape[1], hd.linear_pred.weight.shape[0])


def accelerate(ref_model, nsplit=PARITY, use_graph=True):
    """Drop-in: build the fused wrapper from a REFERENCE TaskPrompterWrapper instance. Parameters and BatchNorm
    statistics are COPIED (`load_state_dict(ref.state_dict(), strict=True)`: same names, so the copy is exact);
    later in-place updates of `ref_model` are not seen -- call `load_state_dict` again (plans re-pack by themselves
    when parameter versions change). Raises for heads this library has no kernels for (FCOS3DHead, task '3ddet' of
    the reference's Cityscapes-3D config)."""
    bb = ref_model.backbone
    p = bb.p
    mine_bb = TaskPrompter(p, list(bb.select_list), img_size=tuple(bb.patch_embed.img_size),
                           patch_size=bb.patch_embed.patch_size[0], embed_dim=bb.embed_dim,
                           depth=len(bb.blocks), num_heads=bb.blocks[0].attn.num_heads,
                           chan_nheads=bb.blocks[0].attn.chan_nheads,
                           drop_path_rate=float(getattr(bb.blocks[-1].drop_path, "drop_prob", 0.0) or 0.0))

    heads = nn.ModuleDict({t: _mirror_head(t, ref_model.heads[t]) for t in ref_model.tasks})
    m = TaskPrompterWrapper(p, mine_bb, heads, nsplit=nsplit, use_graph=use_graph)
    m.load_state_dict(ref_model.state_dict(), strict=True)
    return m.eval()
