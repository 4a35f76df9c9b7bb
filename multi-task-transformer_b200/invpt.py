"""InvPT (ViT backbone + inverted-pyramid multi-task decoder) with the reference's nn.Module
boundaries and a fused sm_90a forward.

Module classes and parameter names mirror the reference so that its checkpoints load unchanged:

  VisionTransformer / Block / Attention        InvPT/models/transformers/vit.py:172-351
  TransformerDecoder / ConvBlock / MLPHead     InvPT/models/transformers/transformer_decoder.py:18-131
  InvPT / InvPTStage / InvPTBlock / SelfAttention / UpEmbed   InvPT/models/transformers/invpt.py:19-544
  TransformerNet                               InvPT/models/transformer_net.py:12-38

The modules own parameters and expose the reference's forward signatures; all arithmetic runs in libmtt_sm90.so
through `ops` (the plan lifecycle and per-module weight caches: plans.py):

  TransformerNet.forward(x)              -> {task: [B,n,H,W], 'inter_preds': {...}}   the fused path, ONE CUDA graph
  VisionTransformer.forward(x)           -> (x [B,P,C], [4 x [B,P,C]])                 vit.py:332-361
  TransformerDecoder.forward(x_list)     -> (x_dict {task: [B,C0,8h,8w]}, inter_pred)  transformer_decoder.py:69-98
  InvPT.forward(x_dict, inter_pred, back_fea) -> x_dict                                invpt.py:502-544
  MLPHead.forward(x)                     -> linear_pred(x)                             transformer_decoder.py:130

The sub-module forwards run segments of the same launch plan eagerly, with NCHW / token tensors in and out like the
reference. Eval-mode only (SyncBatchNorm = running statistics, DropPath = identity). Not reproduced because the
reference never consumes them: scale_embed[2]'s output and `norm_mt` (SURVEY.md section 2.3).
"""
from types import SimpleNamespace

import torch
import torch.nn as nn

from . import ops
from .plans import (Plan, _cached, _check_input, _dev_ctx, _f32, _lin, _pack_stem, _pack_vit_block, _plan_for,
                    _predict_outputs)
from .taskprompter import PARITY, Mlp, PatchEmbed, _trunc_normal_


# --------------------------------------------------------------------------------------------
# parameter containers
# --------------------------------------------------------------------------------------------
class VitAttention(nn.Module):
    def __init__(self, dim, num_heads, qkv_bias=True):
        super().__init__()
        self.num_heads = num_heads
        self.qkv = nn.Linear(dim, dim * 3, bias=qkv_bias)
        self.proj = nn.Linear(dim, dim)


class VitBlock(nn.Module):
    def __init__(self, dim, num_heads, mlp_ratio=4., qkv_bias=True):
        super().__init__()
        self.norm1 = nn.LayerNorm(dim, eps=1e-6)
        self.attn = VitAttention(dim, num_heads, qkv_bias)
        self.norm2 = nn.LayerNorm(dim, eps=1e-6)
        self.mlp = Mlp(dim, int(dim * mlp_ratio))


class VisionTransformer(nn.Module):
    """vit.py:227-330 (same constructor arguments that matter for the forward)."""

    def __init__(self, select_list, img_size=(224, 224), patch_size=16, in_chans=3, embed_dim=768, depth=12,
                 num_heads=12, mlp_ratio=4., qkv_bias=True, **_unused):
        super().__init__()
        if isinstance(img_size, int):
            img_size = (img_size, img_size)
        self.embed_dim = embed_dim
        self.num_heads = num_heads
        self.patch_size = patch_size
        self.in_chans = in_chans
        self.patch_embed = PatchEmbed(img_size, patch_size, in_chans, embed_dim)
        self.cls_token = nn.Parameter(torch.zeros(1, 1, embed_dim))
        self.pos_embed = nn.Parameter(torch.zeros(1, self.patch_embed.num_patches + 1, embed_dim))
        self.blocks = nn.Sequential(*[VitBlock(embed_dim, num_heads, mlp_ratio, qkv_bias) for _ in range(depth)])
        self.norm = nn.LayerNorm(embed_dim, eps=1e-6)
        self.select_list = list(select_list)
        self.nsplit = PARITY
        self.use_graph = False
        _trunc_normal_(self.pos_embed, std=.02)
        _trunc_normal_(self.cls_token, std=.02)
        for m in self.modules():
            if isinstance(m, nn.Linear):
                _trunc_normal_(m.weight, std=.02)
                nn.init.zeros_(m.bias)

    def forward(self, x):
        """vit.py:332-361: (final-norm patch tokens [B,P,C], [x[:,1:] after each selected block ..., the same final
        tokens]). Fresh tensors."""
        _check_input(self, x)
        B, dev = x.shape[0], x.device
        pl = _plan_for(self, (B, dev, self.nsplit, "backbone"), lambda: _Plan(
            self, None, None, None, [], B, dev, self.nsplit, mode="backbone"))
        feats = pl.run(x, graph=self.use_graph)["selected_fea"]
        feats = [f.clone() for f in feats]
        return feats[-1], feats


class ConvBlock(nn.Module):
    """transformer_decoder.py:100-122: conv3x3 (no bias) -> BN -> ReLU."""

    def __init__(self, inplanes, planes):
        super().__init__()
        self.conv = nn.Conv2d(inplanes, planes, 3, padding=1, bias=False)
        self.bn1 = nn.BatchNorm2d(planes)
        self.relu = nn.ReLU(inplace=True)


class MLPHead(nn.Module):
    """transformer_decoder.py:124-131."""

    nsplit = PARITY

    def __init__(self, in_channels, num_classes):
        super().__init__()
        self.linear_pred = nn.Conv2d(in_channels, num_classes, kernel_size=1)

    def forward(self, x):
        """x [B,Cin,h,w] NCHW -> [B,n_out,h,w] (1x1 conv on the wgmma GEMM)."""
        _check_input(self, x)
        B, Cin, h, w = x.shape
        dev, ns = x.device, self.nsplit
        with _dev_ctx(dev):
            lp = _pack_mlp_head(self, dev, ns)
            n = self.linear_pred.weight.shape[0]
            a = ops.Split(B * h * w, Cin, dev, ns)
            ops.nchw_to_nhwc_split(x.contiguous(), a)
            y = torch.empty(B * h * w, ops.round_up(n, 4), device=dev, dtype=torch.float32)
            ops.gemm(a, lp[0], bias=lp[1], out_f32=y[:, :n], N=n)
            out = torch.empty(B, n, h, w, device=dev, dtype=torch.float32)
            ops.nhwc_to_nchw(y, y.stride(0), B, n, h, w, out)
            return out


def _pack_mlp_head(hd, device, ns):
    """MLPHead.linear_pred as (packed weight, bias), cached on the head (shared by MLPHead.forward and the plans)."""
    return _cached(hd, ("pack", device, ns), lambda: _lin(hd.linear_pred, device, ns))


class UpEmbed(nn.Module):
    """invpt.py:19-43; Sequential indices 1,2,4,5 carry the parameters."""

    def __init__(self, in_chans, embed_dim):
        super().__init__()
        self.proj = nn.Sequential(
            nn.Upsample(scale_factor=2, mode='bilinear', align_corners=False),
            nn.Conv2d(in_chans, embed_dim, 3, padding=2, stride=1, bias=False, dilation=2),
            nn.BatchNorm2d(embed_dim), nn.ReLU(inplace=True),
            nn.Conv2d(embed_dim, embed_dim, 3, padding=2, stride=1, bias=False, dilation=2),
            nn.BatchNorm2d(embed_dim), nn.ReLU(inplace=True))


class _DwBn(nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.conv = nn.Conv2d(dim, dim, 3, padding=1, stride=2, bias=False, groups=dim)
        self.bn = nn.BatchNorm2d(dim)


class SelfAttention(nn.Module):
    """invpt.py:68-164 (q_method 'dw_bn', kv_method 'avg')."""

    def __init__(self, fea_no, dim, num_heads, stride_kv):
        super().__init__()
        self.fea_no, self.dim, self.num_heads, self.stride_kv = fea_no, dim, num_heads, stride_kv
        self.scale = dim ** -0.5
        self.conv_proj_q = nn.ModuleList([_DwBn(dim) for _ in range(fea_no)])
        self.proj_q = nn.Linear(dim, dim)
        self.proj_k = nn.Linear(dim, dim)
        self.proj_v = nn.Linear(dim, dim)
        self.proj = nn.Linear(dim, dim)
        self.fuse_attn = nn.Conv2d(num_heads * 2, num_heads, 1)


class InvPTBlock(nn.Module):
    def __init__(self, task_no, dim, num_heads, stride_kv, mlp_ratio=4.):
        super().__init__()
        self.norm1 = nn.LayerNorm(dim)
        self.norm2 = nn.LayerNorm(dim)
        self.mlp = Mlp(dim, int(dim * mlp_ratio))
        self.attn = SelfAttention(task_no, dim, num_heads, stride_kv)


class InvPTStage(nn.Module):
    def __init__(self, task_no, stage_idx, in_chans, embed_dim, num_heads, stride_kv):
        super().__init__()
        self.stage_idx = stage_idx
        self.patch_embed = None if stage_idx == 0 else nn.ModuleList(
            [UpEmbed(in_chans, embed_dim) for _ in range(task_no)])
        self.blocks = nn.ModuleList([InvPTBlock(task_no, embed_dim, num_heads, stride_kv)])
        for m in self.modules():
            if isinstance(m, nn.Linear):
                _trunc_normal_(m.weight, std=0.02)
                nn.init.zeros_(m.bias)


class InvPT(nn.Module):
    """invpt.py:419-500."""

    def __init__(self, p, in_chans, ori_embed_dim):
        super().__init__()
        tasks = list(p.TASKS.NAMES)
        T = len(tasks)
        dims = [in_chans, in_chans // 2, in_chans // 4]
        self.dims = dims
        self.p = p
        self.tasks = tasks
        self.ori_embed_dim = ori_embed_dim
        self.nsplit = PARITY
        self.norm_mts = nn.ModuleList()
        self.redu_chan = nn.ModuleList()
        self.invpt_stages = nn.ModuleList()
        prev = in_chans
        for i in range(3):
            self.invpt_stages.append(InvPTStage(T, i, prev, dims[i], 2, 2 ** (i + 1)))
            prev = dims[i]
            self.norm_mts.append(nn.LayerNorm(dims[i] * T))
            self.redu_chan.append(nn.ModuleList([nn.Conv2d(dims[i], in_chans, 1) for _ in range(T)]))
        self.norm_mt = nn.LayerNorm(T * dims[2])   # never called by the reference forward
        self.mt_proj = nn.ModuleDict({t: nn.Sequential(nn.Conv2d(in_chans, in_chans, 3, padding=1),
                                                       nn.BatchNorm2d(in_chans), nn.ReLU(True)) for t in tasks})
        self.mix_proj = nn.ModuleDict({t: nn.Sequential(nn.Conv2d(ori_embed_dim + p.TASKS.NUM_OUTPUT[t], in_chans, 1))
                                       for t in tasks})

    def forward(self, x_dict, inter_pred, back_fea):
        """invpt.py:502-544. x_dict {task: [B,E,h,w]}, inter_pred {task: [B,n,h,w]}, back_fea [[B,C0/4,4h',4w'],
        [B,C0/2,2h',2w'], ...] (the first two are the skips of stages 2 and 1) -> {task: [B,C0,8h,8w]}."""
        x0 = x_dict[self.tasks[0]]
        _check_input(self, x0)
        B, _, h0, w0 = x0.shape
        dev = x0.device
        pl = _plan_for(self, (B, dev, self.nsplit, "invpt", h0, w0), lambda: _Plan(
            None, None, None, self.p, self.tasks, B, dev, self.nsplit, mode="invpt", inv=self, hw0=(h0, w0)))
        with _dev_ctx(dev):
            pl.load_invpt_inputs(x_dict, inter_pred, back_fea)
            return {t: v.clone() for t, v in pl.run(None, graph=False)["x_dict"].items()}


class TransformerDecoder(nn.Module):
    """transformer_decoder.py:18-67."""

    def __init__(self, p):
        super().__init__()
        self.p = p
        self.nsplit = PARITY
        self.embed_dim = p.embed_dim
        d0 = p.embed_dim + p.PRED_OUT_NUM_CONSTANT
        tasks = list(p.TASKS.NAMES)
        C = p.backbone_channels[-1]
        self.intermediate_head = nn.ModuleDict({t: nn.Conv2d(p.embed_dim, p.TASKS.NUM_OUTPUT[t], 1) for t in tasks})
        self.invpt = InvPT(p, in_chans=d0, ori_embed_dim=p.embed_dim)
        self.preliminary_decoder = nn.ModuleDict(
            {t: nn.Sequential(ConvBlock(C, C), ConvBlock(C, p.embed_dim)) for t in tasks})
        self.scale_embed = nn.ModuleList([
            nn.ConvTranspose2d(p.backbone_channels[0], d0 // 4, kernel_size=3, stride=2, padding=1, output_padding=1),
            nn.Conv2d(p.backbone_channels[1], d0 // 2, 3, padding=1),
            nn.Conv2d(p.backbone_channels[2], d0, 3, padding=1),
            None])

    def forward(self, x_list):
        """transformer_decoder.py:69-98. x_list: the backbone's 4 selected features [B,P,C] ->
        (x_dict {task: [B,C0,8h,8w]}, inter_pred {task: [B,n_out,h,w]}) with (h,w) = the mtt resolution."""
        _check_input(self, x_list[0])
        B, dev = x_list[0].shape[0], x_list[0].device
        tasks = list(self.p.TASKS.NAMES)
        pl = _plan_for(self, (B, dev, self.nsplit, "decoder"), lambda: _Plan(
            None, self, None, self.p, tasks, B, dev, self.nsplit, mode="decoder"))
        with _dev_ctx(dev):
            pl.load_features(x_list)
            out = pl.run(None, graph=False)
            return ({t: v.clone() for t, v in out["x_dict"].items()},
                    {t: v.clone() for t, v in out["inter_pred"].items()})


class TransformerNet(nn.Module):
    """transformer_net.py:12-38. forward(x[B,3,H,W]) -> {task: [B,n_out,H,W], 'inter_preds': {task: ...}}."""

    def __init__(self, p, backbone, backbone_channels, heads, nsplit=PARITY, use_graph=True):
        super().__init__()
        self.p = p
        self.tasks = list(p.TASKS.NAMES)
        self.backbone = backbone
        self.multi_task_decoder = TransformerDecoder(p)
        self.heads = heads
        self.nsplit = nsplit
        self.use_graph = use_graph

    def plan(self, batch, device, postproc=False):
        mode = "postproc" if postproc else "full"
        return _plan_for(self, (int(batch), torch.device(device), int(self.nsplit), mode), lambda: _Plan(
            self.backbone, self.multi_task_decoder, self.heads, self.p, self.tasks, batch, torch.device(device),
            self.nsplit, mode=mode))

    def forward(self, x):
        _check_input(self, x)
        return self.plan(x.shape[0], x.device).run(x, graph=self.use_graph)

    def predict(self, x):
        """forward + the reference's `get_output` post-processing (InvPT/utils/utils.py:18-48) fused into the
        final resize of every task head (no full-resolution logits, no inter_preds)."""
        _check_input(self, x)
        return self.plan(x.shape[0], x.device, postproc=True).run(x, graph=self.use_graph)


# --------------------------------------------------------------------------------------------
# the fused forward
# --------------------------------------------------------------------------------------------
def _pack_decoder(dec, tasks, device, ns):
    """scale_embed, preliminary decoders and intermediate heads (transformer_decoder.py:18-98), BatchNorm folded."""
    def build():
        f = lambda t: _f32(t, device)
        W = SimpleNamespace()
        # ConvTranspose2d(k3,s2,p1,op1) == zero-insert + conv3x3(pad 1) with the spatially flipped,
        # in/out-transposed kernel (mtt_pack_conv_weight transposed = 1)
        W.se0, W.se0_b = ops.pack_conv_weight(f(dec.scale_embed[0].weight), dec.scale_embed[0].bias, None, ns,
                                              transposed=True)
        W.se1, W.se1_b = ops.pack_conv_weight(f(dec.scale_embed[1].weight), dec.scale_embed[1].bias, None, ns)
        W.tasks = []
        for t in tasks:
            tw = SimpleNamespace()
            pd = dec.preliminary_decoder[t]
            tw.pd0, tw.pd0_b = ops.pack_conv_weight(f(pd[0].conv.weight), None, pd[0].bn1, ns)
            tw.pd1, tw.pd1_b = ops.pack_conv_weight(f(pd[1].conv.weight), None, pd[1].bn1, ns)
            tw.ih, tw.ih_b = _lin(dec.intermediate_head[t], device, ns)
            W.tasks.append(tw)
        return W
    return _cached(dec, ("pack_dec", device, ns, tuple(tasks)), build)


def _pack_invpt(inv, tasks, device, ns):
    """mix_proj, the three stages, norm_mts / redu_chan and mt_proj (invpt.py:400-544)."""
    def build():
        f = lambda t: _f32(t, device)
        T, dims = len(tasks), list(inv.dims)
        W = SimpleNamespace(tasks=[], stages=[])
        for t in tasks:
            tw = SimpleNamespace()
            tw.mix, tw.mix_b = _lin(inv.mix_proj[t][0], device, ns)
            tw.mt, tw.mt_b = ops.pack_conv_weight(f(inv.mt_proj[t][0].weight), inv.mt_proj[t][0].bias, inv.mt_proj[t][1], ns)
            W.tasks.append(tw)
        for i, st in enumerate(inv.invpt_stages):
            sw = SimpleNamespace()
            if i > 0:
                sw.up = []
                for k in range(T):
                    pr = st.patch_embed[k].proj
                    wa, ba = ops.pack_conv_weight(f(pr[1].weight), None, pr[2], ns)
                    wb, bb_ = ops.pack_conv_weight(f(pr[4].weight), None, pr[5], ns)
                    sw.up.append((wa, ba, wb, bb_))
            blk = st.blocks[0]
            sw.n1w, sw.n1b, sw.n2w, sw.n2b = f(blk.norm1.weight), f(blk.norm1.bias), f(blk.norm2.weight), f(blk.norm2.bias)
            sw.eps = blk.norm1.eps
            qw, qb = [], []
            for k in range(T):                       # depthwise 3x3 + eval BN: a per-channel fold, kept in fp32
                cq = blk.attn.conv_proj_q[k]
                sc = f(cq.bn.weight) / torch.sqrt(f(cq.bn.running_var) + cq.bn.eps)
                qw.append((f(cq.conv.weight) * sc.reshape(-1, 1, 1, 1)).reshape(dims[i], 9))
                qb.append(f(cq.bn.bias) - f(cq.bn.running_mean) * sc)
            sw.dw_w, sw.dw_b = torch.stack(qw).contiguous(), torch.stack(qb).contiguous()
            sw.proj_q, sw.proj_q_b = _lin(blk.attn.proj_q, device, ns)
            sw.proj_k, sw.proj_k_b = _lin(blk.attn.proj_k, device, ns)
            sw.proj_v, sw.proj_v_b = _lin(blk.attn.proj_v, device, ns)
            sw.proj, sw.proj_b = _lin(blk.attn.proj, device, ns)
            sw.fuse_w = f(blk.attn.fuse_attn.weight).reshape(2, 4).contiguous()
            sw.fuse_b = f(blk.attn.fuse_attn.bias)
            sw.fc1, sw.fc1_b = _lin(blk.mlp.fc1, device, ns)
            sw.fc2, sw.fc2_b = _lin(blk.mlp.fc2, device, ns)
            sw.nmw, sw.nmb, sw.nmeps = f(inv.norm_mts[i].weight), f(inv.norm_mts[i].bias), inv.norm_mts[i].eps
            if i > 0:
                sw.redu = [_lin(inv.redu_chan[i][k], device, ns) for k in range(T)]
            W.stages.append(sw)
        return W
    return _cached(inv, ("pack_inv", device, ns, tuple(tasks)), build)


class _Plan(Plan):
    """Geometry, workspace and launch sequence of one InvPT forward. mode: "full" / "postproc" = TransformerNet
    forward / predict; "backbone" = VisionTransformer.forward; "decoder" = TransformerDecoder.forward on given
    backbone features; "invpt" = InvPT.forward on given task features, preliminary predictions and skips (these two
    take no image: `run(None, graph=False)` after `load_features` / `load_invpt_inputs`)."""

    def __init__(self, bb, dec, heads, p, tasks, B, device, nsplit, mode="full", inv=None, hw0=None):
        self.inv = inv if inv is not None else (dec.invpt if dec is not None else None)
        super().__init__((bb, dec if dec is not None else self.inv, heads), B, device, nsplit, len(tasks))
        device = self.dev
        self.mode = mode
        self.postproc = mode == "postproc"
        self.bb, self.dec, self.heads, self.p = bb, dec, heads, p
        self.tasks = list(tasks)
        self.T = T = len(self.tasks)
        ns = nsplit
        S = lambda r, c, **kw: ops.Split(r, c, device, ns, **kw)
        z = lambda *s: torch.zeros(*s, device=device, dtype=torch.float32)
        with _dev_ctx(device):
            self._repack()
            if bb is not None:
                self.C = C = bb.embed_dim
                self.H = bb.num_heads
                if C // self.H != 64 or C % self.H:
                    raise ValueError(f"InvPT: embed_dim / num_heads = {C} / {self.H} must be 64 (mtt_attention is built for "
                                     "head dim 64: ViT-B 768 / 12, ViT-L 1024 / 16)")
                self.gh, self.gw = bb.patch_embed.grid_size
                self.patch = bb.patch_size
                self.img = (self.gh * self.patch, self.gw * self.patch)
                self.select = list(bb.select_list)
                self.depth = len(bb.blocks)
            elif mode == "decoder":
                self.C = C = p.backbone_channels[-1]
                self.gh, self.gw = p.spatial_dim[-1]
            if mode in ("full", "postproc", "decoder") and (self.gh % 4 or self.gw % 4):
                # the decoder concatenates x2 / x4 / x8 up-sampled maps with stride-2-reduced ones (IP invpt.py:125-147,
                # :524-539, transformer_decoder.py:63-98): they only line up when the token grid is a multiple of 4 x 4.
                # The reference fails for other sizes too (torch.cat size mismatch); say so before any kernel is launched.
                raise ValueError(f"InvPT: token grid {self.gh} x {self.gw} must be a multiple of 4 x 4 (image height and "
                                 f"width multiples of {4 * (self.patch if bb is not None else 16)}); the reference "
                                 "rejects this size as well")
            self.P = P = self.gh * self.gw if mode != "invpt" else 0
            self.N = N = 1 + P
            # ---- backbone workspace
            if bb is not None:
                self.cols = S(B * P, self.patch * self.patch * bb.in_chans)
                self.qkv = S(B * N, 3 * C)
                self.ao = S(B * N, C)
                self.ws_qkv = ops.workspace(ops.workspace_bytes(ops.OP_LN_QKV, rows=B * N, Cdim=C, nsplit=ns), device)
                self.ws_mlp = ops.workspace(ops.workspace_bytes(ops.OP_LN_MLP_RESIDUAL, rows=B * N, Cdim=C,
                                                                hidden=bb.blocks[0].mlp.fc1.out_features, nsplit=ns),
                                            device)
            if mode != "invpt":
                self.xs = z(B * N, C)
                self.xfin = z(B * P, C)
            if mode == "backbone":
                self.sel = [z(B, P, C) for _ in range(len(self.select))]
                self.out = {"selected_fea": self.sel + [self.xfin.view(B, P, C)]}
                return
            # ---- decoder workspace
            inv_ = self.inv
            self.E = E = inv_.ori_embed_dim
            self.dims = dims = list(inv_.dims)
            if mode == "invpt":
                self.h0, self.w0 = hw0
            else:
                down = p.mtt_resolution_downsample_rate
                self.h0, self.w0 = self.gh // down, self.gw // down
            h0, w0 = self.h0, self.w0
            self.th, self.tw = h0 * 8, w0 * 8
            self.n_out = [p.TASKS.NUM_OUTPUT[t] for t in self.tasks]
            if mode != "invpt":
                self.zi = S(B * 4 * P, C)
                self.f1 = S(B * P, C)
                self.x0 = S(B * h0 * w0, C)
                self.p1 = [S(B * h0 * w0, C) for _ in range(T)]   # per task: the task chains run on side streams
                self.back0 = z(B * 4 * P, dims[2])
                self.back1 = z(B * P, dims[1])
            else:
                self.back0 = z(B * 16 * h0 * w0, dims[2])
                self.back1 = z(B * 4 * h0 * w0, dims[1])
            cat_ld = ops.round_up(E + max(self.n_out), 8)     # one row stride for all tasks (grouped launches)
            self.cat = [S(B * h0 * w0, E + n, zero=True, ld=cat_ld) for n in self.n_out]
            self.inter = [z(B * h0 * w0, ops.round_up(n, 4)) for n in self.n_out]
            self.st = []
            for i in range(3):
                h, w = h0 * 2 ** i, w0 * 2 ** i
                Ci = dims[i]
                s = SimpleNamespace(h=h, w=w, C=Ci)
                s.kvs = 2 ** (i + 1)
                s.kh, s.kw = -(-h // s.kvs), -(-w // s.kvs)
                s.Lq = T * (h // 2) * (w // 2)
                s.Tk = T * s.kh * s.kw
                s.xj = z(B * T * h * w, Ci)
                s.xn32 = z(B * T * h * w, Ci)
                s.qin = S(B * s.Lq, Ci)
                s.kvin = S(B * s.Tk, Ci)
                # cross-task attention (2 heads of dim Ci / 2): q, k as split operands of S = Q_h K_h^T, v transposed per image
                # for O_h = P_h V_h; both contractions are grouped launches over (batch, head)
                # (each head's columns start at a multiple of 8 elements: TMA base pointers are 16-byte aligned)
                s.dh = Ci // 2
                s.dhp = ops.round_up(s.dh, 8)
                s.qs, s.ks, s.v32 = S(B * s.Lq, 2 * s.dhp, zero=True), S(B * s.Tk, 2 * s.dhp, zero=True), z(B * s.Tk, Ci)
                s.vt = S(B * Ci, s.Tk, zero=True)
                s.score = z(B, 2, s.Lq, s.Tk)          # raw scores, then (in place) the fused pre-softmax scores
                s.P = S(B * 2 * s.Lq, s.Tk, zero=True)
                s.ao = S(B * s.Lq, Ci)
                s.a32 = z(B * s.Lq, Ci)
                s.ws_mlp = ops.workspace(ops.workspace_bytes(ops.OP_LN_MLP_RESIDUAL, rows=B * T * h * w, Cdim=Ci,
                                                             hidden=4 * Ci, nsplit=ns), device)
                if i == 0:
                    s.ln32 = z(T * B * h * w, Ci)
                else:
                    s.ln = S(T * B * h * w, Ci)
                    s.rc32 = [z(B * h * w, dims[0]) for _ in range(T)]
                    s.ue0 = [S(B * h * w, dims[i - 1]) for _ in range(T)]
                    s.ue1 = [S(B * h * w, Ci) for _ in range(T)]
                self.st.append(s)
            tt = B * self.th * self.tw
            self.mss = [S(tt, dims[0]) for _ in range(T)]
            self.hm = [S(tt, dims[0]) for _ in range(T)]
            if mode in ("decoder", "invpt"):
                self.hm32 = z(tt, dims[0])                       # one NHWC fp32 staging map, reused per task
                self.x_dict = {t: z(B, dims[0], self.th, self.tw) for t in self.tasks}
                self.out = {"x_dict": self.x_dict}
                if mode == "decoder":
                    self.inter_nchw = {t: z(B, n, h0, w0) for t, n in zip(self.tasks, self.n_out)}
                    self.out["inter_pred"] = self.inter_nchw
                return
            self.pred = [z(tt, ops.round_up(n, 4)) for n in self.n_out]
            oh, ow = self.img
            if not self.postproc:
                self.out = {t: z(B, n, oh, ow) for t, n in zip(self.tasks, self.n_out)}
                self.out_inter = {t: z(B, n, oh, ow) for t, n in zip(self.tasks, self.n_out)}
            else:
                self.out = _predict_outputs(self.tasks, B, (oh, ow), device)

    def _pack(self):
        bb, dev, ns = self.bb, self.dev, self.ns
        self.Ws = _pack_stem(bb, dev, ns) if bb is not None else None
        self.Wb = [_pack_vit_block(blk, dev, ns) for blk in bb.blocks] if bb is not None else None
        self.Wd = _pack_decoder(self.dec, self.tasks, dev, ns) if self.dec is not None else None
        self.Wi = _pack_invpt(self.inv, self.tasks, dev, ns) if self.inv is not None else None
        self.Wh = [_pack_mlp_head(self.heads[t], dev, ns) for t in self.tasks] if self.heads is not None else None

    def _result(self):
        out = dict(self.out)
        if self.mode == "full":
            out["inter_preds"] = dict(self.out_inter)
        return out

    def _par(self, fn):
        """Run fn(k) for every task k, each on its own side stream forked from / joined to the current
        stream (the per-task chains are independent and individually too small to fill 132 SMs)."""
        self.streams.par([lambda k=k: fn(k) for k in range(self.T)])

    # ------------------------------------------------------------------------------------------ inputs of the
    # module-boundary modes (copies into the plan's buffers; the fused modes never run these)
    def load_features(self, x_list):
        """TransformerDecoder.forward input: 4 x [B,P,C] token maps (transformer_decoder.py:74-83)."""
        B, P, C = self.B, self.P, self.C
        for which in (0, 1):
            self.xs.view(B, self.N, C)[:, 1:].copy_(x_list[which])
            self._scale_embed(which)
        self.xfin.view(B, P, C).copy_(x_list[3])

    def load_invpt_inputs(self, x_dict, inter_pred, back_fea):
        """InvPT.forward inputs (invpt.py:502-513): NCHW task features + preliminary predictions -> the `cat`
        operands of mix_proj; back_fea[0], [1] -> the NHWC skip maps of stages 2 and 1."""
        B, E = self.B, self.E
        for k, t in enumerate(self.tasks):
            ops.nchw_to_nhwc_split(x_dict[t].contiguous(), self.cat[k])
            ops.nchw_to_nhwc_split(inter_pred[t].contiguous(), self.cat[k], col_offset=E)
        for buf, src in ((self.back0, back_fea[0]), (self.back1, back_fea[1])):
            b_, c_, h_, w_ = src.shape
            buf.view(b_, h_, w_, c_).copy_(src.permute(0, 2, 3, 1))

    # ------------------------------------------------------------------------------------------
    def _vit_block(self, w):
        B, N = self.B, self.N
        ops.ln_qkv(self.xs, w.n1w, w.n1b, w.eps, w.qkv, w.qkv_b, self.qkv, self.ws_qkv)     # vit.py:213, :186
        ops.attention(self.qkv, self.ao, B=B, N=N, H=self.H, scale=64 ** -0.5)             # :189-193
        ops.proj_residual(self.ao, w.proj, w.proj_b, self.xs)                              # :194,:213
        ops.ln_mlp_residual(self.xs, w.n2w, w.n2b, w.eps, w.fc1, w.fc1_b, w.fc2, w.fc2_b, self.ws_mlp)  # :214

    def _scale_embed(self, which):
        B, N, P, C, W = self.B, self.N, self.P, self.C, self.Wd
        if which == 0:      # scale_embed[0]: ConvTranspose2d as zero-insert + flipped 3x3 conv
            ops.zero_insert(self.xs, self.zi, B=B, h=self.gh, w=self.gw, Cdim=C, src_group=N, src_offset=1)
            ops.gemm(self.zi, W.se0, N=self.dims[2], K=C, bias=W.se0_b, out_f32=self.back0,
                     conv=(B, 2 * self.gh, 2 * self.gw, 3, 1))                             # transformer_decoder.py:63,80
        elif which == 1:    # scale_embed[1]
            ops.split_rows(self.xs, self.f1, rows=B * P, cols=C, in_group=P, src_group=N, src_offset=1)
            ops.gemm(self.f1, W.se1, N=self.dims[1], K=C, bias=W.se1_b, out_f32=self.back1,
                     conv=(B, self.gh, self.gw, 3, 1))                                     # :64,:80
        # which == 2: scale_embed[2]'s output is never consumed by the reference

    def _stage(self, i):
        """InvPTStage + InvPTBlock + multi-scale aggregation for stage i (invpt.py:400-417,290-312,522-539)."""
        B, T, W = self.B, self.T, self.Wi
        s, sw = self.st[i], W.stages[i]
        h, w, Ci = s.h, s.w, s.C
        hw = h * w
        if i > 0:
            sp = self.st[i - 1]
            skip = self.back1 if i == 1 else self.back0
            # UpEmbed of the T tasks (invpt.py:32-38): per-task bilinear x2, then the two dilated 3x3 convs of all tasks
            # as grouped launches (T x 96 tiles instead of T single-wave launches); the second adds the backbone skip
            # (:406-411) and writes each task's slice of the joint token buffer
            self._par(lambda k: ops.bilinear(sp.xj, sp.xj.stride(0), B, sp.h, sp.w, sp.C, h, w, out_split=s.ue0[k],
                                             in_batch_rows=T * sp.h * sp.w, in_row_offset=k * sp.h * sp.w))   # :32
            ops.gemm_grouped([(s.ue0[k], sw.up[k][0], dict(N=Ci, K=sp.C, bias=sw.up[k][1], act=ops.ACT_RELU,
                                                          out_split=s.ue1[k], conv=(B, h, w, 3, 2))) for k in range(T)])
            ops.gemm_grouped([(s.ue1[k], sw.up[k][2], dict(N=Ci, K=Ci, bias=sw.up[k][3], act=ops.ACT_RELU, residual=skip,
                                                          res_row_mod=B * hw, out_f32=s.xj[k * hw:], regroup=(hw, T * hw, 0),
                                                          conv=(B, h, w, 3, 2))) for k in range(T)])
        # ---- InvPTBlock
        ops.layernorm(s.xj, sw.n1w, sw.n1b, sw.eps, out_f32=s.xn32)                                    # :298
        ops.dwconv3x3_s2(s.xn32, sw.dw_w, sw.dw_b, s.qin, B=B, T=T, h=h, w=w, Cdim=Ci)                 # :171-173
        ops.avgpool(s.xn32, s.kvin, BT=B * T, h=h, w=w, Cdim=Ci, s=s.kvs)                              # :175-187
        dh, dhp = s.dh, s.dhp
        for src, wq, bq, dst in ((s.qin, sw.proj_q, sw.proj_q_b, s.qs), (s.kvin, sw.proj_k, sw.proj_k_b, s.ks)):   # :200-201
            if dh == dhp:
                ops.gemm(src, wq, bias=bq, out_split=dst)
            else:           # one launch per head so that each head's columns land on an aligned offset
                for hd in range(2):
                    ops.gemm(src, wq, N=dh, bias=bq[hd * dh:], w_row_offset=hd * dh, out_split=dst, out_col_offset=hd * dhp)
        ops.gemm(s.kvin, sw.proj_v, bias=sw.proj_v_b, out_f32=s.v32)                                   # :202
        ops.transpose_split(s.v32, s.vt, B=B, L=s.Tk, Cdim=Ci)
        ops.gemm_grouped([(s.qs, s.ks, dict(M=s.Lq, N=s.Tk, K=dh, a_row_offset=b * s.Lq, a_col_offset=hd * dhp,
                                            w_row_offset=b * s.Tk, w_col_offset=hd * dhp, out_f32=s.score[b, hd]))
                          for b in range(B) for hd in range(2)])                                       # :204 q k^T
        prev = self.st[i - 1].score if i > 0 else None
        ops.invpt_fuse_softmax(s.score, s.P, B=B, Lq=s.Lq, Tk=s.Tk, scale=Ci ** -0.5, prev_score=prev, T=T, qh=h // 2,
                               qw=w // 2, fuse_w=sw.fuse_w, fuse_b=sw.fuse_b,
                               score_out=s.score if i < 2 else None)                                   # :205-232
        ops.gemm_grouped([(s.P, s.vt, dict(M=s.Lq, N=dh, K=s.Tk, a_row_offset=(b * 2 + hd) * s.Lq,
                                           w_row_offset=b * Ci + hd * dh, out_split=s.ao, out_row_offset=b * s.Lq,
                                           out_col_offset=hd * dh)) for b in range(B) for hd in range(2)])   # :234 attn v
        ops.gemm(s.ao, sw.proj, bias=sw.proj_b, out_f32=s.a32)                                         # :238
        qhw = (h // 2) * (w // 2)
        self._par(lambda k: ops.bilinear(                                                              # :299-306
            s.a32, s.a32.stride(0), B, h // 2, w // 2, Ci, h, w, out_f32=s.xj, accumulate=True,
            in_batch_rows=T * qhw, in_row_offset=k * qhw, out_batch_rows=T * hw, out_row_offset=k * hw))
        ops.ln_mlp_residual(s.xj, sw.n2w, sw.n2b, sw.eps, sw.fc1, sw.fc1_b, sw.fc2, sw.fc2_b, s.ws_mlp)  # :307-308
        # ---- joint-channel LayerNorm over all tasks, per-task slices to the common resolution
        ops.layernorm_seg(s.xj, sw.nmw, sw.nmb, sw.nmeps, rows=B * hw, cols=Ci, S=T, in_group=hw, src_group=T * hw,
                          seg_stride=hw, out_f32=s.ln32 if i == 0 else None,
                          out_split=None if i == 0 else s.ln, out_seg_stride=B * hw)                   # :524-526
        d0 = self.dims[0]

        if i > 0:       # per-task slice -> 1x1 redu_chan (:535-536), all tasks in one grouped launch
            ops.gemm_grouped([(s.ln, sw.redu[k][0], dict(M=B * hw, bias=sw.redu[k][1], out_f32=s.rc32[k],
                                                         a_row_offset=k * B * hw)) for k in range(T)])

        def aggregate(k):
            # after the last stage the three per-stage maps of a task are resized to 8h0 x 8w0, summed and written ONCE
            # as the split operand of mt_proj (:528-543)
            s0_, s1_ = self.st[0], self.st[1]
            ops.bilinear_sum3([(s0_.ln32, s0_.h, s0_.w, 0, k * B * s0_.h * s0_.w),
                               (s1_.rc32[k], s1_.h, s1_.w, 0, 0),
                               (s.rc32[k], h, w, 0, 0)],
                              self.mss[k], B=B, Cdim=d0, H2=self.th, W2=self.tw)                       # :537-539
            if self.mode in ("full", "postproc"):
                self._head(k)
        if i == 2:
            self._par(aggregate)
        if i == 2 and self.mode in ("decoder", "invpt"):
            for k, t in enumerate(self.tasks):     # mt_proj -> NCHW x_dict (one fp32 staging map: sequential)
                tw = W.tasks[k]
                ops.gemm(self.mss[k], tw.mt, N=d0, K=d0, bias=tw.mt_b, act=ops.ACT_RELU, out_f32=self.hm32,
                         conv=(B, self.th, self.tw, 3, 1))                                             # :541-543
                ops.nhwc_to_nchw(self.hm32, d0, B, d0, self.th, self.tw, self.x_dict[t])

    def _head(self, k):
        B = self.B
        tw = self.Wi.tasks[k]
        lp, lp_b = self.Wh[k]
        d0 = self.dims[0]
        n = self.n_out[k]
        ops.conv3x3_bn_act(self.mss[k], tw.mt, tw.mt_b, d0, d0, ops.ACT_RELU, B=B, H=self.th, W=self.tw, mid=self.hm[k],
                           w_head=lp, b_head=lp_b, n_out=n, out_f32=self.pred[k][:, :n])               # invpt.py:541-543, MLPHead
        if self.postproc:
            ops.bilinear_postproc(self.pred[k], self.pred[k].stride(0), B, self.th, self.tw, n, self.img[0],
                                  self.img[1], ops.POSTPROC_KIND[self.tasks[k]], self.out[self.tasks[k]])
        else:
            ops.bilinear(self.pred[k], self.pred[k].stride(0), B, self.th, self.tw, n, self.img[0], self.img[1],
                         out_nchw=self.out[self.tasks[k]])                                             # transformer_net.py:35

    def _launch_backbone(self, img):
        B, N, P, C, W = self.B, self.N, self.P, self.C, self.Ws
        ops.im2col_patch(img, self.patch, self.cols)
        ops.gemm(self.cols, W.pe_w, bias=W.pe_b, residual=W.pos, res_row_mod=P, out_f32=self.xs,
                 regroup=(P, N, 1))                                                                    # vit.py:333,339
        ops.broadcast_rows(W.cls, self.xs, B, N)                                                       # :334-339
        for idx, w in enumerate(self.Wb):
            self._vit_block(w)
            if idx + 1 in self.select:
                which = self.select.index(idx + 1)
                if self.mode == "backbone":
                    self.sel[which].copy_(self.xs.view(B, N, C)[:, 1:])                                # :345-346
                else:
                    self._scale_embed(which)
        ops.layernorm_seg(self.xs, W.nw, W.nb, W.neps, rows=B * P, cols=C, S=1, in_group=P, src_group=N,
                          src_offset=1, out_f32=self.xfin)                                             # vit.py:348-349

    def _launch_decoder_front(self):
        B, C, T, W = self.B, self.C, self.T, self.Wd
        h0, w0, E = self.h0, self.w0, self.E
        ops.bilinear(self.xfin, C, B, self.gh, self.gw, C, h0, w0, out_split=self.x0)                  # transformer_decoder.py:85-86

        # preliminary decoders (transformer_decoder.py:88-94): the two ConvBlocks of all tasks as grouped launches
        ops.gemm_grouped([(self.x0, W.tasks[k].pd0, dict(N=C, K=C, bias=W.tasks[k].pd0_b, act=ops.ACT_RELU,
                                                         out_split=self.p1[k], conv=(B, h0, w0, 3, 1))) for k in range(T)])
        ops.gemm_grouped([(self.p1[k], W.tasks[k].pd1, dict(N=E, K=C, bias=W.tasks[k].pd1_b, act=ops.ACT_RELU,
                                                            out_split=self.cat[k], conv=(B, h0, w0, 3, 1)))
                          for k in range(T)])

        def prelim(k):
            tw = W.tasks[k]
            n = self.n_out[k]
            ops.gemm(self.cat[k], tw.ih, K=E, bias=tw.ih_b, out_f32=self.inter[k][:, :n], N=n,
                     out_split=self.cat[k], out_col_offset=E)                                          # :94; invpt.py:511
            if self.mode == "full":
                ops.bilinear(self.inter[k], self.inter[k].stride(0), B, h0, w0, n, self.img[0], self.img[1],
                             out_nchw=self.out_inter[self.tasks[k]])                                   # transformer_net.py:36
            elif self.mode == "decoder":
                ops.nhwc_to_nchw(self.inter[k], self.inter[k].stride(0), B, n, h0, w0, self.inter_nchw[self.tasks[k]])
        self._par(prelim)

    def _launch_invpt(self):
        B, T = self.B, self.T
        s0 = self.st[0]
        hw0 = self.h0 * self.w0
        self._par(lambda k: ops.gemm(self.cat[k], self.Wi.tasks[k].mix, bias=self.Wi.tasks[k].mix_b, out_f32=s0.xj,
                                     regroup=(hw0, T * hw0, k * hw0)))                                 # invpt.py:512
        for i in range(3):
            self._stage(i)

    def _launch(self, img):
        if self.mode in ("full", "postproc", "backbone"):
            self._launch_backbone(img)
        if self.mode in ("full", "postproc", "decoder"):
            self._launch_decoder_front()
        if self.mode != "backbone":
            self._launch_invpt()


def build_from_config(cfg, nsplit=PARITY, use_graph=True):
    """cfg: dict as in oracle/configs.invpt() (mirrors IP/utils/common_config.py:15-21,39-51)."""
    H, Wd = cfg["img_size"]
    gh, gw = H // cfg["patch"], Wd // cfg["patch"]
    p = SimpleNamespace(TASKS=SimpleNamespace(NAMES=list(cfg["tasks"]), NUM_OUTPUT=dict(cfg["num_output"])),
                        embed_dim=cfg["embed_dim"], PRED_OUT_NUM_CONSTANT=cfg["pred_const"],
                        mtt_resolution_downsample_rate=cfg["down"], backbone_channels=[cfg["C"]] * 4,
                        spatial_dim=[[gh, gw]] * 4)
    p.final_embed_dim = cfg["embed_dim"] + cfg["pred_const"]
    bb = VisionTransformer(cfg["select"], img_size=(H, Wd), patch_size=cfg["patch"], embed_dim=cfg["C"],
                           depth=cfg["depth"], num_heads=cfg["heads"])
    heads = nn.ModuleDict({t: MLPHead(p.final_embed_dim, cfg["num_output"][t]) for t in cfg["tasks"]})
    return TransformerNet(p, bb, p.backbone_channels, heads, nsplit=nsplit, use_graph=use_graph)


def accelerate(ref_model, nsplit=PARITY, use_graph=True):
    """Drop-in: build the fused InvPT from a REFERENCE TransformerNet instance (InvPT/models/transformer_net.py).
    Parameters and BatchNorm statistics are COPIED by an exact `load_state_dict(strict=True)`; later in-place updates
    of `ref_model` are not seen (load again; plans re-pack by themselves when parameter versions change)."""
    p = ref_model.multi_task_decoder.p
    bb = ref_model.backbone
    mine_bb = VisionTransformer(list(bb.select_list), img_size=tuple(bb.patch_embed.img_size),
                                patch_size=bb.patch_embed.patch_size[0], embed_dim=bb.embed_dim,
                                depth=len(bb.blocks), num_heads=bb.blocks[0].attn.num_heads)
    heads = nn.ModuleDict({t: MLPHead(ref_model.heads[t].linear_pred.weight.shape[1],
                                      ref_model.heads[t].linear_pred.weight.shape[0]) for t in ref_model.tasks})
    m = TransformerNet(p, mine_bb, p.backbone_channels, heads, nsplit=nsplit, use_graph=use_graph)
    m.load_state_dict(ref_model.state_dict(), strict=True)
    return m.eval()
