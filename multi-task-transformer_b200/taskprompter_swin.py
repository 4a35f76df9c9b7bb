"""TaskPrompter with the Swin backbone (the reference's Cityscapes-3D model family) -- SURVEY.md section 8f N2.

Module classes, constructor arguments and parameter / buffer names mirror
TaskPrompter/models/transformers/taskprompter_swin.py (TP below), so reference checkpoints load unchanged:

  WindowAttention       TP:120-212    relative_position_bias_table, relative_position_index (buffer), qkv, proj
  SwinTransformerBlock  TP:215-405    norm1, attn, norm2, mlp, attn_mask (buffer), chan_q, chan_kv, token_trans, chan_proj,
                                      token_trans1
  PatchMerging          TP:408-481    reduction, norm, process_chan_attn, task_prompts_up, spa_attn_ds
  BasicLayer            TP:484-540    blocks, downsample
  TaskPrompterSwin      TP:542-774    patch_embed (+ norm), task_prompts, fea_fuse / fea_decode_spa / fea_decode_chan,
                                      multi_scale_fuse, layers, norm
used through taskprompter.TaskPrompterWrapper (models/taskprompter_wrapper.py:9-40) with ConvHead / DEConvHead.

The modules own parameters; the forward is `_SwinPlan` (plans.Plan): packed weights + a fixed workspace + one launch
sequence, captured in a CUDA graph. What runs where:
  * every Linear / 1x1 / 3x3 convolution on the wgmma GEMM (mtt_gemm, the named block operators);
  * window partition with cyclic shift and zero padding, with the T task prompts replicated in front of every window:
    one gather kernel writing the joint window stream [B * nW * (T + ws^2), C] (TP:326-340, :177-181);
  * window attention with relative-position bias and shift mask on the patch x patch part (TP:183-204): one kernel per
    block over (window, head), exporting the un-scaled prompt-row logits (TP:189, :351-354);
  * window reverse / un-shift / crop, the residual add and the window-average of the prompt outputs (TP:210, :343-360):
    one scatter kernel; the prompt-row logits land directly in the [B, heads, T, T + H*W] layout the gating kernel of the
    ViT path reads;
  * channel attention between the prompts and the channels of the attention output (TP:372-396): chan_kv as a GEMM over
    the transposed map, the T x C logits / softmax / mixing in one small kernel;
  * PatchMerging (TP:430-472): 2x2 gather, LayerNorm, GEMM; the learned stride-2 3x3 down-sampling of the logit maps and
    the channel-logit up-projection as small direct kernels.
Exact algebraic re-orderings (results equal up to fp32 rounding): the bilinear x2 of the gated maps (TP:747-748) is applied
AFTER the 1x1 decode convs and fea_fuse[0] instead of before -- bilinear resampling and per-pixel linear maps commute --
which runs those convolutions at a quarter of the pixels.
The '3ddet' task of the reference's Cityscapes-3D config (semseg, depth, 3ddet) is an ordinary task in the backbone: its
prompt row takes part in every window attention, channel attention and PatchMerging, and it has gating, decode convs and
fea_fuse at each level. Its level features stay at the level's own resolution (no bilinear x2, TP:741, :764) and are not
fused across scales (no multi_scale_fuse['3ddet'], TP:635, :709-710): the plan writes them as 4 NCHW maps
[B, f, h_l, w_l], and TaskPrompterWrapper hands them to heads['3ddet'] -- the reference's FCOS3DHead (mmcv / mmdet3d), or any
module -- which runs in PyTorch on the same stream. The library has no kernels for that head.
SwinTransformerBlock, PatchMerging and BasicLayer also have the reference's forwards (TP:310-405, :430-477, :527-537),
tensors in and out in its layouts: they run the plan's block and merge launch code (_launch_swin_block, _launch_merge)
eagerly on a _StageSpace sized for the call, with the same packed weights. WindowAttention.forward raises: the reference
returns the full pre-softmax window map from it, which the fused kernel never forms (SURVEY.md section 8b).
Unsupported (raises): absolute position embedding (ape=True; no reference config uses it). Eval mode only.
"""
import math
from types import SimpleNamespace

import torch
import torch.nn as nn

from . import ops
from .plans import (Plan, _cached, _check_input, _dev_ctx, _f32, _lin, _pack_stem, _plan_for, _predict_outputs,
                    _Streams)
from .taskprompter import (PARITY, Mlp, PatchEmbed, _HeadSpace, _launch_head, _mirror_head, _pack_fuse, _pack_head,
                           _trunc_normal_)

STRIDES = (8, 16, 32, 32)          # utils/common_config.py:37: level il lives at 1/STRIDES[il] of the image
DET = "3ddet"                      # the detection task: level maps at their own resolution, no multi-scale fusion


# --------------------------------------------------------------------------------------------
# parameter containers (names = reference state_dict keys)
# --------------------------------------------------------------------------------------------
def relative_position_index(ws):
    """[ws*ws, ws*ws] index into the (2ws-1)^2 bias table (TP:146-157)."""
    ys, xs = torch.meshgrid(torch.arange(ws), torch.arange(ws), indexing="ij")
    ys, xs = ys.flatten(), xs.flatten()
    dy = ys[:, None] - ys[None, :] + ws - 1
    dx = xs[:, None] - xs[None, :] + ws - 1
    return dy * (2 * ws - 1) + dx


def shifted_window_mask(Hp, Wp, ws, shift):
    """[nW, ws*ws, ws*ws]: 0 where two tokens of a cyclically shifted window come from the same image region, -100
    otherwise (TP:276-290)."""
    region = torch.zeros(Hp, Wp)
    cuts = lambda n: [(0, n - ws), (n - ws, n - shift), (n - shift, n)]
    k = 0
    for (y0, y1) in cuts(Hp):
        for (x0, x1) in cuts(Wp):
            region[y0:y1, x0:x1] = k
            k += 1
    win = region.reshape(Hp // ws, ws, Wp // ws, ws).permute(0, 2, 1, 3).reshape(-1, ws * ws)
    diff = win[:, None, :] - win[:, :, None]
    return torch.where(diff != 0, torch.full_like(diff, -100.0), torch.zeros_like(diff))


class WindowAttention(nn.Module):
    def __init__(self, dim, window_size, num_heads, qkv_bias=True):
        super().__init__()
        self.dim, self.window_size, self.num_heads = dim, window_size, num_heads
        self.relative_position_bias_table = nn.Parameter(torch.zeros((2 * window_size - 1) ** 2, num_heads))
        self.register_buffer("relative_position_index", relative_position_index(window_size))
        self.qkv = nn.Linear(dim, dim * 3, bias=qkv_bias)
        self.proj = nn.Linear(dim, dim)
        _trunc_normal_(self.relative_position_bias_table, std=.02)

    def forward(self, *args, **kwargs):
        raise NotImplementedError(
            "mtt_b200 WindowAttention has no forward: the reference's returns the full (B*nW, heads, T + ws^2, T + ws^2) "
            "pre-softmax map, which the fused window-attention kernel never forms (it keeps only the prompt rows, "
            "SURVEY.md H4). Call SwinTransformerBlock.forward: its raw_spa_attn holds those rows on the map")


class SwinTransformerBlock(nn.Module):
    def __init__(self, last_block, p, dim, input_resolution, num_heads, window_size=7, shift_size=0, mlp_ratio=4.,
                 qkv_bias=True):
        super().__init__()
        self.LAST_BLOCK_FLAG = last_block
        self.dim, self.input_resolution, self.num_heads = dim, tuple(input_resolution), num_heads
        self.window_size, self.shift_size = window_size, shift_size
        if min(self.input_resolution) <= self.window_size:       # TP:243-246
            self.shift_size = 0
            self.window_size = min(self.input_resolution)
        H, W = self.input_resolution
        ws = self.window_size
        self.padded = (H + (ws - H % ws) % ws, W + (ws - W % ws) % ws)
        self.norm1 = nn.LayerNorm(dim)
        self.attn = WindowAttention(dim, ws, num_heads, qkv_bias)
        self.norm2 = nn.LayerNorm(dim)
        self.mlp = Mlp(dim, int(dim * mlp_ratio))
        mask = shifted_window_mask(self.padded[0], self.padded[1], ws, self.shift_size) if self.shift_size > 0 else None
        self.register_buffer("attn_mask", mask)
        ce = p.chan_embed_dim
        self.chan_q = nn.Linear(ce, ce, bias=qkv_bias)
        self.chan_kv = nn.Linear(H * W, ce * 2, bias=qkv_bias)
        self.token_trans = nn.Linear(dim, ce)
        if not last_block:
            self.chan_proj = nn.Linear(ce, ce)
            self.token_trans1 = nn.Linear(ce, dim)
        self.chan_nheads = p.chan_nheads

    nsplit = PARITY

    def forward(self, x, task_prompts):
        """TP:310-405: (x [B, H*W, C], [raw_spa_attn [B, heads, T, H, W], raw_chan_attn [B, T, C, nh, nw]],
        task_prompts [B, T, C]), fresh tensors. The model's last block (LAST_BLOCK_FLAG) does not update the prompts and
        returns their window-averaged attention outputs, as the reference does (:344, :399-405)."""
        _check_input(self, x)
        B, T = _check_tokens(self, x, task_prompts, self.dim)
        dev, ns = x.device, self.nsplit
        with _dev_ctx(dev):
            w = _pack_swin_block(self, dev, ns)
            s = _module_space(self, self, B, T, dev, ns)
            _load(s, x, task_prompts)
            spa = torch.zeros(B, T, self.dim, device=dev) if self.LAST_BLOCK_FLAG else None
            _launch_swin_block(s, w, self.shift_size, None if spa is None else spa.view(B * T, self.dim))
            return (s.x.view(B, s.L, s.C).clone(), _attn_out(s, s.logits, s.rc, s.H, s.W),
                    spa if spa is not None else s.p.view(B, T, s.C).clone())


class PatchMerging(nn.Module):
    def __init__(self, p, num_heads, input_resolution, dim):
        super().__init__()
        self.input_resolution, self.dim = tuple(input_resolution), dim
        T = len(p.TASKS.NAMES) * p.prompt_len
        self.reduction = nn.Linear(4 * dim, 2 * dim, bias=False)
        self.norm = nn.LayerNorm(4 * dim)
        self.process_chan_attn = nn.Linear(dim, 2 * dim, bias=False)
        self.task_prompts_up = nn.Linear(dim, 2 * dim, bias=False)
        self.spa_attn_ds = nn.Conv2d(num_heads * T, num_heads * T, kernel_size=3, padding=1, stride=2)
        self.num_heads, self.chan_nheads = num_heads, p.chan_nheads

    nsplit = PARITY

    def forward(self, x, task_prompts, attn_weight):
        """TP:430-477: (x [B, H/2*W/2, 2C], task_prompts [B, T, 2C], [raw_spa_attn [B, heads, T, H/2, W/2],
        raw_chan_attn [B, T, 2C, nh, nw]]), fresh tensors, from attn_weight = [raw_spa_attn [B, heads, T, H, W],
        raw_chan_attn [B, T, C, nh, nw]] of the stage's last block."""
        _check_input(self, x)
        B, T = _check_tokens(self, x, task_prompts, self.dim)
        raw_spa, raw_chan = attn_weight
        H, W = self.input_resolution
        C, nh = self.dim, int(round(math.sqrt(self.chan_nheads)))
        if tuple(raw_spa.shape) != (B, self.num_heads, T, H, W) or tuple(raw_chan.shape) != (B, T, C, nh, nh):
            raise ValueError(f"PatchMerging: expected attn_weight [[{B},{self.num_heads},{T},{H},{W}], [{B},{T},{C},{nh},"
                             f"{nh}]], got {[tuple(raw_spa.shape), tuple(raw_chan.shape)]}")
        dev, ns = x.device, self.nsplit
        with _dev_ctx(dev):
            w = _pack_merge(self, dev, ns)
            s = _module_space(self, None, B, T, dev, ns)
            _load(s, x, task_prompts)
            ops.swin_logit_maps(s.logits, raw_spa.to(device=dev, dtype=torch.float32).contiguous(), T=T, to_maps=False)
            s.rc.copy_(raw_chan)
            return _launch_merge_out(s, w)


class BasicLayer(nn.Module):
    def __init__(self, last_layer, p, dim, input_resolution, depth, num_heads, window_size, mlp_ratio=4., qkv_bias=True,
                 downsample=False):
        super().__init__()
        self.blocks = nn.ModuleList([
            SwinTransformerBlock(last_layer and i == depth - 1, p, dim, input_resolution, num_heads, window_size,
                                 0 if i % 2 == 0 else window_size // 2, mlp_ratio, qkv_bias) for i in range(depth)])
        self.downsample = PatchMerging(p, num_heads, input_resolution, dim) if downsample else None

    nsplit = PARITY

    def forward(self, x, task_prompts):
        """TP:527-537: the blocks in turn, then the PatchMerging if there is one: (x, attn_weight, task_prompts) as the
        last of them returns them (attn_weight = [raw_spa_attn, raw_chan_attn]), fresh tensors. The stage runs on one
        workspace: its maps go from block to block and into the merge without leaving the plan's layout."""
        _check_input(self, x)
        blk0 = self.blocks[0]
        B, T = _check_tokens(self, x, task_prompts, blk0.dim)
        dev, ns = x.device, self.nsplit
        with _dev_ctx(dev):
            Wb = [_pack_swin_block(blk, dev, ns) for blk in self.blocks]
            s = _module_space(self, blk0, B, T, dev, ns)
            _load(s, x, task_prompts)
            spa = torch.zeros(B, T, blk0.dim, device=dev) if self.blocks[-1].LAST_BLOCK_FLAG else None
            for blk, w in zip(self.blocks, Wb):
                _launch_swin_block(s, w, blk.shift_size, None if spa is None else spa.view(B * T, blk0.dim))
            if self.downsample is None:
                return (s.x.view(B, s.L, s.C).clone(), _attn_out(s, s.logits, s.rc, s.H, s.W),
                        spa if spa is not None else s.p.view(B, T, s.C).clone())
            x, task_prompts, attn_weight = _launch_merge_out(s, _pack_merge(self.downsample, dev, ns))
            return x, attn_weight, task_prompts


class SwinPatchEmbed(PatchEmbed):
    """timm PatchEmbed with norm_layer=LayerNorm (TP:592-595, patch_norm=True)."""

    def __init__(self, img_size, patch_size, in_chans, embed_dim):
        super().__init__(img_size, patch_size, in_chans, embed_dim)
        self.norm = nn.LayerNorm(embed_dim)


class TaskPrompterSwin(nn.Module):
    """TP:542-666 (same constructor arguments that matter for the forward; `p` needs TASKS.NAMES, prompt_len,
    chan_embed_dim, chan_nheads, img_ds_ratio, level_embed_dim, final_embed_dim, backbone_channels, ori_spatial_dim)."""

    def __init__(self, p, img_size=224, patch_size=4, in_chans=3, embed_dim=96, depths=(2, 2, 6, 2),
                 num_heads=(3, 6, 12, 24), window_size=7, mlp_ratio=4., qkv_bias=True, ape=False, **_unused):
        super().__init__()
        if ape:
            raise NotImplementedError("mtt_b200 TaskPrompterSwin: absolute position embedding is not supported")
        if isinstance(img_size, int):
            img_size = (img_size, img_size)
        tasks = list(p.TASKS.NAMES)
        self.p = p
        self.num_layers = len(depths)
        self.embed_dim, self.depths, self.heads, self.window_size = embed_dim, tuple(depths), tuple(num_heads), window_size
        self.patch_size, self.in_chans = patch_size, in_chans
        self.img_ds_ratio = p.img_ds_ratio
        self.full_img_size = tuple(img_size)
        self.resolution = [[int(s[0] * self.img_ds_ratio), int(s[1] * self.img_ds_ratio)] for s in p.ori_spatial_dim]
        ds_size = [int(s * self.img_ds_ratio) for s in img_size]                         # TP:590
        self.patch_embed = SwinPatchEmbed(ds_size, patch_size, in_chans, embed_dim)
        self.patch_grid = self.patch_embed.grid_size
        for i in range(self.num_layers - 1):              # PatchMerging halves each map (TP taskprompter_swin.py:438
            gh, gw = self.patch_grid[0] // 2 ** i, self.patch_grid[1] // 2 ** i     # asserts "x size (H*W) are not even")
            if gh % 2 or gw % 2:
                raise ValueError(f"TaskPrompterSwin: the stage-{i} token map {gh} x {gw} (image {tuple(img_size)} x ratio "
                                 f"{self.img_ds_ratio} / patch {patch_size}) must be even on both axes for PatchMerging; the "
                                 "reference asserts the same")
        cnh = int(round(math.sqrt(p.chan_nheads)))
        for i in range(self.num_layers):                  # the channel gate of level i is a cnh x cnh grid of windows over its map
            gh, gw = self.patch_grid[0] // 2 ** i, self.patch_grid[1] // 2 ** i     # (TP taskprompter_swin.py:738-763)
            if cnh * cnh != p.chan_nheads or gh % cnh or gw % cnh:
                raise ValueError(f"TaskPrompterSwin: chan_nheads={p.chan_nheads} must be a perfect square whose root divides "
                                 f"every level's token map (level {i}: {gh} x {gw}); the reference fails on such sizes too")
        assert p.prompt_len == 1, "prompt_len != 1 is unsupported (as in the reference's channel branch)"
        self.prompts_len = len(tasks) * p.prompt_len
        self.task_prompts = nn.Parameter(torch.ones(self.prompts_len, embed_dim))
        _trunc_normal_(self.task_prompts, mean=1., std=1.)
        Lv, f = p.level_embed_dim, p.final_embed_dim
        self.fea_fuse, self.fea_decode_spa, self.fea_decode_chan = nn.ModuleList(), nn.ModuleList(), nn.ModuleList()
        for il in range(self.num_layers):
            cur = p.backbone_channels[il]
            self.fea_fuse.append(nn.ModuleDict({t: nn.Sequential(
                nn.Conv2d(Lv * 2, f, 1), nn.Conv2d(f, f, 3, padding=1), nn.BatchNorm2d(f), nn.GELU(),
                nn.Conv2d(f, f, 3, padding=1)) for t in tasks}))
            self.fea_decode_spa.append(nn.ModuleDict({t: nn.Sequential(nn.Conv2d(cur, Lv, 1)) for t in tasks}))
            self.fea_decode_chan.append(nn.ModuleDict({t: nn.Sequential(nn.Conv2d(cur, Lv, 1)) for t in tasks}))
        # TP:635: no multi-scale fusion for '3ddet', whose head takes the 4 level maps as they are
        self.multi_scale_fuse = nn.ModuleDict({t: nn.Conv2d(f, f, 3, padding=1) for t in tasks if t != DET})
        self.layers = nn.Sequential(*[
            BasicLayer(i == self.num_layers - 1, p, embed_dim * 2 ** i,
                       (self.patch_grid[0] // 2 ** i, self.patch_grid[1] // 2 ** i), depths[i], num_heads[i], window_size,
                       mlp_ratio, qkv_bias, downsample=i < self.num_layers - 1) for i in range(self.num_layers)])
        self.norm = nn.LayerNorm(embed_dim * 2 ** (self.num_layers - 1))
        for m in self.modules():
            if isinstance(m, nn.Linear):
                _trunc_normal_(m.weight, std=.02)
                if m.bias is not None:
                    nn.init.zeros_(m.bias)

    nsplit = PARITY
    use_graph = False

    def forward(self, x):
        """TP:674-718: ({task: [B, final_embed_dim, 2 h0, 2 w0]} after the multi-scale fusion for the 2D tasks, for
        '3ddet' the list of the 4 level maps [B, final_embed_dim, h_l, w_l]; info = {}). Outputs are fresh tensors."""
        _check_input(self, x)
        tasks = list(self.p.TASKS.NAMES)
        pl = _plan_for(self, (x.shape[0], x.device, self.nsplit, "backbone"), lambda: _SwinPlan(
            self, None, tasks, None, x.shape[0], x.device, self.nsplit, mode="backbone"))
        out = pl.run(x, graph=self.use_graph)
        return {t: [m.clone() for m in v] if t == DET else v.clone() for t, v in out.items()}, {}


# --------------------------------------------------------------------------------------------
# packed weights
# --------------------------------------------------------------------------------------------
def _pack_swin_block(blk, device, ns):
    def build():
        f = lambda t: _f32(t, device)
        w = SimpleNamespace()
        w.n1w, w.n1b, w.n2w, w.n2b = f(blk.norm1.weight), f(blk.norm1.bias), f(blk.norm2.weight), f(blk.norm2.bias)
        w.eps = blk.norm1.eps
        w.qkv, w.qkv_b = _lin(blk.attn.qkv, device, ns)
        w.proj, w.proj_b = _lin(blk.attn.proj, device, ns)
        ws = blk.window_size
        L = ws * ws
        idx = blk.attn.relative_position_index.reshape(-1).to(device)
        # bias[h, query, key] (TP:193-195) and the shift mask [nW, query, key], both stored TRANSPOSED for the kernel
        w.biasT = f(blk.attn.relative_position_bias_table)[idx].reshape(L, L, blk.num_heads).permute(2, 1, 0).contiguous()
        w.maskT = f(blk.attn_mask).transpose(1, 2).contiguous() if blk.attn_mask is not None else None
        w.fc1, w.fc1_b = _lin(blk.mlp.fc1, device, ns)
        w.fc2, w.fc2_b = _lin(blk.mlp.fc2, device, ns)
        w.cq, w.cq_b = _lin(blk.chan_q, device, ns)
        w.ckv, w.ckv_b = _lin(blk.chan_kv, device, ns)
        w.tt, w.tt_b = _lin(blk.token_trans, device, ns)
        w.last = blk.LAST_BLOCK_FLAG
        if not w.last:
            w.cp, w.cp_b = _lin(blk.chan_proj, device, ns)
            w.tt1, w.tt1_b = _lin(blk.token_trans1, device, ns)
        return w
    return _cached(blk, ("pack", device, ns), build)


def _pack_merge(dsm, device, ns):
    def build():
        f = lambda t: _f32(t, device)
        w = SimpleNamespace()
        w.red, _ = _lin(dsm.reduction, device, ns)
        w.nw, w.nb, w.eps = f(dsm.norm.weight), f(dsm.norm.bias), dsm.norm.eps
        w.pca = f(dsm.process_chan_attn.weight)                                            # [2C, C] fp32 (small kernel)
        w.tpu, _ = _lin(dsm.task_prompts_up, device, ns)
        w.ds_w, w.ds_b = f(dsm.spa_attn_ds.weight), f(dsm.spa_attn_ds.bias)               # [HT, HT, 3, 3]
        return w
    return _cached(dsm, ("pack", device, ns), build)


def _pack_swin_decoder(bb, tasks, device, ns):
    """levels[il][ti] for every task; msf[k] for the k-th 2D task (the tasks other than '3ddet')."""
    def build():
        W = SimpleNamespace()
        W.levels = [[_pack_fuse(bb, il, t, device, ns) for t in tasks] for il in range(bb.num_layers)]
        W.msf = [ops.pack_conv_weight(_f32(bb.multi_scale_fuse[t].weight, device), bb.multi_scale_fuse[t].bias, None, ns)
                 for t in tasks if t != DET]
        return W
    return _cached(bb, ("decoder", device, ns, tuple(tasks)), build)


# --------------------------------------------------------------------------------------------
# the fused forward
# --------------------------------------------------------------------------------------------
def chan_kv_chunks(rows, ce, L):
    """K chunks of chan_kv, Linear(H*W -> 2 ce) over `rows` = B*C rows: few output tiles, very long K. K is split so that
    about one wave of 148 CTAs is busy (K chunks are multiples of 64, at least 512 columns each). 148 is the B200's SM
    count (the H100 has 132); the chunk count sets the order of the fp32 summation, so a retune changes the results in
    the last bits."""
    tiles = -(-rows // 128) * -(-(2 * ce) // 128)
    return max(1, min(32, 148 // tiles, L // 512))


class _StageSpace:
    """Activations of one Swin stage for one batch size: the token map x [B*L, C] and prompts p [B*T, C] its blocks update
    in place, their intermediates, the prompt-row logit maps in the gating layout logits [B, heads, T, T + L] and the
    channel logits rc [B, T, C, nh, nw] of the last block, and (merge) the PatchMerging scratch and its down-sampled
    maps logits_ds / rc_up. Shared by the blocks of a stage; the buffers only the blocks use are there when blk (a block of
    the stage: window, MLP and channel-attention sizes) is given."""

    def __init__(self, C, res, heads, B, T, chan_nheads, device, ns, streams, blk=None, merge=False):
        S = lambda r, c, **kw: ops.Split(r, c, device, ns, **kw)
        z = lambda *s: torch.zeros(*s, device=device, dtype=torch.float32)
        self.B, self.T, self.ns, self.streams = B, T, ns, streams
        self.nh = self.nw = int(round(math.sqrt(chan_nheads)))
        self.C, self.heads = C, heads
        self.H, self.W = res
        self.L = L = self.H * self.W
        self.x = z(B * L, C)
        self.p = z(B * T, C)
        self.ps = S(B * T, C)
        self.logits = z(B, heads, T, T + L)                 # prompt-row logits in the gating kernel's layout
        self.rc = z(B, T, C, self.nh, self.nw)
        if blk is not None:
            self.ce = ce = blk.chan_q.in_features
            self.ws = ws = blk.window_size
            self.Hp, self.Wp = blk.padded
            self.nW = nW = (self.Hp // ws) * (self.Wp // ws)
            self.wl = wl = ws * ws
            self.rows_w = rows_w = B * nW * (T + wl)
            self.xn32, self.pn32 = z(B * L, C), z(B * T, C)
            self.chan_ps = S(B * T, ce)
            self.sw = S(rows_w, C)
            self.qkv = S(rows_w, 3 * C)
            self.ao = S(rows_w, C)
            self.raw = z(B * nW, heads, T, wl)
            self.o32 = z(rows_w, C)
            self.xa32 = z(B * L, C)
            self.q32 = z(B * T, ce)
            self.xat = S(B * C, L, zero=True)
            self.kv32 = z(B * C, 2 * ce)
            self.kchunks = chan_kv_chunks(B * C, ce, L)
            self.kv_part = z(self.kchunks, B * C, 2 * ce) if self.kchunks > 1 else None
            self.co32, self.cos = z(B * T, ce), S(B * T, ce)
            self.t1 = S(B * T, ce)
            hid = blk.mlp.fc1.out_features
            self.ws_mlp = ops.workspace(ops.workspace_bytes(ops.OP_LN_MLP_RESIDUAL, rows=B * L, Cdim=C, hidden=hid,
                                                            nsplit=ns), device)
            self.ws_mlp_p = ops.workspace(ops.workspace_bytes(ops.OP_LN_MLP_RESIDUAL, rows=B * T, Cdim=C, hidden=hid,
                                                              nsplit=ns), device)
        if merge:
            self.m32 = z(B * L // 4, 4 * C)
            self.ms = S(B * L // 4, 4 * C)
            self.logits_ds = z(B, heads, T, T + L // 4)
            self.rc_up = z(B, T, 2 * C, self.nh, self.nw)


def _launch_swin_block(s, w, shift, spa=None):
    """One SwinTransformerBlock with task prompts (TP:310-405) on the stage space s: s.x [B*L, C] / s.p [B*T, C] are
    updated in place, s.logits and s.rc receive the block's raw_spa_attn / raw_chan_attn. The last block of the model
    (w.last) leaves s.p as it is (the plan reads no prompts after it); spa: zeroed [B*T, C] that then receives the
    window-averaged prompt outputs, which the reference returns as that block's task_prompts (TP:344, :399-405)."""
    B, T, C, ce = s.B, s.T, s.C, s.ce
    ops.layernorm(s.x, w.n1w, w.n1b, w.eps, out_f32=s.xn32)                                    # :322
    ops.layernorm(s.p, w.n1w, w.n1b, w.eps, out_f32=s.pn32)                                    # :317
    ops.split_f32(s.p, s.ns, out=s.ps)
    ops.gemm(s.ps, w.tt, bias=w.tt_b, out_split=s.chan_ps)                                     # :319 token_trans
    ops.swin_window_gather(s.xn32, s.pn32, s.sw, B=B, H=s.H, W=s.W, Cdim=C, T=T, ws=s.ws, shift=shift)   # :326-340
    ops.gemm(s.sw, w.qkv, bias=w.qkv_b, out_split=s.qkv)                                       # :183
    ops.swin_window_attention(s.qkv, s.ao, s.raw, w.biasT, w.maskT, BW=B * s.nW, nW=s.nW, T=T, L=s.wl,
                              heads=s.heads, scale=(C // s.heads) ** -0.5)                      # :185-206
    ops.gemm(s.ao, w.proj, bias=w.proj_b, out_f32=s.o32)                                       # :207
    spa_out = w.last and spa is not None
    ops.swin_window_scatter(s.o32, s.raw, s.xa32, s.x, spa if spa_out else s.p, s.logits, B=B, H=s.H, W=s.W, Cdim=C,
                            T=T, ws=s.ws, shift=shift, heads=s.heads, last=w.last and not spa_out)  # :210, :343-360, :399
    # The prompt path -- channel attention between the prompts and the channels of the attention output (:372-396),
    # then the prompt update and the prompts' own MLP (:403-404) -- is a chain of small launches on B*T rows that
    # only needs xa: it runs on a side stream next to the MLP of the B*H*W patch rows (:400) and joins at the end.
    def prompt_path():
        ops.gemm(s.chan_ps, w.cq, bias=w.cq_b, out_f32=s.q32)
        ops.transpose_split(s.xa32, s.xat, B=B, L=s.L, Cdim=C)
        if s.kchunks > 1:   # C rows x (H*W) columns: a handful of M tiles with thousands of K blocks -> split K
            ops.gemm_splitk(s.xat, w.ckv, s.kv_part, s.kv32, K=s.L, bias=w.ckv_b, chunks=s.kchunks)
        else:
            ops.gemm(s.xat, w.ckv, K=s.L, bias=w.ckv_b, out_f32=s.kv32)
        ops.swin_chan_attention(s.q32, s.kv32, s.co32, s.cos, s.rc, B=B, T=T, Cdim=C, ce=ce, nh=s.nh, nw=s.nw)
        if not w.last:
            ops.gemm(s.cos, w.cp, bias=w.cp_b, out_split=s.t1)                                 # chan_proj
            ops.gemm(s.t1, w.tt1, bias=w.tt1_b, residual=s.p, out_f32=s.p)                     # token_trans1; :403
            ops.ln_mlp_residual(s.p, w.n2w, w.n2b, w.eps, w.fc1, w.fc1_b, w.fc2, w.fc2_b, s.ws_mlp_p)   # :404

    s.streams.par([prompt_path,
                   lambda: ops.ln_mlp_residual(s.x, w.n2w, w.n2b, w.eps, w.fc1, w.fc1_b, w.fc2, w.fc2_b, s.ws_mlp)])


def _launch_merge(s, w, x_out, p_out):
    """PatchMerging (TP:430-472) on the stage space s: s.x, s.p, s.logits, s.rc -> x_out [B*L/4, 2C], p_out [B*T, 2C]
    (fp32), s.logits_ds [B, heads, T, T + L/4] and s.rc_up [B, T, 2C, nh, nw]."""
    B, T = s.B, s.T
    ops.swin_merge_gather(s.x, s.m32, B=B, H=s.H, W=s.W, Cdim=s.C)                             # :441-447
    ops.layernorm(s.m32, w.nw, w.nb, w.eps, out_split=s.ms)
    ops.gemm(s.ms, w.red, out_f32=x_out)                                                       # :449-450
    ops.conv3x3_s2_maps(s.logits, w.ds_w, w.ds_b, s.logits_ds, B=B, Cin=s.heads * T, H=s.H, W=s.W,
                        in_stride=T + s.L, in_offset=T, out_stride=T + s.L // 4, out_offset=T)  # :458-460
    ops.swin_chan_up(s.rc, w.pca, s.rc_up, BT=B * T, Cdim=s.C, nwin=s.nh * s.nw)               # :463-466
    ops.split_f32(s.p, s.ns, out=s.ps)
    ops.gemm(s.ps, w.tpu, out_f32=p_out)                                                       # :469


# --------------------------------------------------------------------------------------------
# the sub-module forwards: the plan's block and merge launches on a workspace sized for the call
# --------------------------------------------------------------------------------------------
def _check_tokens(mod, x, prompts, C):
    """(B, T) of x [B, H*W, C] and task_prompts [B, T, C] for a module over the map `mod.input_resolution`."""
    H, W = mod.input_resolution if hasattr(mod, "input_resolution") else mod.blocks[0].input_resolution
    if x.dim() != 3 or tuple(x.shape[1:]) != (H * W, C) or prompts.dim() != 3 or prompts.shape[0] != x.shape[0] \
            or prompts.shape[2] != C or prompts.shape[1] < 1:
        raise ValueError(f"{type(mod).__name__}: expected x [B,{H * W},{C}] and task_prompts [B,T,{C}], got "
                         f"{tuple(x.shape)} and {tuple(prompts.shape)}")
    return x.shape[0], prompts.shape[1]


def _module_space(mod, blk, B, T, dev, ns):
    """The stage space of a sub-module forward, cached on the module per (device, nsplit, B, T): with the block buffers
    when blk is given, with the PatchMerging scratch when the module is or has a PatchMerging."""
    merge = isinstance(mod, PatchMerging) or getattr(mod, "downsample", None) is not None
    src = blk if blk is not None else mod
    heads = blk.num_heads if blk is not None else mod.num_heads
    chan_nheads = src.chan_nheads
    return _cached(mod, ("space", dev, ns, B, T), lambda: _StageSpace(
        src.dim, src.input_resolution, heads, B, T, chan_nheads, dev, ns, _Streams(dev, 2), blk=blk, merge=merge),
        versioned=False)


def _load(s, x, prompts):
    s.x.copy_(x.reshape(s.B * s.L, s.C))
    s.p.copy_(prompts.reshape(s.B * s.T, s.C))


def _attn_out(s, logits, rc, H, W):
    """[raw_spa_attn [B, heads, T, H, W], raw_chan_attn] (fresh) from the gating-layout logits and the channel logits."""
    maps = torch.empty(s.B, s.heads, s.T, H, W, device=logits.device, dtype=torch.float32)
    ops.swin_logit_maps(logits, maps, T=s.T, to_maps=True)
    return [maps, rc.clone()]


def _launch_merge_out(s, w):
    """PatchMerging on s into fresh tensors: (x [B, L/4, 2C], task_prompts [B, T, 2C], attn_weight)."""
    B, T, C = s.B, s.T, s.C
    x = torch.empty(B, s.L // 4, 2 * C, device=s.x.device, dtype=torch.float32)
    p = torch.empty(B, T, 2 * C, device=s.x.device, dtype=torch.float32)
    _launch_merge(s, w, x.view(B * s.L // 4, 2 * C), p.view(B * T, 2 * C))
    return x, p, _attn_out(s, s.logits_ds, s.rc_up, s.H // 2, s.W // 2)


class _SwinPlan(Plan):
    """Geometry, workspace and launch sequence of one TaskPrompterSwin wrapper forward. mode: "full" = wrapper forward
    (logits at the output size), "postproc" = predict() (get_output fused into the final resize, same launch count),
    "backbone" = TaskPrompterSwin.forward alone (the task features, NCHW). In every mode a '3ddet' task yields the list
    of its 4 level maps [B, f, h_l, w_l] (NCHW fp32, static buffers): the wrapper hands them to the detection head."""

    def __init__(self, bb, heads, tasks, target, B, device, nsplit, mode="full"):
        super().__init__((bb, heads), B, device, nsplit, max(len(tasks), 2))
        if mode not in ("full", "postproc", "backbone"):
            raise NotImplementedError(f"mtt_b200 TaskPrompterSwin: no {mode!r} plan (the wrapper forward, predict() "
                                      "and the backbone forward are built)")
        device = self.dev
        self.bb, self.heads, self.tasks, self.target, self.mode = bb, heads, list(tasks), target, mode
        self.postproc = mode == "postproc"
        self.T = T = len(self.tasks)
        self.det = self.tasks.index(DET) if DET in self.tasks else None
        self.t2 = [t for t in self.tasks if t != DET]          # the 2D tasks: multi-scale fusion and a dense head
        self.i2 = [self.tasks.index(t) for t in self.t2]       # ... and their rows among the T prompts
        T2 = len(self.t2)
        p = bb.p
        self.ce = ce = p.chan_embed_dim
        self.r = int(round(math.sqrt(ce)))
        self.nh = self.nw = int(round(math.sqrt(p.chan_nheads)))
        assert self.r * self.r == ce and self.r % self.nh == 0
        self.Lv, self.f = p.level_embed_dim, p.final_embed_dim
        self.Lv_pad, self.f_ld = ops.round_up(self.Lv, 8), ops.round_up(self.f, 8)
        self.img, self.in_chans = bb.full_img_size, bb.in_chans
        self.ds_img = tuple(bb.patch_embed.img_size)
        ns = nsplit
        S = lambda r, c, **kw: ops.Split(r, c, device, ns, **kw)
        z = lambda *s: torch.zeros(*s, device=device, dtype=torch.float32)
        with _dev_ctx(device):
            self._repack()
            E, patch = bb.embed_dim, bb.patch_size
            gh, gw = bb.patch_grid
            self.img_ds = z(B, bb.in_chans, *self.ds_img) if self.ds_img != self.img else None
            self.cols = S(B * gh * gw, patch * patch * bb.in_chans)
            self.x0 = z(B * gh * gw, E)
            # ---- per stage
            self.st = [_StageSpace(b0.dim, b0.input_resolution, b0.num_heads, B, T, p.chan_nheads, device, ns, self.streams,
                                   blk=b0, merge=layer.downsample is not None)
                       for layer, b0 in ((layer, layer.blocks[0]) for layer in bb.layers)]
            last = self.st[-1]
            self.xfin = z(B * last.L, last.C)
            # ---- decoder levels: level il lives on the map AFTER stage il's merging (the last level: the final norm)
            self.lv = []
            for il in range(bb.num_layers):
                h, w = bb.resolution[il]
                Cl = p.backbone_channels[il]
                d = SimpleNamespace(h=h, w=w, P=h * w, C=Cl, heads=self.st[il].heads)
                d.ws_gate = ops.workspace(ops.workspace_bytes(ops.OP_GATED_CONV1X1, rows=B * d.P, Cdim=Cl, nsplit=ns, T=T),
                                          device)
                d.cat = [S(B * d.P, 2 * self.Lv_pad, zero=True) for _ in range(T)]
                d.g32 = [z(B * d.P, self.f_ld) for _ in range(T2)]
                d.up = [S(B * 4 * d.P, self.f, zero=True) for _ in range(T2)]
                d.mid = [S(B * 4 * d.P, self.f, zero=True) for _ in range(T2)]
                d.out32 = None if il == 0 else [z(B * 4 * d.P, self.f_ld) for _ in range(T2)]
                if self.det is not None:         # fea_fuse of '3ddet' on the level's own map (TP:741, :764: no x2)
                    d.det0, d.det1 = S(B * d.P, self.f, zero=True), S(B * d.P, self.f, zero=True)
                    d.det32 = z(B * d.P, self.f_ld)
                self.lv.append(d)
            h0, w0 = 2 * self.lv[0].h, 2 * self.lv[0].w
            self.fh, self.fw = h0, w0
            self.acc = [z(B * h0 * w0, self.f_ld) for _ in range(T2)]
            self.accs = [S(B * h0 * w0, self.f, zero=True) for _ in range(T2)]
            oh, ow = self.target if self.target is not None else self.img
            self.out_hw = (oh, ow)
            self.det_out = [z(B, self.f, d.h, d.w) for d in self.lv] if self.det is not None else None
            if mode == "backbone":
                self.hs = None
                self.fea32 = [z(B * h0 * w0, self.f_ld) for _ in range(T2)]
                self.out = {t: z(B, self.f, h0, w0) for t in self.t2}
                return
            self.hs = [_HeadSpace(hw, B, h0, w0, device, ns) for hw in self.Wh]
            if self.postproc:
                self.out = _predict_outputs(self.t2, B, (oh, ow), device)
            else:
                self.out = {t: z(B, hw.n_out, oh, ow) for t, hw in zip(self.t2, self.Wh)}

    def _pack(self):
        bb, dev, ns = self.bb, self.dev, self.ns
        self.Ws = _pack_stem(bb, dev, ns)
        self.Wb = [[_pack_swin_block(blk, dev, ns) for blk in layer.blocks] for layer in bb.layers]
        self.Wm = [_pack_merge(layer.downsample, dev, ns) if layer.downsample is not None else None for layer in bb.layers]
        self.Wd = _pack_swin_decoder(bb, self.tasks, dev, ns)
        # the 2D heads; the '3ddet' head (FCOS3D) is the caller's module and runs after the plan (TaskPrompterWrapper)
        self.Wh = [_pack_head(self.heads[t], dev, ns) for t in self.t2] if self.mode != "backbone" else None

    def _result(self):
        return {t: list(self.det_out) if t == DET else self.out[t] for t in self.tasks}

    # ------------------------------------------------------------------------------------------
    def _level(self, il, x_src, logits, rc):
        """cal_task_feature (TP:721-774) at level il on X = x_src [B*P, C]."""
        B, T, d = self.B, self.T, self.lv[il]
        lvw = self.Wd.levels[il]
        ops.gated_conv1x1(x_src, d.P, 0, logits, rc,
                          [(tw.spa, tw.spa_b, tw.chan, tw.chan_b, d.cat[ti]) for ti, tw in enumerate(lvw)],
                          self.Lv, self.Lv_pad, d.ws_gate, B=B, T=T, N=T + d.P, H=d.heads, Cdim=d.C, gh=d.h, gw=d.w,
                          nh=self.nh, nw=self.nw)                                                   # :736-751 (1x1 first)
        if self.t2:      # the 2D tasks; k indexes them, ti the task among all T
            two = [(k, d.cat[ti], lvw[ti]) for k, ti in enumerate(self.i2)]
            K2 = range(len(two))
            ops.gemm_grouped([(cat, tw.f0, dict(bias=tw.f0_b, out_f32=d.g32[k][:, :self.f], N=self.f))
                              for k, cat, tw in two])                                              # fea_fuse[0]
            self.streams.par([lambda k=k: ops.bilinear(d.g32[k], self.f_ld, B, d.h, d.w, self.f, 2 * d.h, 2 * d.w,
                                                       out_split=d.up[k]) for k in K2])            # :747-748 (moved)
            ops.gemm_grouped([(d.up[k], tw.f1, dict(N=self.f, K=self.f, bias=tw.f1_b, act=ops.ACT_GELU,
                                                    out_split=d.mid[k], conv=(B, 2 * d.h, 2 * d.w, 3, 1)))
                              for k, _, tw in two])
            dst = self.acc if il == 0 else d.out32
            ops.gemm_grouped([(d.mid[k], tw.f4, dict(N=self.f, K=self.f, bias=tw.f4_b, out_f32=dst[k][:, :self.f],
                                                     conv=(B, 2 * d.h, 2 * d.w, 3, 1))) for k, _, tw in two])
            if il > 0:                                                                              # TP:713-716
                self.streams.par([lambda k=k: ops.bilinear(d.out32[k], self.f_ld, B, 2 * d.h, 2 * d.w, self.f, self.fh,
                                                           self.fw, out_f32=self.acc[k][:, :self.f], accumulate=True)
                                  for k in K2])
        if self.det is not None:
            self._det_level(il)

    def _det_level(self, il):
        """fea_fuse of '3ddet' at level il on the level's own h x w map (TP:741, :764 skip the bilinear x2), written as
        the NCHW level map the detection head takes (TP:709-710)."""
        B, d, f = self.B, self.lv[il], self.f
        tw = self.Wd.levels[il][self.det]
        ops.gemm(d.cat[self.det], tw.f0, bias=tw.f0_b, out_split=d.det0, N=f)                     # fea_fuse[0]
        ops.gemm(d.det0, tw.f1, N=f, K=f, bias=tw.f1_b, act=ops.ACT_GELU, out_split=d.det1,
                 conv=(B, d.h, d.w, 3, 1))                                                          # fea_fuse[1..3]
        ops.gemm(d.det1, tw.f4, N=f, K=f, bias=tw.f4_b, out_f32=d.det32[:, :f], conv=(B, d.h, d.w, 3, 1))   # [4]
        ops.nhwc_to_nchw(d.det32, self.f_ld, B, f, d.h, d.w, self.det_out[il])

    def _fused(self, k, out_split=None, out_f32=None):
        """multi_scale_fuse of the k-th 2D task on the level sum (TP:711-717)."""
        wm, bm = self.Wd.msf[k]
        ops.split_f32(self.acc[k][:, :self.f], self.ns, out=self.accs[k])
        ops.gemm(self.accs[k], wm, N=self.f, K=self.f, bias=bm, out_split=out_split, out_f32=out_f32,
                 conv=(self.B, self.fh, self.fw, 3, 1))

    def _fea_chain(self, k, t):
        self._fused(k, out_f32=self.fea32[k][:, :self.f])
        ops.nhwc_to_nchw(self.fea32[k], self.f_ld, self.B, self.f, self.fh, self.fw, self.out[t])

    def _head_chain(self, ti, t, hw, hs):
        B = self.B
        oh, ow = self.out_hw
        self._fused(ti, out_split=hs.up)                                                            # :717
        _launch_head(hs, hw)
        if self.postproc:
            ops.bilinear_postproc(hs.pred, hs.pred.stride(0), B, hs.ph, hs.pw, hw.n_out, oh, ow,
                                  ops.POSTPROC_KIND[t], self.out[t])                         # wrapper :35 + utils.py:27-63
        else:
            ops.bilinear(hs.pred, hs.pred.stride(0), B, hs.ph, hs.pw, hw.n_out, oh, ow, out_nchw=self.out[t])  # :35

    def _launch(self, img):
        B, T, bb, W = self.B, self.T, self.bb, self.Ws
        if self.img_ds is not None:                                                                 # TP:676-677
            h, w = self.img
            ops.bilinear(img.view(B * bb.in_chans * h * w, 1), 1, B * bb.in_chans, h, w, 1, self.ds_img[0], self.ds_img[1],
                         out_nchw=self.img_ds.view(B * bb.in_chans, 1, *self.ds_img))
            img = self.img_ds
        s0 = self.st[0]
        ops.im2col_patch(img, bb.patch_size, self.cols)
        ops.gemm(self.cols, W.pe_w, bias=W.pe_b, out_f32=self.x0)                                  # TP:679
        ops.layernorm(self.x0, W.pnw, W.pnb, W.pneps, out_f32=s0.x)                                # patch_embed.norm
        ops.broadcast_rows(W.prompts, s0.p, B, T)                                                  # :685
        n_stage = len(self.st)
        for i, s in enumerate(self.st):
            for j, blk in enumerate(bb.layers[i].blocks):
                _launch_swin_block(s, self.Wb[i][j], blk.shift_size)
            if i < n_stage - 1:
                n = self.st[i + 1]
                _launch_merge(s, self.Wm[i], n.x, n.p)                                             # stage i -> i + 1
                self._level(i, n.x, s.logits_ds, s.rc_up)                                          # :702-707
        last = self.st[-1]
        ops.layernorm(last.x, W.nw, W.nb, W.neps, out_f32=self.xfin)                               # :709
        self._level(n_stage - 1, self.xfin, last.logits, last.rc)
        if self.mode == "backbone":
            self.streams.par([lambda k=k, t=t: self._fea_chain(k, t) for k, t in enumerate(self.t2)])
            return
        self.streams.par([lambda ti=ti, t=t, hw=hw, hs=hs: self._head_chain(ti, t, hw, hs)
                          for ti, (t, hw, hs) in enumerate(zip(self.t2, self.Wh, self.hs))])


def build_from_config(cfg, nsplit=PARITY, use_graph=True, det_head=None):
    """cfg: dict as in configs.taskprompter_swin() (mirrors TP/utils/common_config.py:34-41,64-90). A config with the
    '3ddet' task needs det_head: the nn.Module that takes the 4 level maps (the reference's FCOS3DHead,
    utils/common_config.py:52-57, or any stand-in); it runs in PyTorch after the fused forward."""
    from .taskprompter import ConvHead, DEConvHead, TaskPrompterWrapper
    h, w = cfg["img_size"]
    E = cfg["embed_dim"]
    p = SimpleNamespace(TASKS=SimpleNamespace(NAMES=list(cfg["tasks"]), NUM_OUTPUT=dict(cfg["num_output"])),
                        prompt_len=cfg.get("prompt_len", 1), chan_embed_dim=cfg["chan_embed_dim"],
                        chan_nheads=cfg["chan_nheads"], img_ds_ratio=cfg["img_ds_ratio"],
                        level_embed_dim=cfg["level_embed_dim"], final_embed_dim=cfg["f"],
                        backbone_channels=[2 * E, 4 * E, 8 * E, 8 * E],
                        ori_spatial_dim=[[h // st, w // st] for st in STRIDES])
    if "dd_label_map_size" in cfg:
        p.dd_label_map_size = tuple(cfg["dd_label_map_size"])
    bb = TaskPrompterSwin(p, img_size=(h, w), patch_size=cfg["patch"], embed_dim=E, depths=tuple(cfg["depths"]),
                          num_heads=tuple(cfg["heads"]), window_size=cfg["window"])
    head_cls = DEConvHead if cfg.get("head", "conv") == "deconv" else ConvHead
    if DET in cfg["tasks"] and det_head is None:
        raise ValueError("TaskPrompterSwin: the '3ddet' task needs det_head= (the module that takes the 4 level maps, "
                         "e.g. the reference's FCOS3DHead)")
    heads = nn.ModuleDict({t: det_head if t == DET else head_cls(cfg["f"], cfg["num_output"][t]) for t in cfg["tasks"]})
    return TaskPrompterWrapper(p, bb, heads, nsplit=nsplit, use_graph=use_graph)


def accelerate(ref_model, nsplit=PARITY, use_graph=True):
    """Drop-in for a REFERENCE TaskPrompterWrapper around TaskPrompterSwin (two- or three-task). The geometry is read
    from the instance; the backbone and the 2D heads are COPIED (`load_state_dict(ref.state_dict(), strict=True)`), so a
    later in-place update of `ref_model` is not seen -- call `load_state_dict` again. The '3ddet' head (FCOS3DHead) is
    the reference's module itself, SHARED: the library has no kernels for it, it runs in PyTorch on the 4 level maps."""
    from .taskprompter import TaskPrompterWrapper
    bb = ref_model.backbone
    p = bb.p
    if getattr(bb, "ape", False):
        raise NotImplementedError("mtt_b200 TaskPrompterSwin: absolute position embedding is not supported")
    ratio = p.img_ds_ratio
    img = (p.ori_spatial_dim[0][0] * STRIDES[0], p.ori_spatial_dim[0][1] * STRIDES[0])       # common_config.py:37-39
    if [int(s * ratio) for s in img] != list(bb.patch_embed.img_size):
        raise ValueError(f"accelerate: cannot recover the input size from ori_spatial_dim {p.ori_spatial_dim} and the "
                         f"patch embedding's {tuple(bb.patch_embed.img_size)} at ratio {ratio}")
    blk0 = bb.layers[0].blocks[0]
    mine_bb = TaskPrompterSwin(p, img_size=img, patch_size=bb.patch_embed.patch_size[0],
                               in_chans=bb.patch_embed.proj.in_channels, embed_dim=bb.embed_dim,
                               depths=tuple(len(layer.blocks) for layer in bb.layers),
                               num_heads=tuple(layer.blocks[0].num_heads for layer in bb.layers),
                               # stage 0 has the largest map: its window is the configured one unless every stage clips
                               window_size=blk0.window_size, mlp_ratio=bb.mlp_ratio,
                               qkv_bias=blk0.attn.qkv.bias is not None)
    heads = nn.ModuleDict({t: ref_model.heads[t] if t == DET else _mirror_head(t, ref_model.heads[t])
                           for t in ref_model.tasks})
    m = TaskPrompterWrapper(p, mine_bb, heads, nsplit=nsplit, use_graph=use_graph)
    m.load_state_dict(ref_model.state_dict(), strict=True)
    return m.eval()
