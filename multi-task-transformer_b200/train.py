"""The TaskPrompter training step on the library's kernels (SURVEY.md section 8f N1).

Serves the loop of TaskPrompter/utils/train_utils.py:34-51 (forward -> criterion -> backward -> clip_grad_norm_ ->
optimizer.step) under main.py:92-94 (SyncBatchNorm + DistributedDataParallel) for the ViT TaskPrompter with ConvHead
heads:

* the forward runs in TRAIN mode: BatchNorm2d uses batch statistics (summed over ranks when a process group is given =
  SyncBatchNorm) and updates its running statistics, DropPath applies timm 0.5.4's per-sample masks (drawn with
  torch.rand in the reference's call order, so a seeded run sees the reference's masks);
* the backward is a hand-scheduled reverse pass (no autograd graph inside): every contraction is an mtt_gemm /
  mtt_gemm_grouped launch on transposed split operands (dA = dY W, dW = dY^T A), everything else is a kernel of
  csrc/train_ops.cu; the attention backward recomputes P from q, k (nothing of size N^2 is kept from the forward);
* parameters and gradients live in two flat fp32 arenas: gradient buckets are slices of the arena, all-reduced with NCCL
  on a side stream as soon as the reverse pass has finished the layers they cover, and clip + Adam are two launches over
  the arenas (mtt_sumsq, mtt_adam_step).

`TrainStep.step(images, targets)` is the native loop; `TrainStep.apply(images)` is the torch-facing form (one
autograd.Function: `loss.backward()` runs the reverse pass and hands per-parameter gradients to autograd, so the
reference loop's criterion, clip_grad_norm_, optimizer and DDP hooks work unchanged).
`TrainStep.state_dict()` / `load_state_dict()` save and restore the Adam state in torch.optim.Adam's format (the
checkpoint's 'optimizer' entry, train_utils.py:128, main.py:115-135); the model's own state_dict() is the 'model' entry.
Every write the kernels make to parameters or BatchNorm statistics bumps their version counters, so eval forwards of the
model re-pack the trained weights.

Not covered (raise): DEConvHead / Swin / InvPT models, attention or projection dropout (0 in every reference config).
"""
import math

import torch

from . import ops
from .ops import ACT_GELU, ACT_NONE, Split, round_up
from .taskprompter import ConvHead, TaskPrompter, TaskPrompterWrapper, prompt_row_chunks

__all__ = ["TrainStep"]


def _z(*shape, device):
    return torch.zeros(*shape, dtype=torch.float32, device=device)


def _e(*shape, device):
    return torch.empty(*shape, dtype=torch.float32, device=device)


class _Arena:
    """Flat fp32 storage for a list of named tensors (each start aligned to 64 elements); .view[name] has the tensor's
    shape."""

    def __init__(self, named_shapes, device):
        self.offsets, off = {}, 0
        for name, shape in named_shapes:
            n = int(math.prod(shape))
            self.offsets[name] = (off, n, tuple(shape))
            off += round_up(max(n, 1), 64)
        self.flat = _z(off, device=device)
        self.view = {k: self.flat[o:o + n].view(shape) for k, (o, n, shape) in self.offsets.items()}


class TrainStep:
    """One object per (model, batch geometry is taken per call). `model`: mtt_b200 TaskPrompterWrapper (ViT backbone,
    ConvHead heads). After construction the model's parameters are views of `self.params.flat` and their .grad fields
    views of `self.grads.flat`."""

    def __init__(self, model, *, lr=2e-5, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-6, max_norm=10.0, nsplit=2,
                 process_group=None, bucket_mb=64, use_graph=False):
        if not isinstance(model, TaskPrompterWrapper) or not isinstance(model.backbone, TaskPrompter):
            raise NotImplementedError("mtt_b200 TrainStep: only the ViT TaskPrompter is covered (SURVEY.md 8f N1)")
        for t in model.tasks:
            if not isinstance(model.heads[t], ConvHead):
                raise NotImplementedError("mtt_b200 TrainStep: heads must be ConvHead (taskprompter.py:688-698)")
        self.model, self.bb = model, model.backbone
        bb = self.bb
        self.tasks = list(model.tasks)
        self.T = len(self.tasks)
        self.gh, self.gw = bb.resolution
        self.P = self.gh * self.gw
        self.N = self.T + self.P
        self.C, self.H, self.depth, self.patch = bb.embed_dim, bb.num_heads, bb.depth, bb.patch_size
        if self.C // self.H != 64:
            raise NotImplementedError("mtt_b200 TrainStep: head dim must be 64 (mtt_attention)")
        self.select = list(bb.select_list)
        self.e, self.f = bb.p.embed_dim, bb.p.final_embed_dim
        self.f_ld = round_up(self.f, 8)              # row stride of the per-task feature maps (pad columns stay zero)
        self.nh = self.nw = int(round(math.sqrt(bb.chan_nheads)))
        self.use_ctr = bool(bb.p.use_ctr)
        self.target = model.target_size
        self.ns = nsplit
        self.dev = next(model.parameters()).device
        self.pg = process_group
        self.world = torch.distributed.get_world_size(process_group) if process_group is not None else 1
        self.hyper = dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay)
        self.max_norm = max_norm
        self.step_no = 0
        self.drop_path = [float(x) for x in torch.linspace(0, float(getattr(bb, "drop_path_rate", 0.0)), self.depth)]
        self._dp_keep = torch.tensor([1.0 - d for d in self.drop_path if d > 0.0] or [1.0],
                                     dtype=torch.float32).to(self.dev).view(-1, 1, 1)
        # arenas: parameters in the order the reverse pass finishes them LAST -> FIRST is not needed; buckets are cut by
        # layer group below, so keep module order
        named = [(n, p) for n, p in model.named_parameters()]
        self.names = [n for n, _ in named]
        self.params = _Arena([(n, p.shape) for n, p in named], self.dev)
        self.grads = _Arena([(n, p.shape) for n, p in named], self.dev)
        self.m = torch.zeros_like(self.params.flat)
        self.v = torch.zeros_like(self.params.flat)
        with torch.no_grad():
            for n, p in named:
                self.params.view[n].copy_(p.detach().to(self.dev, torch.float32))
                p.data = self.params.view[n]
                p.grad = self.grads.view[n]
        # the arenas and the BatchNorm statistics are written by kernels torch does not see: their version counters (what
        # the packed-weight caches and launch plans key on, plans._version) are bumped by hand after every such write
        self._param_list = [p for _, p in named]
        self._buffer_list = list(model.buffers())
        self.gnorm = _z((), device=self.dev)
        self.comm = torch.cuda.Stream(device=self.dev) if (self.pg is not None and self.dev.type == "cuda") else None
        self.bucket_elems = int(bucket_mb * (1 << 20) // 4)
        self._pending, self._done = [], set()
        self.ctx = None
        # use_graph: step() captures forward + criterion + reverse pass (about 5000 launches) into ONE CUDA graph per input
        # shape and replays it; clip + Adam stay outside (their bias-correction scalars change every step)
        self.use_graph = bool(use_graph) and self.dev.type == "cuda"      # with a process group the NCCL calls are captured too
        self._graph = None
        # stream-K workspace of the step's GEMMs (one: every kernel of the step runs on one compute stream)
        self.sk_ws = ops.streamk_workspace(self.dev) if self.dev.type == "cuda" else None

    # ---- small helpers -------------------------------------------------------------------------------------------------
    def P_(self, name):
        return self.params.view[name]

    def G_(self, name):
        return self.grads.view[name]

    def _pack(self):
        """Split planes of every GEMM weight and of its transpose (weights change every step)."""
        ns, W, WT = self.ns, {}, {}

        def lin(name, w2d=None):
            w = self.P_(name) if w2d is None else w2d
            w = w.reshape(w.shape[0], -1)
            W[name] = ops.pack_weight(w, ns)
            WT[name] = ops.transpose_planes(W[name], R=w.shape[0], Ccols=w.shape[1])
        bbp = "backbone."
        lin(bbp + "patch_embed.proj.weight")
        for i in range(self.depth):
            b = f"{bbp}blocks.{i}."
            for k in ("attn.qkv", "attn.proj", "attn.token_trans", "attn.token_trans1", "mlp.fc1", "mlp.fc2"):
                lin(b + k + ".weight")
        e = self.e
        for il in range(4):
            for t in self.tasks:
                lin(f"{bbp}fea_decode_spa.{il}.{t}.0.weight")
                lin(f"{bbp}fea_decode_chan.{il}.{t}.0.weight")
                n0 = f"{bbp}fea_fuse.{il}.{t}.0.weight"
                w0 = self.P_(n0).reshape(self.f, 2 * e)
                for key, sl in ((n0 + "#s", w0[:, :e]), (n0 + "#c", w0[:, e:])):
                    W[key] = ops.pack_weight(sl, ns)
                    WT[key] = ops.transpose_planes(W[key], R=self.f, Ccols=e)
                n1 = f"{bbp}fea_fuse.{il}.{t}.1.weight"
                W[n1] = ops.pack_conv_weight(self.P_(n1), None, None, ns)[0]
                WT[n1] = ops.pack_conv_weight(self.P_(n1), None, None, ns, transposed=True)[0]     # dgrad operator
                lin(f"{bbp}fea_fuse.{il}.{t}.4.weight")
        for t in self.tasks:
            n1 = f"heads.{t}.mt_proj.0.weight"
            W[n1] = ops.pack_conv_weight(self.P_(n1), None, None, ns)[0]
            WT[n1] = ops.pack_conv_weight(self.P_(n1), None, None, ns, transposed=True)[0]
            lin(f"heads.{t}.linear_pred.weight")
        self.W, self.WT = W, WT

    def _S(self, x, cols=None):
        return ops.split_f32(x, self.ns, cols_pad=round_up(x.shape[1] if cols is None else cols, 8))

    def _gemm(self, a, w, **kw):
        """ops.gemm on the step's (single) compute stream, with the step's stream-K workspace: the weight-gradient GEMMs
        dW = dY^T A have 48 .. 64 tiles of 256 x 256 for 74 SM pairs and a reduction over all B*N rows, exactly the shape
        whose idle pairs the stream-K schedule puts to work (include/mtt_b200.h, mtt_gemm_desc.sk_ws)."""
        ops.gemm(a, w, sk_ws=self.sk_ws, **kw)

    def _mm(self, a, w, *, M=None, N=None, K=None, bias=None, out=None, **kw):
        M = a.rows if M is None else M
        N = w.rows if N is None else N
        if out is None:
            out = _e(M, N, device=self.dev)
        self._gemm(a, w, M=M, N=N, K=K, bias=bias, out_f32=out, **kw)
        return out

    def _gemms(self, calls):
        """[(a, w, kwargs)]: one problem goes through self._gemm (it has the step's stream-K workspace, which a grouped
        launch cannot take), several go out as grouped launches."""
        if len(calls) == 1:
            a, w, kw = calls[0]
            self._gemm(a, w, **kw)
        else:
            _grouped(calls)

    def _wb(self, layer):
        """The _lin_bwd item of the Linear / 1x1 Conv2d `layer`: (dW as [N, K], db, key of its weight in self.WT)."""
        gW = self.G_(layer + ".weight")
        return gW.reshape(gW.shape[0], -1), self.G_(layer + ".bias"), layer + ".weight"

    def _lin_bwd(self, dy, a_s, items, *, M, N, K, dyT=None, aT=None, dy_s=None, dy_rows=None, dx=None,
                 accumulate_dx=False):
        """The adjoint of len(items) problems Y_t = A_t W_t^T + b_t stacked by rows: dy fp32 [T*M, N] (any row stride),
        a_s Split [T*M, K]; items[t] = (dW view [N, K], db view or None, key of W_t in self.WT or None).
        dW_t += dY_t^T A_t and db_t += colsum(dY_t) accumulate. With a key, dA_t = dY_t W_t goes to rows t*M.. of dx (fp32
        [T*M, K]; None: a new tensor; accumulate_dx: added to what dx holds). Returns (dA or None, dyT, dy_s): the
        transposed / split dY can serve a second call on the same dY.
        A caller whose operands are gathered from a wider buffer passes them in: dyT Split [T*N, M]; aT Split [T*K, M], or
        [K, T*M] with the T blocks side by side (im2col3x3_t of a stacked input); dy_s Split [T*M, N]; and dy_rows =
        (in_group, src_group, src_offset), the rows of dY inside dy as ops.split_rows maps them."""
        Tn, dev, ns = len(items), self.dev, self.ns
        if dyT is None:
            dyT = Split(Tn * N, M, dev, ns)
            ops.transpose_split(dy, dyT, B=Tn, L=M, Cdim=N)
        if aT is None:
            aT = ops.transpose_planes(a_s, B=Tn, R=M, Ccols=K)
        stacked = aT.rows == Tn * K
        self._gemms([(dyT, aT, dict(M=N, N=K, K=M, a_row_offset=t * N, w_row_offset=t * K if stacked else 0,
                                    w_col_offset=0 if stacked else t * M, residual=gW, out_f32=gW))
                     for t, (gW, _, _) in enumerate(items)])                                      # dW += dY^T A
        for t, (_, gb, _) in enumerate(items):
            if gb is not None:
                in_group, src_group, src_offset = dy_rows or ((M, M, t * M) if Tn > 1 else (0, 0, 0))
                ops.colsum(dy, gb, accumulate=True, rows=M, in_group=in_group, src_group=src_group, src_offset=src_offset)
        if items[0][2] is None:
            return None, dyT, dy_s
        dy_s = self._S(dy) if dy_s is None else dy_s
        if dx is None:
            dx = _e(Tn * M, K, device=dev)
        self._gemms([(dy_s, self.WT[key], dict(M=M, N=K, K=N, a_row_offset=t * M, out_f32=dx[t * M:(t + 1) * M],
                                               residual=dx[t * M:(t + 1) * M] if accumulate_dx else None))
                     for t, (_, _, key) in enumerate(items)])                                     # dA = dY W
        return dx, dyT, dy_s

    # ---- forward -------------------------------------------------------------------------------------------------------
    def _drop_scales_batched(self, B, u=None):
        """Per block the two row-scale vectors [B*N] of the joint stream (attention / MLP residual), or (None, None) where
        the rate is 0: timm DropPath's per-sample masks (floor(keep + U[0,1)) / keep per sample and residual branch) for ALL
        blocks from one torch.rand call, ~8 launches per step instead of ~20 per block (1.2 ms of launch time at depth 24).
        `u`: the uniforms [blocks with a non-zero rate, 4, B] to use instead of torch.rand."""
        act = [i for i in range(self.depth) if self.drop_path[i] > 0.0]
        out = [(None, None)] * self.depth
        if not act:
            return out
        keep = self._dp_keep        # device tensor made at construction: nothing here may copy from the host (graph capture)
        if u is None:      # (block, [x attn, x mlp, prompts attn, prompts mlp], sample)
            u = torch.rand((len(act), 4, B), dtype=torch.float32, device=self.dev)
        r = torch.floor(keep + u) / keep
        s = torch.empty(len(act), 2, B, self.N, dtype=torch.float32, device=self.dev)    # (block, [attn, mlp], sample, token)
        s[:, :, :, self.T:] = r[:, 0:2, :, None]
        s[:, :, :, :self.T] = r[:, 2:4, :, None]
        for j, i in enumerate(act):
            out[i] = (s[j, 0].reshape(-1), s[j, 1].reshape(-1))
        return out

    def _bn_fwd(self, x, prefix, act, out_split):
        """Train-mode BatchNorm2d `prefix` (+ act) over NHWC rows x -> out_split; returns the saved statistics. The sums
        (sum x, sum x^2) are float64, all-reduced as such with a process group (SyncBatchNorm), so the variance
        sum x^2 / n - mean^2 does not cancel in fp32 when a channel's |mean| >> std."""
        C_ = x.shape[1]
        sums = torch.empty(2 * C_, dtype=torch.float64, device=self.dev)
        ops.bn_stats(x, sums)
        count = x.shape[0]
        if self.pg is not None:
            torch.distributed.all_reduce(sums, group=self.pg)
            count *= self.world
        mr = _e(2 * C_, device=self.dev)
        bn = self.model.get_submodule(prefix)
        ops.bn_finalize(sums, count, bn.eps, bn.momentum if bn.momentum is not None else 0.1, mr, bn.running_mean,
                        bn.running_var)
        bn.num_batches_tracked += 1
        ops.bn_act(x, mr, self.P_(prefix + ".weight"), self.P_(prefix + ".bias"), act, out_split=out_split)
        return mr, count

    def _bn_bwd(self, x, dy, prefix, act, mr, count, dx=None):
        C_ = x.shape[1]
        sums = _e(2 * C_, device=self.dev)
        g, b = self.P_(prefix + ".weight"), self.P_(prefix + ".bias")
        ops.bn_bwd_reduce(x, dy, mr, g, b, act, sums)
        ops.axpy_rows(self.G_(prefix + ".bias").view(1, -1), sums[:C_].view(1, -1), None, self.G_(prefix + ".bias").view(1, -1))
        ops.axpy_rows(self.G_(prefix + ".weight").view(1, -1), sums[C_:].view(1, -1), None,
                      self.G_(prefix + ".weight").view(1, -1))
        if self.pg is not None:
            torch.distributed.all_reduce(sums, group=self.pg)
        if dx is None:
            dx = _e(x.shape[0], C_, device=self.dev)
        ops.bn_bwd_apply(x, dy, mr, g, b, act, sums, count, dx)
        return dx

    def forward(self, img, drop_rand=None):
        """images fp32 [B,3,H,W] -> {task: fp32 [B,n_out,H,W]} in train mode; keeps what the reverse pass needs.
        `drop_rand`: optional list of the uniform [B,1,1] DropPath draws to use instead of torch.rand, in the reference's
        call order (taskprompter.py:273,274,276,277: x attn, x mlp, prompts attn, prompts mlp per block with a non-zero
        rate); tests replay the reference's."""
        dev, ns = self.dev, self.ns
        B = img.shape[0]
        T, P, N, C, H = self.T, self.P, self.N, self.C, self.H
        M = B * N
        img = img.to(dev, torch.float32).contiguous()
        self._pack()
        W = self.W
        cx = self.ctx = dict(B=B, img=img, blocks=[], levels=[], heads=[])
        bbp = "backbone."
        # stem (taskprompter.py:393-397)
        cols = Split(B * P, 3 * self.patch * self.patch, dev, ns)
        ops.im2col_patch(img, self.patch, cols)
        X = _e(M, C, device=dev)
        pos = self.P_(bbp + "pos_embed")[0, 1:]
        self._gemm(cols, W[bbp + "patch_embed.proj.weight"], bias=self.P_(bbp + "patch_embed.proj.bias"), residual=pos,
                 res_row_mod=P, out_f32=X, regroup=(P, N, T))
        ops.broadcast_rows(self.P_(bbp + "task_prompts"), X, B, N)
        n_act = sum(d > 0.0 for d in self.drop_path)
        u = None
        if drop_rand is not None and n_act:
            u = torch.stack([r.reshape(B) for r in drop_rand[:4 * n_act]]).to(dev, torch.float32).view(n_act, 4, B)
        scales = self._drop_scales_batched(B, u)
        acc = _z(T, B * P, self.f_ld, device=dev)
        logits = rc = None
        for i in range(self.depth):
            sel = (i + 1) in self.select
            want = sel or i == self.depth - 1
            X, logits_i, rc_i = self._block_fwd(i, X, B, want, scales[i])
            if want:
                logits, rc = logits_i, rc_i
            if sel:
                il = sum(1 for s in self.select if i >= s - 1) - 1
                self._level_fwd(il, X, logits, rc, acc, B, i)
        xfin = _e(M, C, device=dev)
        ops.layernorm(X, self.P_(bbp + "norm.weight"), self.P_(bbp + "norm.bias"), self.bb.norm.eps, out_f32=xfin)
        cx["final"] = (X, xfin)
        self._level_fwd(3, xfin, logits, rc, acc, B, self.depth - 1)
        oh, ow = self.target if self.target is not None else img.shape[-2:]
        cx["out_hw"] = (oh, ow)
        out = self._heads_fwd(acc, B, oh, ow)
        torch.autograd.graph.increment_version(self._buffer_list)        # running statistics (mtt_bn_finalize)
        return out

    def _block_fwd(self, i, X, B, want, scales):
        dev, ns = self.dev, self.ns
        T, P, N, C, H = self.T, self.P, self.N, self.C, self.H
        M = B * N
        b = f"backbone.blocks.{i}."
        W = self.W
        eps = self.bb.blocks[i].norm1.eps
        xn = Split(M, C, dev, ns)
        ops.layernorm(X, self.P_(b + "norm1.weight"), self.P_(b + "norm1.bias"), eps, out_split=xn)
        qkv = Split(M, 3 * C, dev, ns)
        self._gemm(xn, W[b + "attn.qkv.weight"], bias=self.P_(b + "attn.qkv.bias"), out_split=qkv)
        ao = Split(M, C, dev, ns)
        logits = _e(B, H, T, N, device=dev) if want else None
        ops.attention(qkv, ao, B=B, N=N, H=H, scale=64 ** -0.5, prompt_logits=logits, T=T)
        o = self._mm(ao, W[b + "attn.proj.weight"], bias=self.P_(b + "attn.proj.bias"))
        # channel-prompt path on the prompt rows (taskprompter.py:217-250)
        cp = _e(B * T, P, device=dev)
        cps = Split(B * T, P, dev, ns)
        for b0, nb in prompt_row_chunks(B, T):
            self._gemm(xn, W[b + "attn.token_trans.weight"], M=nb * T, bias=self.P_(b + "attn.token_trans.bias"),
                     a_gather=(T, N), a_row_offset=b0 * N, out_f32=cp, out_split=cps, regroup=(nb * T, nb * T, b0 * T))
        rc = None
        if want:
            rc = _e(B, T, C, self.nh, self.nw, device=dev)
            ops.chan_logits(cp, xn, rc, B=B, N=N, T=T, Cdim=C, gh=self.gh, gw=self.gw, nh=self.nh, nw=self.nw)
        for b0, nb in prompt_row_chunks(B, T):
            self._gemm(cps, W[b + "attn.token_trans1.weight"], M=nb * T, bias=self.P_(b + "attn.token_trans1.bias"),
                     a_row_offset=b0 * T, residual=o, out_f32=o, regroup=(T, N, b0 * N))
        X1 = _e(M, C, device=dev)
        ops.axpy_rows(X, o, scales[0], X1)
        h = Split(M, C, dev, ns)
        ops.layernorm(X1, self.P_(b + "norm2.weight"), self.P_(b + "norm2.bias"), eps, out_split=h)
        pre = self._mm(h, W[b + "mlp.fc1.weight"], bias=self.P_(b + "mlp.fc1.bias"))
        a = ops.act_split(pre, ACT_GELU, nsplit=ns)
        mo = self._mm(a, W[b + "mlp.fc2.weight"], bias=self.P_(b + "mlp.fc2.bias"))
        X2 = _e(M, C, device=dev)
        ops.axpy_rows(X1, mo, scales[1], X2)
        self.ctx["blocks"].append(dict(X=X, xn=xn, qkv=qkv, ao=ao, cp=cp, cps=cps, X1=X1, h=h, pre=pre, scales=scales,
                                       logits=logits, rc=rc, d_logits=None, d_rc=None))
        return X2, logits, rc

    def _level_fwd(self, il, Xsrc, logits, rc, acc, B, blk):
        """cal_task_feature (taskprompter.py:424-487) in train mode. The T tasks' buffers are stacked by rows ([T*B*P, .]) so
        that their identically shaped GEMMs / convolutions run as ONE grouped launch each and the row-wise kernels as one
        batched launch."""
        dev, ns = self.dev, self.ns
        T, P, N, C, H, e, f = self.T, self.P, self.N, self.C, self.H, self.e, self.f
        Mp = B * P
        W = self.W
        bbp = "backbone."
        pf = [f"{bbp}fea_fuse.{il}.{t}." for t in self.tasks]
        ps = [f"{bbp}fea_decode_spa.{il}.{t}.0." for t in self.tasks]
        pcn = [f"{bbp}fea_decode_chan.{il}.{t}.0." for t in self.tasks]
        rows = lambda t: dict(a_row_offset=t * Mp)
        ys, yc = Split(T * Mp, C, dev, ns), Split(T * Mp, C, dev, ns)
        for t in range(T):
            ops.gate_split(Xsrc, N, T, logits, rc, t, ys.rows_view(t * Mp, Mp), yc.rows_view(t * Mp, Mp), B=B, T=T, N=N,
                           H=H, Cdim=C, gh=self.gh, gw=self.gw, nh=self.nh, nw=self.nw)
        s_s, c_s = Split(T * Mp, e, dev, ns), Split(T * Mp, e, dev, ns)
        _grouped([(ys, W[ps[t] + "weight"], dict(M=Mp, bias=self.P_(ps[t] + "bias"), out_split=s_s, out_row_offset=t * Mp,
                                                 **rows(t))) for t in range(T)] +
                 [(yc, W[pcn[t] + "weight"], dict(M=Mp, bias=self.P_(pcn[t] + "bias"), out_split=c_s, out_row_offset=t * Mp,
                                                  **rows(t))) for t in range(T)])
        y0 = _e(T, Mp, f, device=dev)
        y0s = Split(T * Mp, f, dev, ns)
        _grouped([(s_s, W[pf[t] + "0.weight#s"], dict(M=Mp, K=e, bias=self.P_(pf[t] + "0.bias"), out_f32=y0[t], **rows(t)))
                  for t in range(T)])
        _grouped([(c_s, W[pf[t] + "0.weight#c"], dict(M=Mp, K=e, residual=y0[t], out_f32=y0[t], out_split=y0s,
                                                      out_row_offset=t * Mp, **rows(t))) for t in range(T)])
        y1 = _e(T, Mp, f, device=dev)
        _grouped([(y0s, W[pf[t] + "1.weight"], dict(M=Mp, N=f, K=f, bias=self.P_(pf[t] + "1.bias"), out_f32=y1[t],
                                                    conv=(B, self.gh, self.gw, 3, 1), **rows(t))) for t in range(T)])
        y2s = Split(T * Mp, f, dev, ns)
        bn = [self._bn_fwd(y1[t], pf[t] + "2", ACT_GELU, y2s.rows_view(t * Mp, Mp)) for t in range(T)]
        F_ = _z(T, Mp, self.f_ld, device=dev)
        _grouped([(y2s, W[pf[t] + "4.weight"], dict(M=Mp, bias=self.P_(pf[t] + "4.bias"), out_f32=F_[t][:, :f], **rows(t)))
                  for t in range(T)])
        ctrw = per_ctr = None
        if self.use_ctr:
            pc = [f"{bbp}ctr_attn_conv.{il}.{t}." for t in self.tasks]
            # the T tasks' tiny conv parameters side by side: [T,H,H], [T,H], [T,H], [T]
            c0 = torch.stack([self.P_(p + "0.weight").reshape(H, H) for p in pc])
            c0b = torch.stack([self.P_(p + "0.bias") for p in pc])
            c2 = torch.stack([self.P_(p + "2.weight").reshape(H) for p in pc])
            c2b = torch.stack([self.P_(p + "2.bias").reshape(()) for p in pc])
            ctrw = _e(B, T, T, device=dev)
            ops.ctr_weights(logits, c0, c0b, c2, c2b, ctrw, B=B, H=H, T=T, N=N)
            ops.ctr_mix(F_, ctrw, acc, T=T, M=Mp, Cdim=self.f_ld, ld=self.f_ld, rows_per_batch=P, accumulate=True)
            per_ctr = (c0, c0b, c2)
        else:
            ops.axpy_rows(acc.view(T * Mp, -1), F_.view(T * Mp, -1), None, acc.view(T * Mp, -1))
        self.ctx["levels"].append(dict(il=il, Xsrc=Xsrc, blk=blk, F=F_, ys=ys, yc=yc, s_s=s_s, c_s=c_s, y0=y0, y1=y1, y2s=y2s,
                                       bn=bn, ctrw=ctrw, ctr=per_ctr))

    def _heads_fwd(self, acc, B, oh, ow):
        """ConvHead of every task (taskprompter.py:688-698) on its x4 up-sampled feature map, then the resize to the label
        size (taskprompter_wrapper.py:35); the T 3x3 convolutions are one grouped launch."""
        dev, ns, f, T = self.dev, self.ns, self.f, self.T
        h4, w4 = 4 * self.gh, 4 * self.gw
        M4 = B * h4 * w4
        W = self.W
        up = _e(T, M4, f, device=dev)
        ups = Split(T * M4, f, dev, ns)
        for t in range(T):
            ops.bilinear(acc[t], self.f_ld, B, self.gh, self.gw, f, h4, w4, out_f32=up[t], out_split=ups.rows_view(t * M4, M4))
        ph = [f"heads.{t}." for t in self.tasks]
        z = _e(T, M4, f, device=dev)
        _grouped([(ups, W[ph[t] + "mt_proj.0.weight"], dict(M=M4, N=f, K=f, bias=self.P_(ph[t] + "mt_proj.0.bias"), out_f32=z[t],
                                                            conv=(B, h4, w4, 3, 1), a_row_offset=t * M4)) for t in range(T)])
        z2s = Split(T * M4, f, dev, ns)
        bn = [self._bn_fwd(z[t], ph[t] + "mt_proj.1", ACT_GELU, z2s.rows_view(t * M4, M4)) for t in range(T)]
        out, n_outs = {}, []
        for t, name in enumerate(self.tasks):
            n_out = self.P_(ph[t] + "linear_pred.weight").shape[0]
            y = _e(M4, n_out, device=dev)
            self._gemm(z2s, W[ph[t] + "linear_pred.weight"], M=M4, bias=self.P_(ph[t] + "linear_pred.bias"), out_f32=y,
                     a_row_offset=t * M4)
            out[name] = _e(B, n_out, oh, ow, device=dev)
            ops.bilinear(y, n_out, B, h4, w4, n_out, oh, ow, out_nchw=out[name])
            n_outs.append(n_out)
        self.ctx["heads"] = dict(up=up, z=z, z2s=z2s, bn=bn, n_out=n_outs)
        return out

    # ---- backward ------------------------------------------------------------------------------------------------------
    def backward(self, grad_out):
        """grad_out {task: fp32 [B,n_out,H,W]} (d loss / d prediction). Accumulates into the gradient arena."""
        cx, dev = self.ctx, self.dev
        B = cx["B"]
        T, P, N, C, f = self.T, self.P, self.N, self.C, self.f
        M, Mp = B * N, B * P
        dacc = _z(T, Mp, self.f_ld, device=dev)
        self._heads_bwd(grad_out, dacc, B)
        self._bucket_ready("heads.")
        dX = _z(M, C, device=dev)
        # last level reads LN_final(x)
        X, xfin = cx["final"]
        dxfin = _z(M, C, device=dev)
        self._level_bwd(cx["levels"][-1], dacc, dxfin, B)
        bbp = "backbone."
        ops.layernorm_bwd(X, dxfin, self.P_(bbp + "norm.weight"), self.bb.norm.eps, dX, self.G_(bbp + "norm.weight"),
                          self.G_(bbp + "norm.bias"), accumulate_dx=True)
        lv_by_blk = {lv["blk"]: lv for lv in cx["levels"][:-1]}
        for i in reversed(range(self.depth)):
            if i in lv_by_blk:
                self._level_bwd(lv_by_blk[i], dacc, dX, B)
            dX = self._block_bwd(i, dX, B)
            self._bucket_ready(f"backbone.blocks.{i}.")
        # stem
        gpos = self.G_(bbp + "pos_embed").view(-1)
        dXv = dX.view(B, N * C)
        ops.colsum(dXv[:, :T * C], self.G_(bbp + "task_prompts").view(-1), accumulate=True)
        ops.colsum(dXv[:, T * C:], gpos[C:], accumulate=True)
        dXp = Split(Mp, C, dev, self.ns)
        ops.split_rows(dX, dXp, rows=Mp, cols=C, in_group=P, src_group=N, src_offset=T)
        dXpT = ops.transpose_planes(dXp, R=Mp, Ccols=C)
        colsT = ops.im2col_patch_t(cx["img"], self.patch, self.ns)
        pe = bbp + "patch_embed.proj."
        self._lin_bwd(dX, None, [(self.G_(pe + "weight").reshape(C, -1), self.G_(pe + "bias"), None)], M=Mp, N=C,
                      K=colsT.rows, dyT=dXpT, aT=colsT, dy_rows=(P, N, T))
        self._bucket_ready(None)
        if self.comm is not None:                       # the communication stream rejoins (required when the step is captured)
            torch.cuda.current_stream(self.dev).wait_stream(self.comm)
        self.ctx = None

    def _heads_bwd(self, grad_out, dacc, B):
        dev, f, T, ns = self.dev, self.f, self.T, self.ns
        hc = self.ctx["heads"]
        h4, w4 = 4 * self.gh, 4 * self.gw
        M4 = B * h4 * w4
        oh, ow = self.ctx["out_hw"]
        ph = [f"heads.{t}." for t in self.tasks]
        dz2 = _e(T, M4, f, device=dev)
        for t, name in enumerate(self.tasks):
            n_out = hc["n_out"][t]
            g = grad_out[name].to(dev, torch.float32).contiguous()
            dy = _e(M4, n_out, device=dev)
            ops.bilinear_bwd(g, nchw=True, B=B, h=h4, w=w4, Cdim=n_out, H2=oh, W2=ow, dx=dy)
            self._lin_bwd(dy, hc["z2s"].rows_view(t * M4, M4), [self._wb(ph[t] + "linear_pred")], M=M4, N=n_out, K=f,
                          dx=dz2[t])
        dz = _e(T, M4, f, device=dev)
        for t in range(T):
            self._bn_bwd(hc["z"][t], dz2[t], ph[t] + "mt_proj.1", ACT_GELU, *hc["bn"][t], dx=dz[t])
        dup = self._conv3_bwd_group(dz.view(T * M4, f), hc["up"].view(T * M4, f), [p + "mt_proj.0" for p in ph], B, h4, w4, f, f)
        for t in range(T):
            ops.bilinear_bwd(dup[t * M4:(t + 1) * M4], nchw=False, B=B, h=self.gh, w=self.gw, Cdim=f, H2=h4, W2=w4,
                             dx=dacc[t][:, :f])

    def _conv3_bwd_group(self, dy, x32, prefixes, B, h, w, Cin, Cout):
        """3x3 convs (pad 1) of len(prefixes) tasks stacked by rows: dy fp32 [T*Mx, Cout], inputs x32 fp32 [T*Mx, Cin] ->
        dx fp32 [T*Mx, Cin]; dW and db as the linear adjoint over the transposed im2col operand."""
        Tn, Mx, dev, ns = len(prefixes), B * h * w, self.dev, self.ns
        dyT = Split(Tn * Cout, Mx, dev, ns)
        ops.transpose_split(dy, dyT, B=Tn, L=Mx, Cdim=Cout)
        x9T = ops.im2col3x3_t(x32, B=Tn * B, H=h, W=w, Cdim=Cin, nsplit=ns)              # [Cin*9, Tn*Mx]: task t = columns t*Mx ..
        items = [(self.G_(p + ".weight").reshape(Cout, Cin * 9), self.G_(p + ".bias"), None) for p in prefixes]
        if Mx % 8 == 0:
            self._lin_bwd(dy, None, items, M=Mx, N=Cout, K=Cin * 9, dyT=dyT, aT=x9T)
        else:                                             # column offsets must stay 16-byte aligned for TMA: one task at a time
            for t, it in enumerate(items):
                xt = ops.im2col3x3_t(x32[t * Mx:(t + 1) * Mx], B=B, H=h, W=w, Cdim=Cin, nsplit=ns)
                self._lin_bwd(dy, None, [it], M=Mx, N=Cout, K=Cin * 9, dyT=dyT.rows_view(t * Cout, Cout), aT=xt,
                              dy_rows=(Mx, Mx, t * Mx))
        dys = self._S(dy)
        dx = _e(Tn * Mx, Cin, device=dev)
        _grouped([(dys, self.WT[p + ".weight"], dict(M=Mx, N=Cin, K=Cout, out_f32=dx[t * Mx:(t + 1) * Mx],
                                                     conv=(B, h, w, 3, 1), a_row_offset=t * Mx)) for t, p in enumerate(prefixes)])
        return dx

    def _level_bwd(self, lv, dacc, dXsrc, B):
        """Adjoint of _level_fwd: dacc [T, B*P, f_ld] (the same for every level: acc is their sum) -> dXsrc (+=), the logit
        gradients of the block that exported them, parameter gradients."""
        dev = self.dev
        T, P, N, C, H, e, f = self.T, self.P, self.N, self.C, self.H, self.e, self.f
        Mp = B * P
        il = lv["il"]
        bc = self.ctx["blocks"][lv["blk"]]
        if bc["d_logits"] is None:
            bc["d_logits"] = _z(B, H, T, N, device=dev)
            bc["d_rc"] = _z(B, T, C, self.nh, self.nw, device=dev)
        d_logits, d_rc = bc["d_logits"], bc["d_rc"]
        logits, rc = bc["logits"], bc["rc"]
        bbp = "backbone."
        if self.use_ctr:
            c0, c0b, c2 = lv["ctr"]
            g0, g0b, g2, g2b = torch.zeros_like(c0), torch.zeros_like(c0b), torch.zeros_like(c2), _z(T, device=dev)
            ops.ctr_bwd(dacc, lv["F"], logits, c0, c0b, c2, d_logits, g0, g0b, g2, g2b, T=T, M=Mp, Cdim=f, ld=self.f_ld,
                        rows_per_batch=P, B=B, H=H, N=N)
            for ti, t in enumerate(self.tasks):
                p = f"{bbp}ctr_attn_conv.{il}.{t}."
                for name, src in ((p + "0.weight", g0[ti]), (p + "0.bias", g0b[ti]), (p + "2.weight", g2[ti]),
                                  (p + "2.bias", g2b[ti:ti + 1])):
                    gv = self.G_(name).view(1, -1)
                    ops.axpy_rows(gv, src.reshape(1, -1), None, gv)
            dF = _e(T, Mp, self.f_ld, device=dev)
            ops.ctr_mix(dacc, lv["ctrw"].transpose(1, 2).contiguous(), dF, T=T, M=Mp, Cdim=self.f_ld, ld=self.f_ld,
                        rows_per_batch=P, accumulate=False)
        else:
            dF = dacc
        pf = [f"{bbp}fea_fuse.{il}.{t}." for t in self.tasks]
        G = self.G_
        dFv = dF.view(T * Mp, self.f_ld)[:, :f]
        dy2 = self._lin_bwd(dFv, lv["y2s"], [self._wb(p + "4") for p in pf], M=Mp, N=f, K=f)[0]
        dy1 = _e(T, Mp, f, device=dev)
        for t in range(T):
            self._bn_bwd(lv["y1"][t], dy2[t * Mp:(t + 1) * Mp], pf[t] + "2", ACT_GELU, *lv["bn"][t], dx=dy1[t])
        dy0 = self._conv3_bwd_group(dy1.view(T * Mp, f), lv["y0"].view(T * Mp, f), [p + "1" for p in pf], B, self.gh, self.gw, f, f)
        g0 = [G(p + "0.weight").reshape(f, 2 * e) for p in pf]
        ds, dyT, dy0s = self._lin_bwd(dy0, lv["s_s"], [(g0[t][:, :e], G(pf[t] + "0.bias"), pf[t] + "0.weight#s")
                                                       for t in range(T)], M=Mp, N=f, K=e)
        dc = self._lin_bwd(dy0, lv["c_s"], [(g0[t][:, e:], None, pf[t] + "0.weight#c") for t in range(T)], M=Mp, N=f, K=e,
                           dyT=dyT, dy_s=dy0s)[0]
        dys = self._lin_bwd(ds, lv["ys"], [self._wb(f"{bbp}fea_decode_spa.{il}.{t}.0") for t in self.tasks], M=Mp, N=e,
                            K=C)[0]
        dyc = self._lin_bwd(dc, lv["yc"], [self._wb(f"{bbp}fea_decode_chan.{il}.{t}.0") for t in self.tasks], M=Mp, N=e,
                            K=C)[0]
        for t in range(T):
            ops.gate_bwd(lv["Xsrc"], N, T, logits, rc, t, dys[t * Mp:(t + 1) * Mp], dyc[t * Mp:(t + 1) * Mp], dXsrc, d_logits,
                         d_rc, B=B, T=T, N=N, H=H, Cdim=C, gh=self.gh, gw=self.gw, nh=self.nh, nw=self.nw)

    def _block_bwd(self, i, dX2, B):
        dev, ns = self.dev, self.ns
        T, P, N, C, H = self.T, self.P, self.N, self.C, self.H
        M = B * N
        bc = self.ctx["blocks"][i]
        b = f"backbone.blocks.{i}."
        eps = self.bb.blocks[i].norm1.eps
        sa, sm = bc["scales"]
        # MLP branch: X2 = X1 + sm * fc2(gelu(fc1(LN2(X1))))
        if sm is not None:
            dm = _e(M, C, device=dev)
            ops.axpy_rows(None, dX2, sm, dm)
        else:
            dm = dX2
        a = ops.act_split(bc["pre"], ACT_GELU, nsplit=ns)
        da = self._lin_bwd(dm, a, [self._wb(b + "mlp.fc2")], M=M, N=C, K=bc["pre"].shape[1])[0]
        del a
        ops.act_bwd(bc["pre"], da, ACT_GELU, da)
        dh = self._lin_bwd(da, bc["h"], [self._wb(b + "mlp.fc1")], M=M, N=bc["pre"].shape[1], K=C)[0]
        del da
        dX1 = dX2                                                     # residual path; LN2's input gradient is added to it
        ops.layernorm_bwd(bc["X1"], dh, self.P_(b + "norm2.weight"), eps, dX1, self.G_(b + "norm2.weight"),
                          self.G_(b + "norm2.bias"), accumulate_dx=True)
        # attention branch: X1 = X + sa * o
        if sa is not None:
            do = _e(M, C, device=dev)
            ops.axpy_rows(None, dX1, sa, do)
        else:
            do = dX1
        dxn = _z(M, C, device=dev)
        # token_trans1 (prompt rows of o): o_p += cp W1^T + b1
        dop = Split(B * T, C, dev, ns)
        ops.split_rows(do, dop, rows=B * T, cols=C, in_group=T, src_group=N, src_offset=0)
        dopT = ops.transpose_planes(dop, R=B * T, Ccols=C)
        dcp = self._lin_bwd(do, bc["cps"], [self._wb(b + "attn.token_trans1")], M=B * T, N=C, K=P, dyT=dopT, dy_s=dop,
                            dy_rows=(T, N, 0))[0]
        # raw channel logits
        if bc["d_rc"] is not None:
            dcp2 = _e(B * T, P, device=dev)
            ops.chan_logits_bwd(bc["d_rc"], bc["cp"], bc["xn"], dcp2, dxn, B=B, N=N, T=T, Cdim=C, gh=self.gh, gw=self.gw,
                                nh=self.nh, nw=self.nw)
            ops.axpy_rows(dcp, dcp2, None, dcp)
        # token_trans: cp = pn Wt^T + bt (pn = prompt rows of xn)
        tt = b + "attn.token_trans."
        dcps = self._S(dcp)
        dcpT = Split(P, B * T, dev, ns, zero=(B * T) % 8 != 0)
        ops.transpose_split(dcp, dcpT, B=1, L=B * T, Cdim=P)
        pnT = ops.transpose_planes(bc["xn"], B=B, R=T, Ccols=C, in_batch_rows=N, side_by_side=True)   # [C, B*T]
        self._lin_bwd(dcp, None, [(self.G_(tt + "weight"), self.G_(tt + "bias"), None)], M=B * T, N=P, K=C, dyT=dcpT, aT=pnT)
        for b0, nb in prompt_row_chunks(B, T):       # the data gradient is scattered to the prompt rows of dxn, by chunks
            self._gemm(dcps, self.WT[tt + "weight"], M=nb * T, N=C, K=P, a_row_offset=b0 * T, residual=dxn, out_f32=dxn,
                       regroup=(T, N, b0 * N))
        # proj
        dao = self._lin_bwd(do, bc["ao"], [self._wb(b + "attn.proj")], M=M, N=C, K=C)[0]
        # attention
        dqkv = self._attn_bwd(bc, dao, B)
        # qkv
        self._lin_bwd(dqkv, bc["xn"], [self._wb(b + "attn.qkv")], M=M, N=3 * C, K=C, dx=dxn, accumulate_dx=True)
        # LN1
        dX = dX1
        ops.layernorm_bwd(bc["X"], dxn, self.P_(b + "norm1.weight"), eps, dX, self.G_(b + "norm1.weight"),
                          self.G_(b + "norm1.bias"), accumulate_dx=True)
        self.ctx["blocks"][i] = None
        return dX

    def _attn_bwd(self, bc, dao, B):
        """softmax(q k^T / 8) v backward with P recomputed (taskprompter.py:201-210); dao fp32 [B*N, C] -> dqkv fp32
        [B*N, 3C]. Grouped GEMMs over (image, head): S = q k^T, dP = dO v^T, then dV = P^T dO, dQ = dS k, dK = dS^T q."""
        dev, ns = self.dev, self.ns
        T, N, C, H = self.T, self.N, self.C, self.H
        qkv = bc["qkv"]
        Np = round_up(N, 8)
        BH = B * H
        dao_s = self._S(dao)
        S = _e(BH * N, Np, device=dev)
        dP = _e(BH * N, Np, device=dev)
        dqkv = _e(B * N, 3 * C, device=dev)
        calls_s, calls_p = [], []
        for b_ in range(B):
            for h_ in range(H):
                r0 = (b_ * H + h_) * N
                calls_s.append((qkv, qkv, dict(M=N, N=N, K=64, a_row_offset=b_ * N, a_col_offset=h_ * 64,
                                               w_row_offset=b_ * N, w_col_offset=C + h_ * 64, out_f32=S[r0:r0 + N])))
                calls_p.append((dao_s, qkv, dict(M=N, N=N, K=64, a_row_offset=b_ * N, a_col_offset=h_ * 64,
                                                 w_row_offset=b_ * N, w_col_offset=2 * C + h_ * 64,
                                                 out_f32=dP[r0:r0 + N])))
        _grouped(calls_s)
        _grouped(calls_p)
        dS, PT, dST = Split(BH * N, Np, dev, ns), Split(BH * N, Np, dev, ns), Split(BH * N, Np, dev, ns)
        delta = _e(BH * N, device=dev)
        ops.attn_delta(dao, bc["ao"], delta, B=B, N=N, H=H, head_dim=64)
        ops.attn_softmax_bwd(S, dP, delta, BH=BH, N=N, scale=64 ** -0.5, d_raw=bc["d_logits"], T=T, ds=dS, pt=PT, dst=dST)
        del S, dP
        # operands transposed per image: [B][3C][Np] (q^T | k^T | v^T rows) and [B][C][Np] (dO^T)
        qkvT = Split(B * 3 * C, Np, dev, ns)
        ops.transpose_planes(qkv, B=B, R=N, Ccols=3 * C, in_batch_rows=N, out=qkvT)
        daoT = Split(B * C, Np, dev, ns)
        ops.transpose_planes(dao_s, B=B, R=N, Ccols=C, in_batch_rows=N, out=daoT)
        cq, ck, cv = [], [], []
        for b_ in range(B):
            for h_ in range(H):
                r0 = (b_ * H + h_) * N
                rows = dqkv[b_ * N:(b_ + 1) * N]
                cq.append((dS, qkvT, dict(M=N, N=64, K=N, a_row_offset=r0, w_row_offset=b_ * 3 * C + C + h_ * 64,
                                          out_f32=rows[:, h_ * 64:(h_ + 1) * 64])))
                ck.append((dST, qkvT, dict(M=N, N=64, K=N, a_row_offset=r0, w_row_offset=b_ * 3 * C + h_ * 64,
                                           out_f32=rows[:, C + h_ * 64:C + (h_ + 1) * 64])))
                cv.append((PT, daoT, dict(M=N, N=64, K=N, a_row_offset=r0, w_row_offset=b_ * C + h_ * 64,
                                          out_f32=rows[:, 2 * C + h_ * 64:2 * C + (h_ + 1) * 64])))
        _grouped(cq)
        _grouped(ck)
        _grouped(cv)
        return dqkv

    # ---- gradient all-reduce, clip, Adam -------------------------------------------------------------------------------
    def _bucket_ready(self, prefix):
        """Called when the reverse pass has finished every parameter whose name starts with `prefix` (None = the rest):
        their arena range is all-reduced on the communication stream while the reverse pass goes on."""
        if self.pg is None:
            return
        if prefix is None:
            names = [n for n in self.names if n not in self._done]
        else:
            names = [n for n in self.names if n.startswith(prefix) and n not in self._done]
        if not names:
            return
        self._done.update(names)
        for n in names:                                  # per-parameter ranges; _flush merges the adjacent ones
            o, cnt, _ = self.grads.offsets[n]
            self._pending.append((o, o + round_up(max(cnt, 1), 64)))
        # merge into buckets of >= bucket_elems contiguous elements; flush when big enough or at the end
        if prefix is not None and sum(h - l for l, h in self._pending) < self.bucket_elems:
            return
        self._flush()

    def _flush(self):
        ranges, self._pending = sorted(self._pending), []
        merged = []
        for lo, hi in ranges:
            if merged and lo <= merged[-1][1]:
                merged[-1][1] = max(merged[-1][1], hi)
            else:
                merged.append([lo, hi])
        cur = torch.cuda.current_stream(self.dev) if self.comm is not None else None
        for lo, hi in merged:
            buf = self.grads.flat[lo:hi]
            if self.comm is not None:
                self.comm.wait_stream(cur)
                with torch.cuda.stream(self.comm):
                    torch.distributed.all_reduce(buf, group=self.pg)
            else:
                torch.distributed.all_reduce(buf, group=self.pg)

    def zero_grad(self):
        self.grads.flat.zero_()
        self._done = set()
        self._pending = []

    def optimizer_step(self, lr=None):
        """clip_grad_norm_(max_norm, 2) + Adam over the arenas (train_utils.py:49-50); gradients of the ranks are averaged."""
        if self.comm is not None:
            torch.cuda.current_stream(self.dev).wait_stream(self.comm)
        self.step_no += 1
        h = dict(self.hyper)
        if lr is not None:
            h["lr"] = lr
        gs = 1.0 / self.world
        clip = self.max_norm is not None and self.max_norm > 0
        if clip:
            ops.sumsq(self.grads.flat, self.gnorm)
        ops.adam_step(self.params.flat, self.grads.flat, self.m, self.v, step=self.step_no,
                      gnorm_sq=self.gnorm if clip else None, max_norm=self.max_norm or 0.0, grad_scale=gs, **h)
        torch.autograd.graph.increment_version(self._param_list)

    def _moment(self, flat, name):
        """Parameter `name`'s slice of a moment arena (self.m / self.v share the parameter arena's layout)."""
        o, n, shape = self.params.offsets[name]
        return flat[o:o + n].view(shape)

    def state_dict(self):
        """The optimizer state as torch.optim.Adam(model.parameters(), ...).state_dict() has it: one param group (the
        group keys come from a real torch Adam built with self.hyper), parameters indexed in model.parameters() order,
        state[i] = {'step', 'exp_avg', 'exp_avg_sq'} (copies), no state before the first step. With a process group the
        moments are the same on every rank."""
        h = self.hyper
        sd = torch.optim.Adam(self.model.parameters(), lr=h["lr"], betas=h["betas"], eps=h["eps"],
                              weight_decay=h["weight_decay"]).state_dict()
        if self.step_no:
            sd["state"] = {i: {"step": torch.tensor(float(self.step_no)), "exp_avg": self._moment(self.m, n).clone(),
                               "exp_avg_sq": self._moment(self.v, n).clone()} for i, n in enumerate(self.names)}
        return sd

    def load_state_dict(self, sd):
        """Loads an Adam state dict: what state_dict() returns, what torch.optim.Adam writes for this model (torch 1.10
        stores 'step' as an int), or that of a fresh optimizer (empty state = step 0). The moments are copied into the
        arenas in place (a captured step graph stays valid); step count and hyper-parameters come from the group. The
        parameters themselves are the model's: model.load_state_dict() writes them into the arena."""
        groups = sd["param_groups"]
        if len(groups) != 1:
            raise ValueError(f"TrainStep.load_state_dict: {len(groups)} param groups; TrainStep keeps one")
        g = groups[0]
        for k in ("amsgrad", "maximize", "decoupled_weight_decay"):
            if g.get(k, False):
                raise ValueError(f"TrainStep.load_state_dict: '{k}' is set; TrainStep runs plain Adam")
        ids = list(g["params"])
        if len(ids) != len(self.names):
            raise ValueError(f"TrainStep.load_state_dict: {len(ids)} parameters in the group, the model has "
                             f"{len(self.names)}")
        state = sd["state"]
        have = [i for i in ids if i in state]
        if have and len(have) != len(ids):
            raise ValueError(f"TrainStep.load_state_dict: state for {len(have)} of {len(ids)} parameters (TrainStep keeps "
                             "state for all or none)")
        steps = sorted({int(float(state[i]["step"])) for i in have})
        if len(steps) > 1:
            raise ValueError(f"TrainStep.load_state_dict: step counts {steps} differ between parameters (TrainStep "
                             "keeps one)")
        for i, n in zip(ids, self.names):
            shape = self.params.offsets[n][2]
            for k in ("exp_avg", "exp_avg_sq"):
                if have and tuple(state[i][k].shape) != shape:
                    raise ValueError(f"TrainStep.load_state_dict: {k} of parameter {i} ({n}) has shape "
                                     f"{tuple(state[i][k].shape)}, the parameter {shape}")
        with torch.no_grad():
            if have:
                for i, n in zip(ids, self.names):
                    self._moment(self.m, n).copy_(state[i]["exp_avg"])
                    self._moment(self.v, n).copy_(state[i]["exp_avg_sq"])
            else:
                self.m.zero_()
                self.v.zero_()
        self.step_no = steps[0] if steps else 0
        self.hyper = dict(lr=float(g["lr"]), betas=tuple(float(b) for b in g["betas"]), eps=float(g["eps"]),
                          weight_decay=float(g["weight_decay"]))

    def step(self, images, targets, criterion, tasks=None):
        """One iteration of train_utils.py:34-51 with `criterion` = mtt_b200.losses.MultiTaskLoss (device kernels):
        returns the loss dict (device scalars)."""
        if self.use_graph:
            loss = self._graph_fwd_bwd(images, targets, criterion, tasks)
        else:
            loss = self._fwd_bwd(images, targets, criterion, tasks)
        self.optimizer_step()
        return loss

    def _fwd_bwd(self, images, targets, criterion, tasks):
        self.zero_grad()
        out = self.forward(images)
        leaves = {t: o.requires_grad_(True) for t, o in out.items()}
        with torch.enable_grad():
            loss = criterion(leaves, targets, tasks=tasks or self.tasks)
            grads = torch.autograd.grad(loss["total"], [leaves[t] for t in self.tasks])
        self.backward({t: g for t, g in zip(self.tasks, grads)})
        return {k: v.detach() for k, v in loss.items()}

    def _graph_fwd_bwd(self, images, targets, criterion, tasks):
        key = (tuple(images.shape), tuple(sorted((t, tuple(v.shape)) for t, v in targets.items())))
        if self._graph is None or self._graph[0] != key:
            gx = images.to(self.dev, torch.float32).clone()
            gy = {t: v.to(self.dev).clone() for t, v in targets.items()}
            # one eager pass on a side stream before capture (allocator warm-up); it must not count as a training step:
            # the BatchNorm running statistics it touches are restored
            bufs = [b for b in self.model.buffers()]
            keep = [b.clone() for b in bufs]
            side = torch.cuda.Stream(device=self.dev)
            side.wait_stream(torch.cuda.current_stream(self.dev))
            with torch.cuda.stream(side):
                self._fwd_bwd(gx, gy, criterion, tasks)
            torch.cuda.current_stream(self.dev).wait_stream(side)
            with torch.no_grad():
                for b, k in zip(bufs, keep):
                    b.copy_(k)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                loss = self._fwd_bwd(gx, gy, criterion, tasks)
            self._graph = (key, g, gx, gy, loss)
        _, g, gx, gy, loss = self._graph
        gx.copy_(images, non_blocking=True)
        for t, v in targets.items():
            gy[t].copy_(v, non_blocking=True)
        g.replay()
        torch.autograd.graph.increment_version(self._buffer_list)        # the replayed forward's running statistics
        return loss

    def apply(self, images):
        """Torch-facing forward: {task: prediction} attached to autograd; .backward() of any loss built on them runs the
        reverse pass and delivers per-parameter gradients through autograd (so DDP hooks, clip_grad_norm_ and torch
        optimizers of the reference loop apply)."""
        params = [p for _, p in self.model.named_parameters()]
        outs = _StepFn.apply(self, images, *params)
        return {t: o for t, o in zip(self.tasks, outs)}


def _grouped(calls, limit=32):
    for i in range(0, len(calls), limit):
        ops.gemm_grouped(calls[i:i + limit])


class _StepFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, ts, images, *params):
        ts.zero_grad()
        out = ts.forward(images)
        ctx.ts = ts
        return tuple(out[t] for t in ts.tasks)

    @staticmethod
    def backward(ctx, *gouts):
        ts = ctx.ts
        ts.backward({t: g for t, g in zip(ts.tasks, gouts)})
        grads = tuple(ts.G_(n).clone() for n in ts.names)
        ts.grads.flat.zero_()          # the parameters' .grad fields ARE the arena: autograd adds the clones into it
        return (None, None) + grads
