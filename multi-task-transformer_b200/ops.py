"""Tensor-level wrappers over the C ABI (include/mtt_b200.h).

PyTorch is used for device memory and streams only: every function here enqueues one library
kernel on ``torch.cuda.current_stream()`` and returns. Nothing in this module computes with torch
ops on the hot path.
"""
import ctypes as C

import torch

from . import lib as _L

ACT_NONE, ACT_GELU, ACT_RELU = _L.ACT_NONE, _L.ACT_GELU, _L.ACT_RELU
OP_LN_QKV, OP_ATTN_FWD, OP_PROJ_RESIDUAL, OP_LN_MLP_RESIDUAL, OP_CHAN_PROMPT_LOGITS = (
    _L.OP_LN_QKV, _L.OP_ATTN_FWD, _L.OP_PROJ_RESIDUAL, _L.OP_LN_MLP_RESIDUAL, _L.OP_CHAN_PROMPT_LOGITS)
OP_GATED_CONV1X1, OP_CONV3X3_BN_ACT, OP_BILINEAR_UP, OP_INVPT_ATTN, OP_LAYERNORM = (
    _L.OP_GATED_CONV1X1, _L.OP_CONV3X3_BN_ACT, _L.OP_BILINEAR_UP, _L.OP_INVPT_ATTN, _L.OP_LAYERNORM)


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _launch(name, *args):
    """Call the library's entry point `name` with `args` and the current stream; RuntimeError when it fails."""
    _L.check(getattr(_L.load(), name)(*args, _stream()), name)


def device_check():
    """RuntimeError unless the current device can run the library's kernels."""
    _L.check(_L.load().mtt_device_check(), "mtt_device_check")


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _planes(s, row=0, col=0, lo=True):
    """Split.planes() of an optional operand: NULL planes and ld 0 for None."""
    return (0, 0, 0) if s is None else s.planes(row, col, lo)


def round_up(x, m):
    return (x + m - 1) // m * m


class Split:
    """An fp32-valued [rows, cols] matrix carried as bf16 planes hi (= bf16(x)) and lo (= bf16(x - hi)).

    Storage is one [nsplit, rows, ld] bf16 tensor; ``ld`` (elements) is a multiple of 8 so that TMA
    row strides are 16-byte aligned."""

    __slots__ = ("buf", "rows", "cols", "ld", "nsplit")

    def __init__(self, rows, cols, device, nsplit=2, ld=None, zero=False):
        self.rows, self.cols, self.nsplit = int(rows), int(cols), int(nsplit)
        self.ld = int(ld) if ld is not None else round_up(self.cols, 8)
        alloc = torch.zeros if zero else torch.empty
        self.buf = alloc((self.nsplit, self.rows, self.ld), dtype=torch.bfloat16, device=device)

    @classmethod
    def from_planes(cls, buf, cols):
        """The Split over an existing [nsplit, rows, ld] bf16 tensor (shares its storage)."""
        sp = cls.__new__(cls)
        sp.buf, sp.cols = buf, int(cols)
        sp.nsplit, sp.rows, sp.ld = buf.shape
        return sp

    def rows_view(self, r0, n):
        """Rows [r0, r0 + n) as a Split (shares storage)."""
        return Split.from_planes(self.buf[:, r0:r0 + n], self.cols)

    @property
    def hi(self):
        return self.buf[0]

    @property
    def lo(self):
        return self.buf[1] if self.nsplit == 2 else None

    def planes(self, row=0, col=0, lo=True):
        """(hi address, lo address or 0, ld) from element (row, col) on: the form the C ABI takes a split operand in.
        The lo address is 0 when there is one plane or lo is False."""
        hi = self.buf.data_ptr() + 2 * (row * self.ld + col)
        return hi, (hi + 2 * self.buf.stride(0) if lo and self.nsplit == 2 else 0), self.ld

    def float(self):
        """Reconstruct the fp32 values (testing / debugging only)."""
        x = self.buf[0, :, : self.cols].float()
        if self.nsplit == 2:
            x = x + self.buf[1, :, : self.cols].float()
        return x


def split_f32(x, nsplit=2, cols_pad=None, out=None):
    """fp32 [rows, cols] (last dim contiguous) -> Split. Columns [cols, cols_pad) are zero."""
    assert x.dtype == torch.float32 and x.dim() == 2 and x.stride(1) == 1
    rows, cols = x.shape
    cols_pad = cols if cols_pad is None else cols_pad
    if out is None:
        out = Split(rows, cols_pad, x.device, nsplit, ld=round_up(cols_pad, 8))
    _launch("mtt_split_f32", _ptr(x), x.stride(0), *out.planes(), rows, cols, cols_pad)
    return out


def layernorm(x, gamma, beta, eps, out_f32=None, out_split=None):
    """x fp32 [rows, cols] -> out_f32 (fp32 tensor) and/or out_split (Split)."""
    assert x.dtype == torch.float32 and x.dim() == 2 and x.stride(1) == 1
    rows, cols = x.shape
    _launch("mtt_layernorm", _ptr(x), x.stride(0), _ptr(gamma), _ptr(beta), float(eps),
            _ptr(out_f32), out_f32.stride(0) if out_f32 is not None else 0, *_planes(out_split), rows, cols)


def gemm(a, w, *, sk_ws=None, **kw):
    """D = act(A @ W^T + bias) + residual on the wgmma GEMM.

    a: Split [M, K] (or NHWC activation [B*H*W, C] when ``conv=(B, H, W, ksize, dil)``);
    w: Split [N, K] (conv: [N, ksize*ksize*cin_pad]); outputs: fp32 tensor and/or Split.
    regroup=(in_group, out_group, out_offset[, row_stride]) scatters output rows; a_gather=(group_rows,
    group_stride) gathers A rows in groups (M must be given); w_col_offset selects a K-slice of a wider packed W.
    sk_ws: optional stream-K workspace (streamk_workspace(device)); see mtt_gemm_desc.sk_ws.
    The keyword arguments and their defaults are _fill_gemm_desc's."""
    d = _L.GemmDesc()
    _fill_gemm_desc(d, a, w, **kw)
    if sk_ws is not None:
        d.sk_ws, d.sk_ws_bytes = sk_ws.data_ptr(), sk_ws.numel()
    _launch("mtt_gemm", C.byref(d))


def gemm_grouped(calls):
    """calls: [(a, w, kwargs)] with gemm()'s arguments -- problems of identical geometry that differ only in their
    tensors -- as ONE persistent launch (mtt_gemm_grouped)."""
    arr = (_L.GemmDesc * len(calls))()
    for d, (a, w, kw) in zip(arr, calls):
        _fill_gemm_desc(d, a, w, **kw)
    _launch("mtt_gemm_grouped", arr, len(calls))


def gemm_splitk(a, w, partial, out_f32, *, K, bias=None, chunks):
    """out = A @ W^T + bias for a skinny A with a very long K: `chunks` K-slices run as the problems of ONE grouped
    launch into partial [chunks, M, N] (fp32), then a fixed-order reduction adds them and the bias. K-slices are
    multiples of 64 (the GEMM's K block)."""
    M, N = a.rows, w.rows
    step = round_up(-(-K // chunks), 64)
    calls, k0 = [], 0
    while k0 < K:
        kk = min(step, K - k0)
        calls.append((a, w, dict(M=M, N=N, K=kk, out_f32=partial[len(calls)], a_col_offset=k0, w_col_offset=k0)))
        k0 += kk
    gemm_grouped(calls) if len({c[2]["K"] for c in calls}) == 1 else [gemm(c[0], c[1], **c[2]) for c in calls]
    _launch("mtt_sum_partials", _ptr(partial), len(calls), M, N, partial.stride(-2), _ptr(bias), _ptr(out_f32),
            out_f32.stride(-2))


def _fill_gemm_desc(d, a, w, *, M=None, N=None, K=None, bias=None, act=ACT_NONE, residual=None, res_row_mod=0,
                    out_f32=None, out_split=None, out_col_offset=0, regroup=None, conv=None, a_row_offset=0,
                    a_gather=None, w_col_offset=0, a_col_offset=0, w_row_offset=0, out_row_offset=0):
    """w_row_offset / out_row_offset: first row of the B operand / of the split output (pointer offsets): lets one
    buffer hold the operands of several (batch, head) problems of a grouped launch."""
    nsplit = min(a.nsplit, w.nsplit)
    d.a_hi, d.a_lo, d.lda = a.planes(a_row_offset, a_col_offset, lo=nsplit == 2)
    d.b_hi, d.b_lo, d.ldb = w.planes(w_row_offset, w_col_offset, lo=nsplit == 2)
    d.M = a.rows if M is None else M
    d.N = w.rows if N is None else N
    d.K = a.cols if K is None else K
    d.nsplit = nsplit
    if conv is not None:
        d.mode = 1
        d.B, d.H, d.W, d.ksize, d.dil = conv
    else:
        d.mode = 0
    d.bias = bias.data_ptr() if bias is not None else 0
    d.act = act
    if residual is not None:
        assert residual.dtype == torch.float32 and residual.stride(-1) == 1
        d.residual, d.ldr = residual.data_ptr(), residual.stride(-2)
    d.res_row_mod = res_row_mod
    if out_f32 is not None:
        assert out_f32.dtype == torch.float32 and out_f32.stride(-1) == 1
        d.out_f32, d.ldo_f32 = out_f32.data_ptr(), out_f32.stride(-2)
    if out_split is not None:
        d.out_hi, d.out_lo, d.ldo_bf = out_split.planes(out_row_offset, out_col_offset)
        if nsplit == 2 and out_split.nsplit != 2:
            raise ValueError("nsplit=2 GEMM needs a 2-plane split output")
    if regroup is not None:
        d.in_group, d.out_group, d.out_offset = regroup[:3]
        d.out_row_stride = regroup[3] if len(regroup) > 3 else 1
    if a_gather is not None:    # (group_rows, group_stride): logical row (g, i) at physical row g*stride + i
        d.a_group_rows, d.a_group_stride = a_gather


def attention(qkv, out, *, B, N, H, scale, prompt_logits=None, T=0):
    """Fused softmax(q k^T * scale) v over [B, N] tokens; qkv Split [B*N, 3*H*64], out Split [B*N, H*64].
    prompt_logits: optional fp32 [B, H, T, N] receiving raw q.k^T of the first T query rows."""
    d = _L.AttnDesc()
    nsplit = min(qkv.nsplit, out.nsplit)
    assert qkv.ld == 3 * H * 64 and out.ld == H * 64
    d.qkv_hi, d.qkv_lo, _ = qkv.planes(lo=nsplit == 2)
    d.out_hi, d.out_lo, _ = out.planes()   # lo written in either mode
    if prompt_logits is not None:
        assert prompt_logits.dtype == torch.float32 and prompt_logits.is_contiguous()
        assert tuple(prompt_logits.shape) == (B, H, T, N)
        d.prompt_logits = prompt_logits.data_ptr()
    d.B, d.N, d.H, d.T, d.nsplit, d.scale = B, N, H, T, nsplit, float(scale)
    _launch("mtt_attention", C.byref(d))


def streamk_workspace(device):
    """A zero-filled stream-K workspace for gemm(sk_ws=...): one per stream that issues such launches."""
    with torch.cuda.device(device):
        return workspace(_L.load().mtt_gemm_streamk_bytes(), device)


def set_gemm_streamk(mode):
    """Stream-K policy of the 128x256-tile GEMM: 0 off, 1 automatic (default), 2 whenever legal (tuning / testing knob; env
    MTT_GEMM_STREAMK)."""
    _L.load().mtt_set_gemm_streamk(int(mode))


def set_gemm_variant(v):
    """0 auto, 1 = 128x128 tiles, 2 = 128x256 tiles, 3 = 128x128 tiles (tuning / testing knob)."""
    _L.load().mtt_set_gemm_variant(int(v))


def set_attention_variant(v):
    """0 = default attention kernel; other values select development variants when built (tuning / testing knob)."""
    _L.load().mtt_set_attention_variant(int(v))


def profile_begin():
    """Start per-launch timing of the tensor-core kernels (see mtt_profile_begin)."""
    _L.check(_L.load().mtt_profile_begin(), "mtt_profile_begin")


def profile_end(max_recs=4096):
    """Synchronise and return [(kind, M, N, K, ms, flops)] for every mtt_gemm (kind 0) / mtt_attention (kind 1) launch
    since profile_begin()."""
    arr = (_L.ProfileRec * max_recs)()
    n = C.c_int32(0)
    _L.check(_L.load().mtt_profile_end(arr, max_recs, C.byref(n)), "mtt_profile_end")
    return [(r.kind, r.M, r.N, r.K, r.ms, r.flops) for r in arr[:min(n.value, max_recs)]]


def launch_count(reset=False):
    lib = _L.load()
    n = lib.mtt_launch_count()
    if reset:
        lib.mtt_launch_count_reset()
    return n


def im2col_patch(img, patch, out):
    """img fp32 NCHW -> out Split [B*P, Cin*patch*patch]."""
    assert img.dtype == torch.float32 and img.is_contiguous()
    B, Cin, H, W = img.shape
    _launch("mtt_im2col_patch", _ptr(img), B, Cin, H, W, patch, *out.planes())


def broadcast_rows(src, dst, B, group_rows):
    """dst[(b*group_rows + t), :] = src[t, :] for t < T; dst fp32 [B*group_rows, ld]."""
    T, Cc = src.shape
    assert src.is_contiguous() and src.dtype == torch.float32 and dst.dtype == torch.float32
    _launch("mtt_broadcast_rows", _ptr(src), _ptr(dst), B, T, Cc, group_rows, dst.stride(0))


def chan_logits(cp, xn, out, *, B, N, T, Cdim, gh, gw, nh, nw):
    _launch("mtt_chan_logits", _ptr(cp), *xn.planes(), B, N, T, Cdim, gh, gw, nh, nw, _ptr(out))


def gate_split(x, x_group_rows, x_row_offset, prompt_logits, chan_lg, task, ys, yc, *, B, T, N, H, Cdim, gh,
               gw, nh, nw, ntasks=1, task_stride=0):
    """Gate the patch map for tasks [task, task + ntasks) in one pass; ys / yc are the Splits of the FIRST task, task k's
    planes live k * task_stride elements further on (one task: plain Splits)."""
    assert x.dtype == torch.float32 and x.stride(-1) == 1 and ys.ld == yc.ld
    _launch("mtt_gate_split", _ptr(x), x.stride(-2), x_group_rows, x_row_offset, _ptr(prompt_logits), _ptr(chan_lg),
            task, ntasks, B, T, N, H, Cdim, gh, gw, nh, nw, *ys.planes()[:2], *yc.planes()[:2], ys.ld, task_stride)


def ctr_weights(prompt_logits, w0, b0, w2, b2, out, *, B, H, T, N):
    _launch("mtt_ctr_weights", _ptr(prompt_logits), B, H, T, N, _ptr(w0), _ptr(b0), _ptr(w2), _ptr(b2), _ptr(out))


def ctr_mix(F, w, acc, *, T, M, Cdim, ld, rows_per_batch, accumulate):
    _launch("mtt_ctr_mix", _ptr(F), _ptr(w), _ptr(acc), T, M, Cdim, ld, rows_per_batch, 1 if accumulate else 0)


def bilinear(x, ld_in, B, h, w, Cdim, H2, W2, *, out_f32=None, out_split=None, out_nchw=None,
             accumulate=False, in_batch_rows=0, in_row_offset=0, out_batch_rows=0, out_row_offset=0):
    """x: NHWC fp32 [B*h*w, ld_in] -> NHWC fp32 / NHWC Split / NCHW fp32 [B,C,H2,W2]."""
    _launch("mtt_bilinear", _ptr(x), ld_in, B, h, w, Cdim, H2, W2, _ptr(out_f32),
            out_f32.stride(-2) if out_f32 is not None else 0, *_planes(out_split), _ptr(out_nchw),
            1 if accumulate else 0, in_batch_rows, in_row_offset, out_batch_rows, out_row_offset)


POSTPROC_KIND = {"semseg": 0, "human_parts": 0, "edge": 1, "sal": 2, "normals": 3, "depth": 4}


def bilinear_postproc(x, ld_in, B, h, w, Cdim, H2, W2, kind, out):
    """Bilinear resize fused with get_output's post-processing (TP/utils/utils.py:27-63); `out` is int64
    [B,H2,W2] for kind 0, fp32 otherwise."""
    i64 = out if kind == 0 else None
    f32 = None if kind == 0 else out
    assert out.is_contiguous() and out.dtype == (torch.int64 if kind == 0 else torch.float32)
    _launch("mtt_bilinear_postproc", _ptr(x), ld_in, B, h, w, Cdim, H2, W2, kind, _ptr(i64), _ptr(f32))


METER_CONFUSION, METER_SALIENCY, METER_NORMALS, METER_DEPTH, METER_EDGE = (
    _L.METER_CONFUSION, _L.METER_SALIENCY, _L.METER_NORMALS, _L.METER_DEPTH, _L.METER_EDGE)


def meter_state_bytes(kind, n=0):
    """Bytes of device state a meter of `kind` needs (n = classes or thresholds); ValueError when the library refuses
    the kind or the size."""
    nb = int(_L.load().mtt_meter_state_bytes(int(kind), int(n)))
    if nb == 0:
        raise ValueError(_L.load().mtt_last_error().decode("utf-8", "replace"))
    return nb


def meter_reset(state, kind, n=0):
    _launch("mtt_meter_reset", _ptr(state), int(kind), int(n))


def _meter_inputs(what, pred, pred_dtype, pred_shape, label, label_channels, state, int64_labels=False):
    """Validates a meter update's tensors before any launch: dtypes, shapes (pred_shape(B, H, W) from the label's
    [B, label_channels, H, W], or int64 [B, H, W] where int64_labels allows it), contiguity and device.
    Returns (B, H, W)."""
    if int64_labels and label.dtype == torch.int64 and label.dim() == 3:
        B, H, W = (int(s) for s in label.shape)
    elif label.dtype != torch.float32 or label.dim() != 4 or label.shape[1] != label_channels:
        also = " or int64 [B,H,W]" if int64_labels else ""
        raise ValueError(f"{what}: label must be fp32 [B,{label_channels},H,W]{also}, got {label.dtype} "
                         f"{tuple(label.shape)}")
    else:
        B, _, H, W = (int(s) for s in label.shape)
    if pred.dtype != pred_dtype or tuple(pred.shape) != pred_shape(B, H, W):
        raise ValueError(f"{what}: prediction must be {pred_dtype} {pred_shape(B, H, W)} for a label of shape "
                         f"{tuple(label.shape)}, got {pred.dtype} {tuple(pred.shape)}")
    if not (pred.is_cuda and label.is_cuda and state.is_cuda):
        raise RuntimeError(f"{what}: the meters run on the GPU only; got tensors on {pred.device} / {label.device}")
    if not (pred.is_contiguous() and label.is_contiguous()):
        raise ValueError(f"{what}: prediction and label must be contiguous")
    return B, H, W


def meter_confusion_update(pred, label, n_classes, ignore_index, state):
    """pred int64 [B,H,W] class map, label fp32 [B,1,H,W] (the transforms' format) or int64 [B,H,W] (the Cityscapes-3D
    loader's, TP/data/cityscapes3d.py:227); the reference meter squeezes both the same way (eval_semseg.py:71-81)."""
    B, H, W = _meter_inputs("meter_confusion_update", pred, torch.int64, lambda b, h, w: (b, h, w), label, 1, state,
                            int64_labels=True)
    fn = "mtt_meter_confusion_update_i64" if label.dtype == torch.int64 else "mtt_meter_confusion_update"
    _launch(fn, _ptr(pred), _ptr(label), B, H, W, int(n_classes), float(ignore_index), _ptr(state))


def meter_saliency_update(pred, label, thresholds, ignore_index, state):
    """pred fp32 [B,H,W] (255 * probability), label fp32 [B,1,H,W], thresholds fp32 on the device."""
    B, H, W = _meter_inputs("meter_saliency_update", pred, torch.float32, lambda b, h, w: (b, h, w), label, 1, state)
    assert thresholds.is_cuda and thresholds.dtype == torch.float32 and thresholds.is_contiguous()
    _launch("mtt_meter_saliency_update", _ptr(pred), _ptr(label), B, H, W, _ptr(thresholds), thresholds.numel(),
            float(ignore_index), _ptr(state))


def meter_normals_update(pred, label, ignore_index, state):
    """pred fp32 [B,H,W,3] (predict()'s normals), label fp32 [B,3,H,W]."""
    B, H, W = _meter_inputs("meter_normals_update", pred, torch.float32, lambda b, h, w: (b, h, w, 3), label, 3, state)
    _launch("mtt_meter_normals_update", _ptr(pred), _ptr(label), B, H, W, float(ignore_index), _ptr(state))


def meter_depth_update(pred, label, state, *, min_depth=None, max_depth=None, ignore_index=255):
    """pred fp32 [B,H,W,1] (predict()'s depth) or [B,H,W], label fp32 [B,1,H,W]. The mask is min_depth < gt <
    max_depth when both bounds are given, gt != ignore_index otherwise."""
    shape = (lambda b, h, w: (b, h, w, 1)) if pred.dim() == 4 else (lambda b, h, w: (b, h, w))
    B, H, W = _meter_inputs("meter_depth_update", pred, torch.float32, shape, label, 1, state)
    use_range = min_depth is not None and max_depth is not None
    _launch("mtt_meter_depth_update", _ptr(pred), _ptr(label), B, H, W, int(use_range),
            float(min_depth) if use_range else 0.0, float(max_depth) if use_range else 0.0, float(ignore_index),
            _ptr(state))


def meter_edge_update(pred, label, pos_weight, ignore_index, state):
    """pred fp32 [B,H,W] (255 * sigmoid), label fp32 [B,1,H,W]."""
    B, H, W = _meter_inputs("meter_edge_update", pred, torch.float32, lambda b, h, w: (b, h, w), label, 1, state)
    _launch("mtt_meter_edge_update", _ptr(pred), _ptr(label), B, H, W, float(pos_weight), float(ignore_index),
            _ptr(state))


IMAGENET_MEAN = (0.485, 0.456, 0.406)   # TP/inference.py:99,107
IMAGENET_STD = (0.229, 0.224, 0.225)


def preprocess_image(img_u8, out_hw, *, bgr=True, mean=IMAGENET_MEAN, std=IMAGENET_STD, out=None):
    """The reference's inference pre-processing (TP/inference.py:93-115,127-133) on the device: img_u8 is a CUDA
    uint8 tensor [h,w,3] or [B,h,w,3] as cv2.imread returns it (BGR); returns fp32 [B,3,H,W] normalised and
    bilinearly resized (cv2 INTER_LINEAR), the tensor `model(x)` takes."""
    import ctypes
    if img_u8.dim() == 3:
        img_u8 = img_u8.unsqueeze(0)
    assert img_u8.is_cuda and img_u8.dtype == torch.uint8 and img_u8.is_contiguous() and img_u8.shape[-1] == 3
    B, h, w, _ = img_u8.shape
    H, W = out_hw
    if out is None:
        out = torch.empty(B, 3, H, W, device=img_u8.device, dtype=torch.float32)
    assert out.is_contiguous() and tuple(out.shape) == (B, 3, H, W) and out.dtype == torch.float32
    m3 = (ctypes.c_float * 3)(*mean)
    s3 = (ctypes.c_float * 3)(*std)
    _launch("mtt_preprocess_image", _ptr(img_u8), B, h, w, int(bool(bgr)), m3, s3, _ptr(out), H, W)
    return out


def cityscapes_targets(label_ids, disparity, out_hw, *, semseg=None, depth=None):
    """The reference's Cityscapes-3D targets (mtt_cityscapes_targets): label_ids uint8 [B,h,w] and disparity uint16
    [B,h,w] (or None when no depth is asked for) on the device -> semseg int64 [B,H,W] and / or depth fp32 [B,1,H,W]
    at out_hw = (H, W), written into the given tensors."""
    if label_ids.dtype != torch.uint8 or label_ids.dim() != 3 or not label_ids.is_cuda:
        raise ValueError(f"cityscapes_targets: label ids must be CUDA uint8 [B,h,w], got {label_ids.dtype} "
                         f"{tuple(label_ids.shape)} on {label_ids.device}")
    B, h, w = (int(s) for s in label_ids.shape)
    H, W = (int(s) for s in out_hw)
    if semseg is None and depth is None:
        raise ValueError("cityscapes_targets: no output requested")
    if depth is not None and (disparity is None or disparity.dtype != torch.uint16 or
                              tuple(disparity.shape) != (B, h, w) or not disparity.is_cuda):
        raise ValueError(f"cityscapes_targets: depth needs a CUDA uint16 disparity of shape {(B, h, w)}")
    for name, t, dt, shape in (("semseg", semseg, torch.int64, (B, H, W)), ("depth", depth, torch.float32, (B, 1, H, W))):
        if t is not None and (t.dtype != dt or tuple(t.shape) != shape or not t.is_cuda):
            raise ValueError(f"cityscapes_targets: {name} must be CUDA {dt} {shape}, got {t.dtype} {tuple(t.shape)}")
    for t in (label_ids, disparity, semseg, depth):
        if t is not None and not t.is_contiguous():
            raise ValueError("cityscapes_targets: every tensor must be contiguous")
    _launch("mtt_cityscapes_targets", _ptr(label_ids), _ptr(disparity if depth is not None else None), B, h, w, H, W,
            _ptr(semseg), _ptr(depth))


def augment_workspace_bytes(B):
    return int(_L.load().mtt_augment_workspace_bytes(int(B)))


def augment(samples, data, *, B, H, W, train, crop_hw, tasks, task_out, image_out, workspace,
            mean=IMAGENET_MEAN, std=IMAGENET_STD):
    """The reference's train (train=True) or validation transform chain over a packed ragged batch
    (mtt_augment): samples = device bytes of B mtt_augment_sample records, data = device float32 raw arrays;
    tasks = task names (keys of lib.AUG_TASK_KIND) in the records' offset order, task_out / image_out = fp32 NCHW
    outputs; workspace = int32 device tensor of augment_workspace_bytes(B) bytes."""
    d = _L.AugmentDesc()
    d.samples, d.data = samples.data_ptr(), data.data_ptr()
    d.B, d.H, d.W, d.train = int(B), int(H), int(W), int(bool(train))
    d.crop_h, d.crop_w = (int(crop_hw[0]), int(crop_hw[1])) if train else (0, 0)
    d.ntasks = len(tasks)
    for i, (t, o) in enumerate(zip(tasks, task_out)):
        d.task_kind[i] = _L.AUG_TASK_KIND[t]
        d.task_out[i] = o.data_ptr()
    d.image_out = image_out.data_ptr()
    for c in range(3):
        d.mean[c], d.std[c] = mean[c], std[c]
    d.workspace, d.workspace_bytes = workspace.data_ptr(), workspace.numel() * workspace.element_size()
    _launch("mtt_augment", C.byref(d))


RENDER_ENCODE = {"u8": _L.RENDER_U8, "class": _L.RENDER_CLASS, "palette_bgr": _L.RENDER_PALETTE_BGR,
                 "normals_bgr": _L.RENDER_NORMALS_BGR, "jet": _L.RENDER_JET}
RENDER_CHANNELS = {"u8": 1, "class": 1, "palette_bgr": 3, "normals_bgr": 3, "jet": 3}


def render_workspace_bytes(n_tasks, B):
    return int(_L.load().mtt_render_workspace_bytes(int(n_tasks), int(B)))


def _render_source(what, src, postproc, n_classes):
    """(source kind, C, h, w) of a render source, or ValueError: fp32 NCHW logits when postproc (a get_output kind) is
    given, else predict()'s int64 [B,h,w] class map or fp32 [B,h,w] / [B,h,w,1] / [B,h,w,3] map."""
    if postproc is not None:
        if src.dtype != torch.float32 or src.dim() != 4:
            raise ValueError(f"{what}: logits must be fp32 [B,C,h,w], got {src.dtype} {tuple(src.shape)}")
        return _L.RENDER_SRC_LOGITS, int(src.shape[1]), int(src.shape[2]), int(src.shape[3])
    if src.dtype == torch.int64 and src.dim() == 3:
        return _L.RENDER_SRC_CLASS, int(n_classes or 1), int(src.shape[1]), int(src.shape[2])
    if src.dtype == torch.float32 and (src.dim() == 3 or (src.dim() == 4 and src.shape[3] in (1, 3))):
        return _L.RENDER_SRC_MAP, int(src.shape[3]) if src.dim() == 4 else 1, int(src.shape[1]), int(src.shape[2])
    raise ValueError(f"{what}: a get_output map must be int64 [B,h,w] or fp32 [B,h,w(,1|3)], got {src.dtype} "
                     f"{tuple(src.shape)}")


def render(tasks, workspace):
    """Predictions -> uint8 images (mtt_render): one pre-pass and one main launch for all tasks. `tasks` is a list of
    dicts, one per task, with
      src       fp32 NCHW logits (with postproc = get_output kind, ops.POSTPROC_KIND) or a get_output map (postproc
                None; n_classes = the class count of an int64 map, for the palette check)
      out_hw    the resize target of logits (default: the logits' size); out_sizes: one (h, w) per image instead
      encode    a key of RENDER_ENCODE; table: uint8 CUDA tensor (palette [N,3] RGB, id table [256], JET [256,3])
      crops     host int [B,4] (y0, x0, h, w); offsets: host int [B] byte offsets into out (uint8 CUDA tensor)
      label     optional fp32 CUDA tensor [B,...] with flags (int32 CUDA [B]) and ignore_index: the all-ignore flag.
    Every tensor is checked (dtype, shape, contiguity, device) before anything is launched."""
    import numpy as np
    if not 0 < len(tasks) <= _L.RENDER_MAX_TASKS:
        raise ValueError(f"render: 1..{_L.RENDER_MAX_TASKS} tasks per call, got {len(tasks)}")
    descs = (_L.RenderDesc * len(tasks))()
    keep = []
    for i, t in enumerate(tasks):
        what = f"render(task {i})"
        src, post = t["src"], t.get("postproc")
        kind, Cs, h, w = _render_source(what, src, post, t.get("n_classes"))
        B = int(src.shape[0])
        enc = t["encode"]
        if enc not in RENDER_ENCODE:
            raise ValueError(f"{what}: encode must be one of {sorted(RENDER_ENCODE)}, got {enc!r}")
        out, table, label, flags = t["out"], t.get("table"), t.get("label"), t.get("flags")
        tensors = [src, out] + [x for x in (table, label, flags) if x is not None]
        if not all(isinstance(x, torch.Tensor) and x.is_cuda for x in tensors):
            raise RuntimeError(f"{what}: every tensor must be a CUDA tensor (there is no CPU path)")
        if len({x.device for x in tensors + [workspace]}) != 1:
            raise RuntimeError(f"{what}: tensors on different devices")
        if not all(x.is_contiguous() for x in tensors):
            raise ValueError(f"{what}: tensors must be contiguous")
        if out.dtype != torch.uint8 or (table is not None and table.dtype != torch.uint8):
            raise ValueError(f"{what}: out and table must be uint8")
        if label is not None and (label.dtype != torch.float32 or label.shape[0] != B or flags is None or
                                  flags.dtype != torch.int32 or flags.numel() < B):
            raise ValueError(f"{what}: label must be fp32 [B,...] with int32 flags [B]")
        crops = np.ascontiguousarray(np.asarray(t["crops"], dtype=np.int32).reshape(-1, 4))
        offs = np.ascontiguousarray(np.asarray(t["offsets"], dtype=np.int64).reshape(-1))
        if crops.shape[0] != B or offs.shape[0] != B:
            raise ValueError(f"{what}: {B} images need {B} crops and offsets, got {crops.shape[0]} / {offs.shape[0]}")
        oh, ow = t.get("out_hw") or (h, w)
        sizes = t.get("out_sizes")
        if sizes is not None:
            sizes = np.ascontiguousarray(np.asarray(sizes, dtype=np.int32).reshape(B, 2))
        keep += [crops, offs, sizes]
        d = descs[i]
        d.src_kind, d.src, d.B, d.C, d.h, d.w = kind, src.data_ptr(), B, Cs, h, w
        d.out_h, d.out_w = int(oh), int(ow)
        d.postproc = -1 if post is None else int(post)
        d.encode = RENDER_ENCODE[enc]
        d.table = table.data_ptr() if table is not None else None
        d.table_len = (table.shape[0] if table is not None else 0)
        d.crop = crops.ctypes.data_as(C.POINTER(C.c_int32))
        d.offset = offs.ctypes.data_as(C.POINTER(C.c_int64))
        d.out_size = sizes.ctypes.data_as(C.POINTER(C.c_int32)) if sizes is not None else None
        d.out, d.out_bytes = out.data_ptr(), out.numel()
        d.label = label.data_ptr() if label is not None else None
        d.label_numel = label[0].numel() if label is not None else 0
        d.ignore_index = float(t.get("ignore_index", 255))
        d.flags = flags.data_ptr() if flags is not None else None
    if workspace.numel() * workspace.element_size() < render_workspace_bytes(1, sum(d.B for d in descs)):
        raise ValueError("render: workspace smaller than render_workspace_bytes")
    _launch("mtt_render", descs, len(tasks), _ptr(workspace))


def bilinear_sum3(srcs, out, *, B, Cdim, H2, W2):
    """out (Split [B*H2*W2, C]) = sum_i bilinear(src_i -> H2 x W2); srcs: list of up to three
    (tensor fp32 [rows, ld], h, w, batch_rows, row_offset)."""
    arr = (_L.BilinearSrc * len(srcs))()
    for i, (t, h, w, brows, roff) in enumerate(srcs):
        assert t.dtype == torch.float32 and t.stride(-1) == 1
        arr[i].in_, arr[i].ld_in, arr[i].h, arr[i].w = t.data_ptr(), t.stride(-2), h, w
        arr[i].batch_rows, arr[i].row_offset = brows, roff
    _launch("mtt_bilinear_sum3", arr, len(srcs), B, Cdim, H2, W2, *out.planes())


def split_rows(x, out, *, rows, cols, in_group=0, src_group=0, src_offset=0):
    """Gather fp32 rows of x (row r at (r // in_group) * src_group + src_offset + r % in_group) -> Split."""
    assert x.dtype == torch.float32 and x.stride(-1) == 1
    _launch("mtt_split_rows", _ptr(x), x.stride(-2), in_group, src_group, src_offset, *out.planes(), rows, cols)


def layernorm_seg(x, gamma, beta, eps, *, rows, cols, S=1, in_group=0, src_group=0, src_offset=0,
                  seg_stride=0, out_f32=None, out_split=None, out_seg_stride=0):
    assert x.dtype == torch.float32 and x.stride(-1) == 1
    _launch("mtt_layernorm_seg", _ptr(x), x.stride(-2), in_group, src_group, src_offset, seg_stride, S, _ptr(gamma),
            _ptr(beta), float(eps), _ptr(out_f32), out_f32.stride(-2) if out_f32 is not None else 0,
            *_planes(out_split), out_seg_stride, rows, cols)


def zero_insert(x, out, *, B, h, w, Cdim, src_group, src_offset):
    assert x.dtype == torch.float32 and x.stride(-1) == 1
    _launch("mtt_zero_insert", _ptr(x), x.stride(-2), src_group, src_offset, B, h, w, Cdim, *out.planes())


def dwconv3x3_s2(x, weight, bias, out, *, B, T, h, w, Cdim):
    assert x.dtype == torch.float32 and x.stride(-1) == 1 and weight.is_contiguous() and bias.is_contiguous()
    _launch("mtt_dwconv3x3_s2", _ptr(x), x.stride(-2), B, T, h, w, Cdim, _ptr(weight), _ptr(bias), *out.planes())


def avgpool(x, out, *, BT, h, w, Cdim, s):
    assert x.dtype == torch.float32 and x.stride(-1) == 1
    _launch("mtt_avgpool", _ptr(x), x.stride(-2), BT, h, w, Cdim, s, *out.planes())


def invpt_fuse_softmax(raw, P, *, B, Lq, Tk, scale, prev_score=None, T=0, qh=0, qw=0, fuse_w=None, fuse_b=None,
                       score_out=None):
    """The step between the two GEMMs of InvPT's cross-task attention (invpt.py:204-236): scale, cross-scale fusion with
    the up-sampled previous score, score export, softmax -> P Split [B*2*Lq, Tk]."""
    assert raw.is_contiguous() and raw.dtype == torch.float32
    if prev_score is not None:
        assert prev_score.is_contiguous() and fuse_w.is_contiguous()
    if score_out is not None:
        assert score_out.is_contiguous()
    _launch("mtt_invpt_fuse_softmax", _ptr(raw), B, Lq, Tk, float(scale), _ptr(prev_score), T, qh, qw, _ptr(fuse_w),
            _ptr(fuse_b), _ptr(score_out), *P.planes())


# ------------------------------------------------------------------------------------------------
# named operators of SURVEY.md section 8(b) (block_ops.cu) and the packing / layout entry points
# ------------------------------------------------------------------------------------------------
def _shape(rows=0, Cdim=0, hidden=0, nsplit=2, B=0, N=0, H=0, T=0):
    s = _L.Shape()
    s.rows, s.C, s.hidden, s.nsplit, s.B, s.N, s.H, s.T = rows, Cdim, hidden, nsplit, B, N, H, T
    return s


def _weight(w, nsplit):
    return _L.Weight(*w.planes(lo=nsplit == 2))


def workspace_bytes(op, **shape):
    return int(_L.load().mtt_workspace_bytes(op, C.byref(_shape(**shape))))


def workspace(nbytes, device):
    """A 256-byte aligned, ZERO-FILLED byte buffer (torch's caching allocator aligns to 512). Zero because the stream-K
    flag words inside the LayerNorm-fronted operators' workspaces must start at zero (include/mtt_b200.h, sk_ws)."""
    return torch.zeros(max(int(nbytes), 256), dtype=torch.uint8, device=device)


def ws_split_view(ws, byte_offset, rows, cols, nsplit):
    """The Split living at `byte_offset` of a workspace, laid out as block_ops.cu does: [nsplit][rows][pad8(cols)]."""
    ld = round_up(cols, 8)
    n = nsplit * rows * ld
    return Split.from_planes(ws[byte_offset: byte_offset + 2 * n].view(torch.bfloat16).view(nsplit, rows, ld), cols)


def ln_qkv(x, gamma, beta, eps, wqkv, bias, qkv, ws):
    """qkv = LN(x) @ Wqkv^T + b (taskprompter.py:272,:199,:201); LN(x) stays in `ws` as split planes."""
    rows, Cd = x.shape
    ns = min(wqkv.nsplit, qkv.nsplit)
    _launch("mtt_ln_qkv", _ptr(x), x.stride(0), _ptr(gamma), _ptr(beta), float(eps), C.byref(_weight(wqkv, ns)),
            _ptr(bias), *qkv.planes(), C.byref(_shape(rows, Cd, nsplit=ns)), _ptr(ws), ws.numel())


def proj_residual(ao, wproj, bias, x):
    """x += ao @ Wproj^T + b in place (taskprompter.py:212,:273,:276)."""
    rows, Cd = x.shape
    ns = min(ao.nsplit, wproj.nsplit)
    _launch("mtt_proj_residual", *ao.planes(), C.byref(_weight(wproj, ns)), _ptr(bias), _ptr(x), x.stride(0),
            C.byref(_shape(rows, Cd, nsplit=ns)))


def ln_mlp_residual(x, gamma, beta, eps, w1, b1, w2, b2, ws):
    """x += fc2(gelu(fc1(LN(x)))) in place (taskprompter.py:274,:277)."""
    rows, Cd = x.shape
    ns = min(w1.nsplit, w2.nsplit)
    _launch("mtt_ln_mlp_residual", _ptr(x), x.stride(0), _ptr(gamma), _ptr(beta), float(eps), C.byref(_weight(w1, ns)),
            _ptr(b1), C.byref(_weight(w2, ns)), _ptr(b2), C.byref(_shape(rows, Cd, hidden=w1.rows, nsplit=ns)),
            _ptr(ws), ws.numel())


def gated_conv1x1(x, x_group_rows, x_row_offset, prompt_logits, chan_lg, tasks, e, chan_col, ws, *, B, T, N, H, Cdim,
                  gh, gw, nh, nw):
    """Spatial + channel gating of ALL tasks of a level and their 2 * len(tasks) 1x1 decode convs (taskprompter.py:
    436-471) -- one gating launch, one grouped GEMM launch. tasks: [(w_spa, b_spa, w_chan, b_chan, cat Split)]."""
    cat0 = tasks[0][4]
    ns = min(tasks[0][0].nsplit, cat0.nsplit)
    arr = (_L.GatedTask * len(tasks))()
    for g, (w_spa, b_spa, w_chan, b_chan, cat) in zip(arr, tasks):
        assert cat.ld == cat0.ld
        g.w_spa, g.b_spa, g.w_chan, g.b_chan = _weight(w_spa, ns), b_spa.data_ptr(), _weight(w_chan, ns), b_chan.data_ptr()
        g.cat_hi, g.cat_lo, _ = cat.planes(lo=ns == 2)
    _launch("mtt_gated_conv1x1", _ptr(x), x.stride(-2), x_group_rows, x_row_offset, _ptr(prompt_logits), _ptr(chan_lg),
            len(tasks), arr, gh, gw, nh, nw, e, cat0.ld, chan_col,
            C.byref(_shape(0, Cdim, nsplit=ns, B=B, N=N, H=H, T=T)), _ptr(ws), ws.numel())


def conv3x3_bn_act(a, w3, b3, Cin, Cout, act, *, B, H, W, dil=1, mid=None, w_head=None, b_head=None, n_out=0,
                   out_f32=None, ws=None):
    """3x3 conv + folded BN + act on an NHWC Split (optionally followed by the fused 1x1 head -> out_f32)."""
    ns = min(a.nsplit, w3.nsplit)
    _launch("mtt_conv3x3_bn_act", *a.planes(), B, H, W, Cin, dil, C.byref(_weight(w3, ns)), _ptr(b3), Cout, act,
            *_planes(mid), C.byref(_weight(w_head, ns)) if w_head is not None else None, _ptr(b_head), n_out,
            _ptr(out_f32), out_f32.stride(-2) if out_f32 is not None else 0, ns, _ptr(ws),
            ws.numel() if ws is not None else 0)


def pack_weight(w, nsplit):
    """fp32 [N, K] -> Split [N, K] through mtt_pack_weight."""
    assert w.dtype == torch.float32 and w.dim() == 2 and w.stride(1) == 1
    N, K = w.shape
    out = Split(N, round_up(K, 8), w.device, nsplit)
    out.cols = K
    _launch("mtt_pack_weight", _ptr(w), w.stride(0), N, K, nsplit, *out.planes())
    return out


def pack_conv_weight(w, bias, bn, nsplit, transposed=False):
    """Conv2d [N,Cin,k,k] (or ConvTranspose2d [Cin,N,k,k], transposed=True) + optional eval BatchNorm -> (Split
    [N, k*k*cin_pad] tap-major, folded bias fp32 [N]) through mtt_pack_conv_weight."""
    assert w.dtype == torch.float32 and w.is_contiguous() and w.dim() == 4 and w.shape[2] == w.shape[3]
    N, Cin = (w.shape[1], w.shape[0]) if transposed else (w.shape[0], w.shape[1])
    k = w.shape[2]
    cin_pad = round_up(Cin, 64)
    out = Split(N, k * k * cin_pad, w.device, nsplit)
    bias_out = torch.empty(N, dtype=torch.float32, device=w.device)
    scale = torch.empty(N, dtype=torch.float32, device=w.device)
    f = lambda t: t.detach().to(device=w.device, dtype=torch.float32).contiguous()
    if bn is not None:
        g, b, m, v, eps = f(bn.weight), f(bn.bias), f(bn.running_mean), f(bn.running_var), float(bn.eps)
    else:
        g = b = m = v = None
        eps = 0.0
    bias = f(bias) if bias is not None else None
    _launch("mtt_pack_conv_weight", _ptr(w), _ptr(bias), _ptr(g), _ptr(b), _ptr(m), _ptr(v), eps, N, Cin, k,
            1 if transposed else 0, nsplit, *out.planes(), _ptr(bias_out), _ptr(scale))
    return out, bias_out


def nchw_to_nhwc_split(x, out, col_offset=0):
    """x fp32 NCHW [B,C,H,W] -> columns [col_offset, col_offset + C) of out Split [B*H*W, >= C] (module-boundary
    forwards take NCHW like the reference)."""
    assert x.dtype == torch.float32 and x.is_contiguous() and x.dim() == 4
    B, Cd, H, W = x.shape
    _launch("mtt_nchw_to_nhwc_split", _ptr(x), B, Cd, H, W, *out.planes(col=col_offset))


def nhwc_to_nchw(x, ld_in, B, Cd, H, W, out):
    assert x.dtype == torch.float32 and out.is_contiguous() and tuple(out.shape) == (B, Cd, H, W)
    _launch("mtt_nhwc_to_nchw", _ptr(x), ld_in, B, Cd, H, W, _ptr(out))


# ------------------------------------------------------------------------------------------------
# Swin-backbone TaskPrompter kernels (swin.cu)
# ------------------------------------------------------------------------------------------------
def swin_window_gather(xn, pn, out, *, B, H, W, Cdim, T, ws, shift):
    """LN1 outputs xn [B*H*W, C], pn [B*T, C] (fp32) -> out: split joint window stream [B*nW*(T + ws*ws), C]."""
    _launch("mtt_swin_window_gather", _ptr(xn), xn.stride(0), _ptr(pn), pn.stride(0), B, H, W, Cdim, T, ws, shift,
            *out.planes())


def swin_window_attention(qkv, out, raw, biasT, maskT, *, BW, nW, T, L, heads, scale):
    """Window attention with prompts; biasT [heads, L, L] / maskT [nW, L, L] are stored transposed ([.., key, query])."""
    Cd = out.cols
    assert biasT.is_contiguous() and (maskT is None or maskT.is_contiguous()) and raw.is_contiguous()
    _launch("mtt_swin_window_attention", *qkv.planes(), BW, nW, T, L, heads, Cd // heads, float(scale), _ptr(biasT),
            _ptr(maskT), *out.planes(), _ptr(raw))


def swin_window_scatter(o32, raw, xa, x, p, logits, *, B, H, W, Cdim, T, ws, shift, heads, last):
    """proj output on the joint stream -> xa, x += xa, p += mean prompt rows (unless last), raw -> logits map."""
    _launch("mtt_swin_window_scatter", _ptr(o32), o32.stride(0), _ptr(raw), B, H, W, Cdim, T, ws, shift, heads,
            0 if last else 1, _ptr(xa), xa.stride(0), _ptr(x), x.stride(0), _ptr(p), p.stride(0), _ptr(logits))


def transpose_split(x, out, *, B, L, Cdim):
    """x fp32 [B*L, C] -> out Split [B*C, L] (per-image transpose)."""
    _launch("mtt_transpose_split", _ptr(x), x.stride(0), B, L, Cdim, *out.planes())


def swin_chan_attention(q, kv, co32, cos, rc_out, *, B, T, Cdim, ce, nh, nw):
    _launch("mtt_swin_chan_attention", _ptr(q), q.stride(0), _ptr(kv), kv.stride(0), B, T, Cdim, ce, nh, nw,
            _ptr(co32), co32.stride(0), *cos.planes(), _ptr(rc_out))


def swin_merge_gather(x, out, *, B, H, W, Cdim):
    _launch("mtt_swin_merge_gather", _ptr(x), x.stride(0), B, H, W, Cdim, _ptr(out), out.stride(0))


def conv3x3_s2_maps(x, w, b, out, *, B, Cin, H, W, in_stride, in_offset, out_stride, out_offset):
    assert w.is_contiguous() and x.is_contiguous() and out.is_contiguous()
    _launch("mtt_conv3x3_s2_maps", _ptr(x), _ptr(w), _ptr(b), B, Cin, w.shape[0], H, W, in_stride, in_offset,
            out_stride, out_offset, _ptr(out))


def swin_chan_up(rc_in, w, out, *, BT, Cdim, nwin):
    assert rc_in.is_contiguous() and w.is_contiguous() and out.is_contiguous()
    _launch("mtt_swin_chan_up", _ptr(rc_in), _ptr(w), BT, Cdim, w.shape[0], nwin, _ptr(out))


def swin_logit_maps(logits, maps, *, T, to_maps):
    """Prompt-row logit maps between the gating layout logits [B, heads, T, T + H*W] (the map at column T on) and the
    reference's raw_spa_attn maps [B, heads, T, H, W]; to_maps: logits -> maps, else maps -> logits (the first T
    columns of the logits are not written)."""
    assert logits.is_contiguous() and maps.is_contiguous() and logits.dtype == maps.dtype == torch.float32
    L = logits.shape[-1] - T
    rows = logits.numel() // logits.shape[-1]
    assert maps.numel() == rows * L
    src, dst = (logits, maps) if to_maps else (maps, logits)
    _launch("mtt_swin_logit_maps", _ptr(src), _ptr(dst), rows, T, L, 1 if to_maps else 0)


# ---- training step (csrc/train_ops.cu): fp32 [rows, cols] tensors, last dim contiguous ----------------------------------
def _ld(t):
    assert t.dtype == torch.float32 and t.stride(-1) == 1
    return t.stride(-2) if t.dim() >= 2 else t.shape[-1]


def colsum(x, out, accumulate=False, *, rows=None, in_group=0, src_group=0, src_offset=0):
    """out[c] (+)= sum_r x[row(r), c]; row mapping as split_rows (in_group = 0: the first `rows` rows)."""
    rows = x.shape[0] if rows is None else rows
    _launch("mtt_colsum", _ptr(x), _ld(x), rows, x.shape[1], in_group, src_group, src_offset, _ptr(out),
            int(accumulate))


def layernorm_bwd(x, dy, gamma, eps, dx, dgamma, dbeta, *, accumulate_dx=False):
    """dx (+)= d LN(x) . dy; dgamma / dbeta are ACCUMULATED (None: skip the parameter gradients)."""
    rows, cols = x.shape
    ws = torch.empty(2 * rows, dtype=torch.float32, device=x.device)
    _launch("mtt_layernorm_bwd", _ptr(x), _ld(x), _ptr(dy), _ld(dy), _ptr(gamma), float(eps), rows, cols, _ptr(dx),
            _ld(dx), int(accumulate_dx), _ptr(dgamma), _ptr(dbeta), _ptr(ws))


def act_split(pre, act, out=None, nsplit=2):
    rows, cols = pre.shape
    if out is None:
        out = Split(rows, cols, pre.device, nsplit)
    _launch("mtt_act_split", _ptr(pre), _ld(pre), rows, cols, act, *out.planes())
    return out


def act_bwd(pre, dy, act, dx):
    rows, cols = pre.shape
    _launch("mtt_act_bwd", _ptr(pre), _ld(pre), _ptr(dy), _ld(dy), rows, cols, act, _ptr(dx), _ld(dx))


def axpy_rows(base, src, row_scale, dst):
    """dst = base + row_scale[:, None] * src (base / row_scale may be None)."""
    rows, cols = src.shape
    _launch("mtt_axpy_rows", _ptr(base), _ld(base) if base is not None else 0, _ptr(src), _ld(src), _ptr(row_scale),
            rows, cols, _ptr(dst), _ld(dst))


def transpose_planes(a, *, B=1, R=None, Ccols=None, in_batch_rows=None, out=None, side_by_side=False):
    """Split [B*R(+), C] -> Split: image b (rows b*in_batch_rows ... + R of `a`) transposed to a [C, R] block; blocks are
    stacked by rows ([B*C, ld >= R]) or, side_by_side, along the columns of one [C, B*R] matrix."""
    R = a.rows // B if R is None else R
    Ccols = a.cols if Ccols is None else Ccols
    in_batch_rows = R if in_batch_rows is None else in_batch_rows
    if out is None:
        rows, cols = (Ccols, B * R) if side_by_side else (B * Ccols, R)
        out = Split(rows, cols, a.hi.device, a.nsplit)     # pad columns are never read (TMA bounds)
    _launch("mtt_transpose_planes", *a.planes(), in_batch_rows, B, R, Ccols, *out.planes(), R if side_by_side else 0)
    return out


def bn_stats(x, sums):
    """sums [2C] = (sum x, sum x^2) over the rows of x, accumulated in float64. Keep sums float64 (TrainStep does): a
    float32 buffer receives the rounded sums, and the variance formed from those cancels in fp32 as |mean| / std grows."""
    out = sums if sums.dtype == torch.float64 else torch.empty(sums.shape, dtype=torch.float64, device=sums.device)
    _launch("mtt_bn_stats", _ptr(x), _ld(x), x.shape[0], x.shape[1], _ptr(out))
    if out is not sums:
        sums.copy_(out)


def bn_finalize(sums, count, eps, momentum, mean_rstd, running_mean=None, running_var=None):
    """mean_rstd [2C] fp32 from sums (float64, or float32 widened) / count, the variance formed in float64."""
    s = sums if sums.dtype == torch.float64 else sums.double()
    _launch("mtt_bn_finalize", _ptr(s), float(count), s.numel() // 2, float(eps), float(momentum), _ptr(mean_rstd),
            _ptr(running_mean), _ptr(running_var))


def bn_act(x, mean_rstd, gamma, beta, act, *, out_f32=None, out_split=None):
    rows, cols = x.shape
    _launch("mtt_bn_act", _ptr(x), _ld(x), rows, cols, _ptr(mean_rstd), _ptr(gamma), _ptr(beta), act, _ptr(out_f32),
            _ld(out_f32) if out_f32 is not None else 0, *_planes(out_split))


def bn_bwd_reduce(x, dy, mean_rstd, gamma, beta, act, sums):
    rows, cols = x.shape
    _launch("mtt_bn_bwd_reduce", _ptr(x), _ld(x), _ptr(dy), _ld(dy), rows, cols, _ptr(mean_rstd), _ptr(gamma),
            _ptr(beta), act, _ptr(sums))


def bn_bwd_apply(x, dy, mean_rstd, gamma, beta, act, sums, count, dx):
    rows, cols = x.shape
    _launch("mtt_bn_bwd_apply", _ptr(x), _ld(x), _ptr(dy), _ld(dy), rows, cols, _ptr(mean_rstd), _ptr(gamma),
            _ptr(beta), act, _ptr(sums), float(count), _ptr(dx), _ld(dx))


def attn_delta(dO, o, delta, *, B, N, H, head_dim):
    """delta [B*H*N] = rowdot(dO, O) per head: dO fp32 [B*N, H*head_dim], o = the forward's attention output (Split)."""
    _launch("mtt_attn_delta", _ptr(dO), _ld(dO), *o.planes(), B, N, H, head_dim, _ptr(delta))


def attn_softmax_bwd(S, dP, delta, *, BH, N, scale, d_raw, T, ds, pt=None, dst=None):
    """S, dP fp32 [BH*N, ld] (read only), delta fp32 [BH*N] -> Splits ds [BH*N queries, >= N], and optionally pt = P^T,
    dst = dS^T [BH*N keys, >= N queries] (same ld as ds)."""
    assert (pt is None) == (dst is None) and (pt is None or pt.ld == dst.ld == ds.ld)
    _launch("mtt_attn_softmax_bwd", _ptr(S), _ptr(dP), _ptr(delta), _ld(S), BH, N, float(scale), _ptr(d_raw), T,
            *ds.planes()[:2], *_planes(pt)[:2], *_planes(dst)[:2], ds.ld)


def bilinear_bwd(dy, *, nchw, B, h, w, Cdim, H2, W2, dx, accumulate=False):
    _launch("mtt_bilinear_bwd", _ptr(dy), 0 if nchw else _ld(dy), int(nchw), B, h, w, Cdim, H2, W2, _ptr(dx), _ld(dx),
            int(accumulate))


def gate_bwd(x, x_group_rows, x_row_offset, prompt_logits, chan_lg, task, dys, dyc, dx, d_prompt_logits, d_chan_lg, *, B,
             T, N, H, Cdim, gh, gw, nh, nw):
    _launch("mtt_gate_bwd", _ptr(x), _ld(x), x_group_rows, x_row_offset, _ptr(prompt_logits), _ptr(chan_lg), task, B, T,
            N, H, Cdim, gh, gw, nh, nw, _ptr(dys), _ptr(dyc), _ld(dys), _ptr(dx), _ld(dx), _ptr(d_prompt_logits),
            _ptr(d_chan_lg))


def chan_logits_bwd(d_rc, cp, xn, dcp, dxn, *, B, N, T, Cdim, gh, gw, nh, nw):
    _launch("mtt_chan_logits_bwd", _ptr(d_rc), _ptr(cp), *xn.planes(), B, N, T, Cdim, gh, gw, nh, nw, _ptr(dcp),
            _ptr(dxn), _ld(dxn))


def ctr_bwd(dnew, F, prompt_logits, w0, b0, w2, d_prompt_logits, dw0, db0, dw2, db2, *, T, M, Cdim, ld, rows_per_batch, B,
            H, N):
    ws = torch.empty(B * T * T, dtype=torch.float32, device=dnew.device)
    _launch("mtt_ctr_bwd", _ptr(dnew), _ptr(F), T, M, Cdim, ld, rows_per_batch, _ptr(prompt_logits), B, H, N, _ptr(w0),
            _ptr(b0), _ptr(w2), _ptr(ws), _ptr(d_prompt_logits), _ptr(dw0), _ptr(db0), _ptr(dw2), _ptr(db2))


def im2col3x3_t(x, *, B, H, W, Cdim, nsplit=2):
    """NHWC fp32 [B*H*W, C] -> Split [C*9, B*H*W]: rows (c, ky, kx)."""
    P = B * H * W
    out = Split(Cdim * 9, P, x.device, nsplit)
    _launch("mtt_im2col3x3_t", _ptr(x), _ld(x), B, H, W, Cdim, *out.planes())
    return out


def im2col_patch_t(img, patch, nsplit=2):
    """NCHW fp32 image -> Split [Cin*patch*patch, B*gh*gw]."""
    B, Cin, H, W = img.shape
    cols = B * (H // patch) * (W // patch)
    out = Split(Cin * patch * patch, cols, img.device, nsplit)
    _launch("mtt_im2col_patch_t", _ptr(img), B, Cin, H, W, patch, *out.planes())
    return out


def sumsq(g, out, accumulate=False):
    _launch("mtt_sumsq", _ptr(g), g.numel(), _ptr(out), int(accumulate))


def adam_step(p, g, m, v, *, lr, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, step, gnorm_sq=None, max_norm=0.0,
              grad_scale=1.0):
    _launch("mtt_adam_step", _ptr(p), _ptr(g), _ptr(m), _ptr(v), p.numel(), float(lr), float(betas[0]), float(betas[1]),
            float(eps), float(weight_decay), int(step), _ptr(gnorm_sq), float(max_norm), float(grad_scale))
