"""BEV IoU / NMS of rotated boxes on the device: the functions of the reference's
TaskPrompter/detection_toolbox/iou3d/iou3d_utils.py (`boxes_iou_bev`, `nms_gpu`, `nms_normal_gpu`) with the same
arguments and results, on libmtt_sm90.so instead of the `iou3d_cuda` extension (SURVEY.md section 8f N4).
Unlike the reference (iou3d.cpp:117-143: blocking device-to-host copy of the mask matrix, greedy sweep on the CPU,
cudaMalloc per call) the whole NMS is enqueued on the current stream; the only synchronisation is the caller reading
how many boxes survived, which `nms_gpu` does once to size its result exactly like the reference returns it."""
import torch

from . import lib as _L
from .ops import _launch, _ptr


def _boxes(t):
    if not t.is_cuda:
        raise RuntimeError("mtt_b200.iou3d has no CPU path: boxes must be CUDA tensors")
    assert t.dim() == 2 and t.shape[1] == 5, "boxes are [N, 5] = [x1, y1, x2, y2, ry]"
    return t.detach().float().contiguous()


def boxes_overlap_bev(boxes_a, boxes_b):
    """Overlap area of every pair [M, N] (iou3d.cpp:51-71 boxes_overlap_bev_gpu)."""
    return _pairwise(boxes_a, boxes_b, 0)


def boxes_iou_bev(boxes_a, boxes_b):
    """Rotated IoU in the bird's-eye view of every pair [M, N] (iou3d_utils.py:7-24)."""
    return _pairwise(boxes_a, boxes_b, 1)


def _pairwise(boxes_a, boxes_b, mode):
    a, b = _boxes(boxes_a), _boxes(boxes_b)
    out = a.new_zeros((a.shape[0], b.shape[0]))
    if out.numel() == 0:
        return out
    _launch("mtt_boxes_bev_pairwise", _ptr(a), a.shape[0], _ptr(b), b.shape[0], mode, _ptr(out))
    return out


def nms_sorted(boxes_sorted, thresh, rotated=True):
    """boxes already in descending score order -> (keep int64 [N] on the device, num_keep int32 [1] on the device);
    enqueue-only."""
    b = _boxes(boxes_sorted)
    n = b.shape[0]
    keep = torch.zeros(max(n, 1), dtype=torch.int64, device=b.device)
    num = torch.zeros(1, dtype=torch.int32, device=b.device)
    nbytes = int(_L.load().mtt_nms_workspace_bytes(n))
    ws = torch.empty(nbytes // 8 + 1, dtype=torch.int64, device=b.device)
    _launch("mtt_nms_bev", _ptr(b), n, float(thresh), 1 if rotated else 0, _ptr(keep), _ptr(num), _ptr(ws),
            ws.numel() * 8)
    return keep[:n], num


def nms_gpu(boxes, scores, thresh, pre_maxsize=None, post_max_size=None):
    """iou3d_utils.py:27-52: indices (into `boxes`) of the boxes kept by rotated NMS, best score first."""
    order = scores.sort(0, descending=True)[1]
    if pre_maxsize is not None:
        order = order[:pre_maxsize]
    keep, num = nms_sorted(boxes[order], thresh, rotated=True)
    keep = order[keep[:int(num.item())]].contiguous()
    if post_max_size is not None:
        keep = keep[:post_max_size]
    return keep


def nms_normal_gpu(boxes, scores, thresh):
    """iou3d_utils.py:55-75: axis-aligned NMS on the [x1, y1, x2, y2] part of the boxes."""
    order = scores.sort(0, descending=True)[1]
    keep, num = nms_sorted(boxes[order], thresh, rotated=False)
    return order[keep[:int(num.item())]].contiguous()
