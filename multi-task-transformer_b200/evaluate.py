"""The reference's PerformanceMeter on the device (TP/evaluation/evaluate_utils.py:13-66, IP/evaluation/evaluate_utils.py).

``update(pred, gt)`` enqueues one library kernel per task (csrc/metrics.cu) that adds the batch's statistics into a
device state buffer: no host synchronisation, nothing allocated after the first update, so a validation loop can be
captured in a CUDA graph together with ``predict()``. ``get_score()`` copies the state to the host once and applies the
reference's formulas and guards in Python. ``pred`` is ``predict()``'s dict (or the reference's ``get_output``
results, the same format): int64 class maps, fp32 maps, ``[B,H,W,3]`` normals; ``gt`` the labels as the reference's
loader yields them (fp32 ``[B,C,H,W]``, 255 = ignore). There is no CPU path: ``update`` raises on CPU tensors.

The two reference projects run the same statistics and differ only in (``diff -r TaskPrompter/evaluation
InvPT/evaluation``):
  - ``get_score`` scaling: TaskPrompter reports mIoU and maxF times 100 (TP eval_semseg.py:95, eval_human_parts.py:56,
    eval_sal.py:78), InvPT as fractions (IP eval_semseg.py:85, eval_human_parts.py:56, eval_sal.py:78);
  - the depth mask: ``depth_min < gt < depth_max`` (TP evaluate_utils.py:59, eval_depth.py:36) against
    ``gt != ignore_index`` (IP evaluate_utils.py:59, eval_depth.py DepthMeter);
  - Cityscapes3D semseg (19 classes), which only TaskPrompter has (TP eval_semseg.py:54-57).
``reference=`` selects exactly those.

    from mtt_b200.evaluate import PerformanceMeter      # instead of evaluation.evaluate_utils's
"""
import numpy as np
import torch

from . import ops

REFERENCES = ("TaskPrompter", "InvPT")

VOC_CATEGORY_NAMES = ['background',
                      'aeroplane', 'bicycle', 'bird', 'boat', 'bottle',
                      'bus', 'car', 'cat', 'chair', 'cow',
                      'diningtable', 'dog', 'horse', 'motorbike', 'person',
                      'pottedplant', 'sheep', 'sofa', 'train', 'tvmonitor']
NYU_CATEGORY_NAMES = ['wall', 'floor', 'cabinet', 'bed', 'chair',
                      'sofa', 'table', 'door', 'window', 'bookshelf',
                      'picture', 'counter', 'blinds', 'desk', 'shelves',
                      'curtain', 'dresser', 'pillow', 'mirror', 'floor mat',
                      'clothes', 'ceiling', 'books', 'refridgerator', 'television',
                      'paper', 'towel', 'shower curtain', 'box', 'whiteboard',
                      'person', 'night stand', 'toilet', 'sink', 'lamp',
                      'bathtub', 'bag', 'otherstructure', 'otherfurniture', 'otherprop']
CITYSCAPES_CATEGORY_NAMES = ['road', 'sidewalk', 'building', 'wall', 'fence',
                             'pole', 'traffic_light', 'traffic_sign', 'vegetation', 'terrain',
                             'sky', 'person', 'rider', 'car', 'truck', 'bus', 'train',
                             'motorcycle', 'bicycle']
PART_CATEGORY_NAMES = ['background', 'head', 'torso', 'uarm', 'larm', 'uleg', 'lleg']


def _get(p, key):
    """p[key] or p.key: the reference passes an EasyDict and reads it both ways."""
    try:
        return p[key]
    except (KeyError, TypeError):
        return getattr(p, key)


class _DeviceMeter:
    """One task's statistics in a device buffer of int64 words (layout: csrc/metrics.cu). The buffer is allocated on
    the first update's device, or handed in by a PerformanceMeter that packs all its tasks into one buffer."""
    kind = None

    def __init__(self):
        self.state = None

    @property
    def n(self):
        return 0

    def words(self):
        return ops.meter_state_bytes(self.kind, self.n) // 8

    def _bind(self, state):
        self.state = state

    def _ensure(self, device):
        if self.state is None:
            self._bind(torch.zeros(self.words(), dtype=torch.int64, device=device))
        elif self.state.device != device:
            raise RuntimeError(f"meter state lives on {self.state.device}, the update's tensors on {device}")

    def reset(self):
        if self.state is not None:
            ops.meter_reset(self.state, self.kind, self.n)

    def update(self, pred, gt):
        self._check_device(pred, gt)
        self._ensure(pred.device)
        self._update(pred.contiguous(), gt.contiguous())

    def _check_device(self, pred, gt):
        if not (isinstance(pred, torch.Tensor) and isinstance(gt, torch.Tensor) and pred.is_cuda and gt.is_cuda):
            raise RuntimeError(f"{type(self).__name__}.update: the meters run on the GPU only (no CPU path); got "
                               f"{getattr(pred, 'device', type(pred))} / {getattr(gt, 'device', type(gt))}")

    def host_words(self):
        """One device-to-host copy of the state (int64 numpy array)."""
        if self.state is None:
            return np.zeros(self.words(), dtype=np.int64)
        return self.state.cpu().numpy()

    def get_score(self, verbose=True):
        return self.score(self.host_words(), verbose)

    def score(self, words, verbose=True):
        """The reference's get_score over a host copy of the state words."""
        raise NotImplementedError


def _f64(words, i):
    return float(np.asarray(words[i:i + 1], dtype=np.int64).view(np.float64)[0])


class ConfusionMeter(_DeviceMeter):
    """SemsegMeter (eval_semseg.py:40-107) and HumanPartsMeter (eval_human_parts.py:20-66): tp / fp / fn per class
    from a (gt bin, prediction bin) histogram whose last bin holds every value that is neither a class nor ignore."""
    kind = ops.METER_CONFUSION

    def __init__(self, n_classes, cat_names, ignore_idx=255, scale=100.0, title="Semantic Segmentation", pad=20,
                 always_print=False):
        super().__init__()
        self.n_classes, self.cat_names, self.ignore_idx = int(n_classes), list(cat_names), ignore_idx
        self.scale, self.title, self.pad, self.always_print = scale, title, pad, always_print

    @property
    def n(self):
        return self.n_classes

    def _update(self, pred, gt):
        ops.meter_confusion_update(pred, gt, self.n_classes, self.ignore_idx, self.state)

    def counts(self, words):
        """(tp, fp, fn) int64 arrays of length n_classes, as the reference's per-class == comparisons count them."""
        nb = self.n_classes + 1
        M = np.asarray(words[:nb * nb], dtype=np.int64).reshape(nb, nb)
        d = np.diag(M)[:self.n_classes]
        tp = d
        fp = M.sum(axis=0)[:self.n_classes] - d
        fn = M.sum(axis=1)[:self.n_classes] - d
        return tp, fp, fn

    def score(self, words, verbose=True):
        tp, fp, fn = self.counts(words)
        jac = [0] * self.n_classes
        for i in range(self.n_classes):
            jac[i] = float(tp[i]) / max(float(tp[i] + fp[i] + fn[i]), 1e-8)
        eval_result = {"mIoU": np.mean(jac) * self.scale}             # x * 1.0 == x: InvPT's fraction
        if verbose or self.always_print:
            print('\n{0:s} mIoU: {1:.4f}\n'.format(self.title, 100 * np.mean(jac)))
            for i in range(len(jac)):
                print('{0:s}{1:s}{2:.4f}'.format(self.cat_names[i], ' ' * max(self.pad - len(self.cat_names[i]), 0),
                                                 100 * jac[i]))
        return eval_result


class SaliencyMeter(_DeviceMeter):
    """SaliencyMeter (eval_sal.py:12-79): TP / PP / AP per threshold of sigmoid(pred / 255) over valid pixels."""
    kind = ops.METER_SALIENCY

    def __init__(self, ignore_index=255, threshold_step=0.05, beta_squared=0.3, scale=100.0):
        super().__init__()
        self.ignore_index, self.beta_squared, self.scale = ignore_index, beta_squared, scale
        self.thresholds = torch.arange(threshold_step, 1, threshold_step)      # fp32, as :16
        self._thr_dev = None

    @property
    def n(self):
        return len(self.thresholds)

    def _ensure(self, device):
        super()._ensure(device)
        if self._thr_dev is None:
            self._thr_dev = self.thresholds.to(device)

    def _update(self, pred, gt):
        ops.meter_saliency_update(pred, gt, self._thr_dev, self.ignore_index, self.state)

    def counts(self, words):
        T = self.n
        w = np.asarray(words[:3 * T], dtype=np.int64)
        return w[:T], w[T:2 * T], w[2 * T:]

    def score(self, words, verbose=False):
        tp, pp, ap = (torch.from_numpy(np.ascontiguousarray(c)).float() for c in self.counts(words))
        precision = tp / pp                                                          # :67-76
        recall = tp / ap
        num = (1 + self.beta_squared) * precision * recall
        denom = self.beta_squared * precision + recall
        fscore = num / denom
        fscore[fscore != fscore] = 0
        return {"maxF": fscore.max().item() * self.scale}


class NormalsMeter(_DeviceMeter):
    """NormalsMeter (eval_normals.py:27-51): mean angular error in degrees over valid pixels."""
    kind = ops.METER_NORMALS

    def __init__(self, ignore_index=255):
        super().__init__()
        self.ignore_index = ignore_index

    def _update(self, pred, gt):
        ops.meter_normals_update(pred, gt, self.ignore_index, self.state)

    def counts(self, words):
        return _f64(words, 0), int(words[1])

    def score(self, words, verbose=False):
        sum_deg_diff, total = self.counts(words)
        return {"mean": sum_deg_diff / total}


class DepthMeter(_DeviceMeter):
    """DepthMeter (TP eval_depth.py:19-71 with the range mask; IP eval_depth.py with the ignore mask). Values <= 0
    count as 1e-9 as in :41-42, but the caller's tensors are not modified."""
    kind = ops.METER_DEPTH

    def __init__(self, max_depth=None, min_depth=None, ignore_index=None):
        super().__init__()
        self.max_depth, self.min_depth, self.ignore_index = max_depth, min_depth, ignore_index
        if ignore_index is None and (max_depth is None or min_depth is None):
            raise ValueError("DepthMeter needs min_depth and max_depth (TaskPrompter) or ignore_index (InvPT)")

    def _update(self, pred, gt):
        if self.ignore_index is None:
            ops.meter_depth_update(pred, gt, self.state, min_depth=self.min_depth, max_depth=self.max_depth)
        else:
            ops.meter_depth_update(pred, gt, self.state, ignore_index=self.ignore_index)

    def counts(self, words):
        return (float(words[0]),) + tuple(_f64(words, i) for i in range(1, 5))

    def score(self, words, verbose=True):
        n_valid, total_rmses, total_log_rmses, abs_rel, sq_rel = self.counts(words)
        eval_result = {"rmse": np.sqrt(total_rmses / n_valid), "log_rmse": np.sqrt(total_log_rmses / n_valid),
                       "abs_rel": abs_rel / n_valid, "sq_rel": sq_rel / n_valid}
        if verbose:
            print('Results for depth prediction')
            for x in eval_result:
                print('{0:s}{1:s}{2:.4f}'.format(x, ' ' * max(15 - len(x), 0), eval_result[x]))
        return eval_result


class EdgeMeter(_DeviceMeter):
    """EdgeMeter (eval_edge.py:13-44): the balanced BCE of pred / 255, averaged over all valid pixels of all updates
    (the reference's sum of loss * numel over updates is the sum of the per-pixel losses)."""
    kind = ops.METER_EDGE

    def __init__(self, pos_weight, ignore_index=255):
        super().__init__()
        self.pos_weight, self.ignore_index = pos_weight, ignore_index

    def _update(self, pred, gt):
        ops.meter_edge_update(pred, gt, self.pos_weight, self.ignore_index, self.state)

    def counts(self, words):
        return _f64(words, 0), int(words[1])

    def score(self, words, verbose=True):
        loss, n = self.counts(words)
        eval_dict = {"loss": loss / n}
        if verbose:
            print('\n Edge Detection Evaluation')
            print('Edge Detection Loss %.3f' % (eval_dict['loss']))
        return eval_dict


def get_single_task_meter(p, database, task, reference="TaskPrompter"):
    """Meter for one task (evaluate_utils.py:35-66): the reference's constructor arguments from p."""
    if reference not in REFERENCES:
        raise ValueError(f"reference must be one of {REFERENCES}, got {reference!r}")
    scale = 100.0 if reference == "TaskPrompter" else 1.0
    ignore_index = _get(p, "ignore_index")
    if task == "semseg":
        dbs = {"PASCALContext": (20, VOC_CATEGORY_NAMES, True), "NYUD": (40, NYU_CATEGORY_NAMES, False)}
        if reference == "TaskPrompter":
            dbs["Cityscapes3D"] = (19, CITYSCAPES_CATEGORY_NAMES, False)
        if database not in dbs:
            raise NotImplementedError(f"semseg evaluation on {database!r} ({reference})")
        n, names, has_bg = dbs[database]
        return ConfusionMeter(n + int(has_bg), names, ignore_index, scale)
    elif task == "human_parts":
        if database != "PASCALContext":
            raise NotImplementedError(f"human_parts evaluation on {database!r}")
        return ConfusionMeter(7, PART_CATEGORY_NAMES, ignore_index, scale, title="Human Parts", pad=15,
                              always_print=True)
    elif task == "normals":
        return NormalsMeter(ignore_index=ignore_index)
    elif task == "sal":
        return SaliencyMeter(ignore_index=ignore_index, threshold_step=0.05, beta_squared=0.3, scale=scale)
    elif task == "depth":
        if reference == "TaskPrompter":
            tasks = _get(p, "TASKS")
            return DepthMeter(max_depth=_get(tasks, "depth_max"), min_depth=_get(tasks, "depth_min"))
        return DepthMeter(ignore_index=ignore_index)
    elif task == "edge":
        return EdgeMeter(pos_weight=_get(p, "edge_w"), ignore_index=ignore_index)
    raise NotImplementedError(f"no evaluation meter for task {task!r}")


class PerformanceMeter:
    """A general performance meter which shows performance across one or more tasks (evaluate_utils.py:13-33). All
    tasks share one device state buffer, so get_score() is one device-to-host copy."""

    def __init__(self, p, tasks, reference="TaskPrompter"):
        self.database = _get(p, "train_db_name")
        self.tasks = list(tasks)
        self.reference = reference
        self.meters = {t: get_single_task_meter(p, self.database, t, reference) for t in self.tasks}
        self.state = None

    def _ensure(self, device):
        if self.state is not None:
            return
        sizes = [self.meters[t].words() for t in self.tasks]
        self.state = torch.zeros(sum(sizes), dtype=torch.int64, device=device)
        off = 0
        for t, w in zip(self.tasks, sizes):
            self.meters[t]._bind(self.state[off:off + w])
            off += w

    def reset(self):
        for t in self.tasks:
            self.meters[t].reset()

    def update(self, pred, gt):
        for t in self.tasks:
            self.meters[t]._check_device(pred[t], gt[t])
        self._ensure(pred[self.tasks[0]].device)
        for t in self.tasks:
            self.meters[t].update(pred[t], gt[t])

    def get_score(self, verbose=True):
        host = np.zeros(0, dtype=np.int64) if self.state is None else self.state.cpu().numpy()
        eval_dict, off = {}, 0
        for t in self.tasks:
            m = self.meters[t]
            w = m.words()
            eval_dict[t] = m.score(host[off:off + w] if self.state is not None else np.zeros(w, np.int64), verbose)
            off += w
        return eval_dict
