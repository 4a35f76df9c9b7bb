"""CPU restatement of the reference projects' evaluation meters (TP/evaluation/*.py, IP/evaluation/*.py), written
from the algorithm with the reference's per-class / per-threshold loops and host reads, in plain torch / numpy.
TEST INFRASTRUCTURE: the GPU tests compare mtt_b200.evaluate against it (the GPU machine has no reference tree), and
scripts/eval_throughput.py runs it on CUDA tensors as the reference-style baseline (same syncs as the reference).

PerformanceMeter(p, tasks, reference) mirrors evaluate_utils.py:13-66; reference="TaskPrompter" or "InvPT" selects
the only differences between the two projects: mIoU / maxF times 100 or not, the depth mask (range vs ignore index)
and Cityscapes3D semseg. counters() returns each meter's accumulated statistics under the reference's attribute
names. Deviations: inputs are never modified (TP eval_depth.py:41-42 clamps the caller's tensors in place), and
EdgeMeter accepts batch 1 (the reference's pred[valid_mask] raises an IndexError there: its gt.squeeze() drops the
batch axis and pred keeps it).
"""
import numpy as np
import torch
import torch.nn.functional as F

VOC_N, NYU_N, CS_N, PARTS_N = 21, 40, 19, 7


def _get(p, key):
    try:
        return p[key]
    except (KeyError, TypeError):
        return getattr(p, key)


class ConfusionMeter:
    """SemsegMeter (eval_semseg.py:40-107), HumanPartsMeter (eval_human_parts.py:20-66)."""

    def __init__(self, n_classes, ignore_idx=255, scale=100.0):
        self.n_classes, self.ignore_idx, self.scale = n_classes, ignore_idx, scale
        self.reset()

    def reset(self):
        self.tp = [0] * self.n_classes
        self.fp = [0] * self.n_classes
        self.fn = [0] * self.n_classes

    @torch.no_grad()
    def update(self, pred, gt):                                            # eval_semseg.py:70-81
        pred, gt = pred.squeeze(), gt.squeeze()
        valid = gt != self.ignore_idx
        for i in range(self.n_classes):
            tmp_gt, tmp_pred = gt == i, pred == i
            self.tp[i] += torch.sum(tmp_gt & tmp_pred & valid).item()
            self.fp[i] += torch.sum(~tmp_gt & tmp_pred & valid).item()
            self.fn[i] += torch.sum(tmp_gt & ~tmp_pred & valid).item()

    def counters(self):
        return {"tp": list(self.tp), "fp": list(self.fp), "fn": list(self.fn)}

    def get_score(self, verbose=False):                                    # :88-95
        jac = [float(self.tp[i]) / max(float(self.tp[i] + self.fp[i] + self.fn[i]), 1e-8)
               for i in range(self.n_classes)]
        return {"mIoU": np.mean(jac) * self.scale}


class SaliencyMeter:
    """eval_sal.py:12-79 with threshold_step=0.05, beta_squared=0.3 (evaluate_utils.py:53)."""

    def __init__(self, ignore_index=255, threshold_step=0.05, beta_squared=0.3, scale=100.0):
        self.ignore_index, self.beta_squared, self.scale = ignore_index, beta_squared, scale
        self.thresholds = torch.arange(threshold_step, 1, threshold_step)
        self.reset()

    def reset(self):
        T = len(self.thresholds)
        self.true_positives, self.predicted_positives, self.actual_positives = (torch.zeros(T) for _ in range(3))

    @torch.no_grad()
    def update(self, preds, target):                                       # :22-60
        preds = preds.float() / 255.
        if target.shape[1] == 1:
            target = target.squeeze(1)
        assert preds.shape == target.shape
        preds = torch.sigmoid(preds)                                       # :43, on the post-processed map
        valid = target != self.ignore_index
        for idx, thresh in enumerate(self.thresholds):
            f_preds = torch.masked_select((preds >= thresh).long(), valid)
            f_target = torch.masked_select(target.long(), valid)
            self.true_positives[idx] += torch.sum(f_preds * f_target).cpu()
            self.predicted_positives[idx] += torch.sum(f_preds).cpu()
            self.actual_positives[idx] += torch.sum(f_target).cpu()

    def counters(self):
        return {"true_positives": self.true_positives.clone(), "predicted_positives": self.predicted_positives.clone(),
                "actual_positives": self.actual_positives.clone()}

    def get_score(self, verbose=False):                                    # :63-79
        precision = self.true_positives.float() / self.predicted_positives
        recall = self.true_positives.float() / self.actual_positives
        fscore = (1 + self.beta_squared) * precision * recall / (self.beta_squared * precision + recall)
        fscore[fscore != fscore] = 0
        return {"maxF": fscore.max().item() * self.scale}


def normalize_tensor(x, dim):                                              # eval_normals.py:19-25
    norm = torch.norm(x, p="fro", dim=dim, keepdim=True)
    zero = norm == 0
    out = x.div(torch.where(zero, torch.ones_like(norm), norm))
    return torch.where(zero.expand_as(out), torch.zeros_like(out), out)


class NormalsMeter:
    """eval_normals.py:27-51."""

    def __init__(self, ignore_index=255):
        self.ignore_index = ignore_index
        self.reset()

    def reset(self):
        self.sum_deg_diff, self.total = 0, 0

    @torch.no_grad()
    def update(self, pred, gt):                                            # :33-45
        pred = 2 * pred.permute(0, 3, 1, 2) / 255 - 1
        valid = (gt != self.ignore_index).all(dim=1)
        pred, gt = normalize_tensor(pred, 1), normalize_tensor(gt, 1)
        deg = torch.rad2deg(2 * torch.atan2(torch.norm(pred - gt, dim=1), torch.norm(pred + gt, dim=1)))
        deg = torch.masked_select(deg, valid)
        self.sum_deg_diff += torch.sum(deg).cpu().item()
        self.total += deg.numel()

    def counters(self):
        return {"sum_deg_diff": self.sum_deg_diff, "total": self.total}

    def get_score(self, verbose=False):
        return {"mean": self.sum_deg_diff / self.total}


class DepthMeter:
    """TP eval_depth.py:19-71 (mask min_depth < gt < max_depth) or IP eval_depth.py DepthMeter (mask gt != ignore)."""

    def __init__(self, max_depth=None, min_depth=None, ignore_index=None):
        self.max_depth, self.min_depth, self.ignore_index = max_depth, min_depth, ignore_index
        self.reset()

    def reset(self):
        self.total_rmses = self.total_log_rmses = self.n_valid = self.abs_rel = self.sq_rel = 0.0

    @torch.no_grad()
    def update(self, pred, gt):                                            # :31-54
        pred, gt = pred.squeeze(), gt.squeeze()
        if self.ignore_index is None:
            mask = torch.logical_and(gt < self.max_depth, gt > self.min_depth)
        else:
            mask = gt != self.ignore_index
        self.n_valid += mask.float().sum().item()
        gt = torch.where(gt <= 0, torch.full_like(gt, 1e-9), gt)           # :41-42 on copies
        pred = torch.where(pred <= 0, torch.full_like(pred, 1e-9), pred)
        g, q = gt[mask], pred[mask]
        self.total_log_rmses += torch.pow(torch.log(g) - torch.log(q), 2).sum().item()
        self.total_rmses += torch.pow(g - q, 2).sum().item()
        self.abs_rel += (torch.abs(g - q) / g).sum().item()
        self.sq_rel += (((g - q) ** 2) / g).sum().item()

    def counters(self):
        return {"n_valid": self.n_valid, "total_rmses": self.total_rmses, "total_log_rmses": self.total_log_rmses,
                "abs_rel": self.abs_rel, "sq_rel": self.sq_rel}

    def get_score(self, verbose=False):                                    # :56-61
        return {"rmse": np.sqrt(self.total_rmses / self.n_valid), "log_rmse": np.sqrt(self.total_log_rmses / self.n_valid),
                "abs_rel": self.abs_rel / self.n_valid, "sq_rel": self.sq_rel / self.n_valid}


def balanced_bce(output, label, pos_weight, ignore_index):
    """BalancedBinaryCrossEntropyLoss.forward with a fixed pos_weight (TP/losses/loss_functions.py:57-87)."""
    mask = label != ignore_index
    lab, out = torch.masked_select(label, mask), torch.masked_select(output, mask)
    w = torch.as_tensor(pos_weight, device=output.device)
    factor = 1. / (1 - w)
    return F.binary_cross_entropy_with_logits(out, lab, pos_weight=w * factor, reduction="mean") / factor


class EdgeMeter:
    """eval_edge.py:13-44."""

    def __init__(self, pos_weight, ignore_index=255):
        self.pos_weight, self.ignore_index = pos_weight, ignore_index
        self.reset()

    def reset(self):
        self.loss, self.n = 0, 0

    @torch.no_grad()
    def update(self, pred, gt):                                            # :21-31
        gt = gt.squeeze()
        pred = pred.reshape(gt.shape)
        valid = gt != self.ignore_index
        pred, gt = pred[valid].float() / 255., gt[valid]
        loss = balanced_bce(pred, gt, self.pos_weight, self.ignore_index).item()
        self.n += gt.numel()
        self.loss += gt.numel() * loss

    def counters(self):
        return {"loss": self.loss, "n": self.n}

    def get_score(self, verbose=False):
        return {"loss": self.loss / self.n}


def get_single_task_meter(p, database, task, reference="TaskPrompter"):
    """evaluate_utils.py:35-66 of either project."""
    scale = 100.0 if reference == "TaskPrompter" else 1.0
    ign = _get(p, "ignore_index")
    if task == "semseg":
        n = {"PASCALContext": VOC_N, "NYUD": NYU_N}
        if reference == "TaskPrompter":
            n["Cityscapes3D"] = CS_N
        if database not in n:
            raise NotImplementedError(database)
        return ConfusionMeter(n[database], ign, scale)
    if task == "human_parts":
        assert database == "PASCALContext"
        return ConfusionMeter(PARTS_N, ign, scale)
    if task == "normals":
        return NormalsMeter(ign)
    if task == "sal":
        return SaliencyMeter(ign, 0.05, 0.3, scale)
    if task == "depth":
        if reference == "TaskPrompter":
            t = _get(p, "TASKS")
            return DepthMeter(max_depth=_get(t, "depth_max"), min_depth=_get(t, "depth_min"))
        return DepthMeter(ignore_index=ign)
    if task == "edge":
        return EdgeMeter(_get(p, "edge_w"), ign)
    raise NotImplementedError(task)


class PerformanceMeter:
    def __init__(self, p, tasks, reference="TaskPrompter"):
        self.database = _get(p, "train_db_name")
        self.tasks = list(tasks)
        self.meters = {t: get_single_task_meter(p, self.database, t, reference) for t in self.tasks}

    def reset(self):
        for m in self.meters.values():
            m.reset()

    def update(self, pred, gt):
        for t in self.tasks:
            self.meters[t].update(pred[t], gt[t])

    def counters(self):
        return {t: self.meters[t].counters() for t in self.tasks}

    def get_score(self, verbose=False):
        return {t: self.meters[t].get_score(verbose) for t in self.tasks}


# ---- synthetic batches -------------------------------------------------------------------------------------------
SAL_THRESHOLDS = torch.arange(0.05, 1, 0.05)


def synthetic_batch(tasks, n_classes, B, H, W, g, all_ignore=(), depth_bounds=(0.0, 80.0)):
    """predict()-format predictions and loader-format labels for `tasks`, drawn from the torch CPU generator g. They
    cover ignore pixels, labels outside the class range (and non-integer ones), predictions outside it, zero-norm
    normals (prediction and label), labels ignored in only some normal channels, depth at the range bounds and <= 0,
    and images whose labels are all ignore (batch indices in all_ignore). Saliency maps keep sigmoid(pred / 255) at
    least 1e-6 away from every threshold, so the counts do not depend on the last bit of the sigmoid. Every float
    value lies on the fp16 grid and every class map fits int8, so pack_updates() stores them exactly in little space."""
    pred, gt = {}, {}
    r = lambda *s: torch.rand(*s, generator=g)
    q = lambda x: x.half().float()                                           # onto the fp16 grid
    hole = lambda frac, c=1: (r(B, 1, H, W) < frac).expand(-1, c, -1, -1)
    for t in tasks:
        if t in ("semseg", "human_parts"):
            n = n_classes[t]
            p = torch.randint(0, n, (B, H, W), generator=g)
            p[r(B, H, W) < 0.03] = n + 1                                     # outside the class range
            y = torch.randint(0, n, (B, 1, H, W), generator=g).float()
            y = torch.where(r(B, 1, H, W) < 0.3, p.unsqueeze(1).float(), y)  # some agreement
            y[hole(0.1)] = 255.0
            y[hole(0.02)] = float(n + 3)                                     # neither a class nor ignore
            y[hole(0.01)] = 1.5
        elif t == "sal":
            p = q(r(B, H, W) * 255)
            prob = torch.sigmoid(p / 255.)
            near = (prob.unsqueeze(-1) - SAL_THRESHOLDS).abs().min(dim=-1).values < 1e-6
            p[near] = 255.0                                                  # sigmoid(1) = 0.731, clear of 0.70 / 0.75
            y = (r(B, 1, H, W) < 0.4).float()
            y[hole(0.05)] = 255.0
        elif t == "edge":
            p = q(r(B, H, W) * 255)
            y = (r(B, 1, H, W) < 0.2).float()
            y[hole(0.05)] = 255.0
        elif t == "normals":
            v = F.normalize(torch.randn(B, H, W, 3, generator=g), dim=3)
            v[(r(B, H, W) < 0.03)] = 0.0
            p = q((v + 1.0) * 255 / 2.0)                                     # 127.5 -> exactly 0 after :36
            y = q(F.normalize(torch.randn(B, 3, H, W, generator=g), dim=1))
            y[hole(0.03, 3)] = 0.0                                           # zero-norm label
            y[hole(0.1, 3)] = 255.0
            y[:, 1:2][hole(0.03)] = 255.0                                    # one channel ignored: still invalid
        elif t == "depth":
            lo, hi = depth_bounds
            p = q(r(B, H, W, 1) * 10)
            p[r(B, H, W, 1) < 0.05] = 0.0
            y = q(r(B, 1, H, W) * 12 + 0.01)
            y[hole(0.05)] = lo
            y[hole(0.05)] = hi
            y[hole(0.05)] = -1.0
            y[hole(0.03)] = 0.0
            y[hole(0.1)] = 255.0
        else:
            raise ValueError(t)
        for b in all_ignore:
            y[b] = 255.0
        pred[t], gt[t] = p.contiguous(), y.contiguous()
    return pred, gt


def pack_updates(updates):
    """synthetic_batch() outputs in the fixture's compact form: class maps as int8, float maps as fp16. Exact, since
    synthetic_batch draws every value on those grids; unpack_updates() restores int64 / fp32."""
    def pack(v):
        if v.dtype == torch.int64:
            assert v.min() >= -128 and v.max() <= 127
            return v.to(torch.int8)
        h = v.half()
        assert torch.equal(h.float(), v), "value off the fp16 grid"
        return h
    return [({t: pack(v) for t, v in p.items()}, {t: pack(v) for t, v in y.items()}) for p, y in updates]


def unpack_updates(packed):
    up = lambda v: v.to(torch.int64) if v.dtype == torch.int8 else v.float()
    return [({t: up(v) for t, v in p.items()}, {t: up(v) for t, v in y.items()}) for p, y in packed]
