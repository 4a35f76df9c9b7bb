"""The evaluation meters (csrc/metrics.cu through mtt_b200.evaluate) at every validation geometry the suites run
(plan_calls.runs(("predict",))), against float64 / integer references computed from the same fp32 / int64 inputs.

At these sizes every float meter launch runs the capped grid (512 CTAs, several grid-stride passes) and its last-CTA
fixed-order sum over all 512 partial slots. Counters (confusion bins, saliency tp / pp / ap, valid-pixel counts) are
asserted exact. Each float sum is bounded from the kernel's fp32 operation sequence per pixel (U per rounding, the CUDA
math library's documented maximum errors: logf 1 ulp, expf 2 ulp, atan2f 3 ulp; one ulp is at most 2 U relative). The
per-pixel errors are combined as the rounding errors of f64_checks' model, LAM sqrt(sum b_i^2): the float inputs are
drawn off the fp16 grid, so no two pixels share inputs. A systematic error (the fp32 180 / pi of the normals meter) is
added whole, and the fp64 accumulation adds D U64 sum |t_i| with D its longest chain of additions. The worst-case sum
of the per-pixel bounds is not used: at a million pixels it exceeds what accumulating the block sums in fp32 moves a
sum by, so it could not catch that defect. test_teeth shows, on the CPU, that the bounds catch each defect they are
meant to catch."""
import functools
import math

import numpy as np
import pytest
import torch

from f64_checks import LAM, U, U64, Guarded, bce_term_bound, report
from oracle import configs
from oracle import meters_ref as R
from plan_calls import SwinGeom, run_id, runs

THREADS, MAX_BLOCKS = 256, 512            # csrc/metrics.cu kMeterThreads, kMeterMaxBlocks
PER_THREAD = {"semseg": 16, "human_parts": 16, "sal": 16, "normals": 4, "depth": 4, "edge": 4}   # meter_blocks()
TICKET = {"normals": 2, "depth": 5, "edge": 2}                   # the ticket word: after the header words
FLOAT_TASKS = {"PASCALContext": ("sal", "normals", "edge"), "NYUD": ("depth", "normals", "edge"),
               "Cityscapes3D": ("depth",)}
NCLS = {"PASCALContext": {"semseg": 21, "human_parts": 7}, "NYUD": {"semseg": 40}, "Cityscapes3D": {"semseg": 19}}
IGN = 255
CLAMP = float(np.float32(1e-9))           # the depth meters' clamp, an fp32 constant in the kernel and the reference
C_DEG = 180 / math.pi
C_DEG_F32 = float(np.float32(C_DEG))      # the normals kernel's (float)(180 / pi)
TINY = 2.0 ** -148                        # fp32 underflow of a per-pixel product

GEOMS = runs(("predict",))


def _p(database):
    return dict(train_db_name=database, ignore_index=IGN, edge_w=0.95, TASKS=dict(depth_min=0.0, depth_max=80.0))


def geometry(name, B):
    """(database, project, tasks with a meter, (H, W) of the predictions and labels) of a predict() run."""
    if name.startswith("tps_"):
        sg = SwinGeom(name, B)
        return "Cityscapes3D", "TaskPrompter", tuple(t for t in sg.tasks if t != "3ddet"), tuple(sg.out_hw)
    cfg = configs.invpt(name) if name.startswith("ip_") else configs.taskprompter(name)
    database = "PASCALContext" if "human_parts" in cfg["tasks"] else "NYUD"
    return database, ("InvPT" if name.startswith("ip_") else "TaskPrompter"), tuple(cfg["tasks"]), tuple(cfg["img_size"])


def meter_key(name, B):
    database, project, tasks, hw = geometry(name, B)
    return database, project, tasks, B, hw


# distinct meter geometries (several configs evaluate the same maps), named after their first run
DISTINCT = list({meter_key(n, B): (n, B) for n, B in reversed(GEOMS)}.values())[::-1]


def blocks(npix, task):
    return min(MAX_BLOCKS, max(1, -(-npix // (THREADS * PER_THREAD[task]))))


def chain(npix, task, updates=1):
    """Longest chain of fp64 additions of a float meter's sum: per-thread trips, the 256-thread tree, the last CTA's
    serial sum over the blocks, the add into the state per update."""
    nb = blocks(npix, task)
    return updates * (-(-npix // (nb * THREADS)) + 8 + nb + 1)


# ---- inputs -------------------------------------------------------------------------------------------------------------
def _off_grid(v, keep, g):
    """v moved off the fp16 grid by a relative 2^-11 at most, except where keep: every pixel gets its own fp32 value."""
    j = v * (1 + (torch.rand(v.shape, generator=g) - 0.5) * 2.0 ** -10)
    return torch.where(keep, v, j).contiguous()


@functools.lru_cache(maxsize=3)
def inputs(database, B, H, W):
    """meters_ref.synthetic_batch at the geometry (CPU), plus: predictions -1 and 2^32 + 1 (a 32-bit class would wrap
    into range), labels -0.0 and NaN, int64 Cityscapes labels with -1, 2^32 + 3 and 2^32 + 255 (neither a class nor
    ignore), normals predictions 1 to 4 from 127.5 in all three channels (vectors
    of length 0.014 to 0.055 after 2x / 255 - 1), float maps off the fp16
    grid."""
    tasks = list(NCLS[database]) + list(FLOAT_TASKS[database])
    g = torch.Generator().manual_seed(1000 * B + H + W)
    pred, gt = R.synthetic_batch(tasks, NCLS[database], B, H, W, g)
    r = lambda *s: torch.rand(*s, generator=g)
    for t in NCLS[database]:
        p, y = pred[t], gt[t]
        p[r(p.shape) < 0.01] = -1
        p[r(p.shape) < 0.01] = 2 ** 32 + 1
        if database == "Cityscapes3D":                         # the loader's int64 [B,H,W]
            yi = torch.where(y == y.floor(), y, torch.full_like(y, -1)).squeeze(1).long()
            yi[r(yi.shape) < 0.005] = 2 ** 32 + 3
            yi[r(yi.shape) < 0.005] = 2 ** 32 + IGN
            gt[t] = yi.contiguous()
        else:
            y[r(y.shape) < 0.002] = -0.0
            y[r(y.shape) < 0.002] = float("nan")
    if "normals" in pred:
        p = pred["normals"]
        short = (r(B, H, W) < 0.005).unsqueeze(-1).expand_as(p)
        p = torch.where(short, 127.5 + torch.sign(r(p.shape) - 0.5) * (1 + 3 * r(p.shape)), p)
        pred["normals"] = _off_grid(p, p == 127.5, g)
        gt["normals"] = _off_grid(gt["normals"], (gt["normals"] == 0) | (gt["normals"] == IGN), g)
    if "depth" in pred:
        pred["depth"] = _off_grid(pred["depth"], pred["depth"] == 0, g)
        y = gt["depth"]
        gt["depth"] = _off_grid(y, (y <= 0) | (y == 80.0) | (y == IGN), g)
    if "edge" in pred:
        pred["edge"] = _off_grid(pred["edge"], torch.zeros_like(pred["edge"], dtype=torch.bool), g)
    return pred, gt


def sal_adversarial(B, H, W, thr, seed):
    """A saliency batch whose pixels sit, one in ten, within a few fp32 steps of 255 logit(thr_k) for every threshold:
    the device sigmoid may land on either side there. The rest as synthetic_batch draws them."""
    g = torch.Generator().manual_seed(seed)
    pred, gt = R.synthetic_batch(["sal"], {}, B, H, W, g)
    p = pred["sal"]
    z = 255 * torch.logit(thr.double()).float()                # fp32 preimage of each threshold
    near = torch.rand(p.shape, generator=g) < 0.1
    k = torch.randint(0, len(thr), p.shape, generator=g)
    steps = torch.randint(-40, 41, p.shape, generator=g).float()
    pos = z[k] + steps * torch.where(z[k] == 0, torch.full_like(z[k], 2.0 ** -126), z[k].abs() * 2.0 ** -23)
    return torch.where(near, pos, p).contiguous(), gt["sal"]


# ---- float64 / integer references ----------------------------------------------------------------------------------------
def confusion_ref(pred, label, n):
    """The (n+1)^2 histogram of eval_semseg.py's comparisons: bin i where gt == i (pred == i), bin n where no class
    compares equal; pixels where gt == ignore are left out."""
    p, y = pred.reshape(-1), label.reshape(-1)
    gb, pb = torch.full_like(p, n), torch.full_like(p, n)
    for i in range(n):
        gb[y == i] = i
        pb[p == i] = i
    keep = y != IGN
    return torch.bincount((gb * (n + 1) + pb)[keep], minlength=(n + 1) ** 2)


def sal_bound(z, prob):
    """|fp32 sigmoid(pred / 255) - prob|: pred / 255 rounds (|z| u on exp), expf 2 ulp, 1 + e and the reciprocal one
    rounding each: (|z| + 8) u relative."""
    return (z.abs() + 8) * U * prob


def saliency_ref(pred, label, thr):
    """tp / pp / ap per threshold of eval_sal.py in float64, and per threshold the number of valid pixels within the
    kernel's sigmoid bound of it (amb) and their labels' sum (amb_t)."""
    z = pred.double().reshape(-1) / 255
    prob = torch.sigmoid(z)
    y = label.reshape(-1)
    keep = y != IGN
    z, prob, t = z[keep], prob[keep], y[keep].long()
    th = thr.double().to(prob.device)
    tp, pp, amb, amb_t = [], [], [], []
    d = sal_bound(z, prob)
    for k in range(len(th)):
        f = prob >= th[k]
        a = (prob - th[k]).abs() <= d
        tp.append(int(t[f].sum()))
        pp.append(int(f.sum()))
        amb.append(int(a.sum()))
        amb_t.append(int(t[a].abs().sum()))
    ap = int(t.sum())
    return np.array(tp), np.array(pp), np.full(len(th), ap), np.array(amb), np.array(amb_t)


class FloatRef:
    """A float meter's reference: per-pixel float64 terms of each sum, their bounds b, the valid mask, the pixels whose
    errors are shared (the same rounding of the same values: a zero normals vector, a clamped depth), and the systematic
    relative error of every term. Independent pixels combine as LAM sqrt(sum b_i^2), shared ones add sum b_i."""

    def __init__(self, terms, bounds, keep, shared, systematic=0.0):
        self.terms, self.bounds, self.keep, self.systematic = terms, bounds, keep, systematic
        self.shared = shared & keep

    def sums(self):
        return [float(t[self.keep].sum()) for t in self.terms]

    def count(self):
        return int(self.keep.sum())

    def sum_bounds(self, npix, task, updates=1):
        D = chain(npix, task, updates)
        own = self.keep & ~self.shared
        out = []
        for t, b in zip(self.terms, self.bounds):
            a = float(t[self.keep].abs().sum())
            out.append(LAM * math.sqrt(float((b[own] ** 2).sum())) + float(b[self.shared].sum()) + self.systematic * a +
                       2 * D * U64 * a)
        return out


def normals_ref(pred, label):
    """eval_normals.py in float64. Per pixel (radians): the prediction 2x / 255 - 1 rounds twice, a_k = u (|2x / 255| +
    |p_k|) per channel (0 where x = 127.5: exact), and near x = 127.5 that cancellation turns the direction of a short
    vector by up to 2 |a| / |p| (at most pi); normalising rounds each channel (sqrt(2) u of angle per vector); |p - g| and
    |p + g| carry 3.5 u each (sin(theta) 7 u of angle); atan2f 3 ulp of theta / 2 (6 u theta). Degrees: one rounding
    (u deg); the fp32 180 / pi is a systematic relative error of every term."""
    x = pred.double().reshape(-1, 3)
    gl = label.double().permute(0, 2, 3, 1).reshape(-1, 3)
    keep = (gl != IGN).all(1)
    q = 2 * x / 255
    p = q - 1
    pn, gn = R.normalize_tensor(p, 1), R.normalize_tensor(gl, 1)
    th = 2 * torch.atan2((pn - gn).norm(dim=1), (pn + gn).norm(dim=1))
    deg = th * C_DEG
    a = (U * (q.abs() + p.abs()) * (x != 127.5)).norm(dim=1)
    r = p.norm(dim=1)
    turn = torch.where(r > 0, 2 * a / r.clamp_min(1e-300), torch.zeros_like(r)).clamp(max=math.pi)
    e_th = turn + 3 * U + 7 * U * th.sin() + 6 * U * th
    b = C_DEG * e_th * (1 + 8 * U) + U * deg + TINY
    shared = (r == 0) | (gl.norm(dim=1) == 0)           # 2 atan2f(A, A) of the same A: one value for all of them
    return FloatRef([deg], [b], keep, shared, systematic=abs(C_DEG_F32 - C_DEG) / C_DEG)


def depth_terms(pred, label, use_range, clamp=True):
    gd, pd = label.double().reshape(-1), pred.double().reshape(-1)
    keep = (gd > 0) & (gd < 80) if use_range else gd != IGN
    g = torch.where(gd <= 0, torch.full_like(gd, CLAMP), gd) if clamp else gd
    p = torch.where(pd <= 0, torch.full_like(pd, CLAMP), pd) if clamp else pd
    return g, p, keep


def depth_ref(pred, label, use_range, clamp=True):
    """eval_depth.py in float64 (TaskPrompter: 0 < gt < 80; InvPT: gt != 255, so gt <= 0 counts, as 1e-9). Per pixel:
    d = g - p rounds once; d^2 3u; logf 1 ulp each (2 u |log|), their difference u, so dl^2 within 2 |dl| e + e^2 + u
    dl^2; |d| / g 2u; d^2 / g 4u."""
    g, p, keep = depth_terms(pred, label, use_range, clamp)
    shared = (label.reshape(-1) <= 0) | (pred.reshape(-1) <= 0)        # logf(1e-9): one error for all of them
    d = g - p
    lg, lp = g.log(), p.log()
    dl = lg - lp
    e = 2 * U * (lg.abs() + lp.abs()) + U * dl.abs()
    terms = [d * d, dl * dl, d.abs() / g, d * d / g]
    bounds = [3 * U * d * d + TINY, 2 * dl.abs() * e + e * e + U * dl * dl + TINY, 2 * U * d.abs() / g + TINY,
              4 * U * d * d / g + TINY]
    return FloatRef(terms, bounds, keep, shared)


def edge_ref(pred, label):
    """eval_edge.py in float64 with the fp32 pos_weight: w y softplus(-x) + (1 - w)(1 - y) softplus(x), x = pred / 255.
    Per pixel: the balanced BCE term's bound at x, and x's own rounding (the term's slope in x is at most 1)."""
    x = pred.double().reshape(-1) / 255
    y = label.double().reshape(-1)
    keep = y != IGN
    w = float(np.float32(0.95))
    sp = torch.nn.functional.softplus
    t = w * y * sp(-x) + (1 - w) * (1 - y) * sp(x)
    return FloatRef([t], [bce_term_bound(x) + U * x.abs() + TINY], keep, x == 0)


def float_ref(task, pred, label, project):
    if task == "normals":
        return normals_ref(pred, label)
    if task == "depth":
        return depth_ref(pred, label, project == "TaskPrompter")
    return edge_ref(pred, label)


# ---- device --------------------------------------------------------------------------------------------------------------
def guarded_meter(p, database, task, project):
    """A single-task meter whose state lives inside a Guarded buffer, reset."""
    from mtt_b200 import evaluate as E

    m = E.get_single_task_meter(p, database, task, reference=project)
    gb = Guarded((m.words(),), torch.int64)
    m._bind(gb.view)
    m.reset()
    return m, gb


def _cuda(d):
    return {k: v.cuda() for k, v in d.items()}


def float_words(task, w):
    """A float meter's state words as (float sums, integer count)."""
    f = np.asarray(w, dtype=np.int64).view(np.float64)
    if task == "depth":
        return [float(v) for v in f[1:5]], int(w[0])
    return [float(f[0])], int(w[1])


@pytest.mark.gpu
@pytest.mark.parametrize("name,B", [pytest.param(n, B, id=run_id(n, B)) for n, B in GEOMS])
def test_meters_f64(cuda_dev, name, B):
    """Every meter of the run's tasks, one update of the full validation batch: counters exact, float sums within their
    bounds, scores within the propagated bounds, nothing outside the meter's words written, the ticket back at 0."""
    database, project, tasks, (H, W) = geometry(name, B)
    pred, gt = inputs(database, B, H, W)
    p = _p(database)
    rid = run_id(name, B)
    npix = B * H * W
    for task in tasks:
        m, gb = guarded_meter(p, database, task, project)
        gb.snapshot()
        m.update(pred[task].cuda(), gt[task].cuda())
        gb.unchanged_outside(slice(None), f"{rid} {task}: update")
        w = m.host_words()
        score = m.get_score(verbose=False)
        if task in ("semseg", "human_parts"):
            n = NCLS[database][task]
            ref = confusion_ref(pred[task].cuda(), gt[task].cuda(), n).cpu().numpy()
            assert np.array_equal(w, ref), f"{rid} {task}: {int((w != ref).sum())} confusion bins differ"
            M = ref.reshape(n + 1, n + 1)
            tp = np.diag(M)[:n]
            fp, fn = M.sum(0)[:n] - tp, M.sum(1)[:n] - tp
            jac = [float(tp[i]) / max(float(tp[i] + fp[i] + fn[i]), 1e-8) for i in range(n)]
            want = np.mean(jac) * m.scale
            assert score["mIoU"] == want, f"{rid} {task}: mIoU {score['mIoU']} != {want} (exact counts, same formula)"
            print(f"{rid} {task}: {(n + 1) ** 2} confusion bins exact, {int(ref.sum())} valid pixels")
        elif task == "sal":
            _check_saliency(m, w, pred[task], gt[task], f"{rid} sal", check_score=True)
            adv = sal_adversarial(B, H, W, m.thresholds, seed=B + H)
            m.reset()
            m.update(adv[0].cuda(), adv[1].cuda())
            _check_saliency(m, m.host_words(), *adv, f"{rid} sal (near the thresholds)", check_score=False)
        else:
            assert int(w[TICKET[task]]) == 0, f"{rid} {task}: ticket word {int(w[TICKET[task]])} after the update"
            ref = float_ref(task, pred[task].cuda(), gt[task].cuda(), project)
            sums, count = float_words(task, w)
            assert count == ref.count(), f"{rid} {task}: {count} valid pixels, want {ref.count()}"
            want, bound = ref.sums(), ref.sum_bounds(npix, task)
            ratios = []
            for k, (s, r, e) in enumerate(zip(sums, want, bound)):
                assert abs(s - r) <= e, f"{rid} {task} sum {k}: {s!r} vs float64 {r!r}: error {abs(s - r):.3e} > {e:.3e}"
                ratios.append(abs(s - r) / e)
            ratios.append(_check_float_score(task, score, want, bound, count, f"{rid} {task}"))
            report(f"{rid} {task}", ratios)


def _check_saliency(m, w, pred, label, what, check_score):
    """tp / pp / ap against the float64 reference: exact where no valid pixel is within the sigmoid bound of a
    threshold, otherwise off by at most the ambiguous pixels (pp) and their labels (tp); ap always exact."""
    tp, pp, ap = m.counts(w)
    rtp, rpp, rap, amb, amb_t = saliency_ref(pred.cuda(), label.cuda(), m.thresholds)
    assert np.array_equal(ap, rap), f"{what}: ap {ap[0]} != {rap[0]}"
    assert (np.abs(pp - rpp) <= amb).all(), f"{what}: pp {pp} vs {rpp}, ambiguous {amb}"
    assert (np.abs(tp - rtp) <= amb_t).all(), f"{what}: tp {tp} vs {rtp}, ambiguous {amb_t}"
    if not check_score:
        assert (amb > 0).sum() >= len(amb) - 1, f"{what}: the map puts no pixel near most thresholds: {amb}"
        print(f"{what}: tp / pp within {amb.max()} ambiguous pixels, ap exact")
        return
    assert (amb == 0).all(), f"{what}: the clear map has pixels within the sigmoid bound of a threshold: {amb}"
    assert np.array_equal(tp, rtp) and np.array_equal(pp, rpp), f"{what}: tp {tp} / pp {pp} vs {rtp} / {rpp}"
    # maxF: the counts convert to fp32 (u each), precision / recall 3u, (1 + b) P R 9u, b P + R 6u, the quotient 16u
    P, Rc = rtp / rpp.astype(np.float64), rtp / rap.astype(np.float64)
    with np.errstate(invalid="ignore", divide="ignore"):
        F = (1 + m.beta_squared) * P * Rc / (m.beta_squared * P + Rc)
    F[F != F] = 0
    want = F.max() * m.scale
    got = m.score(w)["maxF"]
    assert abs(got - want) <= 16 * U * want, f"{what}: maxF {got} vs float64 {want}"
    print(f"{what}: tp / pp / ap exact; maxF error / bound = {abs(got - want) / (16 * U * want):.3f}")


def _check_float_score(task, score, sums, bound, count, what):
    """The meter's get_score against the float64 formulas on the reference sums: a mean within E / n (plus the double
    division), a square root within half the relative error of its argument."""
    ratios = []
    if task == "depth":
        pairs = [("rmse", 0, True), ("log_rmse", 1, True), ("abs_rel", 2, False), ("sq_rel", 3, False)]
    else:
        pairs = [("mean" if task == "normals" else "loss", 0, False)]
    for key, k, root in pairs:
        mean = sums[k] / count
        if root:
            want = math.sqrt(mean)
            e = want * (bound[k] / max(abs(sums[k]), 1e-300)) / 2 + 4 * U64 * want
        else:
            want = mean
            e = bound[k] / count + 2 * U64 * abs(want)
        got = float(score[key])
        assert abs(got - want) <= e, f"{what}: {key} {got!r} vs float64 {want!r}, bound {e:.3e}"
        ratios.append(abs(got - want) / e)
    return max(ratios)


@pytest.mark.gpu
@pytest.mark.parametrize("name,B", [pytest.param(n, B, id=run_id(n, B)) for n, B in DISTINCT])
def test_meters_reproducible_and_graph(cuda_dev, name, B):
    """Three full-size updates of every task (the batch, the batch reversed, the batch) through one PerformanceMeter:
    two eager runs give bitwise-equal states, float sums included, and one replay of the sequence captured in a CUDA
    graph gives the same state again."""
    from mtt_b200 import evaluate as E

    database, project, tasks, (H, W) = geometry(name, B)
    pred, gt = inputs(database, B, H, W)
    fwd = (_cuda({t: pred[t] for t in tasks}), _cuda({t: gt[t] for t in tasks}))
    rev = ({t: v.flip(0).contiguous() for t, v in fwd[0].items()}, {t: v.flip(0).contiguous() for t, v in fwd[1].items()})
    seq = [fwd, rev, fwd]
    states = []
    for _ in range(2):
        pm = E.PerformanceMeter(_p(database), tasks, reference=project)
        for p, g in seq:
            pm.update(p, g)
        states.append(pm.state.clone())
    assert torch.equal(states[0], states[1]), f"{run_id(name, B)}: two eager runs differ"
    pm = E.PerformanceMeter(_p(database), tasks, reference=project)
    pm.update(*fwd)                                              # allocates the state outside the capture
    pm.reset()
    graph = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            for p, g in seq:
                pm.update(p, g)
    torch.cuda.current_stream().wait_stream(s)
    pm.reset()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(pm.state, states[0]), f"{run_id(name, B)}: graph replay differs from eager"


@pytest.mark.gpu
def test_counters_past_2_32(cuda_dev):
    """One confusion bin and the saliency tp / pp / ap driven past 2^32 by repeated PASCAL-b6 updates whose pixels all
    fall in that bin (class 5 predicted as 5; label 1 with sigmoid(10) above every threshold): exact products."""
    from mtt_b200 import evaluate as E

    B, H, W = 6, 512, 512
    npix = B * H * W
    K = 2 ** 32 // npix + 1
    cm = E.ConfusionMeter(21, [str(i) for i in range(21)], IGN)
    sm = E.SaliencyMeter(IGN)
    cls_p = torch.full((B, H, W), 5, dtype=torch.int64, device="cuda")
    cls_y = torch.full((B, 1, H, W), 5.0, device="cuda")
    sal_p = torch.full((B, H, W), 2550.0, device="cuda")
    sal_y = torch.ones(B, 1, H, W, device="cuda")
    for _ in range(K):
        cm.update(cls_p, cls_y)
        sm.update(sal_p, sal_y)
    torch.cuda.synchronize()
    want = K * npix
    assert want > 2 ** 32
    w = cm.host_words()
    assert int(w[5 * 22 + 5]) == want and int(w.sum()) == want, (int(w[5 * 22 + 5]), want)
    tp, pp, ap = sm.counts(sm.host_words())
    assert (tp == want).all() and (pp == want).all() and (ap == want).all(), (tp, pp, ap, want)


# ---- teeth (CPU) ---------------------------------------------------------------------------------------------------------
def fp32_block_sum(t, keep, task):
    """The sum as a kernel that adds its 512 block sums in fp32 would make it (grid-stride blocks of the launch)."""
    npix = t.numel()
    nb = blocks(npix, task)
    blk = (torch.arange(npix) % (nb * THREADS)) // THREADS
    bs = torch.zeros(nb, dtype=torch.float64).index_add_(0, blk[keep], t[keep])
    return float(np.add.accumulate(bs.numpy().astype(np.float32), dtype=np.float32)[-1])


@pytest.mark.parametrize("name,B", [pytest.param(n, B, id=run_id(n, B)) for n, B in DISTINCT])
def test_teeth(name, B):
    """On the inputs test_meters_f64 checks, in float64 on the CPU: counting the ignored pixel with the largest term,
    dropping the depth clamp (only the depth meter has one) and accumulating the block sums in fp32 each move some sum
    of the meter by more than twice its bound."""
    database, project, tasks, (H, W) = geometry(name, B)
    pred, gt = inputs(database, B, H, W)
    npix = B * H * W
    for task in tasks:
        if task not in TICKET:
            continue
        ref = float_ref(task, pred[task], gt[task], project)
        bound = ref.sum_bounds(npix, task)
        want = ref.sums()
        defects = {"one ignored pixel": [float(t[~ref.keep].abs().max()) for t in ref.terms],
                   "fp32 block sums": [abs(fp32_block_sum(t, ref.keep, task) - s) for t, s in zip(ref.terms, want)]}
        if task == "depth":
            raw = depth_ref(pred[task], gt[task], project == "TaskPrompter", clamp=False)
            defects["no 1e-9 clamp"] = [abs(s - r) if math.isfinite(s) else math.inf
                                        for s, r in zip(raw.sums(), want)]
        for what, shift in defects.items():
            worst = max(s / e for s, e in zip(shift, bound))
            assert worst > 2, f"{run_id(name, B)} {task}: {what} moves the sums by {shift}, bounds {bound}"
            print(f"{run_id(name, B)} {task}: {what} moves a sum by {worst:.3g}x its bound")
