"""Saving and rendering predictions on the device: the reference's test-phase prediction export
(save_model_pred_for_one_task, TP/evaluation/evaluate_utils.py:69-151, IP/evaluation/evaluate_utils.py:69-105) and its
inference visualisation (vis_pred_for_one_task, TP/utils/visualization_utils.py:80-199).

Both go per task from logits or get_output maps to uint8 images: an optional bilinear resize, get_output, the crop that
undoes PadImage, and an encoding (truncation, class id, palette, normals or JET). ``mtt_render`` (csrc/export.cu) does
that for every (task, image) pair of a batch in two launches; what is left on the host is moving bytes and writing PNGs.

    from mtt_b200.export import PredictionWriter       # test_phase: one writer for the tasks it saves
    writer = PredictionWriter(p, ["edge"], save_dirs)
    writer.update(model.predict(images), batch, batch["meta"])   # or the wrapper's logits dict, as the reference
    writer.close()                                               # waits for every PNG

``update`` enqueues the launches into one slot of a ring of pinned staging buffers, copies the slot to the host on a side
stream after an event and returns without synchronising the host. A small thread pool waits on each slot's event and
writes the files; a slot is reused only after its files are written.
"""
import atexit
import os
import threading
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

REFERENCES = ("TaskPrompter", "InvPT")
GET_OUTPUT_KIND = {"semseg": 0, "human_parts": 0, "edge": 1, "sal": 2, "normals": 3, "depth": 4}   # ops.POSTPROC_KIND

# get_cityscapes_class (TP/utils/utils.py:17-24): train id -> Cityscapes class id
CS_VALID_CLASSES = [7, 8, 11, 12, 13, 17, 19, 20, 21, 22, 23, 24, 25, 26, 27, 28, 31, 32, 33]
# create_cityscapes_label_colormap (TP/utils/visualization_utils.py:13-39): the 19 train-id colours, RGB
CITYSCAPES_COLORS = [(128, 64, 128), (244, 35, 232), (70, 70, 70), (102, 102, 156), (190, 153, 153), (153, 153, 153),
                     (250, 170, 30), (220, 220, 0), (107, 142, 35), (152, 251, 152), (70, 130, 180), (220, 20, 60),
                     (255, 0, 0), (0, 0, 142), (0, 0, 70), (0, 60, 100), (0, 80, 100), (0, 0, 230), (119, 11, 32)]


def labelcolormap(N):
    """The VOC-style palette (visualization_utils.py:46-63): the bits of the class id interleaved into the high bits of
    R, G and B, three at a time. uint8 [N,3] RGB."""
    cmap = np.zeros((N, 3), dtype=np.uint8)
    for i in range(N):
        r = g = b = 0
        cid = i
        for j in range(7):
            r |= (cid & 1) << (7 - j)
            g |= ((cid >> 1) & 1) << (7 - j)
            b |= ((cid >> 2) & 1) << (7 - j)
            cid >>= 3
        cmap[i] = (r, g, b)
    return cmap


def cityscapes_colormap():
    """uint8 [256,3] RGB: the 19 train-id colours, the rest black, as the reference's table."""
    cmap = np.zeros((256, 3), dtype=np.uint8)
    cmap[:19] = CITYSCAPES_COLORS
    return cmap


def cityscapes_id_table():
    """uint8 [256]: train id -> Cityscapes class id for 0..18, identity elsewhere."""
    t = np.arange(256, dtype=np.uint8)
    t[:19] = CS_VALID_CLASSES
    return t


def jet_bgr():
    """cv2.applyColorMap(np.arange(256, dtype=np.uint8), cv2.COLORMAP_JET) as uint8 [256,3] BGR (the library's copy)."""
    from . import lib
    ptr = lib.load().mtt_render_jet_bgr()
    return np.ctypeslib.as_array(ptr, shape=(256 * 3,)).reshape(256, 3).copy()


def _get(p, key, default=None):
    try:
        return p[key]
    except (KeyError, TypeError):
        return getattr(p, key, default)


def _no_3ddet(task):
    if task == "3ddet":
        raise NotImplementedError("task '3ddet' needs mmdet3d (bbox2json / bbox2fig), which mtt_b200 does not provide")


def export_encoding(p, task, reference="TaskPrompter"):
    """(encode, table) of the prediction export: astype(np.uint8) of the get_output map, the Cityscapes class ids for
    TaskPrompter's semseg when p.semseg_save_train_class is false (evaluate_utils.py:74-78). Normals and depth raise
    ValueError: the reference raises on a 3-D prediction (:142-143) before it reaches its .mat branch."""
    _no_3ddet(task)
    if reference not in REFERENCES:
        raise ValueError(f"reference must be one of {REFERENCES}, got {reference!r}")
    if task in ("normals", "depth"):
        raise ValueError(f"the reference cannot export {task!r}: its prediction is 3-D, and evaluate_utils.py raises "
                         "on a 3-D prediction")
    if task not in GET_OUTPUT_KIND:
        raise ValueError(f"no get_output defined for task {task!r}")
    if (task == "semseg" and reference == "TaskPrompter" and not _get(p, "semseg_save_train_class", True)
            and _get(p, "train_db_name") == "Cityscapes3D"):
        return "class", cityscapes_id_table()
    return ("class" if GET_OUTPUT_KIND[task] == 0 else "u8"), None


def vis_encoding(p, task):
    """(encode, table) of vis_pred_for_one_task's parallel branch (visualization_utils.py:158-187)."""
    _no_3ddet(task)
    if task == "semseg":
        db = _get(p, "train_db_name")
        tables = {"NYUD": lambda: labelcolormap(40), "PASCALContext": lambda: labelcolormap(21),
                  "Cityscapes3D": cityscapes_colormap}
        if db not in tables:
            raise NotImplementedError(f"no semseg palette for {db!r}")
        return "palette_bgr", tables[db]()
    if task == "human_parts":
        return "palette_bgr", labelcolormap(7)
    if task == "normals":
        return "normals_bgr", None
    if task == "depth":
        return "jet", None   # the library's JET table
    if task in ("sal", "edge"):
        return "u8", None
    raise ValueError(f"no visualisation defined for task {task!r}")


def crop_window(pred_hw, img_hw):
    """The centre crop that undoes PadImage (evaluate_utils.py:127-138): (y0, x0, h, w). An image larger than the
    prediction is refused, as the reference's assert (:141) refuses it."""
    H, W = (int(v) for v in pred_hw)
    h, w = (int(v) for v in img_hw)
    if h > H or w > W or h <= 0 or w <= 0:
        raise ValueError(f"image size {h}x{w} does not fit in the {H}x{W} prediction")
    return (H - h) // 2, (W - w) // 2, h, w


def pack_offsets(sizes, channels):
    """Byte offsets of ragged [h,w(,channels)] images packed back to back, and the total."""
    offs, total = [], 0
    for h, w in sizes:
        offs.append(total)
        total += int(h) * int(w) * channels
    return offs, total


def _img_sizes(meta, B):
    sizes = meta["img_size"]
    out = []
    for jj in range(B):
        s = sizes[jj]
        out.append((int(s[0]), int(s[1])))
    return out


def _is_logits(x):
    """The wrapper's output (fp32 [B,C,H,W]) rather than a predict() / get_output map."""
    return x.dtype == torch.float32 and x.dim() == 4 and not (x.shape[3] in (1, 3) and x.shape[1] not in (1, 3))


class _Job:
    """One task of one update: what the device renders and where the host writes it."""
    __slots__ = ("task", "save_dir", "names", "suffix", "sizes", "crops", "offsets", "channels", "total", "src",
                 "postproc", "out_hw", "out_sizes", "encode", "table", "n_classes", "label", "ignore_index", "skip",
                 "base")

    def __init__(self, **kw):
        for k in self.__slots__:
            setattr(self, k, kw.get(k))


class _Slot:
    def __init__(self):
        self.future = None
        self.dev = self.host = self.flags_dev = self.flags_host = self.ws = None
        self.event = None


class DeviceEncoder:
    """Renders a slot's jobs with mtt_render on the current stream and copies the bytes into the slot's pinned host
    buffer on a side stream: no host synchronisation. ``wait`` blocks (on a worker thread) until the copy is done."""

    def __init__(self, device=None):
        self.device = torch.device(device) if device is not None else None
        self.stream = None
        self._tables = {}

    def _table(self, arr, device):
        key = (arr.tobytes(), arr.shape, str(device))
        t = self._tables.get(key)
        if t is None:
            t = torch.from_numpy(np.ascontiguousarray(arr)).pin_memory().to(device, non_blocking=True)
            self._tables[key] = t
        return t

    def encode(self, slot, jobs):
        from . import lib, ops
        device = jobs[0].src.device
        if self.stream is None:
            self.stream = torch.cuda.Stream(device=device)
        total = sum(j.total for j in jobs)
        nimg = sum(len(j.names) for j in jobs)
        if slot.dev is None or slot.dev.numel() < total or slot.dev.device != device:
            cap = max(total, 1)
            slot.dev = torch.empty(cap, dtype=torch.uint8, device=device)
            slot.host = torch.empty(cap, dtype=torch.uint8, pin_memory=True)
        if slot.flags_dev is None or slot.flags_dev.numel() < nimg:
            slot.flags_dev = torch.zeros(max(nimg, 1), dtype=torch.int32, device=device)
            slot.flags_host = torch.zeros(max(nimg, 1), dtype=torch.int32, pin_memory=True)
        per = lib.RENDER_MAX_IMAGES
        need_ws = ops.render_workspace_bytes(1, min(nimg, per)) // 4 + 1
        if slot.ws is None or slot.ws.numel() < need_ws:
            slot.ws = torch.empty(need_ws, dtype=torch.int32, device=device)
        # split into calls of at most RENDER_MAX_TASKS tasks / RENDER_MAX_IMAGES images
        calls, cur, n = [], [], 0
        base, fbase = 0, 0
        for j in jobs:
            B = len(j.names)
            for b0 in range(0, B, per):
                b1 = min(B, b0 + per)
                if cur and (len(cur) == lib.RENDER_MAX_TASKS or n + (b1 - b0) > per):
                    calls.append(cur)
                    cur, n = [], 0
                t = dict(src=j.src[b0:b1], postproc=j.postproc, out_hw=j.out_hw, encode=j.encode,
                         crops=j.crops[b0:b1], offsets=[o + base for o in j.offsets[b0:b1]], out=slot.dev,
                         n_classes=j.n_classes, ignore_index=j.ignore_index)
                if j.out_sizes is not None:
                    t["out_sizes"] = j.out_sizes[b0:b1]
                if j.table is not None:
                    t["table"] = self._table(j.table, device)
                elif j.encode == "jet":
                    t["table"] = self._table(jet_bgr(), device)
                if j.label is not None:
                    t["label"] = j.label[b0:b1]
                    t["flags"] = slot.flags_dev[fbase + b0:fbase + b1]
                cur.append(t)
                n += b1 - b0
            j.base = (base, fbase)
            base += j.total
            fbase += B
        if cur:
            calls.append(cur)
        for c in calls:
            ops.render(c, slot.ws)
        main = torch.cuda.current_stream(device)
        ready = torch.cuda.Event()
        ready.record(main)
        self.stream.wait_event(ready)
        with torch.cuda.stream(self.stream):
            slot.host[:total].copy_(slot.dev[:total], non_blocking=True)
            slot.flags_host[:nimg].copy_(slot.flags_dev[:nimg], non_blocking=True)
            slot.event = torch.cuda.Event()
            slot.event.record(self.stream)

    def wait(self, slot):
        slot.event.synchronize()
        return slot.host.numpy(), slot.flags_host.numpy()


def _imwrite(path, arr):
    import cv2
    if not cv2.imwrite(path, arr):
        raise OSError(f"cv2.imwrite failed for {path}")


class PredictionWriter:
    """The drop-in for the save step of test_phase (``mode="export"``: ``'{img_name}.png'`` in save_dirs[task], images
    whose label is all ignore_index skipped) and for vis_pred_for_one_task (``mode="vis"``: the logits resized to the
    image size, ``'{img_name}_{task}.png'``). ``slots`` staging buffers (2 or 3) form the ring; ``workers`` threads
    write files. ``encoder`` / ``imwrite`` replace the device encoder and the PNG writer (tests)."""

    def __init__(self, p, tasks, save_dirs, reference="TaskPrompter", *, mode="export", slots=3, workers=4,
                 encoder=None, imwrite=None):
        if reference not in REFERENCES:
            raise ValueError(f"reference must be one of {REFERENCES}, got {reference!r}")
        if mode not in ("export", "vis"):
            raise ValueError(f"mode must be 'export' or 'vis', got {mode!r}")
        if not 1 <= int(slots):
            raise ValueError("a ring needs at least one slot")
        self.p, self.tasks, self.reference, self.mode = p, list(tasks), reference, mode
        self.save_dirs = dict(save_dirs) if isinstance(save_dirs, dict) else {t: save_dirs for t in self.tasks}
        self.enc = {t: (export_encoding(p, t, reference) if mode == "export" else vis_encoding(p, t))
                    for t in self.tasks}
        for t in self.tasks:
            os.makedirs(self.save_dirs[t], exist_ok=True)
        self.ignore_index = _get(p, "ignore_index", 255)
        self.encoder = encoder if encoder is not None else DeviceEncoder()
        self.imwrite = imwrite if imwrite is not None else _imwrite
        self.ring = [_Slot() for _ in range(int(slots))]
        self.pool = ThreadPoolExecutor(max_workers=int(workers))
        self.count = 0
        self.lock = threading.Lock()

    def _jobs(self, pred, labels, meta):
        jobs = []
        for task in self.tasks:
            x = pred[task]
            encode, table = self.enc[task]
            B = int(x.shape[0])
            names = [str(n) for n in meta["img_name"][:B]]
            logits = _is_logits(x)
            channels = 3 if encode in ("palette_bgr", "normals_bgr", "jet") else 1
            n_classes = len(table) if encode == "palette_bgr" else None
            if self.mode == "vis":
                if not logits:
                    raise ValueError(f"vis_pred_for_one_task resizes the wrapper's logits; {task!r} is a "
                                     f"{x.dtype} {tuple(x.shape)} map")
                sizes = [_img_sizes(meta, 1)[0]] * B   # "We assume all the images have the same size" (:145-147)
                crops = [(0, 0, h, w) for h, w in sizes]
                out_hw, out_sizes = sizes[0], None
            else:
                H, W = (int(x.shape[2]), int(x.shape[3])) if logits else (int(x.shape[1]), int(x.shape[2]))
                sizes = _img_sizes(meta, B)
                crops = [crop_window((H, W), s) for s in sizes]
                out_hw, out_sizes = None, None
            label, skip = None, [False] * B
            if self.mode == "export" and labels is not None and task in labels:
                lab = labels[task]
                if lab.is_cuda:
                    label = lab.contiguous()
                else:   # the reference's loader tensors: the skip rule on the host, as the reference evaluates it
                    skip = [bool(lab[jj].numel() > 0 and bool((lab[jj] == self.ignore_index).all()))
                            for jj in range(B)]
            offs, total = pack_offsets([(c[2], c[3]) for c in crops], channels)
            src = x if (logits or x.dtype != torch.float32 or x.dim() != 4 or x.shape[3] != 1) else x[..., 0]
            jobs.append(_Job(task=task, save_dir=self.save_dirs[task], names=names,
                             suffix=("_" + task) if self.mode == "vis" else "", sizes=sizes, crops=crops,
                             offsets=offs, channels=channels, total=total, src=src,
                             postproc=GET_OUTPUT_KIND[task] if logits else None, out_hw=out_hw, out_sizes=out_sizes,
                             encode=encode, table=table, n_classes=n_classes, label=label,
                             ignore_index=self.ignore_index, skip=skip))
        return jobs

    def update(self, pred, labels=None, meta=None, batch_idx=None):
        """Enqueue one batch: pred = predict()'s dict or the wrapper's logits dict, labels = the batch (or a dict of
        the tasks' labels, CUDA or CPU), meta = batch['meta'] with 'img_name' and 'img_size'. batch_idx is accepted
        for TaskPrompter's call signature and not used."""
        if meta is None:
            meta = labels["meta"]
        jobs = self._jobs(pred, labels, meta)
        with self.lock:
            slot = self.ring[self.count % len(self.ring)]
            self.count += 1
            if slot.future is not None:
                slot.future.result()   # the slot's previous files are written: its buffers may be reused
            self.encoder.encode(slot, jobs)
            slot.future = self.pool.submit(self._write, slot, jobs)

    def _write(self, slot, jobs):
        host, flags = self.encoder.wait(slot)
        for j in jobs:
            base, fbase = j.base
            for jj, name in enumerate(j.names):
                if j.skip[jj] or (j.label is not None and flags[fbase + jj]):
                    continue
                h, w = j.crops[jj][2], j.crops[jj][3]
                o = base + j.offsets[jj]
                arr = host[o:o + h * w * j.channels]
                arr = arr.reshape(h, w, 3) if j.channels == 3 else arr.reshape(h, w)
                self.imwrite(os.path.join(j.save_dir, name + j.suffix + ".png"), arr)

    def flush(self):
        """Wait until every enqueued batch is written (re-raises a writer's exception)."""
        with self.lock:
            for s in self.ring:
                if s.future is not None:
                    s.future.result()

    def close(self):
        self.flush()
        self.pool.shutdown(wait=True)

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


def render(p, output, img_size, tasks=None):
    """The visualisation's images on the device: {task: uint8 CUDA tensor}, [B,h,w,3] BGR or [B,h,w] gray, from the
    wrapper's logits dict. img_size is one (h, w) for the batch (the reference assumes all images have the same size)
    or one per image; with several sizes each task's value is a list of per-image tensors."""
    from . import ops
    tasks = list(tasks if tasks is not None else output)
    for t in tasks:
        _no_3ddet(t)
    first = output[tasks[0]]
    B = int(first.shape[0])
    sizes = [tuple(int(v) for v in img_size)] * B if np.ndim(img_size) == 1 else [tuple(int(v) for v in s)
                                                                                for s in img_size]
    same = len(set(sizes)) == 1
    enc = DeviceEncoder()
    device = first.device
    outs, specs, ws_imgs = {}, [], 0
    for t in tasks:
        encode, table = vis_encoding(p, t)
        ch = ops.RENDER_CHANNELS[encode]
        offs, total = pack_offsets(sizes, ch)
        buf = torch.empty(total, dtype=torch.uint8, device=device)
        spec = dict(src=output[t].contiguous(), postproc=GET_OUTPUT_KIND[t], encode=encode, crops=[(0, 0, h, w) for
                    h, w in sizes], offsets=offs, out=buf)
        if same:
            spec["out_hw"] = sizes[0]
        else:
            spec["out_sizes"] = sizes
        spec["table"] = enc._table(table if table is not None else jet_bgr(), device) if encode != "u8" else None
        if spec["table"] is None:
            del spec["table"]
        specs.append(spec)
        ws_imgs += B
        if same:
            h, w = sizes[0]
            outs[t] = buf.view(B, h, w, 3) if ch == 3 else buf.view(B, h, w)
        else:
            outs[t] = [buf[o:o + h * w * ch].view(h, w, 3) if ch == 3 else buf[o:o + h * w * ch].view(h, w)
                       for o, (h, w) in zip(offs, sizes)]
    ws = torch.empty(ops.render_workspace_bytes(1, ws_imgs) // 4 + 1, dtype=torch.int32, device=device)
    ops.render(specs, ws)
    return outs


_writers = {}
_writers_lock = threading.Lock()


def _writer_for(p, task, save_dir, reference, mode):
    key = (id(p), task, save_dir, reference, mode)
    with _writers_lock:
        w = _writers.get(key)
        if w is None:
            w = PredictionWriter(p, [task], {task: save_dir}, reference, mode=mode)
            _writers[key] = w
        return w


def flush():
    """Wait until every file the module-level save / visualisation functions enqueued is written."""
    with _writers_lock:
        ws = list(_writers.values())
    for w in ws:
        w.flush()


@atexit.register
def _close_all():
    with _writers_lock:
        ws = list(_writers.values())
        _writers.clear()
    for w in ws:
        w.close()


def save_model_pred_for_one_task(p, batch_idx, sample, output, save_dirs, task=None, epoch=None):
    """TaskPrompter's signature (TP/evaluation/evaluate_utils.py:69): enqueues the task's PNGs; export.flush() (or
    interpreter exit) waits for them."""
    _writer_for(p, task, save_dirs[task], "TaskPrompter", "export").update(output, sample, sample["meta"])


def save_model_pred_for_one_task_invpt(p, sample, output, save_dirs, task=None, epoch=None):
    """InvPT's signature (IP/evaluation/evaluate_utils.py:68): as save_model_pred_for_one_task."""
    _writer_for(p, task, save_dirs[task], "InvPT", "export").update(output, sample, sample["meta"])


def vis_pred_for_one_task(p, sample, output, save_dir, task):
    """The reference's signature (TP/utils/visualization_utils.py:80): writes '{img_name}_{task}.png' with
    cv2.imwrite before returning, as the reference's parallel branch does."""
    w = _writer_for(p, task, save_dir, "TaskPrompter", "vis")
    w.update(output, None, sample["meta"])
    w.flush()
