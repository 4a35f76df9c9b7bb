"""CPU: the numpy restatement of the reference's train / validation transform chains (oracle/augment_ref.py) against the
golden data made by the real reference, against the live reference, and its cv2 rules against cv2 itself; the
collate's draw order and packing (augment.py)."""
import ctypes
import os
import random

import numpy as np
import pytest

from oracle import augment_ref as R

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "augment.pt.xz")


def bits_equal(a, b):
    a, b = np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


@pytest.fixture(scope="module")
def golden():
    from oracle import make_augment_golden as G
    return G.load(GOLDEN)


def test_restatement_matches_golden_train(golden):
    for name, s, rec, ref, consumed in zip(golden["names"], golden["samples"], golden["records"], golden["outputs"],
                                           golden["consumed"]):
        got, st = R.train_transform(s, rec, golden["crop"], return_stages=True)
        assert set(got) == set(ref), name
        for k in ref:
            assert bits_equal(got[k], ref[k]), (name, k)
        assert (st["chosen"] is None) == (consumed == 0), name
        if consumed:
            assert st["chosen"] == consumed - 1, name


def test_restatement_matches_golden_valid(golden):
    for s, ref in zip(golden["valid_samples"], golden["valid_outputs"]):
        got = R.valid_transform(s, golden["valid_size"])
        for k in ref:
            assert bits_equal(got[k], ref[k]), k


def test_golden_reaches_every_branch(golden):
    recs, consumed = golden["records"], golden["consumed"]
    scales = [r["scale"] for r in recs]
    assert min(scales) < 1 < max(scales) and 1.0 in scales
    assert {r["flip"] for r in recs} == {True, False}
    for k in ("bright", "contrast", "sat", "hue"):
        assert {r[k] is None for r in recs} == {True, False}, k
    assert {(r["f_mode"], r["contrast"] is not None) for r in recs} >= {(True, True), (False, True)}
    assert 1 in consumed and 11 in consumed and any(1 < c < 11 for c in consumed) and 0 in consumed


def test_restatement_matches_live_reference():
    from oracle import ref_loader
    if not ref_loader.available():
        pytest.skip("reference tree absent")
    import mtt_b200  # noqa: F401
    from mtt_b200 import augment as A
    from oracle import make_augment_golden as G

    rng = np.random.default_rng(4)
    draws = random.Random(9)
    for i in range(24):
        h, w = int(rng.integers(18, 70)), int(rng.integers(18, 70))
        s = G.make_sample(rng, h, w, G.PASCAL if i % 2 else G.NYUD, seg="uniform" if i % 5 == 0 else "mixed",
                          parts_ignore=i % 3 == 0, zero_normals=i % 4 == 0, zero_depth=i % 4 == 1)
        rec = A.draw_params(h, w, G.CROP, rng=draws)
        ref, _ = G.run_reference(s, rec)
        got = R.train_transform(s, rec, G.CROP)
        for k in ref:
            assert bits_equal(got[k], ref[k].numpy()), (i, k)


def test_resize_rules_match_cv2():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(0)
    for h, w in [(375, 500), (281, 500), (480, 640), (17, 23), (3, 5), (333, 477)]:
        img = rng.integers(0, 256, (h, w, 3)).astype(np.float32)
        lab = rng.standard_normal((h, w)).astype(np.float32)
        for s in [0.5, 0.5003, 0.61, 0.97, 1.0, 1.03, 1.6, 1.97, 1.9999, 2.0]:
            dh, dw = int(h * s), int(w * s)
            assert bits_equal(R.resize_linear(img, dh, dw), cv2.resize(img, (dw, dh), interpolation=cv2.INTER_LINEAR))
            assert bits_equal(R.resize_nearest(lab, dh, dw), cv2.resize(lab, (dw, dh), interpolation=cv2.INTER_NEAREST))


def test_rgb2hsv_exhaustive():
    cv2 = pytest.importorskip("cv2")
    a = np.arange(1 << 24, dtype=np.uint32)
    rgb = np.stack([(a >> 16) & 255, (a >> 8) & 255, a & 255], -1).astype(np.uint8).reshape(4096, 4096, 3)
    assert np.array_equal(R.rgb2hsv(rgb), cv2.cvtColor(rgb, cv2.COLOR_RGB2HSV))


def test_hsv2rgb_exhaustive():
    cv2 = pytest.importorskip("cv2")
    H, S, V = np.meshgrid(np.arange(180), np.arange(256), np.arange(256), indexing="ij")
    hsv = np.stack([H, S, V], -1).astype(np.uint8).reshape(180 * 256, 256, 3)
    assert np.array_equal(R.hsv2rgb(hsv), cv2.cvtColor(hsv, cv2.COLOR_HSV2RGB))


def test_draw_order():
    import mtt_b200  # noqa: F401
    from mtt_b200 import augment as A

    log = []

    class Spy(random.Random):
        """Logs the top-level calls (uniform and randint call random / getrandbits themselves)."""
        depth = 0

        def _call(self, entry, fn, *a):
            if self.depth == 0:
                log.append(entry)
            self.depth += 1
            try:
                return fn(*a)
            finally:
                self.depth -= 1

        def uniform(self, a, b):
            return self._call(("uniform", a, b), super().uniform, a, b)

        def randint(self, a, b):
            return self._call(("randint", a, b), super().randint, a, b)

        def random(self):
            return self._call(("random",), super().random)

    for seed in range(40):
        log.clear()
        rec = A.draw_params(375, 500, (512, 512), rng=Spy(seed))
        assert log[0] == ("uniform", 0.5, 2.0)
        sh, sw = int(375 * rec["scale"]), int(500 * rec["scale"])
        n = 0 if rec["crops"] is None else 22
        assert log[1:1 + n] == [("randint", 0, max(sh - 512, 0)), ("randint", 0, max(sw - 512, 0))] * (n // 2)
        rest = [e[0] for e in log[1 + n:]]
        # flip, brightness test (+ beta), f_mode, then the contrast / saturation / hue tests in the reference's order
        expect = ["random", "random"] + (["uniform"] if rec["bright"] is not None else []) + ["random"]
        order = ["contrast", "sat", "hue"] if rec["f_mode"] else ["sat", "hue", "contrast"]
        for k in order:
            expect += ["random"] + ([] if rec[k] is None else ["randint" if k == "hue" else "uniform"])
        assert rest == expect, (seed, rest, expect)
    # the scaled size equals the crop size: no crop draws
    rec = A.draw_params(256, 256, (512, 512), rng=type("Two", (random.Random,), {"uniform": lambda s, a, b: 2.0})(0))
    assert rec["crops"] is None


def test_collate_packing():
    import mtt_b200  # noqa: F401
    from mtt_b200 import augment as A
    from mtt_b200 import lib

    rng = np.random.default_rng(1)
    p = {"train_db_name": "NYUD", "TASKS": {"NAMES": ["semseg", "depth", "normals", "edge"]},
         "TRAIN": {"SCALE": (64, 80)}, "TEST": {"SCALE": (64, 80)}}
    batch = []
    for h, w in [(50, 70), (64, 80), (31, 90)]:
        batch.append({"image": rng.integers(0, 256, (h, w, 3)).astype(np.float32),
                      "semseg": rng.integers(0, 5, (h, w, 1)).astype(np.float32),
                      "depth": rng.random((h, w, 1)).astype(np.float32),
                      "normals": rng.standard_normal((h, w, 3)).astype(np.float32),
                      "edge": rng.random((h, w, 1)).astype(np.float32),
                      "meta": {"img_name": f"s{h}", "img_size": (h, w)}})
    random.seed(3)
    raw = A.make_collate(p)(batch)
    random.seed(3)
    expect = [A.draw_params(s["image"].shape[0], s["image"].shape[1], (64, 80)) for s in batch]
    assert raw["records"] == expect
    assert raw["tasks"] == ["semseg", "depth", "normals", "edge"] and (raw["H"], raw["W"]) == (64, 80)
    assert raw["meta"]["img_name"] == ["s50", "s64", "s31"]
    assert [t.tolist() for t in raw["meta"]["img_size"]] == [[50, 70], [64, 80], [31, 90]]
    buf = raw["buf"].numpy()
    recs = (lib.AugmentSample * 3).from_buffer_copy(buf[:ctypes.sizeof(lib.AugmentSample) * 3].tobytes())
    data = buf[raw["head"]:].view(np.float32)
    assert raw["head"] % 256 == 0
    for s, r, rec in zip(batch, recs, expect):
        h, w = s["image"].shape[:2]
        assert (r.h, r.w) == (h, w)
        assert (r.sh, r.sw) == R.scaled_size(h, w, rec["scale"])
        assert r.ncand == (0 if rec["crops"] is None else 11)
        for i, k in enumerate(["image", "semseg", "depth", "normals", "edge"]):
            a = s[k].reshape(-1)
            assert np.array_equal(data[r.off[i]:r.off[i] + a.size], a), k
    with pytest.raises(NotImplementedError):
        A.make_collate(dict(p, train_db_name="Cityscapes3D"))
