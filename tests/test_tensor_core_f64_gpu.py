"""The wgmma GEMM, the implicit-GEMM convolution and the fused attention at every geometry the benched plans launch,
against float64, element by element.

Recording. A module fixture builds the plan of every forward / predict() run of plan_calls.RUNS (nsplit = 2, no
graph) at the run's batch -- tp_cfg4, tp_cfg2, tp_cfg5, ip_cfg3, tps_swinB at bench.DEFAULT_BATCH, the three-task
tps_swinB3d at batch 1 and 4 (nn.Identity as the 3ddet head: its window GEMMs have M = B nW (3 + 144) rows), the
reference's own model configs tp_nyud_vitL, tp_pascal_vitB, ip_nyud_vitL and tp_cfg4 / ip_cfg3 at its validation batch
6, the PASCAL ones at the ragged last validation batch 5 -- and runs one eager forward; every training run (tp_cfg4 and
tp_cfg2 at batch 4; tp_cfg4, tp_pascal_vitB, tp_nyud_vitL at the reference's training batch 2) runs one eager
TrainStep._fwd_bwd with the bench's criterion and labels. The batch sets every GEMM's M, so its tile count and
stream-K split. Pass-through recorders around ops.gemm, gemm_grouped,
gemm_splitk, attention and the five composites of csrc/block_ops.cu turn every call into a geometry key (call_key): the
shapes, the mode, the epilogue (act, bias, residual kind), the row maps (regroup, a_gather), the offsets, which outputs
are written and every leading dimension. The same runs are bracketed by ops.profile_begin / profile_end, and every
profiled tensor-core launch (kind, M, N, K) must be one a recorded call explains (launches_of expands the composites
into their internal launches as block_ops.cu issues them), so a plan that reaches a kernel another way fails here.

Replay. Every key runs again on fresh buffers of the recorded rows and leading dimensions, in parity (nsplit = 2) and
speed (nsplit = 1) mode, under the production knobs (tile variant and stream-K automatic), with random normal operands
split by ops.split_f32: once plain and once with rows of A and W scaled by 2^u, u uniform in [-20, 20], so that a
small row cannot hide under a large one. Attention runs with q plain and with q scaled by 12 (logits of tens). Every
output lies inside NaN sentinels (pad columns up to ld, rows a regroup does not target, the rest of joint buffers), and
every element the launch must not write keeps its bits. Composites are checked stage by stage against the planes each
stage really consumed, read back from the workspace (ops.ws_split_view) or the mid / hidden buffer.

Reference. The float64 reference is the exact sum of the products the mode issues over the actual bf16 planes:
a_hi w_hi + a_hi w_lo + a_lo w_hi (parity) or a_hi w_hi (speed), so the planes' representation error is not part of
the comparison; convolutions are summed tap by tap from shifted NHWC planes (no im2col). The bound per element rests
on the kernel's arithmetic (gemm_tc.cu mma_piece, gemm_common.cuh epilogue_op):

  * chain: each 64-deep K-stage is summed in a fresh tensor-core accumulator, one wgmma per k16 step and product (12
    per stage in parity, 4 in speed; fewer in the ragged last stage of each tap, k_last_steps). Each wgmma adds its 16
    products to the accumulator and truncates. Its error is at most KAPPA = 2 units of 2^-23 of the partial sum's
    magnitude (one for the truncation of the result, one for aligning the products to the largest exponent), and that
    magnitude is at most the absolute sum of every product added so far in the stage. Summed over the steps this is
    KAPPA 2^-23 sum_k (n_s - j(k)) |t_k|, where step j(k) issues term t_k and n_s is the stage's step count: a
    weighted absolute matmul, computed exactly.
  * fold: stage sums P_s are added to the tile's fp32 sum with round-to-nearest; stream-K pieces start from zero and
    their partials are added in CTA order; gemm_splitk's reduction (mtt_sum_partials) starts from the bias and adds
    its K-slices in a fixed order, so there the bias is one more term of the sum. Depth at most 2 (stages) + 1
    (+ slices + 1), so sum_tol(depth, sum_s |P_s| (+ |bias|)) (tests/f64_checks.py).
  * the float64 reference's own rounding: cuBLAS sums each stage's at most 64 products and the stages are added one
    by one, so it is off by at most (64 + stages) 2^-53 of the absolute sum, which the chain weights (all >= 1)
    bound from above: F64_REF (64 + stages) chain. The float64 softmax and P.V of the attention reference carry
    relative errors near 2^-50, far below the 2^-17 of the split output they are compared through.
  * epilogue, in order: bias add (u |result|); GELU (fp32 erf form: slope < 1.13, and 0.5 |v| 4 2^-23 absolute from
    erff's 2 ulp and the 1 + erf add, which cancels for negative v, plus 4 u |gelu|); ReLU (1-Lipschitz); residual
    add (u |result|).
  * outputs: fp32 within the bound; when a split output is written beside it, hi = RN_bf16(out_f32) and
    lo = RN_bf16(out_f32 - hi) bit for bit; a split output alone within the bound + SPLIT |ref| + SPLIT_ABS.

Attention (attention5_tc.cu) follows the window-attention model of tests/kernel_cases.py: a logit off by d moves a softmax weight by at
most a factor exp(2 d). d is the QK^T chain bound above (one 64-deep stage) times the scale, plus 3 u of the largest
scaled logit (scale * log2 e rounded, the FMA against the running maximum, the maximum itself). Each weight further
carries ex2.approx's relative error (2^-21) once for itself and once per running-maximum rescale (at most one per key
block), the bf16 split of P (2^-16 in parity with the missing p_lo v_lo, 2^-8 more in speed mode), the row sum
(sum_tol of depth 16 + blocks + 2 over weights that sum to 1), the per-block P.V chain (KAPPA 2^-23 per step) and its fused fold into O
(sum_tol over the blocks), and the final 1 / l multiply and split. prompt_logits must hold the raw q.k^T of the first
T rows within the QK^T chain bound.

Teeth. At every key with two or more K-stages the real kernel also runs on altered operands against the unaltered
reference and bound:

  (1) The speed-mode result (dropped lo products) must fail on at least TEETH_FRAC of the elements of every stage
      whose speed-mode output can show it: an fp32 output or a split with both planes written. A speed-mode launch
      of gated_conv1x1 gets no lo plane to write, and a composite's workspace intermediates hold one plane in speed
      mode; a bf16 value cannot show a 2^-9 product drop, so those outputs are left out, and gated_conv1x1's teeth
      are the check below.
  (2) W's lo plane zeroed in the last K-stage of every tap of the final GEMM stage (a ragged-tail defect). The
      defect, computed exactly through the epilogue, must be flagged wherever it moves the result by more than twice
      the bound. At keys with at most TAIL_STAGES K-stages (taps x stages per tap) the defect must also exceed twice
      the bound on at least TEETH_FRAC of the elements, and the result fail it there. Why that limit: for normal
      operands the chain bound is about KAPPA 2^-23 6.5 S (S = 0.64 K sigma_a sigma_w, the weights averaging 6.5 over
      a full stage), while the defect sums 64 products per tap with |w_lo| < 2^-9 |w|, rms about 2^-7.7 sigma_a
      sigma_w per tap. The defect over the bound is then about 76 / stages: 2.4 at 32 stages (twice the bound on
      about 40 % of the elements of a linear epilogue, half that behind a ReLU or the flat side of GELU), and below
      the 10 % line from about 64 stages on. The weight-gradient GEMMs of the training step, with K = B * tokens or
      B * pixels (65 to over 1000 stages), are past it: a bound that must hold for every stage of such a sum is
      larger than any one-stage defect. Their fractions are reported, not asserted.

Attention: the speed-mode result must fail the parity bound on at least TEETH_FRAC of the elements of the draw that
flags more (with q x 1 at N = 8195 the speed-mode weight errors average out over the keys below the per-weight bound;
with q x 12 a few keys carry each row and they do not). The worst err / bound ratio per config and kind, and the
fraction each teeth check flagged, are printed.

The CPU self-checks (no GPU) run the reference builder on integer planes against tests/kernel_cases.py ref_gemm bit for
bit, a CPU model of the kernel's arithmetic (fp32 chains truncated after every k16 step, round-to-nearest fold)
against the bound, and the key builder.
"""
import collections
import math
import time

import pytest
import torch
import torch.nn.functional as F

import kernel_cases as X
from f64_checks import (SENTINEL, SPLIT, SPLIT_ABS, U, bits, check, mtt_ops, planes, sentinel, sentinel_split,
                        split_bound, sum_tol)
from plan_calls import frozen, recording, run_id, runs

pytestmark = [pytest.mark.timeout(1500)]   # the GPU tests are marked one by one: the CPU self-checks are not

KAPPA = 2.0               # units of 2^-23 of the partial-sum magnitude one wgmma step can lose (see the docstring)
UT = 2.0 ** -23           # one ulp of a normalised fp32 value relative to it (the truncating accumulator)
EX2 = 2.0 ** -21          # relative error of ex2.approx.ftz.f32
F64_REF = 2.0 ** -53      # float64 unit roundoff: the reference's own rounding (see the docstring)
TEETH_FRAC = 0.10
TAIL_STAGES = 32          # keys with at most this many K-stages must show the ragged-tail defect (see the docstring)
FORWARD = runs(("forward", "predict"))     # (config, batch): one recorded forward each
TRAIN = runs(("train",))
RECORDED = ["gemm", "gemm_grouped", "gemm_splitk", "attention", "ln_qkv", "proj_residual", "ln_mlp_residual",
            "gated_conv1x1", "conv3x3_bn_act"]


def cdiv(a, b):
    return -(-a // b)


def pad8(x):
    return cdiv(x, 8) * 8


def align256(x):
    return cdiv(x, 256) * 256


# ---- geometry keys ---------------------------------------------------------------------------------------------------
def _sg(s):
    """(rows, cols, ld, planes) of a Split."""
    return None if s is None else (int(s.rows), int(s.cols), int(s.ld), int(s.nsplit))


def _tg(t):
    """(rows, cols, row stride) of a 2-D fp32 tensor view."""
    return None if t is None else (int(t.shape[-2]), int(t.shape[-1]), int(t.stride(-2)))


def gemm_fields(a, w, kw, sk_ws=None):
    """The geometry of one ops.gemm problem: everything that selects a code path or an address."""
    g = dict(kw)
    ns = min(a.nsplit, w.nsplit)
    res, out = g.get("residual"), g.get("out_f32")
    if res is None:
        rk = "none"
    elif g.get("res_row_mod", 0) > 0:
        rk = "row_mod"
    elif out is not None and res.data_ptr() == out.data_ptr() and res.stride() == out.stride():
        rk = "inplace"
    else:
        rk = "separate"
    osp = g.get("out_split")
    regroup, gather, conv = g.get("regroup"), g.get("a_gather"), g.get("conv")
    return frozen(dict(
        M=int(a.rows if g.get("M") is None else g["M"]), N=int(w.rows if g.get("N") is None else g["N"]),
        K=int(a.cols if g.get("K") is None else g["K"]), nsplit=ns, conv=None if conv is None else tuple(conv),
        act=int(g.get("act", 0)), bias=g.get("bias") is not None, res=rk, res_row_mod=int(g.get("res_row_mod", 0)),
        res_geom=_tg(res) if rk in ("separate", "row_mod") else None,
        regroup=None if regroup is None else tuple(int(v) for v in regroup),
        a_gather=None if gather is None else tuple(int(v) for v in gather),
        offsets=tuple(int(g.get(k, 0)) for k in ("a_row_offset", "a_col_offset", "w_row_offset", "w_col_offset",
                                                  "out_row_offset", "out_col_offset")),
        outs=("f32" if out is not None else "") + ("split" if osp is not None else ""),
        out_f32=_tg(out), out_split=_sg(osp), a=_sg(a), w=_sg(w), sk_ws=sk_ws is not None))


def call_key(fn, args):
    """args: the bound arguments of ops.<fn> (defaults applied) -> a hashable key holding the whole geometry."""
    A = args
    if fn == "gemm":
        return ("gemm", (gemm_fields(A["a"], A["w"], A["kw"], A["sk_ws"]),))
    if fn == "gemm_grouped":
        return ("gemm", tuple(gemm_fields(a, w, kw) for a, w, kw in A["calls"]))
    if fn == "gemm_splitk":
        return ("splitk", frozen(dict(a=_sg(A["a"]), w=_sg(A["w"]), partial=tuple(A["partial"].shape),
                                       out_f32=_tg(A["out_f32"]), K=int(A["K"]), chunks=int(A["chunks"]),
                                       bias=A["bias"] is not None, nsplit=min(A["a"].nsplit, A["w"].nsplit))))
    if fn == "attention":
        pl = A["prompt_logits"]
        return ("attention", frozen(dict(B=A["B"], N=A["N"], H=A["H"], T=int(A["T"]), scale=float(A["scale"]),
                                          qkv=_sg(A["qkv"]), out=_sg(A["out"]), logits=pl is not None,
                                          nsplit=min(A["qkv"].nsplit, A["out"].nsplit))))
    if fn == "ln_qkv":
        return ("ln_qkv", frozen(dict(x=_tg(A["x"]), w=_sg(A["wqkv"]), qkv=_sg(A["qkv"]),
                                       nsplit=min(A["wqkv"].nsplit, A["qkv"].nsplit))))
    if fn == "proj_residual":
        return ("proj_residual", frozen(dict(x=_tg(A["x"]), a=_sg(A["ao"]), w=_sg(A["wproj"]),
                                              nsplit=min(A["ao"].nsplit, A["wproj"].nsplit))))
    if fn == "ln_mlp_residual":
        return ("ln_mlp_residual", frozen(dict(x=_tg(A["x"]), w1=_sg(A["w1"]), w2=_sg(A["w2"]),
                                                nsplit=min(A["w1"].nsplit, A["w2"].nsplit))))
    if fn == "gated_conv1x1":
        t0 = A["tasks"][0]
        return ("gated_conv1x1", frozen(dict(
            x=tuple(A["x"].shape) + (int(A["x"].stride(-2)),), x_group_rows=int(A["x_group_rows"]),
            x_row_offset=int(A["x_row_offset"]), logits=tuple(A["prompt_logits"].shape),
            chan_lg=tuple(A["chan_lg"].shape), ntasks=len(A["tasks"]), e=int(A["e"]), chan_col=int(A["chan_col"]),
            w_spa=_sg(t0[0]), w_chan=_sg(t0[2]), cat=_sg(t0[4]), nsplit=min(t0[0].nsplit, t0[4].nsplit),
            shape=tuple(int(A[k]) for k in ("B", "T", "N", "H", "Cdim", "gh", "gw", "nh", "nw")))))
    if fn == "conv3x3_bn_act":
        return ("conv3x3_bn_act", frozen(dict(
            a=_sg(A["a"]), w3=_sg(A["w3"]), Cin=int(A["Cin"]), Cout=int(A["Cout"]), act=int(A["act"]),
            conv=(int(A["B"]), int(A["H"]), int(A["W"]), int(A["dil"])), mid=_sg(A["mid"]), w_head=_sg(A["w_head"]),
            n_out=int(A["n_out"]), out_f32=_tg(A["out_f32"]), nsplit=min(A["a"].nsplit, A["w3"].nsplit))))
    raise KeyError(fn)


SPLIT_FIELDS = {"a", "w", "out_split", "qkv", "out", "mid", "w3", "w_head", "w1", "w2", "w_spa", "w_chan", "cat"}


def without_planes(key):
    """A key with every plane count removed (the nsplit field and the last entry of each Split geometry, found by
    field name): what a speed-mode build must record identically."""
    def strip(fields):
        return tuple((k, v[:3] if k in SPLIT_FIELDS and v is not None else v) for k, v in fields if k != "nsplit")
    kind, body = key
    return (kind, tuple(strip(p) for p in body)) if kind == "gemm" else (kind, strip(body))


def launches_of(key):
    """The profiled tensor-core launches (kind, M, N, K * taps) one recorded call issues (block_ops.cu for composites)."""
    kind, body = key
    if kind == "gemm":
        f = dict(body[0])
        taps = f["conv"][3] ** 2 if f["conv"] else 1
        return [(0, f["M"] * len(body), f["N"], f["K"] * taps)]
    f = dict(body)
    if kind == "splitk":
        M, N, K, chunks = f["a"][0], f["w"][0], f["K"], f["chunks"]
        step = cdiv(cdiv(K, chunks), 64) * 64
        ks = [min(step, K - k0) for k0 in range(0, K, step)]
        return [(0, M * len(ks), N, ks[0])] if len(set(ks)) == 1 and len(ks) > 1 else [(0, M, N, k) for k in ks]
    if kind == "attention":
        return [(1, f["B"] * f["N"], f["N"], f["H"] * 64)]
    if kind == "ln_qkv":
        rows, C = f["x"][:2]
        return [(0, rows, 3 * C, C)]
    if kind == "proj_residual":
        rows, C = f["x"][:2]
        return [(0, rows, C, C)]
    if kind == "ln_mlp_residual":
        rows, C = f["x"][:2]
        hid = f["w1"][0]
        return [(0, rows, hid, C), (0, rows, C, hid)]
    if kind == "gated_conv1x1":
        B, T, N, H, C, gh, gw = f["shape"][:7]
        rows, out = B * gh * gw, []
        for k0 in range(0, f["ntasks"], 6):
            out.append((0, rows * 2 * min(6, f["ntasks"] - k0), f["e"], C))
        return out
    if kind == "conv3x3_bn_act":
        B, H, W, _ = f["conv"]
        out = [(0, B * H * W, f["Cout"], 9 * f["Cin"])]
        if f["w_head"] is not None:
            out.append((0, B * H * W, f["n_out"], f["Cout"]))
        return out
    raise KeyError(kind)


# ---- float64 references ------------------------------------------------------------------------------------------------
def _stage_cols(K, P):
    """Per product kind (P of them), the chain weight n_s - j(k) of every column k of one K-long block (a GEMM, or one
    tap of a convolution): stages of 64, k16 steps, the last stage holding ceil(rem / 16) steps."""
    k = torch.arange(K)
    s = k // 64
    nkb = cdiv(K, 64)
    last = cdiv(K - 64 * (nkb - 1), 16)
    nsteps = torch.where(s == nkb - 1, torch.full_like(s, last), torch.full_like(s, 4)) * P
    ks = (k % 64) // 16
    return [(nsteps - (ks * P + kind)).double() for kind in range(P)]


def gemm_ref(spec, tail=False):
    """Exact float64 sum of the issued products of one GEMM stage and the accumulator's error bound (chain + fold).
    spec: a (Split), w (Split), ns, M, N, K, conv (B, H, W, ks, dil) or None, arow (A rows, plain), aco, wro, wco.
    tail: also return the part the last K-stage of every tap takes from a_hi w_lo (the altered-operand defect)."""
    a, w, ns, M, N, K = spec["a"], spec["w"], spec["ns"], spec["M"], spec["N"], spec["K"]
    aco, wro, wco = spec.get("aco", 0), spec.get("wro", 0), spec.get("wco", 0)
    dev = a.buf.device
    P = 3 if ns == 2 else 1
    pairs = [(0, 0), (0, 1), (1, 0)][:P]                            # (A plane, W plane) in issue order
    wts = [t.to(dev) for t in _stage_cols(K, P)]
    conv = spec.get("conv")
    if conv is None:
        taps = [(None, 0)]
        rows = spec["arow"].to(dev)
        Ablk = lambda p, t: p[rows, aco:aco + K].double()
    else:
        B, H, W, ks, dil = conv
        cp = cdiv(K, 64) * 64
        taps = [((ky, kx), t * cp) for t, (ky, kx) in enumerate((ky, kx) for ky in range(ks) for kx in range(ks))]
        pd = dil * (ks // 2)

        rows = spec["arow"].to(dev)

        def Ablk(p, t):
            x = F.pad(p[rows, aco:aco + K].double().reshape(B, H, W, K), (0, 0, pd, pd, pd, pd))
            ky, kx = t
            return x[:, ky * dil:ky * dil + H, kx * dil:kx * dil + W, :].reshape(M, K)
    Ap, Wp = planes(a, ns), planes(w, ns)
    y = torch.zeros(M, N, dtype=torch.float64, device=dev)
    chain, absP = torch.zeros_like(y), torch.zeros_like(y)
    tl = torch.zeros_like(y) if tail else None
    nkb = cdiv(K, 64)
    for t, c0 in taps:
        As = [Ablk(p, t) for p in Ap]
        Ws = [p[wro:wro + N, wco + c0:wco + c0 + K].double() for p in Wp]
        for kind, (ia, iw) in enumerate(pairs):
            chain += (As[ia].abs() * wts[kind]) @ Ws[iw].abs().t()
        for s in range(nkb):
            sl = slice(64 * s, min(K, 64 * s + 64))
            Ps = sum(As[ia][:, sl] @ Ws[iw][:, sl].t() for ia, iw in pairs)
            y += Ps
            absP += Ps.abs()
            if tail and s == nkb - 1 and ns == 2:
                tl += As[0][:, sl] @ Ws[1][:, sl].t()
    D = 2 * len(taps) * nkb + 1 + spec.get("d_extra", 0)
    E = KAPPA * UT * chain + sum_tol(D, absP) + F64_REF * (64 + len(taps) * nkb) * chain
    return y, E, tl, len(taps) * nkb


def gelu64(v):
    return 0.5 * v * (1.0 + torch.erf(v / math.sqrt(2.0)))


def epilogue(v, E, bias, act, res):
    """epilogue_op in float64: bias add, activation, residual add, each with its fp32 error (see the docstring)."""
    if bias is not None:
        v = v + bias
        E = E + U * (v.abs() + E)
    if act == 1:
        g = gelu64(v)
        E = 1.13 * E + 0.5 * v.abs() * 4 * UT + 4 * U * g.abs()
        v = g
    elif act == 2:
        v = v.clamp_min(0)
    if res is not None:
        v = v + res
        E = E + U * (v.abs() + E)
    return v, E


def stage_check(spec, teeth=None):
    """Check one GEMM stage's outputs against its reference and bound. spec also holds bias (fp32 or None), act,
    res (float64 [M, N] as consumed, or None) and outs: [("f32", tensor, rows, col0) | ("split", Split, rows, col0)].
    teeth=None: assert and return the worst ratio. teeth="speed": return the fraction of elements over the bound.
    teeth="tail": assert every element the tail defect moves by > 2 x bound is flagged; return (fraction flagged,
    fraction the defect moves by > 2 x bound), each the larger over the stage's outputs."""
    M, N = spec["M"], spec["N"]
    y, E, tl, _ = gemm_ref(spec, tail=teeth == "tail")
    bias = spec.get("bias")
    b = None if bias is None else bias[:N].double()[None]
    if b is not None and spec.get("bias_first"):  # mtt_sum_partials starts its sum from the bias: one more term
        E = E + sum_tol(spec["d_extra"], b.abs())
    ref, bound = epilogue(y, E, b, spec.get("act", 0), spec.get("res"))
    moved = None
    if teeth == "tail":
        alt, _ = epilogue(y - tl, E, b, spec.get("act", 0), spec.get("res"))
        moved = (alt - ref).abs()
    worst, frac, detectable = 0.0, 0.0, 0.0
    f32 = [o for o in spec["outs"] if o[0] == "f32"]
    for kind, buf, rows, c0 in spec["outs"]:
        rows = rows.to(ref.device)
        if kind == "f32":
            got = buf[rows, c0:c0 + N].double()
            bnd = bound
        else:
            got = buf.buf[0][rows, c0:c0 + N].double()
            if buf.nsplit == 2:
                got = got + buf.buf[1][rows, c0:c0 + N].double()
            bnd = bound + split_bound(buf.nsplit, ref.abs() + bound)
            if f32 and teeth is None:       # both outputs: the split is the RN split of the fp32 value, bit for bit
                o32 = f32[0][1][f32[0][2].to(ref.device), f32[0][3]:f32[0][3] + N]
                hi = o32.bfloat16()
                assert torch.equal(bits(buf.buf[0][rows, c0:c0 + N]), bits(hi)), "split hi != RN_bf16(out_f32)"
                if buf.nsplit == 2:
                    lo = (o32 - hi.float()).bfloat16()
                    assert torch.equal(bits(buf.buf[1][rows, c0:c0 + N]), bits(lo)), "split lo != RN_bf16(out - hi)"
        if teeth is None:
            worst = max(worst, check(got, ref, bnd, f"{spec['what']} {kind}"))
            continue
        err = (got - ref).abs()
        flagged = ~(err <= bnd)
        frac = max(frac, float(flagged.double().mean()))
        if teeth == "tail":
            must = moved > 2 * bnd
            detectable = max(detectable, float(must.double().mean()))
            missed = must & ~flagged
            assert not missed.any(), (f"{spec['what']}: the last-stage lo defect moves {int(must.sum())} elements by "
                                      f"more than twice their bound, {int(missed.sum())} of them pass it")
    if teeth == "tail":
        return frac, detectable
    return worst if teeth is None else frac


def attn_ref(qkv, B, N, H, ns, scale, b, heads):
    """Float64 softmax(q k^T scale) v of image b, heads `heads`, from the issued products; returns (O, bound of O, S,
    bound of S), O / S as [h, N, 64] / [h, N, N]."""
    C = H * 64
    rows = slice(b * N, (b + 1) * N)
    part = lambda p, off: p[rows, off:off + C].double().view(N, H, 64)[:, heads].permute(1, 0, 2)
    Pq = [part(p, 0) for p in planes(qkv, ns)]
    Pk = [part(p, C) for p in planes(qkv, ns)]
    Pv = [part(p, 2 * C) for p in planes(qkv, 2)]
    P = 3 if ns == 2 else 1
    pairs = [(0, 0), (0, 1), (1, 0)][:P]
    wts = [t.to(qkv.buf.device) for t in _stage_cols(64, P)]
    S = sum(Pq[i] @ Pk[j].transpose(1, 2) for i, j in pairs)
    ch = sum((Pq[i].abs() * wts[kk]) @ Pk[j].abs().transpose(1, 2) for kk, (i, j) in enumerate(pairs))
    eS = KAPPA * UT * ch + F64_REF * 65 * ch
    x = S * scale
    d = (scale * eS).amax(-1, keepdim=True) + 3 * U * x.abs().amax(-1, keepdim=True)
    wgt = torch.softmax(x, -1)
    nkv = cdiv(N, 64)
    p_rel = 2.0 ** -16 + (2.0 ** -8 if ns == 1 else 0.0)
    w_rel = torch.expm1(2 * d) + EX2 * (nkv + 1) + p_rel
    norm = 2 * w_rel / (1 - w_rel) + sum_tol(16 + nkv + 2, 1.0)
    V = Pv[0] + Pv[1] if ns == 2 else Pv[0]
    O = wgt @ V
    Wabs = wgt @ V.abs()
    arith = KAPPA * UT * 4 * P + (2.0 ** -17 if ns == 2 else 0.0) + sum_tol(nkv + 1, 1.0)
    bound = (norm + arith) * Wabs + (2 * U + SPLIT) * O.abs() + SPLIT_ABS
    return O, bound, S, eS


# ---- operands ------------------------------------------------------------------------------------------------------------
class Draw:
    """Random operands of one replay: plain normal, or (scaled) with per-row scales 2^u, u uniform in [-20, 20]."""

    def __init__(self, dev, seed, scaled):
        self.g = torch.Generator(device=dev).manual_seed(seed)
        self.dev, self.scaled = dev, scaled

    def randn(self, *shape):
        return torch.randn(*shape, generator=self.g, device=self.dev)

    def rowscale(self, rows):
        if not self.scaled:
            return torch.ones(rows, 1, device=self.dev)
        return torch.exp2(torch.rand(rows, 1, generator=self.g, device=self.dev) * 40 - 20)

    def split(self, geom, zero_cols=None):
        """A fresh 2-plane Split of the recorded (rows, cols, ld): every column [0, ld) random (pad columns too: a read
        past K adds a wrong term); zero_cols: column ranges that must hold zero (conv weights' cin padding)."""
        rows, cols, ld = geom[:3]
        x = self.randn(rows, ld) * self.rowscale(rows)
        for c0, c1 in zero_cols or ():
            x[:, c0:c1] = 0
        sp = mtt_ops().split_f32(x)
        sp.cols = cols
        return sp


def hi_only(sp):
    return mtt_ops().Split.from_planes(sp.buf[:1], sp.cols)


def sentinel_of(geom, dev):
    """A sentinel-filled Split of a recorded (rows, cols, ld, planes) geometry."""
    rows, cols, ld, ns = geom
    return sentinel_split(rows, cols, dev, ns, ld=ld)


def conv_weight_zeros(K, taps, wco):
    cp = cdiv(K, 64) * 64
    return [(wco + t * cp + K, wco + (t + 1) * cp) for t in range(taps)]


def tail_zeroed(w, K, taps, wco):
    """A copy of W whose lo plane is zero in the last K-stage of every tap."""
    ops = mtt_ops()
    sp = ops.Split.from_planes(w.buf.clone(), w.cols)
    cp = cdiv(K, 64) * 64 if taps > 1 else K
    k0 = 64 * (cdiv(K, 64) - 1)
    for t in range(taps):
        sp.buf[1][:, wco + t * cp + k0:wco + t * cp + K] = 0
    return sp


class Outputs:
    """Output buffers with their initial contents; reset() restores them, untouched() checks every element the launch
    had no business writing."""

    def __init__(self):
        self.items = []            # (buffer tensor, initial copy, written mask)

    def add(self, buf):
        m = torch.zeros(buf.shape, dtype=torch.bool, device=buf.device)
        self.items.append((buf, buf.clone(), m))
        return m

    def reset(self):
        for buf, init, _ in self.items:
            buf.copy_(init)

    def untouched(self, what):
        for buf, init, m in self.items:
            same = bits(buf) == bits(init)
            bad = ~m & ~same
            assert not bad.any(), f"{what}: {int(bad.sum())} elements outside the output written"


# ---- replay of one recorded call ------------------------------------------------------------------------------------------
class Case:
    """A recorded call on fresh buffers: run(ns, tail) launches it (tail: W lo zeroed in the last stage of the final
    GEMM stage), specs(ns) describes each GEMM stage for stage_check."""

    def __init__(self, key, draw, dev):
        self.key, self.draw, self.dev = key, draw, dev
        self.out = Outputs()
        self.kind = key[0]
        getattr(self, "_build_" + self.kind)(key[1])

    # plain / grouped GEMM ------------------------------------------------------------------------------------------
    def _problem(self, fields):
        f = dict(fields)
        d, dev = self.draw, self.dev
        M, N, K = f["M"], f["N"], f["K"]
        aro, aco, wro, wco, oro, oco = f["offsets"]
        taps = f["conv"][3] ** 2 if f["conv"] else 1
        a = d.split(f["a"])
        w = d.split(f["w"], conv_weight_zeros(K, taps, wco) if f["conv"] else None)
        kw = dict(M=M, N=N, K=K, act=f["act"], a_row_offset=aro, a_col_offset=aco, w_row_offset=wro, w_col_offset=wco,
                  out_row_offset=oro, out_col_offset=oco)
        if f["conv"]:
            kw["conv"] = f["conv"]
        if f["regroup"]:
            kw["regroup"] = f["regroup"]
        if f["a_gather"]:
            kw["a_gather"] = f["a_gather"]
        bias = d.randn(N) if f["bias"] else None
        kw["bias"] = bias
        r = torch.arange(M, device=dev)
        ro = X.out_rows(r, f["regroup"])
        outs, res = [], None
        if f["out_f32"] is not None:
            rows, cols, ld = f["out_f32"]
            buf = sentinel((rows, ld), dev=dev)
            if f["res"] == "inplace":
                buf.copy_(d.randn(rows, ld))
            m = self.out.add(buf)
            m[ro[:, None], torch.arange(N, device=dev)[None]] = True
            kw["out_f32"] = buf[:, :cols]
            outs.append(("f32", buf, ro, 0))
        if f["res"] in ("separate", "row_mod"):
            rows, cols, ld = f["res_geom"]
            rbuf = d.randn(rows, ld)
            kw["residual"], kw["res_row_mod"] = rbuf[:, :cols], f["res_row_mod"]
            rr = r % f["res_row_mod"] if f["res_row_mod"] else ro
            res = rbuf[rr, :N].double()
        elif f["res"] == "inplace":
            kw["residual"] = kw["out_f32"]
            res = self.out.items[-1][1][ro, :N].double()
        if f["out_split"] is not None:
            osp = sentinel_of(f["out_split"], dev)
            m = self.out.add(osp.buf)
            m[:, (ro + oro)[:, None], oco + torch.arange(N, device=dev)[None]] = True
            kw["out_split"] = osp
            outs.append(("split", osp, ro + oro, oco))
        if f["a_gather"]:
            arow = aro + (r // f["a_gather"][0]) * f["a_gather"][1] + r % f["a_gather"][0]
        else:
            arow = aro + r
        spec = dict(M=M, N=N, K=K, conv=f["conv"], arow=arow, aco=aco, wro=wro, wco=wco, bias=bias, act=f["act"],
                    res=res, outs=outs, what=f"gemm {M}x{N}x{K}")
        return a, w, kw, spec, taps, f["sk_ws"]

    def _build_gemm(self, body):
        self.probs = [self._problem(p) for p in body]
        self.sk = mtt_ops().streamk_workspace(self.dev) if self.probs[0][5] else None
        self.K, self.taps = self.probs[0][3]["K"], self.probs[0][4]

    def _run_gemm(self, ns, tail):
        ops = mtt_ops()
        calls = []
        for a, w, kw, spec, taps, _ in self.probs:
            if tail:
                w = tail_zeroed(w, spec["K"], taps, spec["wco"])
            if ns == 1:
                a, w = hi_only(a), hi_only(w)
            calls.append((a, w, kw))
        if len(calls) == 1:
            ops.gemm(calls[0][0], calls[0][1], sk_ws=self.sk, **calls[0][2])
        else:
            ops.gemm_grouped(calls)

    def _specs_gemm(self, ns):
        return [dict(p[3], a=p[0], w=p[1], ns=ns) for p in self.probs]

    # split-K -----------------------------------------------------------------------------------------------------------
    def _build_splitk(self, body):
        f = dict(body)
        d, dev = self.draw, self.dev
        self.a, self.w = d.split(f["a"]), d.split(f["w"])
        M, N, K = f["a"][0], f["w"][0], f["K"]
        self.partial = torch.empty(f["partial"], device=dev)
        rows, cols, ld = f["out_f32"]
        buf = sentinel((rows, ld), dev=dev)
        m = self.out.add(buf)
        m[:M, :N] = True
        self.o32 = buf[:, :cols]
        self.bias = d.randn(N) if f["bias"] else None
        self.chunks, self.K, self.taps = f["chunks"], K, 1
        self.spec = dict(M=M, N=N, K=K, conv=None, arow=torch.arange(M, device=dev), bias=self.bias, act=0, res=None,
                         outs=[("f32", buf, torch.arange(M, device=dev), 0)], d_extra=f["chunks"] + 1, bias_first=True,
                         what=f"splitk {M}x{N}x{K}/{f['chunks']}")

    def _run_splitk(self, ns, tail):
        a, w = self.a, tail_zeroed(self.w, self.K, 1, 0) if tail else self.w
        if ns == 1:
            a, w = hi_only(a), hi_only(w)
        mtt_ops().gemm_splitk(a, w, self.partial, self.o32, K=self.K, bias=self.bias, chunks=self.chunks)

    def _specs_splitk(self, ns):
        return [dict(self.spec, a=self.a, w=self.w, ns=ns)]

    # composites ----------------------------------------------------------------------------------------------------------
    def _x(self, geom):
        rows, cols, ld = geom
        buf = self.draw.randn(rows, ld) + 0.5 * self.draw.randn(rows, 1)
        return buf, buf[:, :cols]

    def _ln(self, C):
        return 1 + 0.2 * self.draw.randn(C), 0.2 * self.draw.randn(C)

    def _build_ln_qkv(self, body):
        f = dict(body)
        ops, d, dev = mtt_ops(), self.draw, self.dev
        rows, C = f["x"][:2]
        self.xbuf, self.x = self._x(f["x"])
        self.g, self.b = self._ln(C)
        self.w, self.bias = d.split(f["w"]), d.randn(3 * C)
        self.qkv = sentinel_of(f["qkv"], dev)
        m = self.out.add(self.qkv.buf)
        m[:, :rows, :3 * C] = True
        self.rows, self.C, self.K, self.taps = rows, C, C, 1

    def _run_ln_qkv(self, ns, tail):
        ops = mtt_ops()
        w = tail_zeroed(self.w, self.C, 1, 0) if tail else self.w
        w = hi_only(w) if ns == 1 else w
        self.ws = ops.workspace(ops.workspace_bytes(ops.OP_LN_QKV, rows=self.rows, Cdim=self.C, nsplit=ns), self.dev)
        ops.ln_qkv(self.x, self.g, self.b, 1e-6, w, self.bias, self.qkv, self.ws)

    def _specs_ln_qkv(self, ns):
        r = torch.arange(self.rows, device=self.dev)
        xn = mtt_ops().ws_split_view(self.ws, 0, self.rows, self.C, ns)
        return [dict(a=xn, w=self.w, ns=ns, M=self.rows, N=3 * self.C, K=self.C, conv=None, arow=r, bias=self.bias,
                     act=0, res=None, outs=[("split", self.qkv, r, 0)], what="ln_qkv")]

    def _build_proj_residual(self, body):
        f = dict(body)
        d = self.draw
        rows, C = f["x"][:2]
        self.a, self.w, self.bias = d.split(f["a"]), d.split(f["w"]), d.randn(C)
        xbuf = d.randn(rows, f["x"][2])
        m = self.out.add(xbuf)
        m[:, :C] = True
        self.xbuf, self.x, self.rows, self.C, self.K, self.taps = xbuf, xbuf[:, :C], rows, C, C, 1
        self.x0 = xbuf[:, :C].double().clone()

    def _run_proj_residual(self, ns, tail):
        a, w = self.a, tail_zeroed(self.w, self.C, 1, 0) if tail else self.w
        if ns == 1:
            a, w = hi_only(a), hi_only(w)
        mtt_ops().proj_residual(a, w, self.bias, self.x)

    def _specs_proj_residual(self, ns):
        r = torch.arange(self.rows, device=self.dev)
        return [dict(a=self.a, w=self.w, ns=ns, M=self.rows, N=self.C, K=self.C, conv=None, arow=r, bias=self.bias,
                     act=0, res=self.x0, outs=[("f32", self.xbuf, r, 0)], what="proj_residual")]

    def _build_ln_mlp_residual(self, body):
        f = dict(body)
        d = self.draw
        rows, C, ld = f["x"]
        hid = f["w1"][0]
        self.xbuf = d.randn(rows, ld) + 0.5 * d.randn(rows, 1)
        m = self.out.add(self.xbuf)
        m[:, :C] = True
        self.x, self.x0 = self.xbuf[:, :C], self.xbuf[:, :C].double().clone()
        self.g, self.b = self._ln(C)
        self.w1, self.b1, self.w2, self.b2 = d.split(f["w1"]), d.randn(hid), d.split(f["w2"]), d.randn(C)
        self.rows, self.C, self.hid, self.K, self.taps = rows, C, hid, hid, 1

    def _run_ln_mlp_residual(self, ns, tail):
        ops = mtt_ops()
        w1, w2 = self.w1, tail_zeroed(self.w2, self.hid, 1, 0) if tail else self.w2
        if ns == 1:
            w1, w2 = hi_only(w1), hi_only(w2)
        self.ws = ops.workspace(ops.workspace_bytes(ops.OP_LN_MLP_RESIDUAL, rows=self.rows, Cdim=self.C,
                                                    hidden=self.hid, nsplit=ns), self.dev)
        ops.ln_mlp_residual(self.x, self.g, self.b, 1e-6, w1, self.b1, w2, self.b2, self.ws)

    def _specs_ln_mlp_residual(self, ns):
        ops = mtt_ops()
        r = torch.arange(self.rows, device=self.dev)
        xn = ops.ws_split_view(self.ws, 0, self.rows, self.C, ns)
        h = ops.ws_split_view(self.ws, align256(2 * ns * self.rows * pad8(self.C)), self.rows, self.hid, ns)
        return [dict(a=xn, w=self.w1, ns=ns, M=self.rows, N=self.hid, K=self.C, conv=None, arow=r, bias=self.b1,
                     act=1, res=None, outs=[("split", h, r, 0)], what="ln_mlp fc1"),
                dict(a=h, w=self.w2, ns=ns, M=self.rows, N=self.C, K=self.hid, conv=None, arow=r, bias=self.b2,
                     act=0, res=self.x0, outs=[("f32", self.xbuf, r, 0)], what="ln_mlp fc2")]

    def _build_gated_conv1x1(self, body):
        f = dict(body)
        d, dev = self.draw, self.dev
        B, T, N, H, C, gh, gw, nh, nw = f["shape"]
        xr, xc, xld = f["x"]
        self.xbuf = d.randn(xr, xld)
        self.x = self.xbuf[:, :xc]
        self.logits = d.randn(*f["logits"])
        self.chan = d.randn(*f["chan_lg"])
        self.tasks = []
        for _ in range(f["ntasks"]):
            cat = sentinel_of(f["cat"], dev)
            m = self.out.add(cat.buf)
            m[:, :B * gh * gw, :f["e"]] = True
            m[:, :B * gh * gw, f["chan_col"]:f["chan_col"] + f["e"]] = True
            self.tasks.append([d.split(f["w_spa"]), d.randn(f["e"]), d.split(f["w_chan"]), d.randn(f["e"]), cat])
        self.f, self.rows, self.C, self.K, self.taps = f, B * gh * gw, C, C, 1

    def _run_gated_conv1x1(self, ns, tail):
        ops = mtt_ops()
        f = self.f
        B, T, N, H, C, gh, gw, nh, nw = f["shape"]
        tasks = []
        for ws_, bs, wc, bc, cat in self.tasks:
            if tail:
                ws_, wc = tail_zeroed(ws_, C, 1, 0), tail_zeroed(wc, C, 1, 0)
            if ns == 1:
                ws_, wc = hi_only(ws_), hi_only(wc)
            tasks.append((ws_, bs, wc, bc, cat))
        self.ws = ops.workspace(ops.workspace_bytes(ops.OP_GATED_CONV1X1, rows=self.rows, Cdim=C, nsplit=ns,
                                                    T=len(tasks)), self.dev)
        ops.gated_conv1x1(self.x, f["x_group_rows"], f["x_row_offset"], self.logits, self.chan, tasks, f["e"],
                          f["chan_col"], self.ws, B=B, T=T, N=N, H=H, Cdim=C, gh=gh, gw=gw, nh=nh, nw=nw)

    def _specs_gated_conv1x1(self, ns):
        ops = mtt_ops()
        r = torch.arange(self.rows, device=self.dev)
        pb = align256(2 * ns * self.rows * pad8(self.C))
        out = []
        for k, (ws_, bs, wc, bc, cat) in enumerate(self.tasks):
            for which, (w, b, col) in enumerate(((ws_, bs, 0), (wc, bc, self.f["chan_col"]))):
                a = ops.ws_split_view(self.ws, (2 * k + which) * pb, self.rows, self.C, ns)
                o = cat if ns == 2 else hi_only(cat)      # a speed-mode launch is given no lo plane to write
                out.append(dict(a=a, w=w, ns=ns, M=self.rows, N=self.f["e"], K=self.C, conv=None, arow=r, bias=b,
                                act=0, res=None, outs=[("split", o, r, col)], what=f"gated task {k}.{which}"))
        return out

    def _build_conv3x3_bn_act(self, body):
        f = dict(body)
        d, dev = self.draw, self.dev
        B, H, W, dil = f["conv"]
        M, Cin, Cout = B * H * W, f["Cin"], f["Cout"]
        self.a = d.split(f["a"])
        self.w3, self.b3 = d.split(f["w3"], conv_weight_zeros(Cin, 9, 0)), d.randn(Cout)
        self.mid = None
        if f["mid"] is not None:
            self.mid = sentinel_of(f["mid"], dev)
            m = self.out.add(self.mid.buf)
            m[:, :M, :Cout] = True
        self.wh = self.bh = self.o32 = None
        if f["w_head"] is not None:
            self.wh, self.bh = d.split(f["w_head"]), d.randn(f["n_out"])
            rows, cols, ld = f["out_f32"]
            self.obuf = sentinel((rows, ld), dev=dev)
            m = self.out.add(self.obuf)
            m[:M, :f["n_out"]] = True
            self.o32 = self.obuf[:, :cols]
        self.f, self.M, self.Cin, self.Cout = f, M, Cin, Cout
        self.K, self.taps = (Cout, 1) if self.wh is not None else (Cin, 9)

    def _run_conv3x3_bn_act(self, ns, tail):
        ops = mtt_ops()
        f = self.f
        B, H, W, dil = f["conv"]
        a, w3, wh = self.a, self.w3, self.wh
        if tail:                                  # the final stage's weight: the head when there is one
            if wh is not None:
                wh = tail_zeroed(wh, self.Cout, 1, 0)
            else:
                w3 = tail_zeroed(w3, self.Cin, 9, 0)
        if ns == 1:
            a, w3 = hi_only(a), hi_only(w3)
            wh = hi_only(wh) if wh is not None else None
        self.ws = None
        if self.mid is None:
            self.ws = ops.workspace(ops.workspace_bytes(ops.OP_CONV3X3_BN_ACT, rows=self.M, hidden=self.Cout,
                                                        nsplit=ns), self.dev)
        ops.conv3x3_bn_act(a, w3, self.b3, self.Cin, self.Cout, f["act"], B=B, H=H, W=W, dil=dil, mid=self.mid,
                           w_head=wh, b_head=self.bh, n_out=f["n_out"], out_f32=self.o32, ws=self.ws)

    def _specs_conv3x3_bn_act(self, ns):
        f = self.f
        B, H, W, dil = f["conv"]
        r = torch.arange(self.M, device=self.dev)
        mid = self.mid if self.mid is not None else mtt_ops().ws_split_view(self.ws, 0, self.M, self.Cout, ns)
        out = [dict(a=self.a, w=self.w3, ns=ns, M=self.M, N=self.Cout, K=self.Cin, conv=(B, H, W, 3, dil), arow=r,
                    bias=self.b3,
                    act=f["act"], res=None, outs=[("split", mid, r, 0)], what=f"conv3x3 {B}x{H}x{W} {self.Cin}->{self.Cout}")]
        if self.wh is not None:
            out.append(dict(a=mid, w=self.wh, ns=ns, M=self.M, N=f["n_out"], K=self.Cout, conv=None, arow=r,
                            bias=self.bh, act=0, res=None, outs=[("f32", self.obuf, r, 0)], what="conv3x3 head"))
        return out

    # dispatch -------------------------------------------------------------------------------------------------------------
    def run(self, ns, tail=False):
        self.out.reset()
        getattr(self, "_run_" + self.kind)(ns, tail)
        torch.cuda.synchronize()

    def specs(self, ns):
        return getattr(self, "_specs_" + self.kind)(ns)

    def stages(self):
        return self.taps * cdiv(self.K, 64)


def replay_gemm_key(key, dev, seed):
    """Both modes, both draws, and the teeth on the plain draw. Returns (worst ratio, [(speed-mode fraction flagged or
    None, tail fraction flagged, tail fraction detectable, K-stages)])."""
    ops = mtt_ops()
    worst, teeth = 0.0, []
    for scaled in (False, True):
        case = Case(key, Draw(dev, seed + scaled, scaled), dev)
        case.run(2)
        case.out.untouched(f"{key[0]} parity")
        parity = case.specs(2)
        for sp in parity:
            worst = max(worst, stage_check(sp))
        for sp in parity:        # the planes each parity stage consumed, kept for the speed-mode teeth
            sp["a"] = ops.Split.from_planes(sp["a"].buf.clone(), sp["a"].cols)
        case.run(1)
        case.out.untouched(f"{key[0]} speed")
        for sp in case.specs(1):
            worst = max(worst, stage_check(sp))
        if scaled or case.stages() < 2:
            continue
        # teeth 1: the speed-mode outputs against the parity references and bounds, at every stage whose speed-mode
        # output keeps the precision to show it (fp32, or a split with both planes written)
        speed = [dict(p, outs=q["outs"]) for p, q in zip(parity, case.specs(1))
                 if all(o[0] == "f32" or o[1].nsplit == 2 for o in q["outs"])]
        fr = min(stage_check(sp, "speed") for sp in speed) if speed else None
        assert fr is None or fr >= TEETH_FRAC, f"{key[0]}: the speed-mode result fails the parity bound on only {fr:.3f}"
        # teeth 2: W lo zeroed in the last K-stage of the final GEMM stage's weights
        case.run(2, tail=True)
        specs = case.specs(2)
        final = specs[-1:] if key[0] in ("ln_mlp_residual", "conv3x3_bn_act") else specs
        tails = [stage_check(sp, "tail") for sp in final]
        ft, fd = min(t[0] for t in tails), min(t[1] for t in tails)
        if case.stages() <= TAIL_STAGES:
            assert fd >= TEETH_FRAC and ft >= TEETH_FRAC, (
                f"{key[0]} ({case.stages()} K-stages): the last-stage lo defect exceeds twice the bound on {fd:.3f} "
                f"of the elements and fails it on {ft:.3f}; the bound is too loose to show a ragged-tail defect")
        teeth.append((fr, ft, fd, case.stages()))
    return worst, teeth


def replay_attention_key(key, dev, seed):
    ops = mtt_ops()
    f = dict(key[1])
    B, N, H, T, scale = f["B"], f["N"], f["H"], f["T"], f["scale"]
    worst, teeth = {"attention": 0.0, "prompt_logits": 0.0}, []
    hc = max(1, min(H, (1 << 27) // (N * N)))
    for qs in (1.0, 12.0):
        flagged = total = 0
        d = Draw(dev, seed + int(qs), False)
        x = d.randn(B * N, 3 * H * 64)
        x[:, :H * 64] *= qs
        qkv = ops.split_f32(x)
        out = sentinel_of(f["out"], dev)
        logits = torch.empty(B, H, T, N, device=dev) if f["logits"] else None
        results = {}
        for ns in (2, 1):
            bits(out.buf).fill_(SENTINEL[torch.bfloat16])
            if logits is not None:
                bits(logits).fill_(SENTINEL[torch.float32])
            q = qkv if ns == 2 else hi_only(qkv)
            ops.attention(q, out, B=B, N=N, H=H, scale=scale, prompt_logits=logits, T=T)
            torch.cuda.synchronize()
            results[ns] = (out.buf.clone(), None if logits is None else logits.clone())
        for b in range(B):
            for h0 in range(0, H, hc):
                heads = slice(h0, min(H, h0 + hc))
                for ns in (2, 1):
                    O, bnd, S, eS = attn_ref(qkv, B, N, H, ns, scale, b, heads)
                    ob, lg = results[ns]
                    got = (ob[0, b * N:(b + 1) * N].double() + ob[1, b * N:(b + 1) * N].double()) \
                        .view(N, H, 64)[:, heads].permute(1, 0, 2)
                    worst["attention"] = max(worst["attention"], check(got, O, bnd, f"attention N={N} q*{qs} ns={ns}"))
                    if lg is not None and T:
                        worst["prompt_logits"] = max(worst["prompt_logits"],
                                                     check(lg[b, heads].double(), S[:, :T], eS[:, :T], "prompt_logits"))
                    if ns == 2:                        # teeth: the speed-mode output against the parity bound
                        ob1 = results[1][0]
                        got1 = (ob1[0, b * N:(b + 1) * N].double() + ob1[1, b * N:(b + 1) * N].double()) \
                            .view(N, H, 64)[:, heads].permute(1, 0, 2)
                        flagged += int((~((got1 - O).abs() <= bnd)).sum())
                        total += O.numel()
                    del O, bnd, S, eS
        teeth.append(flagged / total)
    # q x 1 at large N: the speed-mode weight errors average over N keys under the per-weight bound; q x 12 (a few
    # keys dominate each row) does not average, so the teeth are asserted on the draw that flags more
    assert max(teeth) >= TEETH_FRAC, f"attention N={N}: the speed-mode output fails the parity bound on only {teeth}"
    return worst, teeth


# ---- the recording fixture ------------------------------------------------------------------------------------------------
def _build(name, dev, nsplit):
    import bench
    cfg, M, _ = bench.family(name)
    torch.manual_seed(0)
    # a '3ddet' model takes its detection head from the caller; the plan ends at the 4 level maps it hands over
    det = dict(det_head=torch.nn.Identity()) if "3ddet" in cfg["tasks"] and name.startswith("tps_") else {}
    with torch.device(dev):
        return cfg, M.build_from_config(cfg, nsplit=nsplit, use_graph=False, **det)


def _record_run(ops, fn):
    seen = []
    ops.profile_begin()
    try:
        with recording(ops, RECORDED, call_key, seen, outermost_only=True):
            with torch.no_grad():
                fn()
    finally:
        prof = ops.profile_end(max_recs=1 << 16)
    return seen, [tuple(int(v) for v in r[:4]) for r in prof]


def _forward(name, B, dev, nsplit):
    ops = mtt_ops()
    cfg, model = _build(name, dev, nsplit)
    model.eval()
    x = torch.randn(B, 3, *cfg["img_size"], device=dev)
    out = _record_run(ops, lambda: model(x))
    del model
    torch.cuda.empty_cache()
    return out


def _train(name, B, dev):
    import bench
    from mtt_b200.train import TrainStep
    ops = mtt_ops()
    cfg, model = _build(name, dev, 2)
    ts = TrainStep(model, nsplit=2, use_graph=False)
    crit, _ = bench._train_criterion(cfg)
    g = torch.Generator().manual_seed(1)
    x = torch.randn(B, 3, *cfg["img_size"], generator=g).to(dev)
    y = {t: v.to(dev) for t, v in bench._train_labels(cfg, B, g).items()}
    out = _record_run(ops, lambda: ts._fwd_bwd(x, y, crit, None))
    del ts, model
    torch.cuda.empty_cache()
    return out


@pytest.fixture(scope="module")
def recorded(cuda_dev):
    """{(config, batch, "forward" | "train" | "forward_speed"): (recorded keys in call order, profiled launches)}."""
    mtt_ops()
    out = {}
    for name, B in FORWARD:
        out[(name, B, "forward")] = _forward(name, B, cuda_dev, 2)
    out[("tp_cfg4", 4, "forward_speed")] = _forward("tp_cfg4", 4, cuda_dev, 1)
    for name, B in TRAIN:
        out[(name, B, "train")] = _train(name, B, cuda_dev)
    return out


def distinct(seq):
    return list(dict.fromkeys(seq))


# ---- GPU tests ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_recording_explains_every_launch(recorded):
    """Every profiled tensor-core launch of every recorded run is issued by a recorded call, and every recorded call
    issued the launches it should: the multisets are equal."""
    for (name, B, part), (seen, prof) in recorded.items():
        assert seen, f"{name} b{B} {part}: nothing recorded"
        want = collections.Counter(l for k in seen for l in launches_of(k))
        got = collections.Counter(prof)
        extra, missing = got - want, want - got
        assert not extra, f"{name} b{B} {part}: launches no recorded call explains: {sorted(extra.items())[:6]}"
        assert not missing, (f"{name} b{B} {part}: recorded calls whose launches were not profiled: "
                             f"{sorted(missing.items())[:6]}")
        print(f"{name} b{B} {part}: {len(seen)} calls, {len(distinct(seen))} distinct keys, {len(prof)} tensor-core "
              f"launches")
    assert {(n, B, "forward") for n, B in FORWARD} | {(n, B, "train") for n, B in TRAIN} <= set(recorded)
    _assert_reaches(recorded)


def _fields(key):
    """The field dicts of a key (one per problem of a grouped GEMM)."""
    return [dict(p) for p in key[1]] if key[0] == "gemm" else [dict(key[1])]


def _assert_reaches(recorded):
    """The runs reach the geometries they are in the list for."""
    keys = lambda name, B, part="forward": distinct(recorded[(name, B, part)][0])
    # ip_nyud_vitL: 7 x 9 key maps, Tk = 4 * 63 = 252 at every stage: the grouped QK^T has N = 252 and the grouped
    # P.V has K = 252 (a 60-deep last K-stage; ip_cfg3's 320 = 5 x 64 has none)
    ip = [f for k in keys("ip_nyud_vitL", 6) if k[0] == "gemm" and len(k[1]) > 1 for f in _fields(k)]
    assert any(f["K"] == 252 for f in ip) and any(f["N"] == 252 for f in ip), "ip_nyud_vitL: no Tk = 252 GEMM"
    # tp_nyud_vitL: attention over N = 4 + 28 * 36 = 1012 tokens at 16 heads, 6 images
    att = [dict(k[1]) for k in keys("tp_nyud_vitL", 6) if k[0] == "attention"]
    assert {(f["B"], f["N"], f["H"]) for f in att} == {(6, 1012, 16)}, att
    # tp_pascal_vitB: e = 780 columns per gate, the channel gate's at column 784, and f = 1024; tp_cfg4 at valBatch 6:
    # M = 6 * 1029
    gc = [dict(k[1]) for k in keys("tp_pascal_vitB", 6) if k[0] == "gated_conv1x1"]
    assert gc and {(f["e"], f["chan_col"]) for f in gc} == {(780, 784)}, gc
    assert any(f["N"] == 1024 for k in keys("tp_pascal_vitB", 6) if k[0] == "gemm" for f in _fields(k))
    assert any(dict(k[1])["x"][0] == 6 * 1029 for k in keys("tp_cfg4", 6) if k[0] == "ln_qkv")
    assert any(f["M"] == 2 * 1029 for k in keys("tp_pascal_vitB", 2, "train") if k[0] == "gemm" for f in _fields(k))


@pytest.mark.gpu
def test_speed_mode_plan_records_the_same_keys(recorded):
    """tp_cfg4 built with nsplit = 1 issues the same geometries apart from the plane counts: a speed-mode replay of
    the parity keys covers the speed-mode plan."""
    par = {without_planes(k) for k in recorded[("tp_cfg4", 4, "forward")][0]}
    spd = {without_planes(k) for k in recorded[("tp_cfg4", 4, "forward_speed")][0]}
    assert par == spd, (sorted(par - spd, key=str)[:3], sorted(spd - par, key=str)[:3])
    modes = {dict(k[1] if k[0] != "gemm" else k[1][0])["nsplit"] for k in recorded[("tp_cfg4", 4, "forward_speed")][0]}
    assert modes == {1}, modes


def _replay_all(recorded, name, B, part, dev):
    ops = mtt_ops()
    ops.set_gemm_variant(0)
    ops.set_gemm_streamk(1)
    keys = distinct(recorded[(name, B, part)][0])
    worst = collections.defaultdict(float)
    speed, tail, attn = [], [], []
    t0 = time.time()
    for i, key in enumerate(keys):
        if key[0] == "attention":
            w, fr = replay_attention_key(key, dev, 1000 + 10 * i)
            for k, v in w.items():
                worst[k] = max(worst[k], v)
            attn.append(fr)
            print(f"  attention N={dict(key[1])['N']}: speed-mode teeth flag {fr[0]:.3f} (q x 1), {fr[1]:.3f} (q x 12)")
        else:
            kind = key[0]
            if kind == "gemm":
                f = dict(key[1][0])
                kind = ("conv" if f["conv"] else "gemm") + ("_grouped" if len(key[1]) > 1 else "")
            w, th = replay_gemm_key(key, dev, 1000 + 10 * i)
            worst[kind] = max(worst[kind], w)
            speed += [t[0] for t in th if t[0] is not None]
            tail += [t[1:] for t in th]
        torch.cuda.empty_cache()
    print(f"\n{name} b{B} {part}: {len(keys)} distinct keys replayed in {time.time() - t0:.0f} s")
    for k in sorted(worst):
        print(f"  worst err/bound {k:16s} {worst[k]:.3f}")
    fractions = (("speed-mode teeth", speed),
                 (f"last-stage lo teeth, <= {TAIL_STAGES} K-stages", [t[0] for t in tail if t[2] <= TAIL_STAGES]),
                 (f"last-stage lo teeth, > {TAIL_STAGES} K-stages", [t[0] for t in tail if t[2] > TAIL_STAGES]))
    for what, v in fractions:
        if v:
            print(f"  {what}: flagged fraction min {min(v):.3f} median {sorted(v)[len(v) // 2]:.3f} over {len(v)} keys")


@pytest.mark.gpu
@pytest.mark.parametrize("name,B", [pytest.param(n, B, id=run_id(n, B)) for n, B in FORWARD])
def test_forward_launches_f64(recorded, cuda_dev, name, B):
    _replay_all(recorded, name, B, "forward", cuda_dev)


@pytest.mark.gpu
@pytest.mark.parametrize("name,B", [pytest.param(n, B, id=run_id(n, B)) for n, B in TRAIN])
def test_train_launches_f64(recorded, cuda_dev, name, B):
    _replay_all(recorded, name, B, "train", cuda_dev)


# ---- CPU self-checks ---------------------------------------------------------------------------------------------------------
def _spec_of_call(a, w, kw, ns):
    """gemm_ref's spec of an ops.gemm call (host tensors)."""
    M = a.rows if kw.get("M") is None else kw["M"]
    N = w.rows if kw.get("N") is None else kw["N"]
    K = a.cols if kw.get("K") is None else kw["K"]
    r = torch.arange(M)
    g = kw.get("a_gather")
    aro = kw.get("a_row_offset", 0)
    arow = aro + ((r // g[0]) * g[1] + r % g[0] if g else r)
    return dict(a=a, w=w, ns=ns, M=M, N=N, K=K, conv=kw.get("conv"), arow=arow, aco=kw.get("a_col_offset", 0),
                wro=kw.get("w_row_offset", 0), wco=kw.get("w_col_offset", 0))


def test_reference_builder_matches_exact_reference():
    """On integer planes (nothing rounds) gemm_ref + epilogue equals test_tc_exact_gpu.ref_gemm bit for bit: plain,
    regrouped with a row-mod residual, gathered A, and a dilated convolution with a residual, in both modes."""
    builds = [X.plain_case(129, 257, 130, residual=True, act=2, seed=5),
              X.plain_case(127, 129, 130, nsplit=1, residual=True, inplace=True),
              X.regroup_case((100, 105, 5), res_row_mod=100), X.gather_case(10, 32, 40),
              X.conv_case(2, 7, 9, 37, 130, 3, 2, residual=True), X.conv_case(1, 12, 20, 65, 8, 1, 1, nsplit=1)]
    for build in builds:
        calls, outs = build("cpu")
        (a, w, kw), = calls
        ns = min(a.nsplit, w.nsplit)
        res = kw.get("residual")
        res0 = None if res is None else res.clone()
        X.ref_gemm(a, w, **kw)
        spec = _spec_of_call(a, w, kw, ns)
        y, E, _, _ = gemm_ref(spec)
        r = torch.arange(spec["M"])
        ro = X.out_rows(r, kw.get("regroup"))
        rv = None
        if res0 is not None:
            rr = r % kw["res_row_mod"] if kw.get("res_row_mod", 0) > 0 else ro
            rv = res0[rr, :spec["N"]].double()
        b = kw.get("bias")
        v, _ = epilogue(y, E, None if b is None else b[:spec["N"]].double()[None], kw.get("act", 0), rv)
        if kw.get("out_f32") is not None:
            want = kw["out_f32"][ro, :spec["N"]]
            assert torch.equal(bits(v.float()), bits(want)), "reference builder != ref_gemm"
        assert float(E.max()) > 0


def _rz(x):
    """float64 -> the fp32 value rounded toward zero."""
    f = x.float()
    over = f.double().abs() > x.abs()
    return torch.where(over, torch.nextafter(f, torch.zeros_like(f)), f)


def _model_kernel(a, w, ns):
    """The kernel's arithmetic on the host: per 64-deep stage a fresh fp32 accumulator, one step per k16 and product
    (hi.hi, hi.lo, lo.hi), each step's exact sum truncated to fp32; the stages folded with round-to-nearest fp32 adds."""
    M, K = a.rows, a.cols
    pairs = [(0, 0), (0, 1), (1, 0)][:3 if ns == 2 else 1]
    A = [a.buf[i, :, :K].double() for i in range(2)]
    W = [w.buf[i, :, :K].double() for i in range(2)]
    acc = torch.zeros(M, w.rows, dtype=torch.float32)
    for s in range(cdiv(K, 64)):
        part = torch.zeros(M, w.rows, dtype=torch.float32)
        for k0 in range(64 * s, min(K, 64 * s + 64), 16):
            for ia, iw in pairs:
                sl = slice(k0, min(K, k0 + 16))
                part = _rz(part.double() + A[ia][:, sl] @ W[iw][:, sl].t())
        acc = acc + part
    return acc


def test_arithmetic_model_within_bound_and_speed_mode_outside():
    """The CPU model of the kernel (truncating k16 steps, RN fold) stays within gemm_ref's bound at a ragged K with
    both draws; the speed-mode model against the parity reference and bound fails on most elements."""
    ops = mtt_ops()
    g = torch.Generator().manual_seed(3)
    M, N, K = 24, 40, 200
    for scaled in (False, True):
        s = torch.exp2(torch.rand(M, 1, generator=g) * 40 - 20) if scaled else torch.ones(M, 1)
        xa = torch.randn(M, K, generator=g) * s
        xw = torch.randn(N, K, generator=g)
        a, w = ops.Split(M, K, "cpu"), ops.Split(N, K, "cpu")
        for sp, x in ((a, xa), (w, xw)):
            hi = x.bfloat16()
            sp.buf[0, :, :K], sp.buf[1, :, :K] = hi, (x - hi.float()).bfloat16()
        spec = dict(a=a, w=w, ns=2, M=M, N=N, K=K, conv=None, arow=torch.arange(M))
        y, E, _, _ = gemm_ref(spec)
        got = _model_kernel(a, w, 2).double()
        r = float(((got - y).abs() / E).max())
        assert r <= 1.0, r
        assert r > 1e-3, f"the bound is far looser than the modelled error ({r})"
        spd = _model_kernel(a, w, 1).double()
        assert float(((spd - y).abs() > E).double().mean()) > 0.9


def test_keys_tell_apart_what_selects_a_path():
    """Calls differing only in residual kind, regroup or an offset get distinct keys; identical calls one key."""
    ops = mtt_ops()
    a, w = ops.Split(300, 72, "cpu"), ops.Split(136, 72, "cpu")
    out = torch.zeros(400, 136)
    res = torch.zeros(400, 136)
    base = dict(out_f32=out)
    variants = [base, dict(base, residual=res), dict(base, residual=out), dict(base, residual=res[:100], res_row_mod=100),
                dict(base, regroup=(100, 104, 4)), dict(base, regroup=(100, 104, 4, 1)), dict(base, a_row_offset=8),
                dict(base, w_col_offset=8, K=64), dict(base, out_col_offset=8),
                dict(base, out_split=ops.Split(400, 136, "cpu")), dict(out_split=ops.Split(400, 136, "cpu"))]
    keys = [call_key("gemm", dict(a=a, w=w, kw=kw, sk_ws=None)) for kw in variants]
    assert len(set(keys)) == len(keys), "two different calls share a key"
    assert call_key("gemm", dict(a=a, w=w, kw=dict(base), sk_ws=None)) == keys[0]
    sk = call_key("gemm", dict(a=a, w=w, kw=dict(base), sk_ws=torch.zeros(4)))
    assert sk != keys[0]
    grouped = call_key("gemm_grouped", dict(calls=[(a, w, dict(base)), (a, w, dict(base))]))
    assert grouped != keys[0] and launches_of(grouped) == [(0, 600, 136, 72)]
    strict = [call_key("gemm", dict(a=a, w=w, kw=dict(base, regroup=(100, 104, 4, s)), sk_ws=None)) for s in (1, 2)]
    assert without_planes(strict[0]) != without_planes(strict[1]), "a regroup row stride must survive the stripping"
    assert without_planes(keys[0]) == without_planes(call_key("gemm", dict(a=ops.Split(300, 72, "cpu", 1), w=w,
                                                                            kw=dict(base), sk_ws=None)))
