"""-m gpu: the training-step kernels (csrc/train_ops.cu) and the loss kernels (csrc/losses.cu) at the geometries the
training runs of plan_calls.RUNS really run -- tp_cfg4 (ViT-L, PASCAL, 5 tasks) and tp_cfg2 (ViT-B, NYUD, 4 tasks) at
batch 4, and at the reference's training batch 2 tp_cfg4 and its own tp_pascal_vitB (ViT-B, 4 x 4 channel windows with
ctr, f = 1024) and tp_nyud_vitL (ViT-L, 4 x 4 channel windows, f = 768) -- against float64 references written from
each operation's definition: torch autograd in float64 for the adjoints, F.batch_norm / clip_grad_norm_ /
torch.optim.Adam in float64, oracle/loss_ref.py in float64. Then the whole tp_cfg2_d4 reverse pass against autograd of
the train-mode restatement.

Error model: tests/f64_checks.py. The BatchNorm statistics accumulate in double (U64 in place of u). Every assert below
states which bound it uses."""
import math

import pytest
import torch
import torch.nn.functional as F

from f64_checks import (LAM, SPLIT, SPLIT_ABS, U, U64, bce_rel, bce_term_bound, check, gen, ops, randn,  # noqa: F401
                        split_planes, sum_tol)
from oracle import configs, loss_ref
from model_checks import reverse_pass_errors
from plan_calls import TPGeom, run_id, runs

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]

TRAIN = runs(("train",))                                   # (config, batch)
CONFIGS = list(dict.fromkeys(name for name, _ in TRAIN))   # the loss tests run each config's tasks at batch 2


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def colreduce_depth(rows, cols):
    """Longest addition chain of csrc/train_ops.cu colreduce_kernel as launch_colreduce sizes it: serial sum per row lane,
    8 row lanes through shared memory, one atomicAdd per row block."""
    cb = (cols + 31) // 32
    rb = max(1, min((rows + 63) // 64, _sms() * 8 // cb + 1))
    return math.ceil(rows / (8 * rb)) + 8 + rb


@pytest.fixture(scope="module", params=[pytest.param(run, id=run_id(*run)) for run in TRAIN])
def geom(request, cuda_dev):
    import mtt_b200  # noqa: F401
    return TPGeom(*request.param)


def split_of(ops, x):
    """x fp32 [rows, cols] -> device Split (hi + lo planes) and the fp32 value the planes hold."""
    s = ops.split_f32(x.contiguous(), 2)
    return s, s.float()


# ---- BatchNorm ---------------------------------------------------------------------------------------------------------
def _bn_case(ops, rows, cols, r, seed, momentum=0.1):
    """x with per-channel std s_c in [0.5, 2] and mean r * s_c, three constant channels; the kernel chain
    bn_stats -> bn_finalize (float64 sums, as TrainStep keeps them) -> bn_act, bn_bwd_reduce -> bn_bwd_apply against
    F.batch_norm(training) + GELU + autograd in float64."""
    g = gen(seed)
    std = torch.rand(cols, generator=g, device="cuda") * 1.5 + 0.5
    sign = torch.where(torch.rand(cols, generator=g, device="cuda") < 0.5, -1.0, 1.0)
    x = randn(g, rows, cols) * std + sign * r * std
    const = [0, cols // 2, cols - 1]
    x[:, const] = torch.tensor([0.0, 1.5, -r - 0.25], device="cuda")     # var = 0: only eps keeps rstd finite
    dy = randn(g, rows, cols)
    gam, bet = torch.rand(cols, generator=g, device="cuda") + 0.5, randn(g, cols) * 0.5
    rm0, rv0 = randn(g, cols), torch.rand(cols, generator=g, device="cuda") + 0.5
    eps = 1e-5

    sums, mr = torch.empty(2 * cols, dtype=torch.float64, device="cuda"), torch.empty(2 * cols, device="cuda")
    rm, rv = rm0.clone(), rv0.clone()
    ops.bn_stats(x, sums)
    ops.bn_finalize(sums, rows, eps, momentum, mr, rm, rv)
    y = torch.empty(rows, cols, device="cuda")
    ys = ops.Split(rows, cols, "cuda", 2, zero=True)
    ops.bn_act(x, mr, gam, bet, 1, out_f32=y, out_split=ys)
    s2 = torch.empty(2 * cols, device="cuda")
    ops.bn_bwd_reduce(x, dy, mr, gam, bet, 1, s2)
    dx = torch.empty(rows, cols, device="cuda")
    ops.bn_bwd_apply(x, dy, mr, gam, bet, 1, s2, rows, dx)

    # float64 reference: nn.BatchNorm2d in training mode (F.batch_norm) + exact-erf GELU, autograd for the adjoints
    xd = x.double().requires_grad_(True)
    gd, bd = gam.double().requires_grad_(True), bet.double().requires_grad_(True)
    rmd, rvd = rm0.double(), rv0.double()
    z = F.batch_norm(xd, rmd, rvd, gd, bd, training=True, momentum=momentum, eps=eps)
    yd = F.gelu(z)
    yd.backward(dy.double())
    mean, var = xd.detach().mean(0), xd.detach().var(0, unbiased=False)
    rstd = 1.0 / torch.sqrt(var + eps)
    xh = (xd.detach() - mean) * rstd
    ax = xd.detach().abs()

    D = colreduce_depth(rows, cols)
    # sum x and sum x^2 accumulate in double (a float's square is exact there) along the reduction tree of depth D; the
    # variance sum x^2 / n - mean^2 is formed in double, so the cancellation costs ~u64 (mean^2 + E x^2); mean and rstd
    # are then rounded to fp32 (u)
    ex2 = (xd.detach() ** 2).mean(0)
    e_m64 = LAM * math.sqrt(D) * U64 * ax.sum(0) / rows + U64 * mean.abs()
    e_var = LAM * math.sqrt(D) * U64 * ex2 + 2 * mean.abs() * e_m64 + 4 * U64 * (ex2 + mean ** 2)
    e_mean = e_m64 + U * mean.abs()
    check(mr[:cols], mean, e_mean, "batch mean")
    e_rstd = rstd * (0.5 * e_var / (var + eps) + 2 * U64) + U * rstd
    check(mr[cols:], rstd, e_rstd, "batch rstd")
    # running statistics: running_var takes the UNBIASED variance (n / (n - 1))
    # the fp32 update (1 - m) r + m s: m and 1 - m as floats (< u/2 each), two products and a sum
    unb = var * rows / (rows - 1)
    check(rm, rmd, momentum * e_mean + 4 * U * (rmd.abs() + momentum * mean.abs()), "running_mean")
    check(rv, rvd, momentum * e_var * rows / (rows - 1) + 4 * U * (rvd.abs() + momentum * unb), "running_var")
    # y = gelu(gamma xhat + beta): xhat carries e_mean * rstd + |xhat| e_rstd / rstd; GELU's slope is below 1.13 and the
    # fp32 erf-GELU adds a few u of |z|
    e_xh = e_mean * rstd + xh.abs() * (e_rstd / rstd + 2 * U)
    zz = z.detach()
    e_y = 1.13 * (gd.detach() * e_xh + 2 * U * zz.abs()) + 8 * U * (zz.abs() + 1e-30)
    check(y, yd.detach(), e_y, "bn_act fp32")
    check(ys.float(), yd.detach(), e_y + SPLIT * yd.detach().abs() + SPLIT_ABS, "bn_act split planes")
    # parameter gradients (dbeta = sum dz, dgamma = sum dz xhat): reductions of depth D; dz = dy gelu'(z) carries the
    # y-side error through gelu'' (< 0.8)
    zq = zz.clone().requires_grad_(True)
    F.gelu(zq).backward(dy.double())
    dzd = zq.grad
    e_dz = dy.double().abs() * (0.8 * gd.detach() * e_xh + 4 * U)
    check(s2[:cols], bd.grad, sum_tol(D, dzd.abs().sum(0)) + e_dz.sum(0), "dbeta")
    check(s2[cols:], gd.grad, sum_tol(D, (dzd * xh).abs().sum(0)) + (e_dz * xh.abs() + dzd.abs() * e_xh).sum(0), "dgamma")
    # dx = gamma rstd (dz - mean dz - xhat mean(dz xhat)): the two means carry the reductions' bounds / rows
    e_m1 = (sum_tol(D, dzd.abs().sum(0)) + e_dz.sum(0)) / rows
    e_m2 = (sum_tol(D, (dzd * xh).abs().sum(0)) + (e_dz * xh.abs() + dzd.abs() * e_xh).sum(0)) / rows
    m2 = (dzd * xh).mean(0)
    inner = dzd - dzd.mean(0) - xh * m2
    e_dx = gd.detach() * (rstd * (e_dz + e_m1 + xh.abs() * e_m2 + e_xh * m2.abs() + 4 * U * (dzd.abs() + xh.abs() * m2.abs()))
                          + e_rstd * inner.abs())
    check(dx, xd.grad, e_dx, "bn dx")
    return unb


@pytest.mark.parametrize("layer", ["mt_proj.1", "fea_fuse.2"])
@pytest.mark.parametrize("r", [0.0, 3.0, 30.0])
def test_batchnorm_train_f64(ops, geom, layer, r):
    """Train-mode BatchNorm2d + GELU at the rows x channels TrainStep._bn_fwd sees: the heads' mt_proj.1 over
    B * 4gh * 4gw rows and the decoder's fea_fuse.<level>.<task>.2 over B * gh * gw rows, f channels; channel mean /
    std ratio r (a conv bias Adam has moved makes r large: a one-pass variance loses ~1e-6 r^2 of it)."""
    rows = geom.M4 if layer == "mt_proj.1" else geom.Mp
    _bn_case(ops, rows, geom.f, r, seed=int(r) * 7 + (1 if layer == "mt_proj.1" else 2))


def test_batchnorm_running_var_is_unbiased(ops, geom):
    """momentum 1: running_var IS the unbiased batch variance, so n / (n - 1) (2.4e-4 relative at B * gh * gw rows) is
    far above the reduction bound and a biased running_var fails."""
    rows, cols = geom.Mp, geom.f
    g = gen(40)
    x = randn(g, rows, cols) * 2 + 1
    sums, mr = torch.empty(2 * cols, dtype=torch.float64, device="cuda"), torch.empty(2 * cols, device="cuda")
    rm, rv = torch.zeros(cols, device="cuda"), torch.ones(cols, device="cuda")
    ops.bn_stats(x, sums)
    ops.bn_finalize(sums, rows, 1e-5, 1.0, mr, rm, rv)
    want = x.double().var(0, unbiased=True)
    D = colreduce_depth(rows, cols)
    # double sums and variance (as in the BatchNorm case above), then fp32 rounding of unb and of the update
    ex2 = (x.double() ** 2).mean(0)
    e = (LAM * math.sqrt(D) * U64 + 8 * U64) * (ex2 + x.double().mean(0) ** 2) * rows / (rows - 1) + 4 * U * want
    check(rv, want, e, "running_var")
    assert (1.0 / (rows - 1)) * want.min() > 20 * e.max()          # the test can tell n from n - 1


# ---- LayerNorm backward ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("accumulate", [False, True])
def test_layernorm_bwd_f64(ops, geom, accumulate):
    """dx (+)= LN'(x) dy, dgamma / dbeta accumulated, at B * N rows x C (nn.LayerNorm eps 1e-6); a quarter of the rows
    have mean offset 50 x their std."""
    rows, C = geom.B * geom.N, geom.C
    g = gen(3)
    x = randn(g, rows, C) * 0.5
    off = torch.zeros(rows, 1, device="cuda")
    off[::4] = 25.0
    x = x + off
    dy, gam = randn(g, rows, C), torch.rand(C, generator=g, device="cuda") + 0.5
    dx0, dg0, db0 = randn(g, rows, C), randn(g, C), randn(g, C)
    dx, dgm, dbt = dx0.clone(), dg0.clone(), db0.clone()
    ops.layernorm_bwd(x, dy, gam, 1e-6, dx, dgm, dbt, accumulate_dx=accumulate)

    xd, gd = x.double().requires_grad_(True), gam.double().requires_grad_(True)
    bd = torch.zeros(C, dtype=torch.float64, device="cuda", requires_grad=True)
    F.layer_norm(xd, (C,), gd, bd, 1e-6).backward(dy.double())
    mean, var = x.double().mean(1, keepdim=True), x.double().var(1, unbiased=False, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + 1e-6)
    xh = (x.double() - mean) * rstd
    Dr = C // 32 + 5                                         # per-lane serial sum + warp shuffle tree
    e_mean = sum_tol(Dr, x.double().abs().sum(1, keepdim=True)) / C + U * mean.abs()
    e_var = sum_tol(Dr, ((x.double() - mean) ** 2).sum(1, keepdim=True)) / C + 3 * U * var + e_mean ** 2
    e_rr = 0.5 * e_var / (var + 1e-6) + 3 * U                  # relative error of rstd
    e_xh = e_mean * rstd + xh.abs() * (e_rr + 2 * U)
    gg = dy.double() * gd.detach()
    m1, m2 = gg.mean(1, keepdim=True), (gg * xh).mean(1, keepdim=True)
    e_m1 = sum_tol(Dr, gg.abs().sum(1, keepdim=True)) / C
    e_m2 = (sum_tol(Dr, (gg * xh).abs().sum(1, keepdim=True)) + (gg.abs() * e_xh).sum(1, keepdim=True)) / C
    inner = gg - m1 - xh * m2
    e_dx = rstd * (e_m1 + xh.abs() * e_m2 + e_xh * m2.abs() + 4 * U * (gg.abs() + m1.abs() + (xh * m2).abs())) + e_rr * rstd * inner.abs()
    want = xd.grad + (dx0.double() if accumulate else 0)
    check(dx, want, e_dx + (U * want.abs() if accumulate else 0), "layernorm dx")
    D = colreduce_depth(rows, C)
    check(dbt, db0.double() + bd.grad, sum_tol(D, dy.double().abs().sum(0)) + U * (db0.double().abs() + bd.grad.abs()), "dbeta")
    check(dgm, dg0.double() + gd.grad,
          sum_tol(D, (dy.double() * xh).abs().sum(0)) + (dy.double().abs() * e_xh).sum(0) + U * (dg0.double().abs() + gd.grad.abs()),
          "dgamma")


# ---- attention backward: delta + softmax ------------------------------------------------------------------------------------
def test_attn_delta_f64(ops, geom):
    """delta[(b*H + h)*N + i] = dO_i . O_i per head, O given as the forward's split planes, at the real (B, N, H)."""
    B, N, H, dh = geom.B, geom.N, geom.H, geom.dh
    g = gen(5)
    dO = randn(g, B * N, H * dh)
    o_s, o = split_of(ops, randn(g, B * N, H * dh))
    delta = torch.empty(B * H * N, device="cuda")
    ops.attn_delta(dO, o_s, delta, B=B, N=N, H=H, head_dim=dh)
    prod = (dO.double() * o.double()).view(B, N, H, dh)
    want = prod.sum(-1).permute(0, 2, 1).reshape(-1)
    check(delta, want, sum_tol(dh // 32 + 5, prod.abs().sum(-1).permute(0, 2, 1).reshape(-1)), "attn delta")


def test_attn_softmax_bwd_f64(ops, geom):
    """dS = scale P (dP - delta) + d_raw on the first T (prompt) rows, P = softmax(scale S) recomputed, P^T and dS^T, at
    (B*H, N) with N = T + gh*gw (ragged last 64-query tile) and scores like a trained model's (|scale S| up to ~30);
    reference: float64 autograd of softmax."""
    B, N, H, T = geom.B, geom.N, geom.H, geom.T
    BH, scale = B * H, 64 ** -0.5
    ld = (N + 7) // 8 * 8                           # TrainStep._attn_bwd's row stride
    g = gen(6)
    S = torch.zeros(BH * N, ld, device="cuda")
    S[:, :N] = randn(g, BH * N, N) * (8.0 / scale)
    S[:, :N:97] += 22.0 / scale                    # a few strongly preferred keys per row
    dP = torch.zeros(BH * N, ld, device="cuda")
    dP[:, :N] = randn(g, BH * N, N)
    d_raw = randn(g, BH, T, N)
    s3 = S[:, :N].double().view(BH, N, N).requires_grad_(True)
    Pd = torch.softmax(scale * s3, -1)
    delta_d = (Pd.detach() * dP[:, :N].double().view(BH, N, N)).sum(-1)
    delta = delta_d.float().reshape(-1)
    ds, pt, dst = (ops.Split(BH * N, ld, "cuda", 2, zero=True) for _ in range(3))
    S0, dP0 = S.clone(), dP.clone()
    ops.attn_softmax_bwd(S, dP, delta, BH=BH, N=N, scale=scale, d_raw=d_raw, T=T, ds=ds, pt=pt, dst=dst)
    assert torch.equal(S, S0) and torch.equal(dP, dP0)                 # inputs are read only
    Pd.backward(dP[:, :N].double().view(BH, N, N))
    want = s3.grad.clone()
    want[:, :T] += d_raw.double()
    P = Pd.detach()
    # P: __expf(x) is within 2 + 1.173 |x| ulp (CUDA programming guide, intrinsic functions) at x = scale s - m; the
    # row sum (N/32 + 5 deep, with the online rescalings: one more __expf of |m_lane - m| <= max |x| per lane) and the
    # reciprocal add LAM sqrt(N/32 + 5) u + (2 + 1.2 max|x|) 2u + 2u relative
    arg = (scale * s3.detach() - (scale * s3.detach()).amax(-1, keepdim=True)).abs()
    e_sum = LAM * math.sqrt(N // 32 + 5) * U + (2 + 1.2 * arg.amax(-1, keepdim=True)) * 2 * U + 2 * U
    # (plus 2^-126 absolute: probabilities below fp32's normal range are subnormal or flushed to zero)
    e_P = P * ((2 + 1.2 * arg) * 2 * U + e_sum) + 2.0 ** -126
    check(pt.float()[:, :N].view(BH, N, N).transpose(1, 2), P, e_P + SPLIT * P + SPLIT_ABS, "P^T")
    dPd = dP[:, :N].double().view(BH, N, N)
    e_ds = scale * (e_P * (dPd - delta_d[..., None]).abs() + P * U * delta_d.abs()[..., None]) + 4 * U * want.abs()
    e_ds = e_ds + SPLIT * want.abs() + SPLIT_ABS
    check(ds.float()[:, :N].view(BH, N, N), want, e_ds, "dS")
    check(dst.float()[:, :N].view(BH, N, N).transpose(1, 2), want, e_ds, "dS^T")
    assert d_raw.abs().mean() > 1e3 * e_ds[:, :T].mean()               # a missing d_raw term is far outside the bound


# ---- gating adjoints ----------------------------------------------------------------------------------------------------
def _windows(geom):
    return geom.gh // geom.nh, geom.gw // geom.nw


def test_gate_bwd_f64(ops, geom):
    """Adjoint of Ys = X (1 + g_s), Yc = X (1 + g_c) for one task (taskprompter.py:217-250): g_s = the task prompt's
    spatial logit of the pixel for the channel's head, g_c = the task's channel logit of the pixel's nh x nw window
    (1 x 1 windows on 32 x 32 for tp_cfg4, 4 x 4 windows on 28 x 36 for tp_cfg2). dX, d prompt_logits, d chan_logits
    accumulate."""
    B, T, N, H, C, P = geom.B, geom.T, geom.N, geom.H, geom.C, geom.P
    gh, gw, nh, nw = geom.gh, geom.gw, geom.nh, geom.nw
    task = T - 1
    g = gen(8)
    x = randn(g, B * N, C)
    plog, clog = randn(g, B, H, T, N), randn(g, B, T, C, nh, nw)
    dys, dyc = randn(g, B * P, C), randn(g, B * P, C)
    dx0, dl0, dc0 = randn(g, B * N, C), randn(g, B, H, T, N), randn(g, B, T, C, nh, nw)
    dx, dl, dc = dx0.clone(), dl0.clone(), dc0.clone()
    ops.gate_bwd(x, N, T, plog, clog, task, dys, dyc, dx, dl, dc, B=B, T=T, N=N, H=H, Cdim=C, gh=gh, gw=gw, nh=nh, nw=nw)

    X = x.double().view(B, N, C)[:, T:].clone().requires_grad_(True)                 # [B, P, C]
    pl, cl = plog.double().requires_grad_(True), clog.double().requires_grad_(True)
    gs = pl[:, :, task, T:].permute(0, 2, 1).repeat_interleave(C // H, dim=2)        # [B, P, C]
    wh, ww = _windows(geom)
    gc = cl[:, task].reshape(B, C, nh, 1, nw, 1).expand(B, C, nh, wh, nw, ww).reshape(B, C, P).permute(0, 2, 1)
    Ys, Yc = X * (1 + gs), X * (1 + gc)
    dYs, dYc = dys.double().view(B, P, C), dyc.double().view(B, P, C)
    ((Ys * dYs).sum() + (Yc * dYc).sum()).backward()
    wdx = dx0.double().view(B, N, C).clone()
    wdx[:, T:] += X.grad
    e_dx = 4 * U * ((dYs * (1 + gs.detach())).abs() + (dYc * (1 + gc.detach())).abs() + dx0.double().view(B, N, C)[:, T:].abs())
    bound = torch.zeros_like(wdx)
    bound[:, T:] = e_dx
    check(dx.view(B, N, C), wdx, bound, "gate dX")
    assert torch.equal(dx.view(B, N, C)[:, :T], dx0.view(B, N, C)[:, :T])              # prompt rows untouched
    # d prompt_logits at column T + pixel: one warp per pixel sums the head's dh channels
    prod = (dYs * X.detach()).view(B, P, H, -1)
    bl = torch.zeros_like(dl0, dtype=torch.float64)
    bl[:, :, task, T:] = sum_tol(geom.dh // 32 + 6, prod.abs().sum(-1)).permute(0, 2, 1)
    check(dl, dl0.double() + pl.grad, bl + U * dl0.double().abs(), "gate d prompt_logits")
    # d chan_logits: column reduction over the pixels of a window, 8 row lanes + shared memory
    pc = (dYc * X.detach()).abs().view(B, nh, wh, nw, ww, C).sum((2, 4)).permute(0, 3, 1, 2)   # [B, C, nh, nw]
    bc = torch.zeros_like(dc0, dtype=torch.float64)
    bc[:, task] = sum_tol(math.ceil(wh * ww / 8) + 9, pc)
    check(dc, dc0.double() + cl.grad, bc + U * dc0.double().abs(), "gate d chan_logits")


def test_chan_logits_bwd_f64(ops, geom):
    """Adjoint of Rc[b,t,c,win] = sum_{pix in win} cp[b,t,pix] xn[b,T+pix,c] (mtt_chan_logits): dcp (=), dxn (+=) on the
    patch rows, xn as the forward's split planes."""
    B, T, N, C, P = geom.B, geom.T, geom.N, geom.C, geom.P
    gh, gw, nh, nw = geom.gh, geom.gw, geom.nh, geom.nw
    wh, ww = _windows(geom)
    g = gen(9)
    xn_s, xnv = split_of(ops, randn(g, B * N, C))
    cp, d_rc = randn(g, B * T, P), randn(g, B, T, C, nh, nw)
    dxn0 = randn(g, B * N, C)
    dcp, dxn = torch.empty(B * T, P, device="cuda"), dxn0.clone()
    ops.chan_logits_bwd(d_rc, cp, xn_s, dcp, dxn, B=B, N=N, T=T, Cdim=C, gh=gh, gw=gw, nh=nh, nw=nw)
    X = xnv.double().view(B, N, C)[:, T:].clone().requires_grad_(True)
    cpd = cp.double().view(B, T, P).clone().requires_grad_(True)
    Rc = torch.einsum("btihjw,bihjwc->btcij", cpd.view(B, T, nh, wh, nw, ww), X.view(B, nh, wh, nw, ww, C))
    (Rc * d_rc.double()).sum().backward()
    drp = d_rc.double().view(B, T, C, nh, 1, nw, 1).expand(B, T, C, nh, wh, nw, ww).reshape(B, T, C, P)   # dRc per pixel
    bcp = sum_tol(C // 32 + 5, torch.einsum("btcp,bpc->btp", drp.abs(), X.detach().abs()))
    check(dcp.view(B, T, P), cpd.grad, bcp, "dcp")
    want = dxn0.double().view(B, N, C).clone()
    want[:, T:] += X.grad
    bx = torch.zeros_like(want)
    bx[:, T:] = (T + 1) * U * (torch.einsum("btcp,btp->bpc", drp.abs(), cpd.detach().abs()) + dxn0.double().view(B, N, C)[:, T:].abs())
    check(dxn.view(B, N, C), want, bx, "dxn")


def test_ctr_bwd_f64(ops, geom):
    """Cross-task reweighting backward (taskprompter.py:478-482): w[b,t,j] = W2_t . gelu(W0_t a + b0_t) + b2_t with
    a[h] = prompt_logits[b,h,t,j], new[t] = sum_j w[b,t,j] F[j], against float64 autograd of that forward."""
    if not geom.use_ctr:
        pytest.skip(f"{geom.name} has no cross-task reweighting")
    B, T, N, H, P, f = geom.B, geom.T, geom.N, geom.H, geom.P, geom.f
    M, ld = B * P, (f + 7) // 8 * 8
    g = gen(10)
    dnew, Fm = torch.zeros(T, M, ld, device="cuda"), torch.zeros(T, M, ld, device="cuda")
    dnew[..., :f], Fm[..., :f] = randn(g, T, M, f), randn(g, T, M, f)
    plog = randn(g, B, H, T, N)
    w0, b0, w2 = randn(g, T, H, H) * 0.3, randn(g, T, H) * 0.3, randn(g, T, H) * 0.3
    outs0 = [randn(g, B, H, T, N), randn(g, T, H, H), randn(g, T, H), randn(g, T, H), randn(g, T)]
    outs = [o.clone() for o in outs0]
    ops.ctr_bwd(dnew, Fm, plog, w0, b0, w2, *outs, T=T, M=M, Cdim=f, ld=ld, rows_per_batch=P, B=B, H=H, N=N)

    pl = plog.double().requires_grad_(True)
    prm = [p.double().requires_grad_(True) for p in (w0, b0, w2)]
    b2 = torch.zeros(T, dtype=torch.float64, device="cuda", requires_grad=True)
    a = pl[:, :, :, :T]
    w = torch.stack([torch.einsum("o,boj->bj", prm[2][t], F.gelu(torch.einsum("oh,bhj->boj", prm[0][t], a[:, :, t, :])
                                                                            + prm[1][t][None, :, None])) + b2[t]
                     for t in range(T)], 1)                                         # [B, T, T]
    Fd, dn = Fm.double()[..., :f].view(T, B, P, f), dnew.double()[..., :f].view(T, B, P, f)
    new = torch.einsum("btj,jbpc->tbpc", w, Fd)
    (new * dn).sum().backward()
    # dw[b,t,j] = sum over the image's P x f products: reduction depth of ctr_dw_kernel (serial per thread, warp, block,
    # one atomic per row chunk); its error reaches the outputs through |d out / d w|, taken as the float64 gradient
    # of sum |dw-error| * |.| below by scaling
    chunks = min((P + 63) // 64, 32)
    D = math.ceil(P / (chunks * 8)) * math.ceil(f / 32) + 5 + 8 + chunks
    e_dw = sum_tol(D, torch.einsum("tbpc,jbpc->btj", dn.abs(), Fd.abs()))           # [B, T, T]
    dw = torch.einsum("tbpc,jbpc->btj", dn, Fd)
    rel = (e_dw / dw.abs().clamp_min(1e-300)).clamp_max(1.0)
    # every output is a sum over (b, t, j) of dw times a smooth factor: its error is at most the same sum with |dw| rel
    # plus the fp32 evaluation of the factors (H-term dot products, GELU: 8H u relative)
    grads = [pl.grad, prm[0].grad, prm[1].grad, prm[2].grad, b2.grad]
    with torch.enable_grad():
        pl2 = plog.double().requires_grad_(True)
        q = [p.double().requires_grad_(True) for p in (w0, b0, w2)]
        b22 = torch.zeros(T, dtype=torch.float64, device="cuda", requires_grad=True)
        a2 = pl2[:, :, :, :T]
        w2_ = torch.stack([torch.einsum("o,boj->bj", q[2][t], F.gelu(torch.einsum("oh,bhj->boj", q[0][t], a2[:, :, t, :])
                                                                                + q[1][t][None, :, None])) + b22[t]
                           for t in range(T)], 1)
        (w2_ * (dw.abs() * (rel + 8 * H * U))).sum().backward()
    names = ["d prompt_logits", "dw0", "db0", "dw2", "db2"]
    for got, o0, ref, sens, nm in zip(outs, outs0, grads, [pl2.grad, q[0].grad, q[1].grad, q[2].grad, b22.grad], names):
        # the sensitivity gradient has signed factors: bound by its magnitude plus a normwise share of the same size
        bound = sens.abs() + (sens.norm() / math.sqrt(sens.numel())) + U * (o0.double().abs() + ref.abs())
        check(got, o0.double() + ref, bound, f"ctr {nm}")


# ---- bilinear adjoint, column sums, data movement ------------------------------------------------------------------------
def _bilinear_pairs(geom):
    """(h, w) -> (H2, W2) of the step's two bilinear resizes: token grid -> 4x (ConvHead input) and 4x -> image."""
    H_img, W_img = geom.cfg["img_size"]
    return [("tokens->x4", geom.gh, geom.gw, geom.h4, geom.w4, geom.f, False),
            ("x4->image", geom.h4, geom.w4, H_img, W_img, max(geom.cfg["num_output"].values()), True)]


@pytest.mark.parametrize("which", [0, 1])
def test_bilinear_bwd_f64(ops, geom, which):
    """Adjoint of the align_corners=False bilinear resize at the decoder's (h, w) -> (H2, W2): NHWC for the up-sampling
    in front of the heads, NCHW for the resize of the predictions to the label size; accumulate on and off."""
    name, h, w, H2, W2, C, nchw = _bilinear_pairs(geom)[which]
    B = geom.B
    g = gen(11 + which)
    dy = randn(g, B, C, H2, W2) if nchw else randn(g, B * H2 * W2, C)
    base = randn(g, B * h * w, C)
    xin = torch.zeros(B, C, h, w, dtype=torch.float64, device="cuda", requires_grad=True)
    yd = F.interpolate(xin, size=(H2, W2), mode="bilinear", align_corners=False)
    dyd = dy.double() if nchw else dy.double().view(B, H2, W2, C).permute(0, 3, 1, 2)
    yd.backward(dyd)
    want = xin.grad.permute(0, 2, 3, 1).reshape(B * h * w, C)
    ones = torch.zeros_like(xin, requires_grad=True)
    F.interpolate(ones, size=(H2, W2), mode="bilinear", align_corners=False).backward(dyd.abs())
    absum = ones.grad.permute(0, 2, 3, 1).reshape(B * h * w, C)
    # every input pixel receives at most 4 * ceil(H2 / h + 1) * ceil(W2 / w + 1) atomic adds; weights carry ~4u
    D = 4 * (math.ceil(H2 / h) + 1) * (math.ceil(W2 / w) + 1) + 1
    for acc in (False, True):
        dx = base.clone()
        ops.bilinear_bwd(dy, nchw=nchw, B=B, h=h, w=w, Cdim=C, H2=H2, W2=W2, dx=dx, accumulate=acc)
        ref = want + (base.double() if acc else 0)
        check(dx, ref, sum_tol(D, absum + (base.double().abs() if acc else 0)) + 6 * U * absum, f"bilinear_bwd {name} acc={acc}")


def test_colsum_step_mappings_f64(ops, geom):
    """The bias / pos_embed / task-prompt gradient column sums with the row mappings the step uses: plain rows, the per-task
    rows of a stacked [T*M, N] dY (in_group = src_group = M, src_offset = t*M), the patch rows of the joint stream
    (in_group = P, src_group = N, src_offset = T), and the [B, N*C] view summed over the batch (pos_embed, task_prompts)."""
    B, T, N, C, P, f, Mp = geom.B, geom.T, geom.N, geom.C, geom.P, geom.f, geom.Mp
    g = gen(13)
    dX = randn(g, B * N, C)
    stacked = randn(g, T * Mp, f)
    cases = [("plain", dX, dict(), dX.double()),
             ("task t of stacked", stacked, dict(rows=Mp, in_group=Mp, src_group=Mp, src_offset=(T - 1) * Mp),
              stacked.double()[(T - 1) * Mp:]),
             ("patch rows", dX, dict(rows=B * P, in_group=P, src_group=N, src_offset=T), dX.double().view(B, N, C)[:, T:].reshape(-1, C)),
             ("task_prompts over batch", dX.view(B, N * C)[:, :T * C], dict(), dX.double().view(B, N * C)[:, :T * C]),
             ("pos_embed over batch", dX.view(B, N * C)[:, T * C:], dict(), dX.double().view(B, N * C)[:, T * C:])]
    for name, x, kw, rows_ref in cases:
        out0 = randn(g, x.shape[1])
        out = out0.clone()
        ops.colsum(x, out, accumulate=True, **kw)
        D = colreduce_depth(rows_ref.shape[0], x.shape[1]) + 1
        check(out, out0.double() + rows_ref.sum(0), sum_tol(D, rows_ref.abs().sum(0) + out0.double().abs()), f"colsum {name}")


def test_im2col_and_transpose_bit_exact(ops, geom):
    """im2col3x3_t (conv weight-gradient operand of the decoder's 3x3 convs and the heads' mt_proj.0), im2col_patch_t
    (patch embedding) and transpose_planes at the step's shapes: bit for bit against F.unfold + the split."""
    B, f = geom.B, geom.f
    g = gen(14)
    for (H, W) in ((geom.gh, geom.gw), (geom.h4, geom.w4)):
        x = randn(g, B * H * W, f)
        got = ops.im2col3x3_t(x, B=B, H=H, W=W, Cdim=f)
        cols = F.unfold(x.view(B, H, W, f).permute(0, 3, 1, 2), 3, padding=1).permute(1, 0, 2).reshape(f * 9, B * H * W)
        hi, lo = split_planes(cols)
        assert torch.equal(got.hi[:, :B * H * W], hi) and torch.equal(got.lo[:, :B * H * W], lo), f"im2col3x3_t {H}x{W}"
    img = randn(g, B, 3, *geom.cfg["img_size"])
    got = ops.im2col_patch_t(img, geom.cfg["patch"])
    cols = F.unfold(img, geom.cfg["patch"], stride=geom.cfg["patch"])
    cols = cols.permute(1, 0, 2).reshape(cols.shape[1], -1)
    hi, lo = split_planes(cols)
    assert torch.equal(got.hi[:, :cols.shape[1]], hi) and torch.equal(got.lo[:, :cols.shape[1]], lo), "im2col_patch_t"
    # the attention operands: per image [N, 3C] -> [3C, N] (TrainStep._attn_bwd), and [Mp, C] -> [C, Mp]
    N, C = geom.N, geom.C
    a_s, _ = split_of(ops, randn(g, B * N, 3 * C))
    t = ops.transpose_planes(a_s, B=B, R=N, Ccols=3 * C)
    want = a_s.buf[:, :, :3 * C].view(2, B, N, 3 * C).transpose(2, 3).reshape(2, B * 3 * C, N)
    assert torch.equal(t.buf[:, :, :N], want), "transpose_planes per image"
    t = ops.transpose_planes(a_s, B=B, R=N, Ccols=3 * C, side_by_side=True)
    want = a_s.buf[:, :, :3 * C].view(2, B, N, 3 * C).permute(0, 3, 1, 2).reshape(2, 3 * C, B * N)
    assert torch.equal(t.buf[:, :, :B * N], want), "transpose_planes side by side"


# ---- clip + Adam over the parameter arena ---------------------------------------------------------------------------------
def test_sumsq_and_adam_over_the_arena_f64(ops, cuda_dev):
    """mtt_sumsq + mtt_adam_step over a buffer the size of tp_cfg4's real gradient arena, two steps with clipping active,
    against clip_grad_norm_ + torch.optim.Adam in float64."""
    from mtt_b200 import taskprompter as TP
    from mtt_b200.train import TrainStep

    cfg = configs.taskprompter("tp_cfg4")
    with torch.device(cuda_dev):
        model = TP.build_from_config(cfg, nsplit=1, use_graph=False)
    n = TrainStep(model, nsplit=1).grads.flat.numel()
    del model
    torch.cuda.empty_cache()
    g = gen(15)
    p0, grads = randn(g, n) * 0.05, [randn(g, n) * 1e-2, randn(g, n) * 1e-2]
    lr, wd, max_norm, betas, eps = 2e-5, 1e-6, 10.0, (0.9, 0.999), 1e-8
    p, m, v, ss = p0.clone(), torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda"), torch.zeros((), device="cuda")
    q = torch.nn.Parameter(p0.double())
    opt = torch.optim.Adam([q], lr=lr, betas=betas, eps=eps, weight_decay=wd)
    blocks = min((n + 255) // 256, _sms() * 8)
    D = math.ceil(n / (blocks * 256)) + 5 + 8 + blocks        # serial per thread, warp, block, one atomic per block
    em = ev = 0.0
    for step, gr in enumerate(grads, 1):
        ops.sumsq(gr, ss)
        ops.adam_step(p, gr, m, v, lr=lr, betas=betas, eps=eps, weight_decay=wd, step=step, gnorm_sq=ss, max_norm=max_norm,
                      grad_scale=1.0)
        want_ss = (gr.double() ** 2).sum()
        e_ss = sum_tol(D, want_ss) + 2 * U * want_ss
        check(ss, want_ss, e_ss, f"sumsq step {step}")
        q.grad = gr.double().clone()
        total = torch.nn.utils.clip_grad_norm_([q], max_norm)
        assert total > 2 * max_norm                                # clipping is active
        clip = float(q.grad.norm() / gr.double().norm())
        opt.step()
        st = opt.state[q]
        # error propagation in float64 alongside the reference: gi = g clip + wd p carries the clip factor's error (half of
        # sumsq's relative bound) relative to |g clip| + wd |p| (the two can cancel); m and v accumulate it (v through
        # 2 |gi| e_gi) plus 2u of their own rounding per step
        e_clip = 0.5 * e_ss / want_ss + 4 * U
        pd = p.double() if step == 1 else q_prev
        e_gi = (e_clip + 3 * U) * (gr.double().abs() * clip + wd * pd.abs())
        gi = gr.double() * clip + wd * pd
        mr, vr = st["exp_avg"], st["exp_avg_sq"]
        em = betas[0] * em + (1 - betas[0]) * e_gi + 2 * U * mr.abs()
        ev = betas[1] * ev + (1 - betas[1]) * (2 * gi.abs() * e_gi + e_gi ** 2) + 2 * U * vr
        check(m, mr, em, f"adam m step {step}")
        check(v, vr, ev, f"adam v step {step}")
        # p -= lr / bc1 m / (sqrt(v) / sqrt(bc2) + eps): first order in em, ev (sqrt's error: min(ev / 2 sqrt(v), sqrt(ev))),
        # 6u relative of the step for the fp32 operations, and the rounding of p itself
        bc1, bc2 = 1 - betas[0] ** step, 1 - betas[1] ** step
        den = vr.sqrt() / math.sqrt(bc2) + eps
        e_den = torch.minimum(0.5 * ev / vr.sqrt().clamp_min(1e-300), ev.sqrt()) / math.sqrt(bc2) + 4 * U * den
        stp = lr / bc1 * mr / den
        e_step = lr / bc1 * (em / den + mr.abs() * e_den / den ** 2) + 6 * U * stp.abs()
        check(p, q.detach(), U * q.detach().abs() + e_step, f"adam p step {step}")
        q_prev = p.double()
        q.data.copy_(q_prev)                                       # continue from the same fp32 parameters


# ---- loss kernels ---------------------------------------------------------------------------------------------------------
def _labels(task, nout, B, H, W, g):
    """Labels as the datasets give them, with ignore regions; image 0 is fully ignored."""
    if task in ("semseg", "human_parts", "sal"):
        y = torch.randint(0, nout, (B, 1, H, W), generator=g, device="cuda").float()
        y[torch.rand(B, 1, H, W, generator=g, device="cuda") < 0.1] = 255.0
    elif task == "edge":
        y = (torch.rand(B, 1, H, W, generator=g, device="cuda") < 0.1).float()
        y[torch.rand(B, 1, H, W, generator=g, device="cuda") < 0.05] = 255.0
    elif task == "normals":
        y = F.normalize(torch.randn(B, 3, H, W, generator=g, device="cuda"), dim=1)
        y[:, :, :H // 8] = 255.0
    else:                                                           # depth, invalid area -1
        y = torch.rand(B, 1, H, W, generator=g, device="cuda") * 9 + 0.5
        y[torch.rand(B, 1, H, W, generator=g, device="cuda") < 0.1] = -1.0
    ign = -1.0 if task == "depth" else 255.0
    y[0] = ign
    return y


def _device_loss(task):
    from mtt_b200 import losses as ML
    p = dict(edge_w=0.95, ignore_index=255, ignore_invalid_area_depth=True)
    return ML.get_loss(p, task)


def _ref_loss(task, pred, label):
    return loss_ref.task_loss(task, pred, label, edge_w=0.95, ignore_invalid_area_depth=True)


def _run_loss(task, pred, label, gscale=1.0):
    """mtt_b200 loss value and d loss / d pred (fp32 device) and the float64 reference's."""
    x = pred.clone().requires_grad_(True)
    val = _device_loss(task)(x, label)
    (val * gscale).backward()
    xd = pred.double().requires_grad_(True)
    ref = _ref_loss(task, xd, label.double())
    if ref.requires_grad:
        (ref * gscale).backward()
    refg = xd.grad if xd.grad is not None else torch.zeros_like(xd)
    return val.detach(), x.grad, ref.detach(), refg


def _loss_bounds(task, pred, label, gscale):
    """Error bounds of the device loss value and of d loss / d pred. Per pixel the kernels evaluate in fp32 and sum the
    per-pixel losses in double.
    CE (C classes): lse = max + log sum exp over C terms carries (C + 4) u + u |lse|; softmax = expf(x - lse) then
    (|x| + 2 |lse| + C + 8) u relative; (softmax - onehot) * w * gs adds 4 u of |softmax - onehot|.
    BCE: softplus / sigmoid of x within (|x| + 8) u of the weighted terms. L1: sign() is exact, gs rounds (2u); with the
    normalisation n = x / r carries 4u and (g - n (n . g)) / r (C + 8) u of (1 + C) / r.
    The value's bound is the mean over valid pixels of the per-pixel bound times the term's magnitude."""
    x, y = pred.double(), label.double()
    C = x.shape[1]
    ign = -1.0 if task == "depth" else 255.0
    if task in ("semseg", "human_parts", "sal"):
        keep = (y != ign)
        nv = max(int(keep.sum()), 1)
        lse = torch.logsumexp(x, 1, keepdim=True)
        sm = torch.softmax(x, 1)
        tgt = y.clamp(0, C - 1).long()
        onehot = torch.zeros_like(x).scatter_(1, tgt, 1.0)
        w = torch.ones_like(y)
        if task == "sal":
            w_pos = float((1 - y)[keep].sum()) / nv
            w = torch.where(y == 1, w_pos, 1 - w_pos)
        gsw = gscale * w * keep / nv
        k = (x.abs().amax(1, keepdim=True) + 2 * lse.abs() + C + 8) * U
        e_grad = (k * sm + 4 * U * (sm - onehot).abs()) * gsw
        e_val = float(((k * (lse.abs() + x.abs().amax(1, keepdim=True))) * w * keep).sum()) / nv
    elif task == "edge":
        keep = (y != ign)
        nv = max(int(keep.sum()), 1)
        e_grad = bce_rel(x) * gscale * keep / nv
        e_val = float((bce_term_bound(x) * keep).sum()) / nv
    else:
        keep = (y != ign).all(1, keepdim=True)
        nv = max(int(keep.sum()), 1)
        if task == "normals":
            r = x.norm(dim=1, keepdim=True).clamp_min(1e-12)
            e_grad = (C + 8) * U * (1 + C) / r * gscale * keep / nv + 0 * x
            e_val = float(((C + 8) * U * (C + 2) * keep).sum()) / nv
        else:
            e_grad = 2 * U * gscale * keep / nv + 0 * x
            e_val = float((4 * U * ((x - y).abs() + x.abs()) * keep).sum()) / nv
    return e_val + 1e-300, e_grad


@pytest.mark.parametrize("name", CONFIGS)
def test_losses_at_the_training_sizes_f64(cuda_dev, name):
    """Every task loss of the config at its image size, batch 2, image 0 fully ignored: value and elementwise d loss / d
    prediction against oracle/loss_ref.py in float64. Normals: pixels whose normalised prediction is within the forward's
    bound of the label (sign() ambiguous) are left out of the elementwise check."""
    import mtt_b200  # noqa: F401

    cfg = configs.taskprompter(name)
    H, W = cfg["img_size"]
    g = torch.Generator(device="cuda").manual_seed(20)
    for task in cfg["tasks"]:
        nout = cfg["num_output"][task]
        pred = torch.randn(2, nout, H, W, generator=g, device="cuda") * 3
        label = _labels(task, nout, 2, H, W, g)
        if task == "depth":                                        # exact hits: sign(0) = 0
            hit = torch.rand(2, 1, H, W, generator=g, device="cuda") < 0.05
            pred[hit] = label[hit]
        val, grad, rv, rg = _run_loss(task, pred, label, gscale=0.7)
        e_val, e_grad = _loss_bounds(task, pred, label, 0.7)
        assert abs(float(val) - float(rv)) <= e_val, (name, task, float(val), float(rv), e_val)
        mask = torch.ones_like(rg, dtype=torch.bool)
        if task == "normals":
            n = F.normalize(pred.double(), dim=1)
            mask = ((n - label.double()).abs() > 64 * U).all(1, keepdim=True).expand_as(rg)
        assert grad[0].abs().max() == 0, (task, "fully ignored image got a gradient")
        check(grad[mask], rg[mask], e_grad[mask], f"{name} {task} d loss / d pred")
        if task == "depth":
            assert (grad[hit] == 0).all() and (rg[hit] == 0).all(), "sign(0) must be 0 at exact label hits"


def test_loss_edge_cases_f64(cuda_dev):
    """All-ignored batches, HED / balanced-CE without positives or negatives, exactly zero normals vectors.
    Deliberate deviation: the reference's BalancedBinaryCrossEntropyLoss returns NaN (the mean of an empty tensor) on an
    all-ignored batch; the device loss returns 0 with a zero gradient, like CrossEntropyLoss and L1Loss do there."""
    import mtt_b200  # noqa: F401
    from mtt_b200 import losses as ML

    g = torch.Generator(device="cuda").manual_seed(21)
    H, W = 64, 96
    rnd = lambda *s: torch.randn(*s, generator=g, device="cuda")
    # whole batch ignored
    for task, nout, ign in (("semseg", 21, 255.0), ("depth", 1, -1.0), ("normals", 3, 255.0)):
        pred = rnd(2, nout, H, W)
        val, grad, rv, rg = _run_loss(task, pred, torch.full((2, nout if task == "normals" else 1, H, W), ign, device="cuda"))
        assert float(val) == 0.0 and float(rv) == 0.0 and grad.abs().max() == 0 and rg.abs().max() == 0, task
    pred = rnd(2, 1, H, W)
    y = torch.full((2, 1, H, W), 255.0, device="cuda")
    val, grad, rv, _ = _run_loss("edge", pred, y)
    assert float(val) == 0.0 and grad.abs().max() == 0 and math.isnan(float(rv))       # the deliberate deviation
    x = pred.clone().requires_grad_(True)
    hed = ML.BalancedBinaryCrossEntropyLoss()(x, y)
    hed.backward()
    assert float(hed) == 0.0 and x.grad.abs().max() == 0
    # HED weighting without a positive pixel (reference: 0) and without a negative one (w = 0)
    for fill in (0.0, 1.0):
        y = torch.full((2, 1, H, W), fill, device="cuda")
        y[:, :, :4] = 255.0
        x = pred.clone().requires_grad_(True)
        v = ML.BalancedBinaryCrossEntropyLoss()(x, y)
        v.backward()
        xd = pred.double().requires_grad_(True)
        r = loss_ref.balanced_bce(xd, y.double())
        if r.requires_grad:
            r.backward()
        rg = xd.grad if xd.grad is not None else torch.zeros_like(xd)
        assert abs(float(v) - float(r)) <= 1e-6 * max(1.0, abs(float(r))), (fill, float(v), float(r))
        check(x.grad, rg, _loss_bounds("edge", pred, y, 1.0)[1], f"hed fill={fill}")
    # balanced CE (sal) with no positive / no negative pixel
    for fill in (0.0, 1.0):
        y = torch.full((2, 1, H, W), fill, device="cuda")
        y[:, :, :4] = 255.0
        pred2 = rnd(2, 2, H, W)
        val, grad, rv, rg = _run_loss("sal", pred2, y)
        assert abs(float(val) - float(rv)) <= 1e-6 * max(1.0, abs(float(rv))), (fill, float(val), float(rv))
        check(grad, rg, _loss_bounds("sal", pred2, y, 1.0)[1], f"sal fill={fill}")
    # normals with exactly-zero prediction vectors: F.normalize's eps path (x / 1e-12)
    pred3 = rnd(2, 3, H, W)
    pred3[:, :, ::5, ::7] = 0.0
    y = F.normalize(rnd(2, 3, H, W), dim=1)
    val, grad, rv, rg = _run_loss("normals", pred3, y)
    assert abs(float(val) - float(rv)) <= 1e-6 * float(rv)
    zero = (pred3 == 0).all(1, keepdim=True).expand_as(rg)
    e_grad = _loss_bounds("normals", pred3, y, 1.0)[1]
    check(grad[zero], rg[zero], e_grad[zero], "normals at zero vectors")
    n = F.normalize(pred3.double(), dim=1)
    far = ((n - y.double()).abs() > 64 * U).all(1, keepdim=True).expand_as(rg) & ~zero
    check(grad[far], rg[far], e_grad[far], "normals elsewhere")


def test_losses_golden_criterion_on_the_device(cuda_dev):
    """tests/golden/losses.pt part (a): the reference criterion's inputs through the device losses; the loss values and
    the d loss / d prediction the reference's own autograd stored, elementwise."""
    import os

    import mtt_b200  # noqa: F401
    from mtt_b200 import losses as ML

    fx = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "losses.pt"), weights_only=False)
    c = fx["criterion"]
    p = {"TASKS": {"NAMES": c["tasks"]}, "edge_w": 0.95, "ignore_index": 255, "ignore_invalid_area_depth": True,
         "loss_kwargs": {"loss_weights": fx["weights"]}}
    preds = {t: c["preds"][t].to(cuda_dev).requires_grad_() for t in c["tasks"]}
    out = ML.get_criterion(p)(preds, {t: c["labels"][t].to(cuda_dev) for t in c["tasks"]}, tasks=c["tasks"])
    out["total"].backward()
    for k, want in c["losses"].items():
        # the reference evaluated in fp32 too: twice the device bound (its sum over pixels in fp32: + LAM sqrt(n) u)
        if k != "total":
            lab = c["labels"][k].to(cuda_dev)
            e_val = 2 * _loss_bounds(k, c["preds"][k].to(cuda_dev), lab, 1.0)[0] + sum_tol(lab.numel(), abs(want))
            assert abs(float(out[k].detach()) - want) <= e_val, (k, float(out[k].detach()), want, e_val)
    for t in c["tasks"]:
        ref = c["dpreds"][t].to(cuda_dev).double()
        e_grad = 2 * _loss_bounds(t, c["preds"][t].to(cuda_dev), c["labels"][t].to(cuda_dev), fx["weights"][t])[1]
        check(preds[t].grad, ref, e_grad + 2 * U * ref.abs(), f"golden d loss / d pred {t}")


# ---- the tp_cfg2 reverse pass -----------------------------------------------------------------------------------------------
def test_training_step_reverse_pass_tp_cfg2_d4(cuda_dev):
    """tp_cfg2_d4 (ViT-B width, 448 x 576, the 4 NYUD tasks, 4 x 4 channel windows, e = f = 768, no ctr), batch 2: the
    same d loss / d prediction through TrainStep.backward and through float64 autograd of the train-mode restatement
    (pinned to the reference by test_train.py::test_train_mode_restatement_is_pinned_to_the_reference), every parameter
    gradient elementwise (tests/model_checks.py reverse_pass_errors). DropPath draws come from a CPU generator in the
    reference's call order."""
    fwd, bad, n = reverse_pass_errors("tp_cfg2_d4", cuda_dev, seed=31, B=2)
    for t, err in fwd.items():
        assert err < 2e-4, f"train-mode forward {t}: rel-L2 {err:.3e}"
    assert not bad, f"{len(bad)} of {n} parameter gradients off: {bad[:8]}"
