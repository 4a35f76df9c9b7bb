"""Float64 references and case builders that more than one kernel test runs: the forward glue kernels (LayerNorm,
gating, bilinear, post-processing), the Swin kernels (window attention, gather / scatter, channel attention, stride-2
convolution, channel up-projection) and the integer-valued GEMM / convolution cases that make the tensor-core
arithmetic exact. Bounds follow f64_checks."""
import math

import torch
import torch.nn.functional as F

from f64_checks import (U, Guarded, assert_planes_bit_exact, bits, check, check_planes, decode, gen,
                        guarded_split, is_sentinel, mtt_ops, padded, pad_cols, randn, round_up, sentinel,
                        sentinel_split, split_bound, sum_tol)
from oracle import taskprompter_swin_ref as R

E_BIL = 6 * U             # one bilinear value: 4 products and 3 sums, each term rounded at most 4 times (plus slack)


# ---- bilinear references -------------------------------------------------------------------------------------------------
def rows_of(B, n, batch_rows, offset, device):
    """Physical rows of image b's n logical rows: b * batch_rows + offset + i."""
    return (torch.arange(B, device=device)[:, None] * batch_rows + offset + torch.arange(n, device=device)[None]).reshape(-1)


def fp32_scale(n, n2):
    """The kernels' resize scale: fp32(n) / fp32(n2), correctly rounded (computed on the host)."""
    return float(torch.tensor(n, dtype=torch.float32) / torch.tensor(n2, dtype=torch.float32))


def fp32_coords_exact(n, n2):
    """True when the fp32 scale equals n / n2 and every source coordinate scale (d + 0.5) - 0.5, d < n2, is exact in
    fp32 (power-of-two ratios, but also 384 -> 512): then float64 F.interpolate computes the kernel's coordinates."""
    sc = fp32_scale(n, n2)
    if sc != n / n2:
        return False
    p = sc * (torch.arange(n2, dtype=torch.float64) + 0.5)
    return bool(torch.equal(p.float().double(), p) and torch.equal((p - 0.5).float().double(), p - 0.5))


def ref_bilinear(x, rows, B, h, w, C, H2, W2):
    """NHWC rows `rows` of x (float64) resized to H2 x W2, align_corners=False: (y, the same resize of |x|), NCHW.
    Only where the fp32 coordinates are exact (ref_bilinear_any covers the other ratios)."""
    assert fp32_coords_exact(h, H2) and fp32_coords_exact(w, W2), \
        f"resize {h}x{w} -> {H2}x{W2}: the fp32 coordinates are not exact, so float64 F.interpolate is no reference " \
        f"for the kernel's; use ref_bilinear_any"
    img = x[rows, :C].reshape(B, h, w, C).permute(0, 3, 1, 2)
    it = lambda v: F.interpolate(v, size=(H2, W2), mode="bilinear", align_corners=False)
    return it(img), it(img.abs())


def _bil_axis(n, n2, device):
    """bilin_coord (postproc.cuh) along one axis in float64 from the kernel's fp32 scale: (i0, i1, l1, e_s). e_s is one
    ulp of the coordinate s = scale (d + 0.5) - 0.5: the fp32 rounding of the product and of the subtraction (or of the
    one fused multiply-add) is at most 2^-24 (|s| + 0.5) + 2^-24 |s| <= 2^-23 (|s| + 1); the clamp at 0 does not add."""
    s = fp32_scale(n, n2) * (torch.arange(n2, dtype=torch.float64, device=device) + 0.5) - 0.5
    e_s = 2.0 ** -23 * (s.abs() + 1)
    s = s.clamp(min=0)
    i0 = s.floor().long().clamp(max=n - 1)
    return i0, (i0 + 1).clamp(max=n - 1), s - i0, e_s


def _nbr_max(G, ry, rx):
    """max of G [B, C, h, w] over the rows ry x columns rx (lists of [H2] / [W2] index tensors, clamped): [B, C, H2, W2]."""
    h, w = G.shape[-2:]
    m = torch.stack([G[:, :, r.clamp(0, h - 1)] for r in ry]).amax(0)
    return torch.stack([m[..., c.clamp(0, w - 1)] for c in rx]).amax(0)


def ref_bilinear_any(x, rows, B, h, w, C, H2, W2):
    """ref_bilinear at any ratio: the interpolation in float64 at the coordinates the kernel derives from its fp32
    scale, (y, |.| resize, e_coord), NCHW. The kernel rounds each coordinate in fp32 (at most e_s off, _bil_axis); the
    resize is continuous and piecewise linear in each coordinate, so a coordinate off by e moves the value by at most
    e times the largest difference of neighbouring source values it can see: rows i0 - 1 .. i0 + 2 (the shifted
    coordinate may cross into the next cell) by columns j0 - 1 .. j0 + 2. e_coord is that term for both axes; the
    kernel's arithmetic on its own weights is E_BIL of the |.| resize, as with exact coordinates."""
    img = x[rows, :C].reshape(B, h, w, C).permute(0, 3, 1, 2)
    y0, y1, ly, ey = _bil_axis(h, H2, x.device)
    x0, x1, lx, ex = _bil_axis(w, W2, x.device)

    def it(v):
        r0, r1 = v[:, :, y0], v[:, :, y1]
        top = r0[..., x0] * (1 - lx) + r0[..., x1] * lx
        bot = r1[..., x0] * (1 - lx) + r1[..., x1] * lx
        return top * (1 - ly)[:, None] + bot * ly[:, None]

    gy = F.pad((img[:, :, 1:] - img[:, :, :-1]).abs(), (0, 0, 0, 1))
    gx = F.pad((img[..., 1:] - img[..., :-1]).abs(), (0, 1))
    dy = _nbr_max(gy, [y0 - 1, y0, y0 + 1], [x0 - 1, x0, x0 + 1, x0 + 2])
    dx = _nbr_max(gx, [y0 - 1, y0, y0 + 1, y0 + 2], [x0 - 1, x0, x0 + 1])
    return it(img), it(img.abs()), ey[:, None] * dy + ex[None, :] * dx


def ref_bilinear_kernel(x, rows, B, h, w, C, H2, W2):
    """(y, |.| resize, coordinate term): float64 F.interpolate with a zero coordinate term where the fp32 coordinates
    are exact, ref_bilinear_any elsewhere."""
    if fp32_coords_exact(h, H2) and fp32_coords_exact(w, W2):
        y, a = ref_bilinear(x, rows, B, h, w, C, H2, W2)
        return y, a, torch.zeros_like(y)
    return ref_bilinear_any(x, rows, B, h, w, C, H2, W2)


def ref_im2col(img, patch):
    B, Cin = img.shape[:2]
    return F.unfold(img, patch, stride=patch).transpose(1, 2).reshape(-1, Cin * patch * patch)


def ref_gates(logits, rc, B, T, H, C, gh, gw, nh, nw, task):
    """(g_s, g_c) [B, P, C] of one task: the prompt's spatial logit of the pixel for the channel's head, and the task's
    channel logit of the pixel's window."""
    P = gh * gw
    gs = logits[:, :, task, T:].permute(0, 2, 1).repeat_interleave(C // H, dim=2)
    gc = rc[:, task].reshape(B, C, nh, 1, nw, 1).expand(B, C, nh, gh // nh, nw, gw // nw).reshape(B, C, P)
    return gs, gc.permute(0, 2, 1)


def ref_layernorm(x, gamma, beta, eps):
    return F.layer_norm(x, (x.shape[1],), gamma, beta, eps)


def ref_postproc(y, kind):
    """get_output (TP/utils/utils.py:27-63) of NCHW logits y: kind 0 argmax, 1 255 sigmoid, 2 255 softmax[1],
    3 (normalize + 1) 255 / 2 as [B,H,W,3], 4 clamp(min 0) as [B,H,W,1]."""
    if kind == 0:
        return y.argmax(1)
    if kind == 1:
        return 255 * torch.sigmoid(y[:, 0])
    if kind == 2:
        return 255 * torch.softmax(y[:, :2], 1)[:, 1]
    if kind == 3:
        return ((F.normalize(y[:, :3], dim=1) + 1) * 255 / 2).permute(0, 2, 3, 1)
    return y[:, :1].clamp(min=0).permute(0, 2, 3, 1)


# ---- forward glue cases --------------------------------------------------------------------------------------------------
def ln_input(g, rows, cols):
    """Rows of std 0.5 around a per-row offset: a quarter at 25 (50 x their std: the two-pass variance's cancellation)."""
    x = randn(g, rows, cols, scale=0.5)
    off = torch.zeros(rows, 1, device="cuda")
    off[::4] = 25.0
    off[1::4] = -3.0
    return x + off


def ln_bound(xd, gam, bet, eps, D):
    """LayerNorm in float64 and its elementwise fp32 bound: mean and the centred sum of squares are reductions of
    depth D, rstd = 1 / sqrt(var + eps) adds 3u, y = (x - mean) rstd gamma + beta 4u."""
    n = xd.shape[1]
    mean, var = xd.mean(1, keepdim=True), xd.var(1, unbiased=False, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + eps)
    xh = (xd - mean) * rstd
    e_mean = sum_tol(D, xd.abs().sum(1, keepdim=True)) / n + U * mean.abs()
    e_var = sum_tol(D, ((xd - mean) ** 2).sum(1, keepdim=True)) / n + 3 * U * var + e_mean ** 2
    e_rr = 0.5 * e_var / (var + eps) + 3 * U
    e_xh = e_mean * rstd + xh.abs() * (e_rr + 2 * U)
    y = xh * gam + bet
    return y, gam.abs() * e_xh + 4 * U * ((xh * gam).abs() + y.abs())


def layernorm_case(ops, d, seed, ns=2):
    """One mtt_layernorm call of a table (rows x cols, input ld): fp32 out (ld = ld_in) or split out (ns planes)."""
    rows, cols = d["rows"], d["cols"]
    gg = gen(seed)
    x = torch.full((rows, d["ld_in"]), float("nan"), device="cuda")[:, :cols]      # NaN input pad columns
    x.copy_(ln_input(gg, rows, cols))
    gam, bet = torch.rand(cols, generator=gg, device="cuda") + 0.5, randn(gg, cols, scale=0.5)
    eps = 1e-6
    fast = cols % 128 == 0 and cols <= 1024
    D = (cols // 128 + 7) if fast else (math.ceil(cols / 32) + 5)   # per-lane serial chain + 5 shuffle levels
    want, e = ln_bound(x.double(), gam.double(), bet.double(), eps, D)
    assert torch.allclose(want, ref_layernorm(x.double(), gam.double(), bet.double(), eps), rtol=1e-12, atol=1e-12)
    if d.get("split"):
        gb, sp, reg = guarded_split(ops, ns, rows, cols)
        gb.snapshot()
        ops.layernorm(x, gam, bet, eps, out_split=sp)
        gb.unchanged_outside(reg, "layernorm split")
        return check_planes(sp, want, e, f"layernorm {rows}x{cols} split (LN bound, D={D})")
    gb = Guarded((rows, d["ld_in"]), torch.float32)
    gb.snapshot()
    ops.layernorm(x, gam, bet, eps, out_f32=gb.view)
    gb.unchanged_outside((slice(None), slice(0, cols)), "layernorm")
    return check(gb.view[:, :cols], want, e, f"layernorm {rows}x{cols} (LN bound, D={D})")


def gate_case(ops, d, ns, name, seed=40):
    """One gating launch of a table entry (the gating stage of gated_conv1x1: all its tasks, x rows of image b at
    b * x_group_rows + x_row_offset); err / bound ratios per task and gate."""
    B, T, N, H, C, gh, gw, nh, nw = (d[k] for k in ("B", "T", "N", "H", "C", "gh", "gw", "nh", "nw"))
    xg, xo = d["x_group_rows"], d["x_row_offset"]
    P, rows, ldy = gh * gw, B * gh * gw, round_up(C, 8)
    gg = gen(seed)
    x = randn(gg, B * xg, d["ldx"])
    logits = randn(gg, B, H, T, N, scale=1.5)
    rc = randn(gg, B, T, C, nh, nw, scale=1.5)
    pbe = round_up(ns * rows * ldy * 2, 256) // 2        # elements of one task's ys (or yc) plane set
    gb = Guarded((2 * T + 1, pbe), torch.bfloat16)        # one spare plane set after the last task
    flat = gb.view.reshape(-1)
    ys = ops.Split.from_planes(flat[:ns * rows * ldy].view(ns, rows, ldy), C)
    yc = ops.Split.from_planes(flat[pbe:pbe + ns * rows * ldy].view(ns, rows, ldy), C)
    gb.snapshot()
    ops.gate_split(x, xg, xo, logits, rc, 0, ys, yc, B=B, T=T, N=N, H=H, Cdim=C, gh=gh, gw=gw, nh=nh, nw=nw,
                   ntasks=d["ntasks"], task_stride=2 * pbe)
    gb.unchanged_outside((slice(0, 2 * T), slice(0, ns * rows * ldy)), "gate_split")
    X = x.double()[rows_of(B, P, xg, xo, "cuda"), :C].view(B, P, C)
    ratios = []
    for t in range(T):
        gs, gc = ref_gates(logits.double(), rc.double(), B, T, H, C, gh, gw, nh, nw, t)
        for which, gate in ((0, gs), (1, gc)):
            want = (X * (1 + gate)).reshape(rows, C)
            e = 2 * U * (X.abs() * (1 + gate).abs()).reshape(rows, C)      # fl(1 + g), then the product
            k = 2 * t + which
            sp = ops.Split.from_planes(gb.view[k, :ns * rows * ldy].view(ns, rows, ldy), C)
            ratios.append(check_planes(sp, want, e, f"gate_split {name} task {t} {'Yc' if which else 'Ys'} (2u)"))
    return ratios


def bilinear_case(ops, d, ns, seed):
    """One bilinear call of a table (plan_calls.bil fields) in its output form, inside sentinels; its err / bound
    ratio. The bound is E_BIL of the |.| resize plus, at a ratio whose fp32 coordinates are inexact, ref_bilinear_any's
    coordinate term."""
    B, h, w, C, H2, W2 = d["B"], d["h"], d["w"], d["C"], d["H2"], d["W2"]
    ibr = d["ibr"] or h * w
    nin = (B - 1) * ibr + d["ioff"] + h * w
    x = randn(gen(seed), nin, d["ld_in"])
    rin = rows_of(B, h * w, ibr, d["ioff"], "cuda")
    want, absr, ec = ref_bilinear_kernel(x.double(), rin, B, h, w, C, H2, W2)
    what = f"bilinear {h}x{w}->{H2}x{W2} C={C} {d['form']} ioff={d['ioff']} ooff={d['ooff']}"
    kw = dict(in_batch_rows=d["ibr"], in_row_offset=d["ioff"], out_batch_rows=d["obr"], out_row_offset=d["ooff"])
    if d["form"] == "nchw":
        gb = Guarded((B, C, H2, W2), torch.float32)
        gb.snapshot()
        ops.bilinear(x, d["ld_in"], B, h, w, C, H2, W2, out_nchw=gb.view, **kw)
        gb.unchanged_outside((slice(None),), what)
        return check(gb.view, want, E_BIL * absr + ec, f"{what} (6u of the |.| resize + coordinate term)")
    obr = d["obr"] or H2 * W2
    nout = (B - 1) * obr + d["ooff"] + H2 * W2
    rout = rows_of(B, H2 * W2, obr, d["ooff"], "cuda")
    wn = want.permute(0, 2, 3, 1).reshape(-1, C)
    an = (E_BIL * absr + ec).permute(0, 2, 3, 1).reshape(-1, C)
    if d["form"] == "f32":
        gb = Guarded((nout, d["ld_out"]), torch.float32)
        base = randn(gen(seed + 30), nout, d["ld_out"])
        gb.view.copy_(base)
        gb.snapshot()
        ops.bilinear(x, d["ld_in"], B, h, w, C, H2, W2, out_f32=gb.view, accumulate=d["acc"], **kw)
        gb.unchanged_outside((rout, slice(0, C)), what)
        old = base.double()[rout, :C] if d["acc"] else 0
        ref = wn + old
        return check(gb.view[rout, :C], ref, an + U * ref.abs(), f"{what} (6u + u of the sum)")
    gb, sp, reg = guarded_split(ops, ns, nout, C, ld=d["ld_out"])
    gb.snapshot()
    ops.bilinear(x, d["ld_in"], B, h, w, C, H2, W2, out_split=sp, **kw)
    region = torch.zeros(gb.view.shape, dtype=torch.bool, device="cuda")
    region[:ns, 16 + rout, :C] = True
    gb.unchanged_outside(region, what)
    return check(decode(sp)[rout], wn, an + split_bound(ns, wn.abs() + an), f"{what} ns={ns} (6u + split bound)")


def postproc_case(ops, d, seed):
    """One bilinear_postproc call of a table; its err / bound ratio (None for the argmax, which is checked exactly
    where the top-2 margin is clear)."""
    B, h, w, C, H2, W2, kind = (d[k] for k in ("B", "h", "w", "C", "H2", "W2", "kind"))
    x = randn(gen(seed), B * h * w, d["ld_in"], scale=3.0)
    y, ya, ec = ref_bilinear_kernel(x.double(), torch.arange(B * h * w, device="cuda"), B, h, w, C, H2, W2)
    ev = E_BIL * ya + ec                                         # bound of each resized logit
    shape = {0: (B, H2, W2), 3: (B, H2, W2, 3), 4: (B, H2, W2, 1)}.get(kind, (B, H2, W2))
    gb = Guarded(shape, torch.int64 if kind == 0 else torch.float32)
    gb.snapshot()
    ops.bilinear_postproc(x, d["ld_in"], B, h, w, C, H2, W2, kind, gb.view)
    gb.unchanged_outside((slice(None),), f"bilinear_postproc kind {kind}")
    what = f"bilinear_postproc {h}x{w}->{H2}x{W2} kind {kind} C={C}"
    got = gb.view
    if kind == 0:
        top2 = y.topk(2, dim=1)
        margin = top2.values[:, 0] - top2.values[:, 1]
        emax = ev.amax(1)
        clear = margin > 2 * emax
        assert torch.equal(got[clear], top2.indices[:, 0][clear]), f"{what}: class off where the top-2 margin is clear"
        picked = y.gather(1, got.clamp(0, C - 1)[:, None])[:, 0]
        assert ((got >= 0) & (got < C)).all() and (picked >= top2.values[:, 0] - 2 * emax).all(), \
            f"{what}: class outside the tied set"
        print(f"{what}: {int((~clear).sum())} of {clear.numel()} pixels within the tie margin")
        return None
    want = ref_postproc(y, kind)
    if kind == 1:        # sigmoid' <= 1/4; expf, 1 +, reciprocal and * 255: 6u
        e = 255 * 0.25 * ev[:, 0] + 6 * U * want.abs()
    elif kind == 2:      # d softmax[1] / d x_c <= 1/4 each; two expf, a sum, a division, * 255: 8u
        e = 255 * 0.25 * (ev[:, 0] + ev[:, 1]) + 8 * U * want.abs()
    elif kind == 3:      # d (x / |x|) moves by at most 2 |e| / |x|; sqrt, divisions, + 1, * 255 / 2: 8u of 255
        n = y[:, :3].norm(dim=1, keepdim=True).clamp_min(1e-12)
        e = (255 / 2 * 2 * ev[:, :3].norm(dim=1, keepdim=True) / n + 8 * U * 255).permute(0, 2, 3, 1).expand_as(want)
    else:                # clamp is exact
        e = ev[:, :1].permute(0, 2, 3, 1)
    return check(got, want, e, f"{what} (logit bound through the post-processing)")


# ---- Swin kernel cases ---------------------------------------------------------------------------------------------------
# Split inputs are decoded in float64 (hi + lo), so the only difference left is the kernel's own fp32 arithmetic: a dot
# product of n fp32 FMAs is off by at most n u sum |a_i b_i|, a softmax weight whose logit is off by d by a factor of at
# most exp(2 d) (the running maximum moves too). Every output lies in sentinels (pad columns, a trailing row or slot),
# inputs carry the sentinel NaN in their pad columns, so a read past C shows up in the result.
def f32(x):
    """The fp32 value the kernel receives for a Python float scale."""
    return float(torch.tensor(x, dtype=torch.float32))


def nan_split(rows, cols, dev, ns=2):
    """A sentinel Split of ns planes with one trailing row and 8 pad columns past round_up(cols, 8)."""
    return sentinel_split(rows + 1, cols, dev, ns, ld=round_up(cols, 8) + 8)


def split_in(ops, x, pad=8, ns=2):
    """x fp32 [rows, cols] -> Split of ns planes with sentinel pad columns (what the kernel reads) and its float64
    decoding."""
    rows, cols = x.shape
    sp = sentinel_split(rows, cols, x.device, ns, ld=round_up(cols, 8) + pad)
    ops.split_f32(x, ns, out=sp)
    return sp, decode(sp, rows)


def assert_untouched(sp, rows, cols):
    """Pad columns [cols, ld) and every row past `rows` of both planes still hold the sentinel."""
    assert is_sentinel(sp.buf[:, :rows, cols:]), "pad columns written"
    assert is_sentinel(sp.buf[:, rows:]), "rows past the output written"


def attention_case(ops, dev, *, B, nWy, nWx, ws, shift, T, heads, dh, seed, ns=2):
    """B images of nWy x nWx windows; q of every other query row scaled 12x so that its logits span about +-50 (the
    online softmax rescales many times); bias table at std 0.5; shift mask (-100) when shift > 0. qkv and the output
    as ns planes. Returns the worst err / bound ratios of the output and the raw logits."""
    g = torch.Generator(device=dev).manual_seed(seed)
    C, L = heads * dh, ws * ws
    N, nW = T + L, nWy * nWx
    BW, rows = B * nW, B * nW * N
    x = torch.randn(rows, 3 * C, device=dev, generator=g)
    qs = torch.where(torch.arange(rows, device=dev) % N % 2 == 0, 12.0, 1.0)
    x[:, :C] *= qs[:, None]
    qkv, X = split_in(ops, x, ns=ns)
    table = torch.randn((2 * ws - 1) ** 2, heads, device=dev, generator=g) * 0.5
    bias = table[R.relative_position_index(ws).reshape(-1).to(dev)].reshape(L, L, heads).permute(2, 0, 1)  # [h, q, k]
    biasT = bias.transpose(1, 2).contiguous()                                                 # the kernel's [h, key, query]
    mask = R.shifted_window_mask(nWy * ws, nWx * ws, ws, shift).to(dev) if shift else None    # [nW, q, k]
    maskT = mask.transpose(1, 2).contiguous() if shift else None
    out = nan_split(rows, C, dev, ns=ns)
    raw_buf = sentinel((BW * heads * T * L + 16,), dev=dev)
    raw = raw_buf[:BW * heads * T * L].view(BW, heads, T, L)
    scale = f32(dh ** -0.5)
    ops.swin_window_attention(qkv, out, raw, biasT, maskT, BW=BW, nW=nW, T=T, L=L, heads=heads, scale=scale)
    torch.cuda.synchronize()

    q, k, v = X.view(BW, N, 3, heads, dh).permute(2, 0, 3, 1, 4)              # [BW, h, N, dh] each
    dot, A = q @ k.transpose(-1, -2), q.abs() @ k.abs().transpose(-1, -2)      # raw q.k and sum |q_d k_d|
    s, As = dot * scale, A * scale
    extra = bias.double()[None].expand(BW, -1, -1, -1)
    if shift:
        extra = extra + mask.double().repeat(B, 1, 1)[:, None]                 # window w of every image gets mask[w]
    s[..., T:, T:] += extra                                                    # patch x patch entries only (TP:196, :201)
    As[..., T:, T:] += extra.abs()
    o = torch.softmax(s, -1) @ v                                               # [BW, h, N, dh]
    # logit error per query row: the dot product (dh FMAs + the pair sum), the scale and the bias / mask adds; __expf adds
    # at most (2 + 1.2|x|) ulp to a weight exp(-|x|), < 2^-21 of the largest weight. Output: the weights shift by
    # exp(2 d) - 1 ~ 2 d, times |v_j - o| <= 2 max|v|; the fp32 accumulation of N weighted v rows and 1/l; the split.
    d = U * (dh + 4) * As.amax(-1, keepdim=True) + 2.0 ** -21
    vmax = v.abs().amax((-1, -2), keepdim=True)
    bound = (4 * d + (N + 3) * U) * vmax + split_bound(ns, o.abs())
    got = decode(out, rows).view(BW, N, heads, dh).transpose(1, 2)
    ratios = [check(got, o, bound, f"attention out (B={B} nW={nW} ws={ws} shift={shift} T={T} dh={dh} ns={ns})",
                    block=2)]
    assert_untouched(out, rows, C)
    if T:
        rb = U * (dh + 1) * A[..., :T, T:]
        ratios.append(check(raw, dot[..., :T, T:], rb, "raw prompt logits", block=2))
    assert is_sentinel(raw_buf[raw.numel():]) and (T or is_sentinel(raw_buf)), "raw written past its end"
    return ratios


def _windows(m, ws, shift):
    """[B, H, W, ...] -> [B * nW, ws*ws, ...]: zero pad after the norm, roll by -shift, row-major windows (TP:326-340)."""
    B, H, W = m.shape[:3]
    Hp, Wp = -(-H // ws) * ws, -(-W // ws) * ws
    m = F.pad(m, (0, 0, 0, Wp - W, 0, Hp - H))
    if shift:
        m = torch.roll(m, (-shift, -shift), (1, 2))
    return R.to_windows(m, ws)


def _unwindow(w, ws, shift, B, H, W):
    """Inverse of _windows, cropped to H x W (TP:343-360)."""
    Hp, Wp = -(-H // ws) * ws, -(-W // ws) * ws
    m = R.from_windows(w, ws, B, Hp, Wp)
    if shift:
        m = torch.roll(m, (shift, shift), (1, 2))
    return m[:, :H, :W]


def gather_scatter_case(ops, dev, *, B, H, W, C, T, heads, ws, shift, ns=2, lasts=(False, True)):
    """Window gather into ns planes (bit-exact), and the scatter with last = each of `lasts`: xa and x += xa bit-exact,
    the logits map [B, heads, T, T + H*W] bit-exact with its T prefix columns untouched, the prompt mean within its
    bound. Returns the prompt mean's worst err / bound."""
    g = torch.Generator(device=dev).manual_seed(H * W + C + shift)
    rnd = lambda *s: torch.randn(*s, device=dev, generator=g)
    Hp, Wp = -(-H // ws) * ws, -(-W // ws) * ws
    nW, wl = (Hp // ws) * (Wp // ws), ws * ws
    rows = B * nW * (T + wl)
    # gather: split rows of the joint window stream, bit-exact
    xn, pn = padded(B * H * W, C, dev), padded(B * T, C, dev)
    xn.copy_(rnd(B * H * W, C))
    pn.copy_(rnd(B * T, C))
    sw = nan_split(rows, C, dev, ns=ns)
    ops.swin_window_gather(xn, pn, sw, B=B, H=H, W=W, Cdim=C, T=T, ws=ws, shift=shift)
    torch.cuda.synchronize()
    win = _windows(xn.reshape(B, H, W, C), ws, shift)
    pr = pn.reshape(B, 1, T, C).expand(B, nW, T, C).reshape(B * nW, T, C)
    assert_planes_bit_exact(sw, torch.cat([pr, win], 1).reshape(rows, C), "window gather")   # the T prompts first
    assert_untouched(sw, rows, C)
    del sw, win, pr

    # scatter: xa = window reverse (copy), x += xa (torch's fp32 add), p += window mean of the prompt rows, logits map
    o = padded(rows, C, dev)
    o.copy_(rnd(rows, C))
    raw = rnd(B * nW, heads, T, wl)
    ow = o.reshape(B * nW, T + wl, C)
    xa_ref = _unwindow(ow[:, T:], ws, shift, B, H, W).reshape(B * H * W, C)
    lg_ref = _unwindow(raw.reshape(B * nW, heads * T, wl).transpose(1, 2), ws, shift, B, H, W)     # [B, H, W, heads*T]
    lg_ref = lg_ref.reshape(B, H * W, heads, T).permute(0, 2, 3, 1)
    pm = ow[:, :T].double().reshape(B, nW, T, C)
    x0, p0 = rnd(B * H * W, C), rnd(B * T, C)
    ratio = 0.0
    for last in lasts:
        xa, x, p = padded(B * H * W, C, dev), padded(B * H * W, C, dev, fill=7.0), padded(B * T, C, dev, fill=7.0)
        x.copy_(x0)
        p.copy_(p0)
        lg = sentinel((B, heads, T, T + H * W), dev=dev)
        ops.swin_window_scatter(o, raw, xa, x, p, lg, B=B, H=H, W=W, Cdim=C, T=T, ws=ws, shift=shift, heads=heads,
                                last=last)
        torch.cuda.synchronize()
        assert torch.equal(bits(xa), bits(xa_ref)) and is_sentinel(pad_cols(xa))
        assert torch.equal(bits(x), bits(x0 + xa_ref)) and (pad_cols(x) == 7.0).all()
        assert torch.equal(bits(lg[..., T:]), bits(lg_ref)), "logits map"
        assert is_sentinel(lg[..., :T]), "logits columns [0, T) written"
        assert (pad_cols(p) == 7.0).all()
        if last:
            assert torch.equal(bits(p), bits(p0)), "the last block leaves the prompts alone"
        else:
            # 4 window groups of ceil(nW / 4) sequential fp32 adds, the 4-way sum, the division and the += of p
            want = p0.double() + pm.mean(1).reshape(B * T, C)
            bound = U * ((-(-nW // 4) + 4) * pm.abs().mean(1).reshape(B * T, C) + p0.double().abs() + want.abs())
            ratio = max(ratio, check(p, want, bound, "prompt mean", block=1))
    return ratio


def chan_attention_case(ops, dev, *, B, T, C, nh, ns=2):
    """swin_chan_attention at ce = 256 with nh x nh channel windows, the split output as ns planes: raw_chan and
    chan_out within their bounds, the split bit-exact. Returns the worst err / bound of raw_chan and chan_out."""
    ce = 256
    r = 16
    wh = ww = r // nh
    G, we = nh * nh, wh * ww
    gen = torch.Generator(device=dev).manual_seed(C + nh)
    q = padded(B * T, ce, dev)
    q.copy_(torch.randn(B * T, ce, device=dev, generator=gen))
    q[0::2] *= 15.0                          # even prompts: logits span about +-50 at one window of 256 entries
    kv = padded(B * C, 2 * ce, dev)
    kv.copy_(torch.randn(B * C, 2 * ce, device=dev, generator=gen))
    co = padded(B * T, ce, dev)
    cs = nan_split(B * T, ce, dev, ns=ns)
    rc_buf = sentinel((B * T * C * G + 16,), dev=dev)
    rc = rc_buf[:B * T * C * G].view(B, T, C, nh, nh)
    ops.swin_chan_attention(q, kv, co, cs, rc, B=B, T=T, Cdim=C, ce=ce, nh=nh, nw=nh)
    torch.cuda.synchronize()

    def grid(t):   # [B, n, ce] with ce = (nh, wh, nw, ww) -> [B, nh*nw, n, wh*ww] (TP:383-388)
        return t.reshape(B, t.shape[1], nh, wh, nh, ww).permute(0, 2, 4, 1, 3, 5).reshape(B, G, t.shape[1], we)

    qg = grid(q.double().reshape(B, T, ce))
    kvd = kv.double().reshape(B, C, 2, ce)
    kg, vg = grid(kvd[:, :, 0]), grid(kvd[:, :, 1])
    scale = f32(1.0) / math.sqrt(ce)                                         # 1/16, exact in fp32
    raw = qg @ kg.transpose(-1, -2)                                          # [B, G, T, C]
    A = qg.abs() @ kg.abs().transpose(-1, -2)
    out = torch.softmax(raw * scale, -1) @ vg                                # [B, G, T, we]
    # raw: ceil(we / 32) FMAs per lane and a 5-step shuffle tree. Output: logit error d -> weights off by ~2 d, times
    # |v - o| <= 2 max|v|, __expf < 2^-21 of the largest weight, C / 8 + 8 fp32 adds of the weighted v and 1/sum.
    rb = U * (-(-we // 32) + 6) * A
    d = scale * rb.amax(-1, keepdim=True) + 2.0 ** -21
    vmax = vg.abs().amax((-1, -2), keepdim=True)
    bound = (4 * d + (C // 8 + 12) * U) * vmax
    ratios = [check(rc.permute(0, 3, 4, 1, 2).reshape(B, G, T, C), raw, rb, "raw_chan", block=3),
              check(grid(co.reshape(B, T, ce)), out, bound, "chan_out", block=3)]
    assert is_sentinel(pad_cols(co)) and is_sentinel(rc_buf[rc.numel():])
    assert_planes_bit_exact(cs, co.contiguous(), "chan_out split")          # the split output is the split of chan_out
    assert_untouched(cs, B * T, ce)
    return ratios


def conv3x3_s2_case(ops, dev, *, B, T, H, W, Cin, seed):
    """conv3x3_s2_maps over [B, Cin, T + H*W] logit maps (the T prompt columns first) into [B, Cin, T + H*W/4]:
    within 9 Cin + 2 FMAs of the absolute conv, the T prefix columns untouched. Returns the worst err / bound."""
    L = H * W
    g = torch.Generator(device=dev).manual_seed(seed)
    x = torch.randn(B, Cin, T + L, device=dev, generator=g)
    w = torch.randn(Cin, Cin, 3, 3, device=dev, generator=g) * 0.2
    b = torch.randn(Cin, device=dev, generator=g)
    out = sentinel((B, Cin, T + L // 4), dev=dev)
    ops.conv3x3_s2_maps(x, w, b, out, B=B, Cin=Cin, H=H, W=W, in_stride=T + L, in_offset=T, out_stride=T + L // 4,
                        out_offset=T)
    torch.cuda.synchronize()
    xm = x[..., T:].double().reshape(B, Cin, H, W)
    want = F.conv2d(xm, w.double(), b.double(), stride=2, padding=1)
    absum = F.conv2d(xm.abs(), w.double().abs(), b.double().abs(), stride=2, padding=1)
    ratio = check(out[..., T:].reshape(want.shape), want, U * (9 * Cin + 2) * absum,   # 9 Cin FMAs after the bias
                  f"conv3x3_s2 B={B} Cin={Cin} {H}x{W}", block=2)
    assert is_sentinel(out[..., :T])
    return ratio


def chan_up_case(ops, dev, *, BT, C, nwin, seed):
    """swin_chan_up C -> 2C over the channel axis of raw_chan [BT, C, nwin]; nothing past the output written. Returns
    the worst err / bound."""
    Cout = 2 * C
    g = torch.Generator(device=dev).manual_seed(seed)
    rc = torch.randn(BT, C, nwin, device=dev, generator=g)
    w = torch.randn(Cout, C, device=dev, generator=g) * 0.05
    buf = sentinel((BT * Cout * nwin + 16,), dev=dev)
    out = buf[:BT * Cout * nwin].view(BT, Cout, nwin)
    ops.swin_chan_up(rc, w, out, BT=BT, Cdim=C, nwin=nwin)
    torch.cuda.synchronize()
    want = w.double() @ rc.double()
    ratio = check(out, want, U * (C + 1) * (w.double().abs() @ rc.double().abs()), f"chan_up BT={BT} C={C}", block=1)
    assert is_sentinel(buf[out.numel():])
    return ratio


# ---- integer-valued GEMM / convolution cases ------------------------------------------------------------------------------
# Every plane holds small integers, so every product and partial sum is an integer below 2^24 and the kernels' fp32
# arithmetic is exact: ref_gemm states ops.gemm in float64 and the result must match bit for bit.
BOUND = 2 ** 22


def ints(g, shape, r):
    return torch.randint(-r, r + 1, shape, generator=g).float()


def int_range(k_eff):
    """Largest value range r (|hi|, |lo| <= r) that keeps sum|terms| of a k_eff-deep product well below BOUND."""
    return max(1, min(16, math.isqrt(2 ** 19 // k_eff)))


def to_dev(sp, dev):
    return mtt_ops().Split.from_planes(sp.buf.to(dev, copy=True), sp.cols)


def int_split(dev, g, rows, cols, r, nsplit=2, ld=None, pad=0.0, lo_zero=False):
    """Split [rows, cols] with integer planes in [-r, r], written straight into Split.buf (split_f32 would give lo = 0
    for small integers); columns [cols, ld) hold `pad` (NaN: a poisoned pad)."""
    sp = mtt_ops().Split(rows, cols, "cpu", nsplit, ld=ld)
    sp.buf.fill_(pad)
    sp.buf[0, :, :cols] = ints(g, (rows, cols), r).bfloat16()
    if nsplit == 2:
        sp.buf[1, :, :cols] = 0 if lo_zero else ints(g, (rows, cols), r).bfloat16()
    return to_dev(sp, dev)


def conv_weight(dev, g, Cout, Cin, ks, r, nsplit=2):
    """Packed conv weight [Cout, ks*ks*cin_pad] with integer hi and lo planes: pack_conv_weight of an integer hi tensor
    and of an integer lo tensor, the second's hi plane copied into the first's lo plane (pad columns stay zero)."""
    ops = mtt_ops()
    wh = ints(g, (Cout, Cin, ks, ks), r)
    wl = ints(g, (Cout, Cin, ks, ks), r) if nsplit == 2 else None
    if dev == "cpu":    # the host copy for the reference: the packed layout written out in torch
        cp = (Cin + 63) // 64 * 64
        sp = ops.Split(Cout, ks * ks * cp, "cpu", nsplit, zero=True)
        for i, t in enumerate((wh, wl)[:nsplit]):
            sp.buf[i].view(Cout, ks * ks, cp)[:, :, :Cin] = t.permute(0, 2, 3, 1).reshape(Cout, ks * ks, Cin).bfloat16()
        return sp
    hi, _ = ops.pack_conv_weight(wh.to(dev), None, None, nsplit)
    if nsplit == 2:
        lo, _ = ops.pack_conv_weight(wl.to(dev), None, None, 2)
        hi.buf[1] = lo.buf[0]
    return hi


def out_rows(r, regroup):
    """The output row of GEMM row r under ops.gemm's regroup (in_group, out_group, offset[, row stride])."""
    if regroup is None or regroup[0] == 0:
        return r
    stride = regroup[3] if len(regroup) > 3 else 1
    return (r // regroup[0]) * regroup[1] + regroup[2] + (r % regroup[0]) * stride


def _im2col(x, B, H, W, ks, dil):
    """NHWC [B*H*W, K] -> [B*H*W, ks*ks*K], tap-major (the packed weight's column order), zero padding."""
    K = x.shape[1]
    p = dil * (ks // 2)
    xp = F.pad(x.reshape(B, H, W, K), (0, 0, p, p, p, p))
    cols = [xp[:, ky * dil:ky * dil + H, kx * dil:kx * dil + W, :] for ky in range(ks) for kx in range(ks)]
    return torch.stack(cols, 3).reshape(B * H * W, ks * ks * K)


def ref_gemm(a, w, *, M=None, N=None, K=None, bias=None, act=0, residual=None, res_row_mod=0, out_f32=None,
             out_split=None, out_col_offset=0, regroup=None, conv=None, a_row_offset=0, a_gather=None, w_col_offset=0,
             a_col_offset=0, w_row_offset=0, out_row_offset=0, sk_ws=None):
    """Exact float64 restatement of ops.gemm on host tensors (a, w: Splits; outputs updated in place). Asserts the
    sum|terms| bound that makes the kernel's fp32 arithmetic exact."""
    nsplit = min(a.nsplit, w.nsplit)
    M = a.rows if M is None else M
    N = w.rows if N is None else N
    K = a.cols if K is None else K
    r = torch.arange(M)
    if a_gather is not None:
        arow = a_row_offset + (r // a_gather[0]) * a_gather[1] + r % a_gather[0]
    else:
        arow = a_row_offset + r
    planes64 = lambda sp: [sp.buf[0].double(), sp.buf[1].double() if nsplit == 2 else None]
    A = [None if p is None else p[arow][:, a_col_offset:a_col_offset + K] for p in planes64(a)]
    if conv is None:
        Wp = [None if p is None else p[w_row_offset:w_row_offset + N, w_col_offset:w_col_offset + K]
              for p in planes64(w)]
    else:
        B, H, Wd, ks, dil = conv
        cp = (K + 63) // 64 * 64
        A = [None if p is None else _im2col(p, B, H, Wd, ks, dil) for p in A]
        Wp = [None if p is None else p[w_row_offset:w_row_offset + N, :ks * ks * cp].reshape(N, ks * ks, cp)[:, :, :K]
              .reshape(N, ks * ks * K) for p in planes64(w)]
    (ah, al), (wh, wl) = A, Wp
    y = ah @ wh.t()
    if nsplit == 2:
        y = y + ah @ wl.t() + al @ wh.t()
    # sum|terms| <= (largest row sum of |a_hi| + |a_lo|) * (largest |w_hi| + |w_lo|) + |bias| + |residual|
    amag = ah.abs() + (al.abs() if nsplit == 2 else 0)
    wmag = wh.abs() + (wl.abs() if nsplit == 2 else 0)
    mag = float(amag.sum(1).max()) * float(wmag.max()) if M and N else 0.0
    ro = out_rows(r, regroup)
    if bias is not None:
        b = bias[:N].double().cpu()
        y, mag = y + b, mag + float(b.abs().max())
    if act == 2:
        y = y.clamp_min(0)
    else:
        assert act == 0, "integer cases: no activation or ReLU"
    if residual is not None:
        rr = r % res_row_mod if res_row_mod > 0 else ro
        res = residual.cpu()[rr, :N].double()
        y, mag = y + res, mag + float(res.abs().max())
    assert not torch.isnan(y).any() and mag <= BOUND, f"case out of the exact range: {mag}"
    y32 = y.float()
    if out_f32 is not None:
        out_f32[ro, :N] = y32.to(out_f32.device)
    if out_split is not None:
        hi = y32.bfloat16()
        rows, cols = ro + out_row_offset, slice(out_col_offset, out_col_offset + N)
        out_split.buf[0, rows.to(out_split.buf.device), cols] = hi.to(out_split.buf.device)
        if out_split.nsplit == 2:
            out_split.buf[1, rows.to(out_split.buf.device), cols] = (y32 - hi.float()).bfloat16().to(out_split.buf.device)


# Each builder is a function of the device returning ([(a, w, gemm kwargs)], [output tensors]); the operands come from a
# fixed seed on the host, so the same case is built once on the host for the reference and once on the device.
def plain_case(M, N, K, *, nsplit=2, w_nsplit=None, bias=True, act=0, residual=False, inplace=False, seed=0,
               a_lo_zero=False, out_split_nsplit=2):
    """One GEMM into a sentinel fp32 output and a sentinel split output with pad columns [N, ld)."""
    w_nsplit = nsplit if w_nsplit is None else w_nsplit

    def build(dev):
        g = torch.Generator().manual_seed(seed * 7919 + M * 31 + N * 7 + K)
        r = int_range(K)
        a = int_split(dev, g, M, K, r, nsplit, lo_zero=a_lo_zero)
        w = int_split(dev, g, N, K, r, w_nsplit)
        kw = dict(act=act)
        if bias:
            kw["bias"] = ints(g, (N,), 64).to(dev)
        of = sentinel((M, N), dev=dev)
        if residual:
            res = ints(g, (M, N), 4096).to(dev)
            if inplace:
                of.copy_(res)
                res = of
            kw["residual"] = res
        osp = sentinel_split(M, N, dev, out_split_nsplit, ld=(N + 7) // 8 * 8)
        kw.update(out_f32=of, out_split=osp)
        return [(a, w, kw)], [of, osp.buf]
    return build


def conv_case(B, H, W, Cin, Cout, ks, dil, *, nsplit=2, residual=False, seed=0, a_lo_zero=False):
    def build(dev):
        g = torch.Generator().manual_seed(seed * 104729 + B * 1000003 + H * 1009 + W * 17 + Cin * 3 + Cout + ks + dil)
        r = int_range(ks * ks * Cin)
        M = B * H * W
        a = int_split(dev, g, M, Cin, r, nsplit, lo_zero=a_lo_zero)
        w = conv_weight(dev, g, Cout, Cin, ks, r, nsplit)
        of = sentinel((M, Cout), dev=dev)
        osp = sentinel_split(M, Cout, dev, 2)
        kw = dict(N=Cout, K=Cin, bias=ints(g, (Cout,), 64).to(dev), act=2, out_f32=of, out_split=osp,
                  conv=(B, H, W, ks, dil))
        if residual:
            kw["residual"] = ints(g, (M, Cout), 4096).to(dev)
        return [(a, w, kw)], [of, osp.buf]
    return build


def gather_case(G, T, stride, N=72, K=136, a_lo_zero=False):
    """token_trans-style gathered A: rows (g, i) at g * stride + i, i < T; every row that is not gathered is NaN."""
    def build(dev):
        g = torch.Generator().manual_seed(24 + T)
        a = int_split("cpu", g, G * stride, K, int_range(K), lo_zero=a_lo_zero)
        keep = torch.zeros(G * stride, dtype=torch.bool)
        keep[(torch.arange(G)[:, None] * stride + torch.arange(T)[None]).reshape(-1)] = True
        a.buf[:, ~keep] = float("nan")
        a = to_dev(a, dev)
        w = int_split(dev, g, N, K, int_range(K))
        of = sentinel((G * T, N), dev=dev)
        osp = sentinel_split(G * T, N, dev)
        return [(a, w, dict(M=G * T, a_gather=(T, stride), bias=ints(g, (N,), 64).to(dev), out_f32=of,
                            out_split=osp))], [of, osp.buf]
    return build


def regroup_case(regroup, M=300, N=136, K=72, res_row_mod=0, a_lo_zero=False):
    ig, og = regroup[:2]

    def build(dev):
        g = torch.Generator().manual_seed(31 + og)
        rows_out = (M // ig) * og
        a = int_split(dev, g, M, K, int_range(K), lo_zero=a_lo_zero)
        w = int_split(dev, g, N, K, int_range(K))
        of = sentinel((rows_out, N), dev=dev)
        osp = sentinel_split(rows_out, N, dev)
        kw = dict(bias=ints(g, (N,), 64).to(dev), out_f32=of, out_split=osp, regroup=regroup)
        if res_row_mod:
            kw.update(residual=ints(g, (res_row_mod, N), 4096).to(dev), res_row_mod=res_row_mod)
        return [(a, w, kw)], [of, osp.buf]
    return build
