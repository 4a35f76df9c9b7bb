"""-m gpu: the kernels of csrc/swin.cu (and the split-K chan_kv GEMM) at the geometries the Swin-B TaskPrompter launches,
against float64 statements of the reference's semantics (TP/models/transformers/taskprompter_swin.py) written here:

  * roll by -shift after padding the normed map, row-major windows with the T prompts first in every window;
  * relative-position bias from oracle.taskprompter_swin_ref.relative_position_index, shift mask from its
    shifted_window_mask (both checked against the reference by test_oracle.py);
  * softmax attention / channel attention / PatchMerging / stride-2 convolution in float64 on the device.

Split inputs are decoded in float64 (hi + lo), so the only difference left is the kernel's own fp32 arithmetic. Every
fp32 result is checked element by element against a bound computed from its own operands: a dot product of n fp32
FMAs is off by at most n * 2^-24 * sum |a_i b_i|, a softmax weight whose logit is off by d is off by a factor of at most
exp(2 d) (the running maximum moves too), and a split output adds its 2^-17 rounding (asserted here as 2^-16 |ref|).
A bound per element, not one relative to the global maximum, means a wrong window, head or row of small magnitude cannot
hide. Failures report the worst block's error over that block's own max |ref|.

Copies (window gather / scatter, transpose, merge, logits scatter) and splits of copies are bit-exact. Every output
buffer is NaN-filled first, with pad columns [C, ld) and a trailing row or slot the kernel must not write; the test
asserts they survive. Inputs carry NaN in their pad columns, so a read past C shows up in the result.

Swin-B at 1024x2048 (0.75 input scale, patch 4): stage maps 192x384 / 96x192 / 48x96 / 24x48, C 128 / 256 / 512 / 1024,
heads 4 / 8 / 16 / 32 (head dim 32), window 12 (144 tokens + T = 2 prompts: N = 146), 512 / 128 / 32 / 8 windows per
image, chan_embed_dim 256 with one channel window.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import taskprompter_swin_ref as R

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]

U = 2.0 ** -24               # unit roundoff of fp32
NAN = float("nan")
SWINB = [  # (H, W, C, heads) per stage, window 12, T 2
    (192, 384, 128, 4), (96, 192, 256, 8), (48, 96, 512, 16), (24, 48, 1024, 32)]


@pytest.fixture(scope="module")
def ops(cuda_dev):
    import mtt_b200  # noqa: F401
    from mtt_b200 import ops
    return ops


def f32(x):
    """The fp32 value the kernel receives for a Python float scale."""
    return float(torch.tensor(x, dtype=torch.float32))


def nan_split(ops, rows, cols, dev, extra_ld=8, ns=2):
    """A NaN-filled Split of ns planes with one trailing row and extra_ld pad columns past round_up(cols, 8)."""
    sp = ops.Split(rows + 1, cols, dev, ns, ld=ops.round_up(cols, 8) + extra_ld)
    sp.buf.fill_(NAN)
    return sp


def padded(rows, cols, dev, pad=3, fill=NAN):
    """A [rows, cols] fp32 view of a [rows, cols + pad] buffer whose pad columns hold `fill`."""
    buf = torch.full((rows, cols + pad), fill, device=dev)
    return buf[:, :cols]


def pad_cols(v):
    """The pad columns of a `padded` view."""
    return torch.as_strided(v, (v.shape[0], v.stride(0) - v.shape[1]), (v.stride(0), 1), v.storage_offset() + v.shape[1])


def split_in(ops, x, pad=8, ns=2):
    """x fp32 [rows, cols] -> Split of ns planes with NaN pad columns (what the kernel reads) and its float64 decoding."""
    rows, cols = x.shape
    sp = ops.Split(rows, cols, x.device, ns, ld=ops.round_up(cols, 8) + pad)
    sp.buf.fill_(NAN)
    ops.split_f32(x, ns, out=sp)
    return sp, decode(sp, rows, cols)


def decode(sp, rows, cols):
    """float64 value of the planes: hi + lo, or hi alone."""
    v = sp.buf[0, :rows, :cols].double()
    return v + sp.buf[1, :rows, :cols].double() if sp.nsplit == 2 else v


def split_rel(ns):
    """Relative error of storing a value as ns planes (asserted as 2^-16 for hi + lo, 2^-8 for hi alone)."""
    return 2.0 ** -16 if ns == 2 else 2.0 ** -8


def assert_split_of(sp, x, what):
    """The planes are the split of fp32 x bit for bit (hi alone when there is one plane)."""
    rows, cols = x.shape
    hi, lo = split_exact(x)
    assert torch.equal(sp.buf[0, :rows, :cols], hi), f"{what}: hi plane"
    assert sp.nsplit == 1 or torch.equal(sp.buf[1, :rows, :cols], lo), f"{what}: lo plane"


def split_exact(x):
    """The split of fp32 x: hi = bf16(x) and lo = bf16(x - hi), both round-to-nearest-even."""
    hi = x.bfloat16()
    return hi, (x - hi.float()).bfloat16()


def assert_untouched(sp, rows, cols):
    """Pad columns [cols, ld) and every row past `rows` of both planes still hold the NaN sentinel."""
    assert torch.isnan(sp.buf[:, :rows, cols:].float()).all(), "pad columns written"
    assert torch.isnan(sp.buf[:, rows:].float()).all(), "rows past the output written"


def assert_bounded(got, ref, bound, block, what):
    """|got - ref| <= bound elementwise (all float64, same shape); `block` = number of leading dims that index a block,
    for the report."""
    assert torch.isfinite(got).all(), f"{what}: non-finite output (unwritten sentinel or NaN read)"
    err = (got - ref).abs()
    bad = err > bound
    if bad.any():
        e = err.flatten(block).amax(-1)
        m = ref.abs().flatten(block).amax(-1).clamp_min(1e-300)
        worst = (e / m).flatten().argmax()
        raise AssertionError(f"{what}: {int(bad.sum())} of {err.numel()} elements over the bound; worst block "
                             f"{tuple(int(i) for i in torch.unravel_index(worst, e.shape))}: error / block max |ref| = "
                             f"{(e / m).flatten()[worst].item():.3e}, max error / bound = {(err / bound).max().item():.3e}")


# ---------------------------------------------------------------------------------------------------------------------
# window attention
# ---------------------------------------------------------------------------------------------------------------------
def _attention_case(ops, dev, *, B, nWy, nWx, ws, shift, T, heads, dh, seed, ns=2):
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
    out = nan_split(ops, rows, C, dev, ns=ns)
    raw_buf = torch.full((BW * heads * T * L + 16,), NAN, device=dev)
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
    # exp(2 d) - 1 ~ 2 d, times |v_j - o| <= 2 max|v|; the fp32 accumulation of N weighted v rows and 1/l; split 2^-16.
    d = U * (dh + 4) * As.amax(-1, keepdim=True) + 2.0 ** -21
    vmax = v.abs().amax((-1, -2), keepdim=True)
    bound = (4 * d + (N + 3) * U) * vmax + split_rel(ns) * o.abs()
    got = decode(out, rows, C).view(BW, N, heads, dh).transpose(1, 2)
    assert_bounded(got, o, bound, 2, f"attention out (B={B} nW={nW} ws={ws} shift={shift} T={T} dh={dh} ns={ns})")
    assert_untouched(out, rows, C)
    ratios = [float(((got - o).abs() / bound).max())]
    if T:
        rb = U * (dh + 1) * A[..., :T, T:]
        assert_bounded(raw.double(), dot[..., :T, T:], rb, 2, "raw prompt logits")
        ratios.append(float(((raw.double() - dot[..., :T, T:]).abs() / rb).max()))
    assert torch.isnan(raw_buf[raw.numel():]).all() and (T or torch.isnan(raw_buf).all()), "raw written past its end"
    return ratios


@pytest.mark.parametrize("stage", range(4))
@pytest.mark.parametrize("shift", [0, 6])
def test_window_attention_swinB_stages(ops, cuda_dev, stage, shift):
    """The four Swin-B stages exactly: ws 12, T 2, head dim 32, N = 146 (the 192-thread launch). Two images in the
    small stages, so the mask is indexed by the window within its image."""
    H, W, C, heads = SWINB[stage]
    _attention_case(ops, cuda_dev, B=1 if stage < 2 else 2, nWy=H // 12, nWx=W // 12, ws=12, shift=shift, T=2,
                    heads=heads, dh=C // heads, seed=10 * stage + shift)


@pytest.mark.parametrize("ws,T,dh,heads", [
    (7, 15, 8, 3),     # N = 64: the 64-thread launch, full
    (8, 1, 16, 2),     # N = 65: 128 threads
    (11, 7, 64, 2),    # N = 128
    (11, 8, 32, 2),    # N = 129: 192 threads
    (13, 23, 8, 4),    # N = 192
    (14, 3, 64, 2),    # N = 199 > 192: threads loop over query rows
    (20, 4, 16, 2),    # N = 404: three row passes
    (6, 0, 32, 2),     # T = 0: no prompts, no raw logits
    (4, 0, 64, 1),     # T = 0, N = 16
])
def test_window_attention_geometries(ops, cuda_dev, ws, T, dh, heads):
    """Every head_dim instantiation (8, 16, 32, 64) and N on both sides of each thread-count branch, 2 images of 2 x 3
    shifted windows."""
    _attention_case(ops, cuda_dev, B=2, nWy=2, nWx=3, ws=ws, shift=ws // 2, T=T, heads=heads, dh=dh, seed=ws * 100 + T)


@pytest.mark.parametrize("ws,T,dh,why", [(4, 2, 24, "head_dim=24"), (20, 4, 64, "window too large")])
def test_window_attention_refusals(ops, cuda_dev, ws, T, dh, why):
    """head_dim outside {8, 16, 32, 64}, and K + V of a window over the 200 KB of shared memory (N = 404 at head dim 64:
    202 KB), are refused with the library's error and nothing is launched."""
    heads, L = 2, ws * ws
    N, C = T + L, heads * dh
    qkv, _ = split_in(ops, torch.randn(N, 3 * C, device=cuda_dev))
    out = nan_split(ops, N, C, cuda_dev)
    raw = torch.full((1, heads, T, L), NAN, device=cuda_dev)
    biasT = torch.zeros(heads, L, L, device=cuda_dev)
    torch.cuda.synchronize()
    n0 = ops.launch_count()
    with pytest.raises(RuntimeError, match=why):
        ops.swin_window_attention(qkv, out, raw, biasT, None, BW=1, nW=1, T=T, L=L, heads=heads, scale=dh ** -0.5)
    torch.cuda.synchronize()
    assert ops.launch_count() == n0
    assert torch.isnan(out.buf.float()).all() and torch.isnan(raw).all()


# ---------------------------------------------------------------------------------------------------------------------
# window gather / scatter (partition, reverse, residual add, prompt mean, logits map)
# ---------------------------------------------------------------------------------------------------------------------
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


@pytest.mark.parametrize("B,H,W,C,T,heads,shift", [
    (1, 192, 384, 128, 2, 4, 6),     # Swin-B stage 1 map: 512 windows
    (2, 24, 48, 1024, 2, 32, 6),     # Swin-B stage 4 map: 8 windows
    (2, 25, 49, 97, 3, 3, 6),        # padded to 36 x 60: 15 windows (not a multiple of 4), odd C, C % 64 != 0
    (2, 25, 49, 97, 3, 3, 0),
])
def test_window_gather_scatter(ops, cuda_dev, B, H, W, C, T, heads, shift):
    _gather_scatter_case(ops, cuda_dev, B=B, H=H, W=W, C=C, T=T, heads=heads, ws=12, shift=shift)


def _gather_scatter_case(ops, dev, *, B, H, W, C, T, heads, ws, shift, ns=2, lasts=(False, True)):
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
    sw = nan_split(ops, rows, C, dev, ns=ns)
    ops.swin_window_gather(xn, pn, sw, B=B, H=H, W=W, Cdim=C, T=T, ws=ws, shift=shift)
    torch.cuda.synchronize()
    win = _windows(xn.reshape(B, H, W, C), ws, shift)
    pr = pn.reshape(B, 1, T, C).expand(B, nW, T, C).reshape(B * nW, T, C)
    assert_split_of(sw, torch.cat([pr, win], 1).reshape(rows, C), "window gather")   # the T prompts first in every window
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
        lg = torch.full((B, heads, T, T + H * W), NAN, device=dev)
        ops.swin_window_scatter(o, raw, xa, x, p, lg, B=B, H=H, W=W, Cdim=C, T=T, ws=ws, shift=shift, heads=heads,
                                last=last)
        torch.cuda.synchronize()
        assert torch.equal(xa, xa_ref) and torch.isnan(pad_cols(xa)).all()
        assert torch.equal(x, x0 + xa_ref) and (pad_cols(x) == 7.0).all()
        assert torch.equal(lg[..., T:], lg_ref), "logits map"
        assert torch.isnan(lg[..., :T]).all(), "logits columns [0, T) written"
        assert (pad_cols(p) == 7.0).all()
        if last:
            assert torch.equal(p, p0), "the last block leaves the prompts alone"
        else:
            # 4 window groups of ceil(nW / 4) sequential fp32 adds, the 4-way sum, the division and the += of p
            want = p0.double() + pm.mean(1).reshape(B * T, C)
            bound = U * ((-(-nW // 4) + 4) * pm.abs().mean(1).reshape(B * T, C) + p0.double().abs() + want.abs())
            assert_bounded(p.double(), want, bound, 1, "prompt mean")
            ratio = max(ratio, float(((p.double() - want).abs() / bound).max()))
    return ratio


# ---------------------------------------------------------------------------------------------------------------------
# channel attention: transpose_split -> chan_kv (split-K GEMM) -> swin_chan_attention
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,L,C", [(1, 73728, 128), (2, 1001, 45)])
def test_transpose_split(ops, cuda_dev, B, L, C):
    """[B, L, C] fp32 -> split [B*C, L], bit-exact: Swin-B stage 1 (L = 192 * 384) and ragged L and C (tiles of 64 x 32
    cut on both axes, odd L: the last column is written alone)."""
    x = padded(B * L, C, cuda_dev)
    x.copy_(torch.randn(B * L, C, device=cuda_dev, generator=torch.Generator(device=cuda_dev).manual_seed(L)))
    out = nan_split(ops, B * C, L, cuda_dev)
    ops.transpose_split(x, out, B=B, L=L, Cdim=C)
    torch.cuda.synchronize()
    hi, lo = split_exact(x.reshape(B, L, C).transpose(1, 2).reshape(B * C, L))
    assert torch.equal(out.buf[0, :B * C, :L], hi) and torch.equal(out.buf[1, :B * C, :L], lo)
    assert_untouched(out, B * C, L)


@pytest.mark.parametrize("stage", range(4))
def test_chan_kv_splitk_swinB(ops, cuda_dev, stage):
    """chan_kv at Swin-B: M = C rows, N = 2 * 256, K = L = H * W, in the number of K chunks the plan chooses
    (taskprompter_swin.chan_kv_chunks), against float64 of the decoded split operands."""
    from mtt_b200 import taskprompter_swin as TS

    H, W, C, _ = SWINB[stage]
    K, N, dev = H * W, 512, cuda_dev
    chunks = TS.chan_kv_chunks(C, 256, K)
    g = torch.Generator(device=dev).manual_seed(stage)
    a, A = split_in(ops, torch.randn(C, K, device=dev, generator=g))
    w = ops.pack_weight(torch.randn(N, K, device=dev, generator=g) * K ** -0.5, 2)
    bias = torch.randn(N, device=dev, generator=g)
    part = torch.full((chunks, C, N), NAN, device=dev)
    out = padded(C, N, dev)
    ops.gemm_splitk(a, w, part, out, K=K, bias=bias, chunks=chunks)
    torch.cuda.synchronize()
    want = A @ decode(w, N, K).t() + bias.double()
    assert torch.isfinite(out).all() and torch.isnan(pad_cols(out)).all()
    # Per output row, relative to that row's max |ref| (unit-scale rows: the bias is as large as the product). The split
    # GEMM drops lo * lo (<= 2^-18 |a w| per product, random signs: ~2^-18 of the row's rms), and accumulates K / chunks
    # products per chunk in fp32 before the fixed-order sum of the chunks (random walk: ~2^-24 sqrt(K / chunks) = 3e-6 of
    # the rms at 2304 products). Observed errors are a few 1e-6 of the row max; 3e-5 leaves a margin of about 10.
    err = ((out.double() - want).abs().amax(1) / want.abs().amax(1)).max().item()
    assert err < 3e-5, (stage, chunks, err)


@pytest.mark.parametrize("B,T,C,nh", [
    (1, 2, 128, 1), (1, 2, 256, 1), (1, 2, 512, 1), (1, 2, 1024, 1),   # Swin-B: ce 256, one channel window (8 y blocks)
    (2, 3, 256, 2),                                                      # 2 x 2 windows of 8 x 8: 2 y blocks
    (2, 3, 1003, 4),                                                     # 4 x 4 windows of 4 x 4; C % 8 != 0
])
def test_chan_attention(ops, cuda_dev, B, T, C, nh):
    _chan_attention_case(ops, cuda_dev, B=B, T=T, C=C, nh=nh)


def _chan_attention_case(ops, dev, *, B, T, C, nh, ns=2):
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
    cs = nan_split(ops, B * T, ce, dev, ns=ns)
    rc_buf = torch.full((B * T * C * G + 16,), NAN, device=dev)
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
    got_rc = rc.double().permute(0, 3, 4, 1, 2).reshape(B, G, T, C)
    got_co = grid(co.double().reshape(B, T, ce))
    assert_bounded(got_rc, raw, rb, 3, "raw_chan")
    assert_bounded(got_co, out, bound, 3, "chan_out")
    assert torch.isnan(pad_cols(co)).all() and torch.isnan(rc_buf[rc.numel():]).all()
    assert_split_of(cs, co.contiguous(), "chan_out split")                  # the split output is the split of chan_out
    assert_untouched(cs, B * T, ce)
    return [float(((got_rc - raw).abs() / rb).max()), float(((got_co - out).abs() / bound).max())]


# ---------------------------------------------------------------------------------------------------------------------
# PatchMerging helpers
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("stage", range(3))
def test_merge_gather(ops, cuda_dev, stage):
    """2 x 2 merge in the order (0,0), (1,0), (0,1), (1,1) (TP:441-444), exact, two images, ldo > 4C."""
    H, W, C, _ = SWINB[stage]
    B = 2
    x = padded(B * H * W, C, cuda_dev)
    x.copy_(torch.randn(B * H * W, C, device=cuda_dev, generator=torch.Generator(device=cuda_dev).manual_seed(stage)))
    out = padded(B * H * W // 4, 4 * C, cuda_dev, pad=5)
    ops.swin_merge_gather(x, out, B=B, H=H, W=W, Cdim=C)
    torch.cuda.synchronize()
    m = x.reshape(B, H, W, C)
    want = torch.cat([m[:, 0::2, 0::2], m[:, 1::2, 0::2], m[:, 0::2, 1::2], m[:, 1::2, 1::2]], -1)
    assert torch.equal(out, want.reshape(B * H * W // 4, 4 * C))
    assert torch.isnan(pad_cols(out)).all()


@pytest.mark.parametrize("stage", range(3))
def test_conv3x3_s2_maps(ops, cuda_dev, stage):
    """spa_attn_ds (TP:458-460) at the three Swin-B merges: Cin = Cout = heads * T = 8 / 16 / 32 over the full-size
    logit maps stored behind T prompt columns; columns before out_offset stay untouched."""
    H, W, _, heads = SWINB[stage]
    _conv3x3_s2_case(ops, cuda_dev, B=1, T=2, H=H, W=W, Cin=heads * 2, seed=stage)


def _conv3x3_s2_case(ops, dev, *, B, T, H, W, Cin, seed):
    """conv3x3_s2_maps over [B, Cin, T + H*W] logit maps (the T prompt columns first) into [B, Cin, T + H*W/4]:
    within 9 Cin + 2 FMAs of the absolute conv, the T prefix columns untouched. Returns the worst err / bound."""
    L = H * W
    g = torch.Generator(device=dev).manual_seed(seed)
    x = torch.randn(B, Cin, T + L, device=dev, generator=g)
    w = torch.randn(Cin, Cin, 3, 3, device=dev, generator=g) * 0.2
    b = torch.randn(Cin, device=dev, generator=g)
    out = torch.full((B, Cin, T + L // 4), NAN, device=dev)
    ops.conv3x3_s2_maps(x, w, b, out, B=B, Cin=Cin, H=H, W=W, in_stride=T + L, in_offset=T, out_stride=T + L // 4,
                        out_offset=T)
    torch.cuda.synchronize()
    xm = x[..., T:].double().reshape(B, Cin, H, W)
    want = F.conv2d(xm, w.double(), b.double(), stride=2, padding=1)
    absum = F.conv2d(xm.abs(), w.double().abs(), b.double().abs(), stride=2, padding=1)
    got = out[..., T:].double().reshape(want.shape)
    bound = U * (9 * Cin + 2) * absum
    assert_bounded(got, want, bound, 2, f"conv3x3_s2 B={B} Cin={Cin} {H}x{W}")   # 9 Cin FMAs after the bias
    assert torch.isnan(out[..., :T]).all()
    return float(((got - want).abs() / bound).max())


@pytest.mark.parametrize("nwin", [1, 4])
def test_chan_up(ops, cuda_dev, nwin):
    """process_chan_attn (TP:463-466) at the last merge: C 1024 -> 2048 over the channel axis of raw_chan."""
    _chan_up_case(ops, cuda_dev, BT=2, C=1024, nwin=nwin, seed=nwin)


def _chan_up_case(ops, dev, *, BT, C, nwin, seed):
    """swin_chan_up C -> 2C over the channel axis of raw_chan [BT, C, nwin]; nothing past the output written. Returns
    the worst err / bound."""
    Cout = 2 * C
    g = torch.Generator(device=dev).manual_seed(seed)
    rc = torch.randn(BT, C, nwin, device=dev, generator=g)
    w = torch.randn(Cout, C, device=dev, generator=g) * 0.05
    buf = torch.full((BT * Cout * nwin + 16,), NAN, device=dev)
    out = buf[:BT * Cout * nwin].view(BT, Cout, nwin)
    ops.swin_chan_up(rc, w, out, BT=BT, Cdim=C, nwin=nwin)
    torch.cuda.synchronize()
    want = w.double() @ rc.double()
    bound = U * (C + 1) * (w.double().abs() @ rc.double().abs())
    assert_bounded(out.double(), want, bound, 1, f"chan_up BT={BT} C={C}")
    assert torch.isnan(buf[out.numel():]).all()
    return float(((out.double() - want).abs() / bound).max())
