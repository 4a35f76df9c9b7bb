"""-m gpu: every HBM-bound "glue" kernel and every composite operator of the C ABI against its plain-torch
restatement (tests/emul_ops.py -- the same functions the CPU tests use to stand in for the kernels), on random
inputs at shapes with ragged edges. The wgmma GEMM / conv / attention kernels have their own file
(test_kernels_gpu.py); this one covers gate_split, ctr_weights, ctr_mix, bilinear (all output forms, row offsets,
accumulate), bilinear_postproc (all kinds), zero_insert, dwconv3x3_s2, avgpool (ceil mode), InvPT's cross-task attention
(grouped GEMMs + fuse / softmax kernel, with and without cross-scale fusion), split_rows, layernorm_seg, the packing entry points (BatchNorm folding, transposed
kernels), the NCHW <-> NHWC layout kernels, the strided row scatter of mtt_gemm and the named block operators
(ln_qkv, proj_residual, ln_mlp_residual, gated_conv1x1, conv3x3_bn_act).

Tolerance: split outputs carry 16 significant bits (2^-17 relative), fp32 outputs differ by summation order only.
"""
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]


class _Emu:
    """emu[name](...) runs the torch restatement `name` of tests/emul_ops.py: the emulation is installed over
    mtt_b200.ops only for the duration of the call (the restatements of the composite operators call the primitive
    restatements through the ops module), the real wrappers are back afterwards."""

    def __getitem__(self, name):
        import emul_ops
        from mtt_b200 import ops

        def call(*a, **k):
            mp = pytest.MonkeyPatch()
            emul_ops.install(mp)
            try:
                return getattr(ops, name)(*a, **k)
            finally:
                mp.undo()
        return call


@pytest.fixture(scope="module")
def both(cuda_dev):
    """(ops = the real library wrappers, emu[name] = torch restatement of ops.name on CPU tensors)."""
    import mtt_b200  # noqa: F401
    from mtt_b200 import ops
    return ops, _Emu()


def relerr(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).abs().max() / b.abs().max().clamp_min(1e-30)).item()


def cpu_split(ops, sp):
    """CPU twin of a device Split (same shape / ld), zero-filled."""
    c = ops.Split(sp.rows, sp.cols, "cpu", sp.nsplit, ld=sp.ld, zero=True)
    return c


def rnd(*shape, dev, scale=1.0):
    return torch.randn(*shape, device=dev) * scale


def test_gate_split(both, cuda_dev):
    """All tasks in one launch (X read once) against the per-task restatement; 1x1 and 2x2 channel windows."""
    ops, emu = both
    torch.manual_seed(1)
    for (B, T, H, dh, gh, gw, nh) in [(2, 3, 2, 64, 4, 6, 2), (1, 5, 4, 32, 8, 8, 1)]:
        C, P = H * dh, gh * gw
        N = T + P
        x = rnd(B * N, C, dev=cuda_dev)
        lg = rnd(B, H, T, N, dev=cuda_dev)
        rc = rnd(B, T, C, nh, nh, dev=cuda_dev)
        ys = [ops.Split(B * P, C, cuda_dev) for _ in range(T)]
        yc = [ops.Split(B * P, C, cuda_dev) for _ in range(T)]
        big = torch.zeros(T, 2, 2, B * P, C, dtype=torch.bfloat16, device=cuda_dev)      # [task][ys|yc][plane]
        y0, c0 = ops.Split.from_planes(big[0, 0], C), ops.Split.from_planes(big[0, 1], C)
        ops.gate_split(x, N, T, lg, rc, 0, y0, c0, B=B, T=T, N=N, H=H, Cdim=C, gh=gh, gw=gw, nh=nh, nw=nh, ntasks=T,
                       task_stride=big.stride(0))
        torch.cuda.synchronize()
        for task in range(T):
            eys, eyc = cpu_split(ops, ys[task]), cpu_split(ops, yc[task])
            emu["gate_split"](x.cpu(), N, T, lg.cpu(), rc.cpu(), task, eys, eyc, B=B, T=T, N=N, H=H, Cdim=C, gh=gh, gw=gw,
                              nh=nh, nw=nh)
            got_s = big[task, 0, 0].float() + big[task, 0, 1].float()
            got_c = big[task, 1, 0].float() + big[task, 1, 1].float()
            assert relerr(got_s, eys.float()) < 2e-5 and relerr(got_c, eyc.float()) < 2e-5


def test_gemm_splitk(both, cuda_dev):
    """Skinny M with a long K (Swin chan_kv): K chunks as one grouped launch + fixed-order reduction == one GEMM."""
    ops, emu = both
    torch.manual_seed(13)
    for (M, N, K, chunks) in [(96, 64, 4608, 9), (256, 96, 2304, 4), (64, 40, 1000, 3)]:   # last: unequal chunks
        a, w = ops.split_f32(rnd(M, K, dev=cuda_dev)), ops.pack_weight(rnd(N, K, dev=cuda_dev, scale=0.05), 2)
        bias = rnd(N, dev=cuda_dev)
        ref = torch.zeros(M, N, device=cuda_dev)
        ops.gemm(a, w, bias=bias, out_f32=ref)
        part, out = torch.zeros(chunks, M, N, device=cuda_dev), torch.zeros(M, N, device=cuda_dev)
        ops.gemm_splitk(a, w, part, out, K=K, bias=bias, chunks=chunks)
        torch.cuda.synchronize()
        assert relerr(out, ref) < 3e-5          # same products, different fp32 summation order
        want = a.float().double() @ w.float()[:, :K].double().t() + bias.double()
        assert relerr(out, want) < 2e-5


@pytest.mark.parametrize("variant", [1, 2], ids=["bn128", "bn256"])
def test_gemm_grouped_equals_separate_launches(both, cuda_dev, variant):
    """mtt_gemm_grouped == the same problems launched one by one on the same kernel variant, bit for bit (linear and
    3x3 conv, ragged N: the last N tile is partial), and both agree with float64."""
    ops, emu = both
    ops.set_gemm_variant(variant)
    try:
        _grouped_case(ops, cuda_dev)
    finally:
        ops.set_gemm_variant(0)


def _grouped_case(ops, cuda_dev):
    torch.manual_seed(12)
    G, M, N, K = 5, 4 * 96, 300, 200
    A = [ops.split_f32(rnd(M, K, dev=cuda_dev)) for _ in range(G)]
    W = [ops.pack_weight(rnd(N, K, dev=cuda_dev, scale=0.05), 2) for _ in range(G)]
    bias = [rnd(N, dev=cuda_dev) for _ in range(G)]
    res = [rnd(M, 304, dev=cuda_dev) for _ in range(G)]
    o1 = [torch.zeros(M, 304, device=cuda_dev) for _ in range(G)]
    o2 = [torch.zeros(M, 304, device=cuda_dev) for _ in range(G)]
    s1 = [ops.Split(M, 304, cuda_dev, zero=True) for _ in range(G)]
    s2 = [ops.Split(M, 304, cuda_dev, zero=True) for _ in range(G)]
    kw = lambda g, o, sp: dict(N=N, bias=bias[g], act=ops.ACT_GELU, residual=res[g], out_f32=o[g], out_split=sp[g])
    for g in range(G):
        ops.gemm(A[g], W[g], **kw(g, o1, s1))
    ops.gemm_grouped([(A[g], W[g], kw(g, o2, s2)) for g in range(G)])
    torch.cuda.synchronize()
    for g in range(G):
        assert torch.equal(o1[g], o2[g]) and torch.equal(s1[g].buf, s2[g].buf)
        want = torch.nn.functional.gelu(A[g].float().double() @ W[g].float()[:, :K].double().t() + bias[g].double()) \
            + res[g][:, :N].double()
        assert relerr(o2[g][:, :N], want) < 3e-5
    B, H, Wd, Cin, Cout = 2, 8, 12, 70, 44
    X = [ops.split_f32(rnd(B * H * Wd, Cin, dev=cuda_dev)) for _ in range(G)]
    Wc = [ops.pack_conv_weight(rnd(Cout, Cin, 3, 3, dev=cuda_dev, scale=0.05), rnd(Cout, dev=cuda_dev), None, 2) for _ in range(G)]
    c1 = [ops.Split(B * H * Wd, Cout, cuda_dev, zero=True) for _ in range(G)]
    c2 = [ops.Split(B * H * Wd, Cout, cuda_dev, zero=True) for _ in range(G)]
    ckw = lambda g, sp: dict(N=Cout, K=Cin, bias=Wc[g][1], act=ops.ACT_RELU, out_split=sp[g], conv=(B, H, Wd, 3, 1))
    for g in range(G):
        ops.gemm(X[g], Wc[g][0], **ckw(g, c1))
    ops.gemm_grouped([(X[g], Wc[g][0], ckw(g, c2)) for g in range(G)])
    torch.cuda.synchronize()
    for g in range(G):
        assert torch.equal(c1[g].buf, c2[g].buf)
    with pytest.raises(RuntimeError):       # geometry must match
        ops.gemm_grouped([(A[0], W[0], dict(N=N, out_f32=o1[0])), (A[1], W[1], dict(N=N - 8, out_f32=o1[1]))])


def test_ctr_weights_and_mix(both, cuda_dev):
    ops, emu = both
    torch.manual_seed(2)
    B, H, T, P, f = 3, 4, 5, 24, 28
    N = T + P
    lg = rnd(B, H, T, N, dev=cuda_dev)
    w0, b0, w2, b2 = rnd(T, H, H, dev=cuda_dev), rnd(T, H, dev=cuda_dev), rnd(T, H, dev=cuda_dev), rnd(T, dev=cuda_dev)
    out = torch.empty(B, T, T, device=cuda_dev)
    ops.ctr_weights(lg, w0, b0, w2, b2, out, B=B, H=H, T=T, N=N)
    ref = torch.empty(B, T, T)
    emu["ctr_weights"](lg.cpu(), w0.cpu(), b0.cpu(), w2.cpu(), b2.cpu(), ref, B=B, H=H, T=T, N=N)
    torch.cuda.synchronize()
    assert relerr(out, ref) < 1e-5
    ld = ops.round_up(f, 8)
    Fm = rnd(T, B * P, ld, dev=cuda_dev)
    for accumulate in (False, True):
        acc = rnd(T, B * P, ld, dev=cuda_dev)
        racc = acc.cpu().clone()
        ops.ctr_mix(Fm, out, acc, T=T, M=B * P, Cdim=ld, ld=ld, rows_per_batch=P, accumulate=accumulate)
        emu["ctr_mix"](Fm.cpu(), ref, racc, T=T, M=B * P, Cdim=ld, ld=ld, rows_per_batch=P, accumulate=accumulate)
        torch.cuda.synchronize()
        assert relerr(acc, racc) < 1e-5


@pytest.mark.parametrize("h,w,H2,W2", [(4, 6, 16, 24), (8, 8, 5, 11), (6, 10, 6, 10), (3, 5, 12, 7)])
def test_bilinear_forms(both, cuda_dev, h, w, H2, W2):
    ops, emu = both
    torch.manual_seed(3)
    B, C, T = 2, 20, 3
    x = rnd(B * T * h * w, C + 4, dev=cuda_dev)          # strided rows (ld > C), T task slices per image
    k = 1
    kw = dict(in_batch_rows=T * h * w, in_row_offset=k * h * w)
    o32 = torch.zeros(B * H2 * W2, C + 4, device=cuda_dev)
    osp = ops.Split(B * H2 * W2, C, cuda_dev)
    onc = torch.zeros(B, C, H2, W2, device=cuda_dev)
    ops.bilinear(x, x.stride(0), B, h, w, C, H2, W2, out_f32=o32, out_split=osp, out_nchw=onc, **kw)
    r32, rsp, rnc = torch.zeros(B * H2 * W2, C + 4), cpu_split(ops, osp), torch.zeros(B, C, H2, W2)
    emu["bilinear"](x.cpu(), x.stride(0), B, h, w, C, H2, W2, out_f32=r32, out_split=rsp, out_nchw=rnc, **kw)
    torch.cuda.synchronize()
    assert relerr(o32, r32) < 1e-5 and relerr(onc, rnc) < 1e-5 and relerr(osp.float(), rsp.float()) < 2e-5
    # accumulate into a task slice of a joint token buffer
    acc = rnd(B * T * H2 * W2, C, dev=cuda_dev)
    racc = acc.cpu().clone()
    kw2 = dict(kw, accumulate=True, out_batch_rows=T * H2 * W2, out_row_offset=2 * H2 * W2)
    ops.bilinear(x, x.stride(0), B, h, w, C, H2, W2, out_f32=acc, **kw2)
    emu["bilinear"](x.cpu(), x.stride(0), B, h, w, C, H2, W2, out_f32=racc, **kw2)
    torch.cuda.synchronize()
    assert relerr(acc, racc) < 1e-5


@pytest.mark.parametrize("h,w,H2,W2,C,pad", [(32, 32, 128, 128, 350, 2), (9, 7, 18, 37, 21, 0), (16, 24, 40, 50, 130, 3),
                                             (20, 33, 10, 17, 66, 0)])
def test_bilinear_runs(both, cuda_dev, h, w, H2, W2, C, pad):
    """The NHWC form walks runs of 16 output pixels per warp with the corner columns kept in registers: several 64-channel
    chunks (C = 350: the last one partial), odd C (a single-channel lane), odd row strides (scalar loads), rows that are
    not a multiple of the run length, x2 / x4 / fractional up-sampling and down-sampling."""
    ops, emu = both
    torch.manual_seed(5)
    B = 2
    x = rnd(B * h * w, C + pad, dev=cuda_dev)
    o32 = torch.zeros(B * H2 * W2, C + 1, device=cuda_dev)
    osp = ops.Split(B * H2 * W2, C, cuda_dev, zero=True)
    ops.bilinear(x, x.stride(0), B, h, w, C, H2, W2, out_f32=o32, out_split=osp)
    r32, rsp = torch.zeros(B * H2 * W2, C + 1), cpu_split(ops, osp)
    emu["bilinear"](x.cpu(), x.stride(0), B, h, w, C, H2, W2, out_f32=r32, out_split=rsp)
    torch.cuda.synchronize()
    ref = F.interpolate(x[:, :C].reshape(B, h, w, C).permute(0, 3, 1, 2).double().cpu(), size=(H2, W2), mode="bilinear",
                        align_corners=False).permute(0, 2, 3, 1).reshape(B * H2 * W2, C)
    assert relerr(o32[:, :C], ref) < 1e-5 and (o32[:, C:] == 0).all()
    assert relerr(o32, r32) < 1e-5 and relerr(osp.float(), rsp.float()) < 2e-5


@pytest.mark.parametrize("kind,C", [(0, 7), (1, 1), (2, 2), (3, 3), (4, 1)])
def test_bilinear_postproc(both, cuda_dev, kind, C):
    ops, emu = both
    torch.manual_seed(4)
    B, h, w, H2, W2 = 2, 6, 9, 24, 36
    ld = ops.round_up(C, 4)
    x = rnd(B * h * w, ld, dev=cuda_dev, scale=2.0)
    shape = {0: (B, H2, W2), 1: (B, H2, W2), 2: (B, H2, W2), 3: (B, H2, W2, 3), 4: (B, H2, W2, 1)}[kind]
    dt = torch.int64 if kind == 0 else torch.float32
    out = torch.zeros(shape, device=cuda_dev, dtype=dt)
    ref = torch.zeros(shape, dtype=dt)
    ops.bilinear_postproc(x, ld, B, h, w, C, H2, W2, kind, out)
    emu["bilinear_postproc"](x.cpu(), ld, B, h, w, C, H2, W2, kind, ref)
    torch.cuda.synchronize()
    if kind == 0:
        assert (out.cpu() == ref).float().mean().item() > 0.999      # near ties may flip with the summation order
    else:
        assert relerr(out, ref) < 2e-5


def test_zero_insert_dwconv_avgpool_split_rows(both, cuda_dev):
    ops, emu = both
    torch.manual_seed(5)
    B, T, h, w, C = 2, 3, 6, 10, 40
    N = 1 + h * w
    x = rnd(B * N, C, dev=cuda_dev)
    zi, rz = ops.Split(B * 4 * h * w, C, cuda_dev), None
    ops.zero_insert(x, zi, B=B, h=h, w=w, Cdim=C, src_group=N, src_offset=1)
    rz = cpu_split(ops, zi)
    emu["zero_insert"](x.cpu(), rz, B=B, h=h, w=w, Cdim=C, src_group=N, src_offset=1)
    sr, rsr = ops.Split(B * h * w, C, cuda_dev), None
    ops.split_rows(x, sr, rows=B * h * w, cols=C, in_group=h * w, src_group=N, src_offset=1)
    rsr = cpu_split(ops, sr)
    emu["split_rows"](x.cpu(), rsr, rows=B * h * w, cols=C, in_group=h * w, src_group=N, src_offset=1)
    torch.cuda.synchronize()
    assert relerr(zi.float(), rz.float()) < 2e-5 and relerr(sr.float(), rsr.float()) < 2e-5
    xt = rnd(B * T * h * w, C, dev=cuda_dev)
    wq, bq = rnd(T, C, 9, dev=cuda_dev, scale=0.3), rnd(T, C, dev=cuda_dev)
    q = ops.Split(B * T * (h // 2) * (w // 2), C, cuda_dev)
    ops.dwconv3x3_s2(xt, wq, bq, q, B=B, T=T, h=h, w=w, Cdim=C)
    rq = cpu_split(ops, q)
    emu["dwconv3x3_s2"](xt.cpu(), wq.cpu(), bq.cpu(), rq, B=B, T=T, h=h, w=w, Cdim=C)
    torch.cuda.synchronize()
    assert relerr(q.float(), rq.float()) < 2e-5
    for s in (2, 4, 8):                                    # 6x10 with stride 4 / 8: ceil_mode partial windows
        kh, kw_ = -(-h // s), -(-w // s)
        kv = ops.Split(B * T * kh * kw_, C, cuda_dev)
        ops.avgpool(xt, kv, BT=B * T, h=h, w=w, Cdim=C, s=s)
        rkv = cpu_split(ops, kv)
        emu["avgpool"](xt.cpu(), rkv, BT=B * T, h=h, w=w, Cdim=C, s=s)
        torch.cuda.synchronize()
        assert relerr(kv.float(), rkv.float()) < 2e-5, s


def test_layernorm_seg(both, cuda_dev):
    ops, emu = both
    torch.manual_seed(6)
    B, T, hw, C = 2, 3, 12, 48
    x = rnd(B * T * hw, C, dev=cuda_dev)
    g, b = rnd(T * C, dev=cuda_dev), rnd(T * C, dev=cuda_dev)
    o32 = torch.zeros(T * B * hw, C, device=cuda_dev)
    osp = ops.Split(T * B * hw, C, cuda_dev)
    kw = dict(rows=B * hw, cols=C, S=T, in_group=hw, src_group=T * hw, seg_stride=hw, out_seg_stride=B * hw)
    ops.layernorm_seg(x, g, b, 1e-5, out_f32=o32, out_split=osp, **kw)
    r32, rsp = torch.zeros(T * B * hw, C), cpu_split(ops, osp)
    emu["layernorm_seg"](x.cpu(), g.cpu(), b.cpu(), 1e-5, out_f32=r32, out_split=rsp, **kw)
    torch.cuda.synchronize()
    assert relerr(o32, r32) < 1e-5 and relerr(osp.float(), rsp.float()) < 2e-5


@pytest.mark.parametrize("fused", [False, True])
def test_invpt_attention_as_two_grouped_gemms(both, cuda_dev, fused):
    """InvPT cross-task attention (invpt.py:204-236) the way the plan runs it: S = Q_h K_h^T as a grouped launch over
    (batch, head), mtt_invpt_fuse_softmax (scale, cross-scale fusion, score export, softmax), O_h = P_h V_h as a second
    grouped launch -- against softmax(fuse(q k^T * scale)) v in float64."""
    ops, emu = both
    import torch.nn.functional as F
    torch.manual_seed(7)
    B, T, qh, qw, C = 2, 3, 4, 6, 48
    Lq, Tk, dh = T * qh * qw, T * 4, C // 2
    q, k, v = rnd(B * Lq, C, dev=cuda_dev), rnd(B * Tk, C, dev=cuda_dev), rnd(B * Tk, C, dev=cuda_dev)
    qs, ks = ops.split_f32(q), ops.split_f32(k)
    vt = ops.Split(B * C, Tk, cuda_dev, zero=True)
    ops.transpose_split(v, vt, B=B, L=Tk, Cdim=C)
    score = torch.zeros(B, 2, Lq, Tk, device=cuda_dev)
    ops.gemm_grouped([(qs, ks, dict(M=Lq, N=Tk, K=dh, a_row_offset=b * Lq, a_col_offset=h * dh, w_row_offset=b * Tk,
                                    w_col_offset=h * dh, out_f32=score[b, h])) for b in range(B) for h in range(2)])
    kw = {}
    if fused:
        kw = dict(prev_score=rnd(B, 2, T * (qh // 2) * (qw // 2), Tk, dev=cuda_dev), T=T, qh=qh, qw=qw,
                  fuse_w=rnd(2, 4, dev=cuda_dev), fuse_b=rnd(2, dev=cuda_dev))
    P = ops.Split(B * 2 * Lq, Tk, cuda_dev, zero=True)
    raw = score.clone()
    ops.invpt_fuse_softmax(score, P, B=B, Lq=Lq, Tk=Tk, scale=C ** -0.5, score_out=score, **kw)      # in place
    out = ops.Split(B * Lq, C, cuda_dev)
    ops.gemm_grouped([(P, vt, dict(M=Lq, N=dh, K=Tk, a_row_offset=(b * 2 + h) * Lq, w_row_offset=b * C + h * dh,
                                   out_split=out, out_row_offset=b * Lq, out_col_offset=h * dh))
                      for b in range(B) for h in range(2)])
    torch.cuda.synchronize()
    # the fuse / softmax kernel against its restatement on the same raw scores
    rP, rsc = cpu_split(ops, P), torch.zeros(B, 2, Lq, Tk)
    ckw = {n: (t.cpu() if torch.is_tensor(t) else t) for n, t in kw.items()}
    emu["invpt_fuse_softmax"](raw.cpu(), rP, B=B, Lq=Lq, Tk=Tk, scale=C ** -0.5, score_out=rsc, **ckw)
    assert relerr(score, rsc) < 2e-5 and relerr(P.float(), rP.float()) < 3e-5
    # the whole chain against float64
    sp = lambda t, L: t.double().cpu().reshape(B, L, 2, dh).transpose(1, 2)
    sref = (sp(q, Lq) @ sp(k, Tk).transpose(-2, -1)) * C ** -0.5
    if fused:
        sh, sw = qh // 2, qw // 2
        ups = []
        for i in range(T):
            s_ = ckw["prev_score"].double()[:, :, sh * sw * i: sh * sw * (i + 1), :].permute(0, 1, 3, 2).reshape(B * 2, Tk, sh, sw)
            ups.append(F.interpolate(s_, scale_factor=2, mode="bilinear", align_corners=False)
                       .reshape(B, 2, Tk, -1).permute(0, 1, 3, 2))
        sref = F.conv2d(torch.cat([sref, torch.cat(ups, dim=2)], dim=1), ckw["fuse_w"].double().reshape(2, 4, 1, 1),
                        ckw["fuse_b"].double())
    oref = (sref.softmax(-1) @ sp(v, Tk)).transpose(1, 2).reshape(B * Lq, C)
    assert relerr(score, sref) < 3e-5 and relerr(out.float(), oref) < 5e-5


def test_pack_conv_weight_folds_batchnorm(both, cuda_dev):
    """mtt_pack_conv_weight against the fold in plain torch, for Conv2d + BN, bare Conv2d, and ConvTranspose2d."""
    ops, emu = both
    torch.manual_seed(8)
    bn = nn.BatchNorm2d(24).to(cuda_dev).eval()
    with torch.no_grad():
        bn.weight.normal_(1, 0.2), bn.bias.normal_(), bn.running_mean.normal_(), bn.running_var.uniform_(0.5, 2)
    cases = [(rnd(24, 70, 3, 3, dev=cuda_dev), rnd(24, dev=cuda_dev), bn, False),
             (rnd(24, 70, 3, 3, dev=cuda_dev), None, bn, False),
             (rnd(24, 64, 1, 1, dev=cuda_dev), rnd(24, dev=cuda_dev), None, False),
             (rnd(70, 24, 3, 3, dev=cuda_dev), rnd(24, dev=cuda_dev), None, True),
             (rnd(70, 24, 1, 1, dev=cuda_dev), rnd(24, dev=cuda_dev), bn, True)]
    for w, b, n, tr in cases:
        got, gb = ops.pack_conv_weight(w, b, n, 2, transposed=tr)
        ref, rb = emu["pack_conv_weight"](w.cpu(), None if b is None else b.cpu(), None if n is None else n.cpu(), 2,
                                         transposed=tr)
        if n is not None:
            n.to(cuda_dev)
        torch.cuda.synchronize()
        assert got.rows == ref.rows and got.ld == ref.ld
        assert relerr(got.float(), ref.float()) < 2e-5 and relerr(gb, rb) < 1e-5


def test_layout_kernels_and_strided_scatter(both, cuda_dev):
    ops, emu = both
    torch.manual_seed(9)
    B, C, H, W = 2, 37, 5, 9
    x = rnd(B, C, H, W, dev=cuda_dev)
    sp = ops.Split(B * H * W, C + 11, cuda_dev, zero=True)
    ops.nchw_to_nhwc_split(x, sp, col_offset=8)
    torch.cuda.synchronize()
    want = x.permute(0, 2, 3, 1).reshape(B * H * W, C)
    assert relerr(sp.float()[:, 8:8 + C], want) < 2e-5 and sp.float()[:, :8].abs().max() == 0
    y = rnd(B * H * W, C + 3, dev=cuda_dev)
    out = torch.zeros(B, C, H, W, device=cuda_dev)
    ops.nhwc_to_nchw(y, y.stride(0), B, C, H, W, out)
    torch.cuda.synchronize()
    assert torch.equal(out, y[:, :C].reshape(B, H, W, C).permute(0, 3, 1, 2))
    # ConvTranspose2d(k2, s2) as four GEMMs with a strided row scatter (DEConvHead, taskprompter.py:704)
    Cin, Cout = 40, 24
    ct = nn.ConvTranspose2d(Cin, Cout, 2, stride=2).to(cuda_dev)
    xin = rnd(B, Cin, H, W, dev=cuda_dev)
    a = ops.Split(B * H * W, Cin, cuda_dev)
    ops.nchw_to_nhwc_split(xin, a)
    o = ops.Split(B * 4 * H * W, Cout, cuda_dev, zero=True)
    for dy in range(2):
        for dx in range(2):
            wp, bp = ops.pack_conv_weight(ct.weight.detach()[:, :, dy, dx].contiguous().reshape(Cin, Cout, 1, 1),
                                          ct.bias.detach(), None, 2, transposed=True)
            ops.gemm(a, wp, N=Cout, K=Cin, bias=bp, out_split=o, regroup=(W, 4 * W, 2 * W * dy + dx, 2))
    torch.cuda.synchronize()
    ref = ct(xin).permute(0, 2, 3, 1).reshape(-1, Cout)
    assert relerr(o.float(), ref) < 3e-5


def test_named_block_operators(both, cuda_dev):
    """ln_qkv / proj_residual / ln_mlp_residual / gated_conv1x1 / conv3x3_bn_act: the C launch sequences against the
    same sequences of torch restatements (identical workspace layout)."""
    ops, emu = both
    import mtt_b200.lib as L
    torch.manual_seed(10)
    B, T, H, dh, gh, gw, e = 2, 3, 2, 64, 4, 6, 20
    C, P, hid = H * dh, gh * gw, 4 * H * dh
    N = T + P
    rows = B * N
    dev = cuda_dev

    def twin(sp):
        c = cpu_split(ops, sp)
        c.buf.copy_(sp.buf.cpu())
        return c

    x = rnd(rows, C, dev=dev)
    g, b = rnd(C, dev=dev) * 0.1 + 1, rnd(C, dev=dev) * 0.1
    wqkv, bqkv = ops.pack_weight(rnd(3 * C, C, dev=dev, scale=0.05), 2), rnd(3 * C, dev=dev)
    ws = ops.workspace(ops.workspace_bytes(L.OP_LN_QKV, rows=rows, Cdim=C, nsplit=2), dev)
    qkv = ops.Split(rows, 3 * C, dev)
    ops.ln_qkv(x, g, b, 1e-6, wqkv, bqkv, qkv, ws)
    rws, rqkv = torch.zeros(ws.numel(), dtype=torch.uint8), cpu_split(ops, qkv)
    emu["ln_qkv"](x.cpu(), g.cpu(), b.cpu(), 1e-6, twin(wqkv), bqkv.cpu(), rqkv, rws)
    torch.cuda.synchronize()
    assert relerr(qkv.float(), rqkv.float()) < 3e-5
    assert relerr(ops.ws_split_view(ws, 0, rows, C, 2).float(), ops.ws_split_view(rws, 0, rows, C, 2).float()) < 2e-5

    ao = ops.split_f32(rnd(rows, C, dev=dev))
    wp, bp = ops.pack_weight(rnd(C, C, dev=dev, scale=0.05), 2), rnd(C, dev=dev)
    x1, rx1 = x.clone(), x.cpu().clone()
    ops.proj_residual(ao, wp, bp, x1)
    emu["proj_residual"](twin(ao), twin(wp), bp.cpu(), rx1)
    torch.cuda.synchronize()
    assert relerr(x1, rx1) < 3e-5

    w1, b1 = ops.pack_weight(rnd(hid, C, dev=dev, scale=0.05), 2), rnd(hid, dev=dev)
    w2, b2 = ops.pack_weight(rnd(C, hid, dev=dev, scale=0.05), 2), rnd(C, dev=dev)
    ws2 = ops.workspace(ops.workspace_bytes(L.OP_LN_MLP_RESIDUAL, rows=rows, Cdim=C, hidden=hid, nsplit=2), dev)
    x2, rx2 = x.clone(), x.cpu().clone()
    ops.ln_mlp_residual(x2, g, b, 1e-6, w1, b1, w2, b2, ws2)
    emu["ln_mlp_residual"](rx2, g.cpu(), b.cpu(), 1e-6, twin(w1), b1.cpu(), twin(w2), b2.cpu(),
                           torch.zeros(ws2.numel(), dtype=torch.uint8))
    torch.cuda.synchronize()
    assert relerr(x2, rx2) < 5e-5

    lg, rc = rnd(B, H, T, N, dev=dev), rnd(B, T, C, 2, 2, dev=dev)
    e_pad = ops.round_up(e, 8)
    tasks, rtasks = [], []
    for _ in range(T):
        wsp, bsp = ops.pack_weight(rnd(e, C, dev=dev, scale=0.05), 2), rnd(e, dev=dev)
        wch, bch = ops.pack_weight(rnd(e, C, dev=dev, scale=0.05), 2), rnd(e, dev=dev)
        cat = ops.Split(B * P, 2 * e_pad, dev, zero=True)
        tasks.append((wsp, bsp, wch, bch, cat))
        rtasks.append((twin(wsp), bsp.cpu(), twin(wch), bch.cpu(), cpu_split(ops, cat)))
    ws3 = ops.workspace(ops.workspace_bytes(L.OP_GATED_CONV1X1, rows=B * P, Cdim=C, nsplit=2, T=T), dev)
    kw = dict(B=B, T=T, N=N, H=H, Cdim=C, gh=gh, gw=gw, nh=2, nw=2)
    ops.gated_conv1x1(x, N, T, lg, rc, tasks, e, e_pad, ws3, **kw)
    emu["gated_conv1x1"](x.cpu(), N, T, lg.cpu(), rc.cpu(), rtasks, e, e_pad, torch.zeros(ws3.numel(), dtype=torch.uint8),
                         **kw)
    torch.cuda.synchronize()
    for tk, rt in zip(tasks, rtasks):
        assert relerr(tk[4].float(), rt[4].float()) < 3e-5

    Cin, Cout, n_out, Hh, Ww = 40, 24, 5, 7, 9
    a = ops.split_f32(rnd(B * Hh * Ww, Cin, dev=dev))
    w3, b3 = ops.pack_conv_weight(rnd(Cout, Cin, 3, 3, dev=dev, scale=0.05), rnd(Cout, dev=dev), None, 2)
    wh, bh = ops.pack_weight(rnd(n_out, Cout, dev=dev, scale=0.1), 2), rnd(n_out, dev=dev)
    out = torch.zeros(B * Hh * Ww, 8, device=dev)
    ws4 = ops.workspace(ops.workspace_bytes(L.OP_CONV3X3_BN_ACT, rows=B * Hh * Ww, hidden=Cout, nsplit=2), dev)
    ops.conv3x3_bn_act(a, w3, b3, Cin, Cout, ops.ACT_GELU, B=B, H=Hh, W=Ww, w_head=wh, b_head=bh, n_out=n_out,
                       out_f32=out[:, :n_out], ws=ws4)                        # hidden map in the workspace
    rout = torch.zeros(B * Hh * Ww, 8)
    emu["conv3x3_bn_act"](twin(a), twin(w3), b3.cpu(), Cin, Cout, ops.ACT_GELU, B=B, H=Hh, W=Ww, w_head=twin(wh),
                          b_head=bh.cpu(), n_out=n_out, out_f32=rout[:, :n_out],
                          ws=torch.zeros(ws4.numel(), dtype=torch.uint8))
    torch.cuda.synchronize()
    assert relerr(out, rout) < 5e-5
