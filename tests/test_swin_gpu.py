"""Swin-backbone TaskPrompter (SURVEY.md 8f N2). CPU: the launch plan with the kernels replaced by tests/emul_ops.py
against the oracle restatement (host logic: window bookkeeping, level wiring, packing). gpu: every Swin kernel against
its torch restatement, and the fused CUDA forward through the C ABI against the golden vectors of the UNMODIFIED
reference (tests/golden/tps_*.pt: shifted, clipped and padded windows, 1x1 and 2x2 channel windows, ConvHead and
DEConvHead) and against the oracle at the reference config's window 12 / shift 6 / 0.75 input scaling (tps_mid).
Tolerances as in test_taskprompter_gpu.py: rel-L2 < 2e-4, max-abs < 1e-3 max|ref|, arg-max exact away from near ties."""
import os

import pytest
import torch

from oracle import configs
from oracle import taskprompter_swin_ref as R

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _model(name, seed, graph=False):
    import mtt_b200  # noqa: F401
    from mtt_b200 import taskprompter_swin as TS

    cfg = configs.taskprompter_swin(name)
    sd = R.init_state_dict(cfg, seed=seed)
    m = TS.build_from_config(cfg, nsplit=2, use_graph=graph).eval()
    missing, unexpected = m.load_state_dict(sd, strict=False)
    assert not unexpected and all("relative_position_index" in k or "attn_mask" in k for k in missing)
    return cfg, sd, m


@pytest.mark.parametrize("name", ["tps_tiny", "tps_tiny4", "tps_mid"])
def test_swin_plan_matches_oracle_emulated(monkeypatch, name):
    import emul_ops

    emul_ops.install(monkeypatch)
    cfg, sd, m = _model(name, 11)
    x = torch.randn(2, 3, *cfg["img_size"], generator=torch.Generator().manual_seed(5))
    with torch.no_grad():
        ref = R.forward(sd, cfg, x)
        got = m.plan(2, torch.device("cpu")).run(x, graph=False)
    for t in cfg["tasks"]:
        assert got[t].shape == ref[t].shape
        assert ((got[t] - ref[t]).norm() / ref[t].norm()).item() < 2e-4, (name, t)


def test_swin_state_dict_matches_reference_names():
    """Parameter names / shapes equal the oracle's (which equal the reference module's, tests/test_oracle.py), the
    derived buffers of the reference (relative_position_index, attn_mask) are present as buffers, and equal its values."""
    for name in ("tps_tiny", "tps_tiny4", "tps_swinB"):
        cfg = configs.taskprompter_swin(name)
        if name == "tps_swinB":
            cfg["img_size"] = (256, 512)         # same module structure, small maps
            cfg["dd_label_map_size"] = (128, 256)
        import mtt_b200  # noqa: F401
        from mtt_b200 import taskprompter_swin as TS
        m = TS.build_from_config(cfg)
        want = R.param_shapes(cfg)
        mine = {k: tuple(v.shape) for k, v in m.state_dict().items()}
        extra = set(mine) - set(want)
        assert set(want) <= set(mine), sorted(set(want) - set(mine))[:5]
        assert all(("relative_position_index" in k or "attn_mask" in k) for k in extra), sorted(extra)[:5]
        assert all(mine[k] == tuple(want[k]) for k in want)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["tps_tiny", "tps_tiny4"])
def test_swin_golden_parity(cuda_dev, name):
    from model_checks import check_parity as _check

    fx = torch.load(os.path.join(GOLD, f"{name}.pt"), weights_only=False)
    cfg, sd, m = _model(fx["cfg"], fx["seed"])
    m = m.cuda()
    with torch.no_grad():
        got = m(fx["x"].cuda())
    torch.cuda.synchronize()
    _check(got, fx["out"], cfg["tasks"], 2e-4, 1e-3)


@pytest.mark.gpu
def test_swin_reference_window_geometry_and_graph_replay(cuda_dev):
    from model_checks import check_parity as _check

    cfg, sd, m = _model("tps_mid", 13, graph=True)
    m = m.cuda()
    x = torch.randn(2, 3, *cfg["img_size"], generator=torch.Generator().manual_seed(6))
    with torch.no_grad():
        ref = R.forward(sd, cfg, x)
        m(x.cuda())
        got = m(x.cuda())                    # pure graph replay
    torch.cuda.synchronize()
    _check(got, ref, cfg["tasks"], 2e-4, 1e-3)


@pytest.mark.gpu
def test_swin_kernels_against_restatements(cuda_dev):
    """Each kernel of swin.cu against tests/emul_ops.py on ragged geometry: 6 x 10 map, window 4 (padded to 8 x 12),
    shift 2, 3 prompts, 2 heads of dim 16; 2 x 2 channel windows."""
    import mtt_b200  # noqa: F401
    from mtt_b200 import ops
    from test_glue_kernels_gpu import _Emu, cpu_split, relerr, rnd

    emu = _Emu()
    dev = cuda_dev
    torch.manual_seed(21)
    B, H, W, C, T, ws, heads = 2, 6, 10, 32, 3, 4, 2
    dh = C // heads
    for shift in (0, 2):
        Hp, Wp = 8, 12
        nW, wl = (Hp // ws) * (Wp // ws), ws * ws
        rows = B * nW * (T + wl)
        xn, pn = rnd(B * H * W, C, dev=dev), rnd(B * T, C, dev=dev)
        sw = ops.Split(rows, C, dev)
        ops.swin_window_gather(xn, pn, sw, B=B, H=H, W=W, Cdim=C, T=T, ws=ws, shift=shift)
        rsw = cpu_split(ops, sw)
        emu["swin_window_gather"](xn.cpu(), pn.cpu(), rsw, B=B, H=H, W=W, Cdim=C, T=T, ws=ws, shift=shift)
        torch.cuda.synchronize()
        assert relerr(sw.float(), rsw.float()) < 2e-5
        qkv = ops.split_f32(rnd(rows, 3 * C, dev=dev))
        biasT = rnd(heads, wl, wl, dev=dev)
        maskT = None
        if shift:
            maskT = torch.where(torch.rand(nW, wl, wl, device=dev) < 0.3, -100.0, 0.0)
            maskT = torch.minimum(maskT, maskT.transpose(1, 2)).contiguous()
        ao, raw = ops.Split(rows, C, dev), torch.zeros(B * nW, heads, T, wl, device=dev)
        ops.swin_window_attention(qkv, ao, raw, biasT, maskT, BW=B * nW, nW=nW, T=T, L=wl, heads=heads, scale=dh ** -0.5)
        rq = cpu_split(ops, qkv)
        rq.buf.copy_(qkv.buf.cpu())
        rao, rraw = cpu_split(ops, ao), torch.zeros(B * nW, heads, T, wl)
        emu["swin_window_attention"](rq, rao, rraw, biasT.cpu(), None if maskT is None else maskT.cpu(), BW=B * nW, nW=nW,
                                     T=T, L=wl, heads=heads, scale=dh ** -0.5)
        torch.cuda.synchronize()
        assert relerr(ao.float(), rao.float()) < 3e-5 and relerr(raw, rraw) < 1e-5
        o32 = rnd(rows, C, dev=dev)
        xa, x, p = torch.zeros(B * H * W, C, device=dev), rnd(B * H * W, C, dev=dev), rnd(B * T, C, dev=dev)
        lg = torch.zeros(B, heads, T, T + H * W, device=dev)
        rxa, rx, rp, rlg = xa.cpu().clone(), x.cpu().clone(), p.cpu().clone(), lg.cpu().clone()
        for last in (False, True):
            ops.swin_window_scatter(o32, raw, xa, x, p, lg, B=B, H=H, W=W, Cdim=C, T=T, ws=ws, shift=shift, heads=heads, last=last)
            emu["swin_window_scatter"](o32.cpu(), rraw, rxa, rx, rp, rlg, B=B, H=H, W=W, Cdim=C, T=T, ws=ws, shift=shift,
                                       heads=heads, last=last)
        torch.cuda.synchronize()
        assert relerr(xa, rxa) < 1e-6 and relerr(x, rx) < 1e-6 and relerr(p, rp) < 1e-5 and relerr(lg, rlg) < 1e-5
    # transpose_split (L not a multiple of 8), channel attention, merge gather, stride-2 conv, channel up-projection
    L = H * W
    xa = rnd(B * L, C, dev=dev)
    xat = ops.Split(B * C, L, dev, zero=True)
    ops.transpose_split(xa, xat, B=B, L=L, Cdim=C)
    rxat = cpu_split(ops, xat)
    emu["transpose_split"](xa.cpu(), rxat, B=B, L=L, Cdim=C)
    torch.cuda.synchronize()
    assert relerr(xat.float(), rxat.float()) < 2e-5
    ce, nh = 16, 2
    q, kv = rnd(B * T, ce, dev=dev), rnd(B * C, 2 * ce, dev=dev)
    co, cos, rc = torch.zeros(B * T, ce, device=dev), ops.Split(B * T, ce, dev), torch.zeros(B, T, C, nh, nh, device=dev)
    ops.swin_chan_attention(q, kv, co, cos, rc, B=B, T=T, Cdim=C, ce=ce, nh=nh, nw=nh)
    rco, rcos, rrc = torch.zeros(B * T, ce), cpu_split(ops, cos), torch.zeros(B, T, C, nh, nh)
    emu["swin_chan_attention"](q.cpu(), kv.cpu(), rco, rcos, rrc, B=B, T=T, Cdim=C, ce=ce, nh=nh, nw=nh)
    torch.cuda.synchronize()
    assert relerr(co, rco) < 2e-5 and relerr(cos.float(), rcos.float()) < 3e-5 and relerr(rc, rrc) < 1e-5
    x = rnd(B * H * W, C, dev=dev)
    m32 = torch.zeros(B * L // 4, 4 * C, device=dev)
    ops.swin_merge_gather(x, m32, B=B, H=H, W=W, Cdim=C)
    rm = torch.zeros(B * L // 4, 4 * C)
    emu["swin_merge_gather"](x.cpu(), rm, B=B, H=H, W=W, Cdim=C)
    torch.cuda.synchronize()
    assert torch.equal(m32.cpu(), rm)
    Cin = heads * T
    lg = rnd(B, Cin, T + L, dev=dev)
    w, b = rnd(Cin, Cin, 3, 3, dev=dev, scale=0.2), rnd(Cin, dev=dev)
    out = torch.zeros(B, Cin, T + L // 4, device=dev)
    kw = dict(B=B, Cin=Cin, H=H, W=W, in_stride=T + L, in_offset=T, out_stride=T + L // 4, out_offset=T)
    ops.conv3x3_s2_maps(lg, w, b, out, **kw)
    rout = torch.zeros(B, Cin, T + L // 4)
    emu["conv3x3_s2_maps"](lg.cpu(), w.cpu(), b.cpu(), rout, **kw)
    torch.cuda.synchronize()
    assert relerr(out, rout) < 1e-5
    rcin, wup = rnd(B, T, C, nh, nh, dev=dev), rnd(2 * C, C, dev=dev, scale=0.2)
    up = torch.zeros(B, T, 2 * C, nh, nh, device=dev)
    ops.swin_chan_up(rcin, wup, up, BT=B * T, Cdim=C, nwin=nh * nh)
    rup = torch.zeros(B, T, 2 * C, nh, nh)
    emu["swin_chan_up"](rcin.cpu(), wup.cpu(), rup, BT=B * T, Cdim=C, nwin=nh * nh)
    torch.cuda.synchronize()
    assert relerr(up, rup) < 1e-5
