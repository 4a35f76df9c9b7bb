"""-m gpu: the wgmma GEMM, the implicit-GEMM convolution and the fused attention, checked bit for bit.

The kernels see bf16 planes, never fp32 inputs. Parity mode (nsplit = 2) sums a_hi*b_hi + a_hi*b_lo + a_lo*b_hi in fp32,
speed mode (nsplit = 1) sums a_hi*b_hi. Every plane here holds small integers (bf16 holds integers up to 256 exactly),
and so do the bias and the residual. Each product is then an exact integer and every partial sum, in any order, is an
integer below 2^24, which fp32 represents exactly: the tensor core's truncating accumulate, the per-stage fold, the
stream-K partial sums and the epilogue's adds have nothing to round. The output must therefore equal, bit for bit, the
same three-term (or one-term) sum computed in float64, whatever the summation order, tile shape or schedule.

Every case keeps sum|terms| <= 2^22 per output element (asserted from the generated operands); the factor-4 margin below
2^24 covers any internal alignment of the tensor core's adder. The lo planes are NOT smaller than one ulp of hi: they
hold integers of the same size as hi, so that the three issued products are told apart, and a swapped plane or an
extra lo*lo product changes the result.

Outputs are compared as raw bits over the WHOLE buffer: every byte the kernel must not write keeps its sentinel
(tests/f64_checks.py), so a stray store or a store to the wrong row fails too. The float64 references are written in plain
torch on the host (im2col + matmul for the convolutions); test_reference_builder_matches_emulation checks them against
tests/emul_ops.py without a GPU.
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from f64_checks import assert_bits_equal, mtt_ops, sentinel, sentinel_split
from kernel_cases import (BOUND, conv_case, conv_weight, gather_case, int_range, int_split, ints, plain_case,
                          ref_gemm, regroup_case, to_dev)

LN2 = float(np.float32(math.log(2.0)))   # scale * log2(e) == 1 in fp32: the kernel's exp2 argument is exact


def check_gemm(build, dev, run=None):
    """build(dev) -> (calls [(a, w, kwargs)], outputs [tensors]): the same case built twice from its seed, once on the
    host for the reference, once on `dev` for the launch (one problem: ops.gemm, several: ops.gemm_grouped)."""
    ops = mtt_ops()
    calls_ref, outs_ref = build("cpu")
    for a, w, kw in calls_ref:
        ref_gemm(a, w, **kw)
    calls, outs = build(dev)
    if run is not None:
        run(calls)
    elif len(calls) == 1:
        ops.gemm(calls[0][0], calls[0][1], **calls[0][2])
    else:
        ops.gemm_grouped(calls)
    if dev != "cpu":
        torch.cuda.synchronize()
    for i, (got, want) in enumerate(zip(outs, outs_ref)):
        assert_bits_equal(got, want, f"output {i}")


@pytest.fixture(params=[1, 2], ids=["bn128", "bn256"])
def tile(request, cuda_dev):
    """The GEMM's 128 x 128 (1) or 128 x 256 (2) tile, forced."""
    ops = mtt_ops()
    ops.set_gemm_variant(request.param)
    try:
        yield request.param
    finally:
        ops.set_gemm_variant(0)


# ------------------------------------------------------------------------------------------------------------------
# 1. GEMM, every instantiation
# ------------------------------------------------------------------------------------------------------------------
# every k_last_steps value 1..4, K below one k16 step, one stage, a long ring; M and N at and around the tile edges
SHAPES = [(1, 1, 1), (127, 8, 15), (128, 127, 16), (129, 128, 17), (300, 129, 40), (1, 255, 63), (127, 256, 64),
          (128, 257, 65), (129, 520, 130), (300, 1, 63), (1, 520, 4096), (129, 255, 1), (300, 8, 65), (128, 1, 130),
          (1, 128, 17), (300, 256, 15), (129, 257, 40), (128, 520, 64), (127, 1, 16), (300, 257, 4096)]


@pytest.mark.gpu
@pytest.mark.parametrize("nsplit", [2, 1])
@pytest.mark.parametrize("M,N,K", SHAPES, ids=[f"{m}x{n}x{k}" for m, n, k in SHAPES])
def test_gemm_shapes(cuda_dev, tile, nsplit, M, N, K):
    """Bias on every case; ReLU and a residual on alternate ones. The split output has two planes in both modes: a
    speed-mode GEMM writes its lo plane as bf16(v - hi) too."""
    i = SHAPES.index((M, N, K))
    check_gemm(plain_case(M, N, K, nsplit=nsplit, act=2 * (i % 2), residual=i % 3 == 0, seed=i), cuda_dev)


@pytest.mark.gpu
@pytest.mark.parametrize("nsplit", [2, 1])
def test_gemm_persistent(cuda_dev, tile, nsplit):
    """More than 2 x 132 tiles on either tile shape, so each CTA runs several tiles, and 7 k-blocks, not a multiple of
    any stage count (3 / 6 stages on 128 x 128, 2 / 4 on 128 x 256): the stage phase carries across tiles at every
    offset."""
    check_gemm(plain_case(2200, 3600, 420, nsplit=nsplit, residual=True, seed=1), cuda_dev)


@pytest.mark.gpu
@pytest.mark.parametrize("nsplit", [2, 1])
@pytest.mark.parametrize("M,N,K", [(300, 257, 130), (129, 520, 64)])
def test_gemm_residual_is_output(cuda_dev, tile, nsplit, M, N, K):
    """x += relu(A W^T + b): the residual buffer is the fp32 output."""
    check_gemm(plain_case(M, N, K, nsplit=nsplit, act=2, residual=True, inplace=True, seed=2), cuda_dev)


@pytest.mark.gpu
def test_gemm_mixed_planes_run_speed_mode(cuda_dev, tile):
    """A with two planes and W with one: nsplit = 1, the result is hi * hi and A_lo is ignored."""
    check_gemm(plain_case(300, 257, 130, nsplit=2, w_nsplit=1, residual=True, seed=3), cuda_dev)


@pytest.mark.gpu
@pytest.mark.parametrize("what", ["gemm", "attention"])
def test_speed_mode_writes_lo_plane(cuda_dev, what):
    """A speed-mode GEMM or attention writing into a 2-plane Split leaves no stale lo plane behind: a parity-mode
    consumer of that Split reads hi + lo."""
    if what == "gemm":
        check_gemm(plain_case(129, 200, 72, nsplit=1, seed=4), cuda_dev)
    else:
        _check_retrieval(cuda_dev, "first_middle_last", nsplit=1, out_nsplit=2)


# ------------------------------------------------------------------------------------------------------------------
# 2. operand addressing: the memory next to each operand is poisoned; TMA clipping must keep it out of the result
# ------------------------------------------------------------------------------------------------------------------
def k_slice_case(a_lo_zero=False):
    """gemm_splitk-style K-slices: A and W hold two slices side by side; the neighbouring slice is NaN."""
    M, N, K0, K = 200, 136, 64, 72

    def build(dev):
        g = torch.Generator().manual_seed(21)
        r = int_range(K)
        a = int_split("cpu", g, M, K0 + K + 40, r, lo_zero=a_lo_zero)
        w = int_split("cpu", g, N, K0 + K + 40, r)
        for sp in (a, w):
            sp.buf[:, :, :K0] = float("nan")
            sp.buf[:, :, K0 + K:] = float("nan")
        a, w = to_dev(a, dev), to_dev(w, dev)
        of = sentinel((M, N), dev=dev)
        return [(a, w, dict(M=M, N=N, K=K, a_col_offset=K0, w_col_offset=K0, out_f32=of))], [of]
    return build


def row_offset_case(a_lo_zero=False):
    """Three stacked problems in one A and one W buffer: the middle one is computed; its neighbours hold NaN."""
    M, N, K = 130, 136, 40

    def build(dev):
        g = torch.Generator().manual_seed(22)
        r = int_range(K)
        a = int_split("cpu", g, 3 * M, K, r, lo_zero=a_lo_zero)
        w = int_split("cpu", g, 3 * N, K, r)
        for sp, n in ((a, M), (w, N)):
            sp.buf[:, :n] = float("nan")
            sp.buf[:, 2 * n:] = float("nan")
        a, w = to_dev(a, dev), to_dev(w, dev)
        of = sentinel((M, N), dev=dev)
        return [(a, w, dict(M=M, N=N, K=K, a_row_offset=M, w_row_offset=N, out_f32=of))], [of]
    return build


def pad_columns_case(a_lo_zero=False):
    """A's and W's pad columns [K, ld) hold NaN (K = 70, ld = 80)."""
    M, N, K = 200, 130, 70

    def build(dev):
        g = torch.Generator().manual_seed(23)
        a = int_split(dev, g, M, K, int_range(K), ld=80, pad=float("nan"), lo_zero=a_lo_zero)
        w = int_split(dev, g, N, K, int_range(K), ld=80, pad=float("nan"))
        of = sentinel((M, N), dev=dev)
        return [(a, w, dict(out_f32=of, bias=ints(g, (N,), 64).to(dev)))], [of]
    return build


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["k_slice", "row_offset", "pad_columns"])
def test_operand_addressing(cuda_dev, tile, case):
    check_gemm({"k_slice": k_slice_case, "row_offset": row_offset_case, "pad_columns": pad_columns_case}[case](),
               cuda_dev)


@pytest.mark.gpu
@pytest.mark.parametrize("G,T,stride", [(4, 5, 69), (37, 8, 11), (10, 32, 40)], ids=["T5_one_tile", "T8_tiles",
                                                                                   "T32_tiles"])
def test_gathered_a(cuda_dev, tile, G, T, stride):
    """T = 5: all groups in one tile. T = 8, 32: 16 / 4 groups per tile over 3 tiles, the last one ragged."""
    check_gemm(gather_case(G, T, stride), cuda_dev)


# ------------------------------------------------------------------------------------------------------------------
# 3. output addressing: every output byte outside the problem keeps its sentinel
# ------------------------------------------------------------------------------------------------------------------
def out_offset_case(a_lo_zero=False):
    """The split output is a window of a wider buffer: out_row_offset 3, out_col_offset 24 (like a task's columns of a
    concatenated map), split pad columns [N, ld) of a second split output."""
    M, N, K = 200, 130, 72

    def build(dev):
        g = torch.Generator().manual_seed(33)
        a = int_split(dev, g, M, K, int_range(K), lo_zero=a_lo_zero)
        w = int_split(dev, g, N, K, int_range(K))
        big = sentinel_split(M + 7, N + 40, dev)
        of = sentinel((M, N + 9), dev=dev)
        return [(a, w, dict(N=N, out_split=big, out_row_offset=3, out_col_offset=24, out_f32=of[:, :N]))], [big.buf, of]
    return build


@pytest.mark.gpu
@pytest.mark.parametrize("regroup,res_row_mod", [((100, 104, 4), 0), ((60, 130, 5, 2), 0), ((100, 105, 5), 100)],
                         ids=["scatter", "row_stride_2", "res_row_mod"])
def test_output_regroup(cuda_dev, tile, regroup, res_row_mod):
    check_gemm(regroup_case(regroup, res_row_mod=res_row_mod), cuda_dev)


@pytest.mark.gpu
def test_output_offsets(cuda_dev, tile):
    check_gemm(out_offset_case(), cuda_dev)


# ------------------------------------------------------------------------------------------------------------------
# 4. implicit-GEMM convolution (pick_conv_tile's patch shapes: single pixel, W > 128, H > 128 with W = 1, ragged)
# ------------------------------------------------------------------------------------------------------------------
CONVS = [(1, 1, 1, 8, 8, 3, 1), (2, 1, 200, 37, 130, 3, 2), (1, 200, 1, 65, 8, 3, 1), (2, 7, 9, 64, 264, 3, 2),
         (1, 12, 20, 200, 130, 3, 1), (3, 16, 16, 65, 264, 1, 1), (1, 33, 130, 37, 8, 3, 2), (2, 7, 9, 200, 130, 1, 1),
         (1, 12, 20, 8, 264, 3, 2), (3, 16, 16, 37, 130, 3, 1), (2, 1, 200, 64, 8, 1, 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("nsplit", [2, 1])
@pytest.mark.parametrize("B,H,W,Cin,Cout,ks,dil", CONVS, ids=[f"{b}x{h}x{w}_c{ci}-{co}_k{k}d{d}"
                                                                for b, h, w, ci, co, k, d in CONVS])
def test_conv(cuda_dev, tile, nsplit, B, H, W, Cin, Cout, ks, dil):
    check_gemm(conv_case(B, H, W, Cin, Cout, ks, dil, nsplit=nsplit, residual=Cin % 2 == 1), cuda_dev)


# ------------------------------------------------------------------------------------------------------------------
# 5. grouped launches
# ------------------------------------------------------------------------------------------------------------------
def grouped_case(count, M=130, N=136, K=72, a_lo_zero=False):
    """`count` problems, each with its own operands, bias, residual and outputs."""
    def build(dev):
        g = torch.Generator().manual_seed(40 + count)
        calls, outs = [], []
        for _ in range(count):
            a = int_split(dev, g, M, K, int_range(K), lo_zero=a_lo_zero)
            w = int_split(dev, g, N, K, int_range(K))
            of = sentinel((M, N), dev=dev)
            osp = sentinel_split(M, N, dev)
            calls.append((a, w, dict(bias=ints(g, (N,), 64).to(dev), act=2, residual=ints(g, (M, N), 4096).to(dev),
                                     out_f32=of, out_split=osp)))
            outs += [of, osp.buf]
        return calls, outs
    return build


def upembed_case(T=3, B=2, h=6, w=10, Cin=40, Ci=72, a_lo_zero=False):
    """InvPT's UpEmbed: the T tasks' dilated 3x3 convs as one grouped launch; each writes its task's rows of the joint
    token buffer (regroup (hw, T hw, 0)) and adds the backbone skip (res_row_mod = B hw)."""
    hw = h * w

    def build(dev):
        g = torch.Generator().manual_seed(50)
        r = int_range(9 * Cin)
        skip = ints(g, (B * hw, Ci), 4096).to(dev)
        xj = sentinel((T * B * hw + 5, Ci), dev=dev)
        calls = []
        for k in range(T):
            a = int_split(dev, g, B * hw, Cin, r, lo_zero=a_lo_zero)
            wt = conv_weight(dev, g, Ci, Cin, 3, r)
            calls.append((a, wt, dict(N=Ci, K=Cin, bias=ints(g, (Ci,), 64).to(dev), act=2, residual=skip,
                                      res_row_mod=B * hw, out_f32=xj[k * hw:], regroup=(hw, T * hw, 0),
                                      conv=(B, h, w, 3, 2))))
        return calls, [xj]
    return build


@pytest.mark.gpu
@pytest.mark.parametrize("count", [2, 5, 32])
def test_grouped(cuda_dev, tile, count):
    check_gemm(grouped_case(count), cuda_dev)


@pytest.mark.gpu
def test_grouped_upembed(cuda_dev, tile):
    check_gemm(upembed_case(), cuda_dev)


@pytest.mark.gpu
def test_grouped_count_limit(cuda_dev):
    """33 problems are refused on the host with the library's error; nothing is launched."""
    ops = mtt_ops()
    calls, _ = grouped_case(2, M=8, N=8, K=8)(cuda_dev)
    with pytest.raises(RuntimeError, match="33 problems"):
        ops.gemm_grouped([calls[0]] * 33)


# ------------------------------------------------------------------------------------------------------------------
# 6. stream-K (128 x 256 tile, the ragged last round split along K over all CTAs)
# ------------------------------------------------------------------------------------------------------------------
def _streamk_pieces(dev, tiles, k_iters):
    from mtt_b200 import lib

    L = lib.load()
    units = torch.cuda.get_device_properties(dev).multi_processor_count
    buf = (C.c_int32 * 96)()
    pieces = []
    for u in range(units):
        n = L.mtt_debug_streamk_schedule(tiles, k_iters, units, u, buf, 32)
        pieces += [tuple(buf[3 * i:3 * i + 3]) for i in range(min(n, 32))]
    return pieces


def _cdiv(a, b):
    return -(-a // b)


def _streamk_geometry(M, N, K, conv=None):
    """(tiles, k-blocks per tile, k-blocks per tap) of the 128 x 256-tile launch of this case: 64-deep k-blocks, 256
    columns per tile, and 128 rows per tile, or, for a convolution, the TH x TW pixel patch that pick_conv_tile in
    gemm_host.cu chooses (restated here: the fewest MMA rows wasted, ties to the wider patch)."""
    num_kb = _cdiv(K, 64)
    if conv is None:
        return _cdiv(M, 128) * _cdiv(N, 256), num_kb, num_kb
    B, H, W, ks, _ = conv
    best, tw_, th_ = -1.0, 1, 1
    for tw in range(1, min(128, W) + 1):
        th = min(128 // tw, H)
        eff = H * W / (_cdiv(W, tw) * _cdiv(H, th) * 128.0)
        if eff > best + 1e-9 or (eff > best - 1e-9 and tw > tw_):
            best, tw_, th_ = eff, tw, th
    return B * _cdiv(W, tw_) * _cdiv(H, th_) * _cdiv(N, 256), ks * ks * num_kb, num_kb


def _run_streamk(dev, geometry, mid_tap):
    """Runs the case on the stream-K schedule; before the launch, the library's own schedule for the case's geometry
    must split some tile along K (and, for mid_tap, start a piece inside a filter tap)."""
    ops = mtt_ops()
    tiles, k_iters, num_kb = geometry
    ws = ops.streamk_workspace(dev)

    def run(calls):
        a, w, kw = calls[0]
        ops.set_gemm_variant(2)
        ops.set_gemm_streamk(2)
        try:
            pieces = _streamk_pieces(dev, tiles, k_iters)
            assert any(kb > 0 or ke < k_iters for _, kb, ke in pieces), "the shape must split along K"
            if mid_tap:
                assert any(kb % num_kb for _, kb, _ in pieces), "a piece must start inside a tap"
            ops.gemm(a, w, sk_ws=ws, **kw)
            torch.cuda.synchronize()
        finally:
            ops.set_gemm_variant(0)
            ops.set_gemm_streamk(1)
        assert int(ws[:16384].view(torch.int32).abs().sum()) == 0, "stream-K flags must be zero after a launch"
    return run


@pytest.mark.gpu
@pytest.mark.parametrize("nsplit", [2, 1])
@pytest.mark.parametrize("inplace", [False, True], ids=["res", "inplace"])
def test_streamk(cuda_dev, nsplit, inplace):
    M, N, K = 1029, 1000, 1000        # 9 x 4 tiles, 16 k-blocks
    check_gemm(plain_case(M, N, K, nsplit=nsplit, act=2, residual=True, inplace=inplace, seed=60), cuda_dev,
               run=_run_streamk(cuda_dev, _streamk_geometry(M, N, K), False))


@pytest.mark.gpu
@pytest.mark.parametrize("nsplit", [2, 1])
def test_streamk_conv(cuda_dev, nsplit):
    """3 x 16 x 16 pixels in 16 x 8 patches (6 row tiles) x 3 column tiles, 9 taps x 4 k-blocks: pieces of about
    4.9 k-blocks, several of which start inside a tap."""
    conv = (3, 16, 16, 3, 1)
    check_gemm(conv_case(*conv[:3], 200, 520, *conv[3:], nsplit=nsplit, residual=True, seed=61), cuda_dev,
               run=_run_streamk(cuda_dev, _streamk_geometry(3 * 16 * 16, 520, 200, conv), True))


# ------------------------------------------------------------------------------------------------------------------
# 7. attention
# ------------------------------------------------------------------------------------------------------------------
def _qkv_ref_planes(qkv, B, N, H, nsplit):
    """[3][B, H, N, 64] float64 (hi, lo or None) of q, k, v."""
    def part(p):
        return None if p is None else p[:, :3 * H * 64].double().reshape(B, N, 3, H, 64).permute(2, 0, 3, 1, 4)
    return part(qkv.buf[0].cpu()), part(qkv.buf[1].cpu() if nsplit == 2 else None)


def _logits(qkv, B, N, H, nsplit):
    hi, lo = _qkv_ref_planes(qkv, B, N, H, nsplit)
    s = hi[0] @ hi[1].transpose(-2, -1)
    mag = hi[0].abs() @ hi[1].abs().transpose(-2, -1)
    if nsplit == 2:
        s = s + hi[0] @ lo[1].transpose(-2, -1) + lo[0] @ hi[1].transpose(-2, -1)
        mag = mag + hi[0].abs() @ lo[1].abs().transpose(-2, -1) + lo[0].abs() @ hi[1].abs().transpose(-2, -1)
    assert float(mag.max()) <= BOUND, "logits out of the exact range"
    return s, hi, lo


ATTN = [(1, 1, 1, 1), (2, 1, 2, 2), (1, 2, 63, 5), (2, 1, 64, 1), (1, 1, 65, 5), (1, 2, 127, 1), (2, 1, 128, 5),
        (1, 1, 129, 1), (1, 2, 517, 5), (2, 2, 1029, 1), (5, 16, 1029, 5), (1, 1, 200, 0)]


@pytest.mark.gpu
@pytest.mark.parametrize("nsplit", [2, 1])
@pytest.mark.parametrize("B,H,N,T", ATTN, ids=[f"B{b}H{h}N{n}T{t}" for b, h, n, t in ATTN])
def test_attention_prompt_logits(cuda_dev, nsplit, B, H, N, T):
    """The exported raw logits of the first T query rows are exactly the integer q.k^T (three-term or one-term); the
    rest of the export buffer keeps its sentinel. B = 5, H = 16 at N = 1029: more items than one wave of CTAs."""
    ops = mtt_ops()
    g = torch.Generator().manual_seed(70 + N)
    qkv = int_split(cuda_dev, g, B * N, 3 * H * 64, 16, nsplit)
    out = ops.Split(B * N, H * 64, cuda_dev, nsplit)
    big = sentinel((B * H * T * N + 64,), dev=cuda_dev)
    logits = big[:B * H * T * N].view(B, H, T, N) if T else None
    ops.attention(qkv, out, B=B, N=N, H=H, scale=0.125, prompt_logits=logits, T=T)
    torch.cuda.synchronize()
    s, _, _ = _logits(qkv, B, N, H, nsplit)
    want = sentinel(big.shape, dev="cpu")
    if T:
        want[:B * H * T * N] = s[:, :, :T, :].reshape(-1).float()
    assert_bits_equal(big, want, "prompt logits")
    assert not torch.isnan(out.hi.float()).any()


def _retrieval_qkv(dev, B, N, H, nsplit, winners, negative):
    """Integer q, k, v whose scaled logits are -4 beta_j + 1000 [j in winners(class(i))]: query i of head h belongs to
    class (i + h) % len(winners); key j carries beta_j >= 0. Planes: q_lo lives only on the class dims and k_lo only on
    the beta dims, so q_lo.k_lo = 0 and parity logits equal the logits of hi + lo.
    negative[b]: image b's logits are all negative (winners at beta 260), so a zero key (logit 0) would win."""
    ncls = len(winners)
    assert ncls <= 62
    g = torch.Generator().manual_seed(80 + N)
    buf = torch.zeros(2, B * N, 3 * H * 64)
    q = buf[:, :, :H * 64].view(2, B, N, H, 64)
    k = buf[:, :, H * 64:2 * H * 64].view(2, B, N, H, 64)
    v = buf[:, :, 2 * H * 64:].view(2, B, N, H, 64)
    blk = torch.arange(N) // 64
    for b in range(B):
        if negative[b]:
            beta = (250 - 40 * blk).clamp_min(48)
            bw = 260
        else:
            beta = (200 - 40 * blk).clamp_min(0)
            bw = 0
            if b > 0 and negative[b - 1]:
                beta[0] = 0        # for image b - 1's queries this key (logit 0) beats their winners (logit -40)
        for h in range(H):
            cls = (torch.arange(N) + h) % ncls
            q_eff = torch.zeros(N, 64)
            q_eff[:, 0] = q_eff[:, 63] = 4
            q_eff[torch.arange(N), 1 + cls] = 200
            bt = beta.clone().float()
            k_eff = torch.zeros(N, 64)
            for c, ws in enumerate(winners):
                for j in ws:
                    if j < N:
                        k_eff[j, 1 + c] = 5
                        bt[j] = bw
            k_eff[:, 0] = k_eff[:, 63] = -bt / 2
            if nsplit == 2:   # q: class dims 100 + 100; k: beta dims split across hi and lo
                q[0, b, :, h] = torch.where(q_eff == 200, torch.full_like(q_eff, 100), q_eff)
                q[1, b, :, h] = torch.where(q_eff == 200, torch.full_like(q_eff, 100), torch.zeros_like(q_eff))
                kh = torch.where(k_eff < 0, torch.trunc(k_eff / 2), k_eff)
                k[0, b, :, h], k[1, b, :, h] = kh, k_eff - kh
            else:
                q[0, b, :, h], k[0, b, :, h] = q_eff, k_eff
                q[1, b, :, h] = ints(g, (N, 64), 200)     # ignored in speed mode
                k[1, b, :, h] = ints(g, (N, 64), 200)
            v[0, b, :, h] = ints(g, (N, 64), 256)     # wide enough that means of 2 or 4 rows need a lo part
            v[1, b, :, h] = ints(g, (N, 64), 256)
    ops = mtt_ops()
    sp = ops.Split(B * N, 3 * H * 64, "cpu", 2)
    sp.buf.copy_(buf.bfloat16())
    assert torch.equal(sp.buf.float(), buf)
    return to_dev(sp, dev)


RETRIEVAL = {
    # N = 517: 9 key blocks, the last one 5 keys long
    "first_middle_last": (1, 517, 1, [[3], [300], [515], [63, 64], [10, 130, 250, 516], [100, 101]], [False]),
    "all_negative": (1, 517, 2, [[3], [300], [516], [64, 127], [0, 200, 400, 512]], [True]),
    "images_back_to_back": (3, 130, 2, [[0], [129], [64, 65], [1, 63, 66, 128]], [True, False, True]),
    "single_block": (2, 40, 1, [[39], [0, 1], [5, 6, 7, 8]], [False, True]),
    "many_items": (5, 1029, 16, [[7], [500], [1028], [1000, 1025], [2, 600, 700, 1027]], [True, False, True, False,
                                                                                          True]),
}


@pytest.mark.gpu
@pytest.mark.parametrize("nsplit", [2, 1])
@pytest.mark.parametrize("case", list(RETRIEVAL))
def test_attention_retrieval(cuda_dev, nsplit, case):
    """One-hot attention, exactly. scale = ln 2 makes the kernel's log2-domain scale exactly 1, so the winning keys'
    exponent is exactly 0 (ex2.approx(0) = 1) and every other real key is >= 150 below it (ex2.approx.ftz flushes to 0).
    The output row is then the mean of the winners' V rows (hi + lo in parity mode, hi in speed mode): exact for 1, 2 or
    4 winners. The winners sit in the first, a middle and the ragged last key block and tie across blocks; the running
    maximum rises by >= 150 from block to block, so the rescale factor 0 must wipe the earlier blocks; where all real
    logits are negative, a key past N (zero-filled, logit 0) or a key of the next image would win if it were let in."""
    _check_retrieval(cuda_dev, case, nsplit, nsplit)


def _check_retrieval(dev, case, nsplit, out_nsplit):
    """nsplit 1 with out_nsplit 1: qkv carries a junk lo plane the kernel must ignore; with out_nsplit 2: qkv has one
    plane and the output's lo plane must be written."""
    ops = mtt_ops()
    assert np.float32(LN2) * np.float32(1.4426950408889634) == np.float32(1.0)
    B, N, H, winners, negative = RETRIEVAL[case]
    qkv = _retrieval_qkv(dev, B, N, H, nsplit, winners, negative)
    if nsplit == 1 and out_nsplit == 2:
        qkv.buf, qkv.nsplit = qkv.buf[:1].clone(), 1
    out = sentinel_split(B * N, H * 64, dev, out_nsplit)
    ops.attention(qkv, out, B=B, N=N, H=H, scale=LN2)
    torch.cuda.synchronize()

    s, hi, lo = _logits(qkv, B, N, H, nsplit)
    m = s.max(-1, keepdim=True).values
    win = s == m
    cnt = win.sum(-1)
    assert bool(((cnt == 1) | (cnt == 2) | (cnt == 4)).all()), "1, 2 or 4 winners per query"
    assert bool((s[~win] <= (m.expand_as(s)[~win] - 150)).all()), "every other key >= 150 below the winners"
    if any(negative):
        assert bool((m[torch.tensor(negative)] < 0).all())
    vv = hi[2] + lo[2] if nsplit == 2 else hi[2]
    assert float((win.double() @ vv.abs()).max()) <= BOUND
    o = (win.double() @ vv) / cnt[..., None].double()                   # [B, H, N, 64]
    o = o.permute(0, 2, 1, 3).reshape(B * N, H * 64).float()
    h_ = o.bfloat16()
    assert_bits_equal(out.hi, h_, "attention output hi")
    if out_nsplit == 2:
        lo_want = (o - h_.float()).bfloat16()
        assert bool((lo_want != 0).any()), "the case must need a lo part"
        assert_bits_equal(out.lo, lo_want, "attention output lo")


# ------------------------------------------------------------------------------------------------------------------
# 8. the references above against tests/emul_ops.py, without a GPU
# ------------------------------------------------------------------------------------------------------------------
def test_reference_builder_matches_emulation(monkeypatch):
    """ref_gemm (float64, im2col) against emul_ops' gemm (fp32, F.conv2d) on the host, A_lo = 0 so that the emulation's
    extra lo*lo term vanishes: checks the references' indexing (regroup, gather, offsets, conv tap layout)."""
    import emul_ops

    emul_ops.install(monkeypatch)
    cases = [plain_case(129, 257, 65, residual=True, act=2, a_lo_zero=True),
             plain_case(1, 8, 17, a_lo_zero=True),
             plain_case(127, 129, 130, residual=True, inplace=True, a_lo_zero=True),
             k_slice_case(a_lo_zero=True), row_offset_case(a_lo_zero=True), pad_columns_case(a_lo_zero=True),
             gather_case(4, 5, 69, a_lo_zero=True), gather_case(10, 32, 40, a_lo_zero=True),
             regroup_case((60, 130, 5, 2), a_lo_zero=True), regroup_case((100, 105, 5), res_row_mod=100, a_lo_zero=True),
             out_offset_case(a_lo_zero=True),
             conv_case(2, 7, 9, 37, 130, 3, 2, residual=True, a_lo_zero=True),
             conv_case(1, 12, 20, 65, 8, 1, 1, a_lo_zero=True),
             conv_case(2, 1, 200, 8, 16, 3, 1, a_lo_zero=True),
             grouped_case(3, a_lo_zero=True), upembed_case(a_lo_zero=True)]
    for build in cases:
        check_gemm(build, "cpu")
