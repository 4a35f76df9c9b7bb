"""-m gpu: the GEMM's fused epilogue against the same fp32 operations applied in torch to the raw product.

Each case runs twice on the same kernel: once raw (no bias, no activation, no residual, fp32 output only) and once
fused. The fused fp32 output must equal (raw + bias) -> act -> + residual computed in fp32 by torch: exactly for no
activation and ReLU, within 2 ulp for GELU (torch's erf may differ from erff). The split-bf16 output must be exactly
hi = bf16_rn(v), lo = bf16_rn(v - hi) of the fused fp32 value v.
"""
import pytest
import torch

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300)]


def _ops():
    from mtt_b200 import ops

    return ops


def _post(raw, bias, act, res):
    ops = _ops()
    v = raw.clone()
    if bias is not None:
        v = v + bias
    if act == ops.ACT_RELU:
        v = torch.relu(v)
    elif act == ops.ACT_GELU:
        v = 0.5 * v * (1.0 + torch.erf(v * 0.70710678118654752440))
    if res is not None:
        v = v + res
    return v


def _check(got, osp, ref, act, rows=None):
    """got: fused fp32 output [rows, N]; osp: fused split output; ref: torch's fp32 restatement."""
    ops = _ops()
    N = got.shape[1]
    if rows is not None:
        got, ref = got[rows], ref[rows]
    assert not torch.isnan(ref).any()
    if act == ops.ACT_GELU:
        a = ref.abs()
        ulp = torch.nextafter(a, torch.full_like(a, float("inf"))) - a
        d = (got - ref).abs()
        assert bool((d <= 2 * ulp).all()), f"GELU: {(d / ulp).max().item():.1f} ulp"
    else:
        assert torch.equal(got, ref), f"max |diff| {(got - ref).abs().max().item()}"
    hi, lo = osp.hi[:, :N], osp.lo[:, :N]
    if rows is not None:
        hi, lo = hi[rows], lo[rows]
    h = got.bfloat16()
    assert torch.equal(hi, h)
    assert torch.equal(lo, (got - h.float()).bfloat16())


def _operands(dev, M, N, K, seed):
    ops = _ops()
    g = torch.Generator(device=dev).manual_seed(seed)
    a = torch.randn(M, K, device=dev, generator=g)
    w = torch.randn(N, K, device=dev, generator=g) * 0.05
    bias = torch.randn(N, device=dev, generator=g)
    res = torch.randn(M, N, device=dev, generator=g)
    return ops.split_f32(a, 2), ops.split_f32(w, 2), bias, res


def _run(dev, A, W, M, N, bias, act, res, inplace=False, **kw):
    """(raw, fused fp32, fused split) of one problem."""
    ops = _ops()
    raw = torch.full((M, N), float("nan"), device=dev)
    ops.gemm(A, W, out_f32=raw, **kw)
    osp = ops.Split(M, N, dev, 2, zero=True)
    if inplace:
        out = res.clone()
        ops.gemm(A, W, bias=bias, act=act, residual=out, out_f32=out, out_split=osp, **kw)
    else:
        out = torch.full((M, N), float("nan"), device=dev)
        ops.gemm(A, W, bias=bias, act=act, residual=res, out_f32=out, out_split=osp, **kw)
    torch.cuda.synchronize()
    return raw, out, osp


@pytest.fixture(params=[1, 2], ids=["bn128", "bn256"])
def tile(request, cuda_dev):
    ops = _ops()
    ops.set_gemm_variant(request.param)
    yield request.param
    ops.set_gemm_variant(0)


# (M, N, K): ragged M; N = 200 (vector path, column tail inside a chunk); N = 201 (odd: the scalar path)
@pytest.mark.parametrize("M,N,K", [(300, 200, 136), (389, 201, 200), (1029, 1024, 512)])
@pytest.mark.parametrize("act", [0, 1, 2], ids=["none", "gelu", "relu"])
@pytest.mark.parametrize("with_res", [False, True], ids=["nores", "res"])
def test_fused_equals_raw_then_torch(cuda_dev, tile, M, N, K, act, with_res):
    A, W, bias, res = _operands(cuda_dev, M, N, K, seed=M + N + K + act)
    res = res if with_res else None
    raw, out, osp = _run(cuda_dev, A, W, M, N, bias, act, res)
    _check(out, osp, _post(raw, bias, act, res), act)
    # without a bias
    raw, out, osp = _run(cuda_dev, A, W, M, N, None, act, res)
    _check(out, osp, _post(raw, None, act, res), act)


@pytest.mark.parametrize("M,N,K", [(300, 200, 136), (389, 201, 200), (1029, 1024, 512)])
@pytest.mark.parametrize("act", [0, 2], ids=["none", "relu"])
def test_residual_is_the_output(cuda_dev, tile, M, N, K, act):
    """x += f(x): the residual read of every element precedes its store."""
    A, W, bias, res = _operands(cuda_dev, M, N, K, seed=3 * M + N)
    raw, out, osp = _run(cuda_dev, A, W, M, N, bias, act, res, inplace=True)
    _check(out, osp, _post(raw, bias, act, res), act)


def test_grouped(cuda_dev):
    ops = _ops()
    M, N, K = 389, 520, 264
    probs = [_operands(cuda_dev, M, N, K, seed=11 + i) for i in range(3)]
    raws = [torch.full((M, N), float("nan"), device=cuda_dev) for _ in probs]
    ops.gemm_grouped([(A, W, dict(out_f32=r)) for (A, W, _, _), r in zip(probs, raws)])
    outs = [torch.full((M, N), float("nan"), device=cuda_dev) for _ in probs]
    osps = [ops.Split(M, N, cuda_dev, 2, zero=True) for _ in probs]
    inplace = probs[2][3].clone()  # the last problem adds its residual in place
    calls = []
    for i, (A, W, b, r) in enumerate(probs):
        o = inplace if i == 2 else outs[i]
        calls.append((A, W, dict(bias=b, act=ops.ACT_RELU, residual=o if i == 2 else r, out_f32=o, out_split=osps[i])))
    ops.gemm_grouped(calls)
    torch.cuda.synchronize()
    for i, (A, W, b, r) in enumerate(probs):
        _check(inplace if i == 2 else outs[i], osps[i], _post(raws[i], b, ops.ACT_RELU, r), ops.ACT_RELU)


@pytest.mark.parametrize("act,inplace", [(0, True), (1, False)], ids=["none_inplace", "gelu"])
def test_streamk(cuda_dev, act, inplace):
    """The stream-K owner runs the epilogue on the sum of the partials; the raw run splits the same way."""
    ops = _ops()
    M, N, K = 1029, 1024, 2048
    A, W, bias, res = _operands(cuda_dev, M, N, K, seed=5 + act)
    ws = ops.streamk_workspace(cuda_dev)
    ops.set_gemm_variant(2)
    ops.set_gemm_streamk(2)
    try:
        raw, out, osp = _run(cuda_dev, A, W, M, N, bias, act, res, inplace=inplace, sk_ws=ws)
    finally:
        ops.set_gemm_variant(0)
        ops.set_gemm_streamk(1)
    _check(out, osp, _post(raw, bias, act, res), act)


@pytest.mark.parametrize("ksize", [3, 1])
def test_conv(cuda_dev, tile, ksize):
    """Implicit-GEMM convolution: output rows come from image patches (row_info's conv mode)."""
    ops = _ops()
    from mtt_b200.pack import pack_conv_weight

    g = torch.Generator(device=cuda_dev).manual_seed(ksize)
    B, H, W_, Cin, Cout = 2, 12, 20, 72, 264
    x = torch.randn(B * H * W_, Cin, device=cuda_dev, generator=g)
    w = torch.randn(Cout, Cin, ksize, ksize, device=cuda_dev, generator=g) * 0.05
    bias = torch.randn(Cout, device=cuda_dev, generator=g)
    res = torch.randn(B * H * W_, Cout, device=cuda_dev, generator=g)
    A, Wp = ops.split_f32(x, 2), pack_conv_weight(w, 2)
    raw, out, osp = _run(cuda_dev, A, Wp, B * H * W_, Cout, bias, ops.ACT_RELU, res, conv=(B, H, W_, ksize, 1))
    _check(out, osp, _post(raw, bias, ops.ACT_RELU, res), ops.ACT_RELU)


def test_regroup_and_rowmod(cuda_dev, tile):
    """Patch-embedding style: output rows scattered behind 5 prompt rows per image, residual rows taken mod 64."""
    ops = _ops()
    M, N, K, ig, og, off = 2 * 64, 256, 768, 64, 69, 5
    A, W, bias, _ = _operands(cuda_dev, M, N, K, seed=17)
    pos = torch.randn(ig, N, device=cuda_dev, generator=torch.Generator(device=cuda_dev).manual_seed(18))
    rows_out = (M // ig) * og
    idx = torch.arange(M, device=cuda_dev)
    oidx = (idx // ig) * og + off + idx % ig
    raw = torch.full((rows_out, N), float("nan"), device=cuda_dev)
    ops.gemm(A, W, out_f32=raw, regroup=(ig, og, off))
    out = torch.full((rows_out, N), float("nan"), device=cuda_dev)
    osp = ops.Split(rows_out, N, cuda_dev, 2, zero=True)
    ops.gemm(A, W, bias=bias, residual=pos, res_row_mod=ig, out_f32=out, out_split=osp, regroup=(ig, og, off))
    torch.cuda.synchronize()
    ref = torch.full_like(raw, float("nan"))
    ref[oidx] = _post(raw[oidx], bias, ops.ACT_NONE, pos[idx % ig])
    _check(out, osp, ref, ops.ACT_NONE, rows=oidx)
    untouched = torch.ones(rows_out, dtype=torch.bool, device=cuda_dev)
    untouched[oidx] = False
    assert torch.isnan(out[untouched]).all()
