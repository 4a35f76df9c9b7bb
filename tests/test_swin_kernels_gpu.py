"""-m gpu: the kernels of csrc/swin.cu (and the split-K chan_kv GEMM) at the geometries the Swin-B TaskPrompter launches,
against float64 statements of the reference's semantics (TP/models/transformers/taskprompter_swin.py) written here:

  * roll by -shift after padding the normed map, row-major windows with the T prompts first in every window;
  * relative-position bias from oracle.taskprompter_swin_ref.relative_position_index, shift mask from its
    shifted_window_mask (both checked against the reference by test_oracle.py);
  * softmax attention / channel attention / PatchMerging / stride-2 convolution in float64 on the device.

The cases themselves (tests/kernel_cases.py) decode split inputs in float64 and check every fp32 result element by
element against a bound computed from its own operands (tests/f64_checks.py), so a wrong window, head or row of small
magnitude cannot hide; failures report the worst block. Copies (window gather / scatter, transpose,
merge, logits scatter) and splits of copies are bit-exact. Every output buffer is sentinel-filled first, with pad
columns and a trailing row or slot the kernel must not write; the tests assert they keep their bits. Inputs carry the
sentinel NaN in their pad columns, so a read past C shows up in the result.

Swin-B at 1024x2048 (0.75 input scale, patch 4): stage maps 192x384 / 96x192 / 48x96 / 24x48, C 128 / 256 / 512 / 1024,
heads 4 / 8 / 16 / 32 (head dim 32), window 12 (144 tokens + T = 2 prompts: N = 146), 512 / 128 / 32 / 8 windows per
image, chan_embed_dim 256 with one channel window.
"""
import pytest
import torch

from f64_checks import assert_planes_bit_exact, decode, is_sentinel, ops, pad_cols, padded, sentinel  # noqa: F401
from kernel_cases import (assert_untouched, attention_case, chan_attention_case, chan_up_case, conv3x3_s2_case,
                          gather_scatter_case, nan_split, split_in)

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]

SWINB = [  # (H, W, C, heads) per stage, window 12, T 2
    (192, 384, 128, 4), (96, 192, 256, 8), (48, 96, 512, 16), (24, 48, 1024, 32)]


# ---------------------------------------------------------------------------------------------------------------------
# window attention
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("stage", range(4))
@pytest.mark.parametrize("shift", [0, 6])
def test_window_attention_swinB_stages(ops, cuda_dev, stage, shift):
    """The four Swin-B stages exactly: ws 12, T 2, head dim 32, N = 146 (the 192-thread launch). Two images in the
    small stages, so the mask is indexed by the window within its image."""
    H, W, C, heads = SWINB[stage]
    attention_case(ops, cuda_dev, B=1 if stage < 2 else 2, nWy=H // 12, nWx=W // 12, ws=12, shift=shift, T=2,
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
    attention_case(ops, cuda_dev, B=2, nWy=2, nWx=3, ws=ws, shift=ws // 2, T=T, heads=heads, dh=dh, seed=ws * 100 + T)


@pytest.mark.parametrize("ws,T,dh,why", [(4, 2, 24, "head_dim=24"), (20, 4, 64, "window too large")])
def test_window_attention_refusals(ops, cuda_dev, ws, T, dh, why):
    """head_dim outside {8, 16, 32, 64}, and K + V of a window over the 200 KB of shared memory (N = 404 at head dim 64:
    202 KB), are refused with the library's error and nothing is launched."""
    heads, L = 2, ws * ws
    N, C = T + L, heads * dh
    qkv, _ = split_in(ops, torch.randn(N, 3 * C, device=cuda_dev))
    out = nan_split(N, C, cuda_dev)
    raw = sentinel((1, heads, T, L), dev=cuda_dev)
    biasT = torch.zeros(heads, L, L, device=cuda_dev)
    torch.cuda.synchronize()
    n0 = ops.launch_count()
    with pytest.raises(RuntimeError, match=why):
        ops.swin_window_attention(qkv, out, raw, biasT, None, BW=1, nW=1, T=T, L=L, heads=heads, scale=dh ** -0.5)
    torch.cuda.synchronize()
    assert ops.launch_count() == n0
    assert is_sentinel(out.buf) and is_sentinel(raw)


# ---------------------------------------------------------------------------------------------------------------------
# window gather / scatter (partition, reverse, residual add, prompt mean, logits map)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,H,W,C,T,heads,shift", [
    (1, 192, 384, 128, 2, 4, 6),     # Swin-B stage 1 map: 512 windows
    (2, 24, 48, 1024, 2, 32, 6),     # Swin-B stage 4 map: 8 windows
    (2, 25, 49, 97, 3, 3, 6),        # padded to 36 x 60: 15 windows (not a multiple of 4), odd C, C % 64 != 0
    (2, 25, 49, 97, 3, 3, 0),
])
def test_window_gather_scatter(ops, cuda_dev, B, H, W, C, T, heads, shift):
    gather_scatter_case(ops, cuda_dev, B=B, H=H, W=W, C=C, T=T, heads=heads, ws=12, shift=shift)


# ---------------------------------------------------------------------------------------------------------------------
# channel attention: transpose_split -> chan_kv (split-K GEMM) -> swin_chan_attention
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,L,C", [(1, 73728, 128), (2, 1001, 45)])
def test_transpose_split(ops, cuda_dev, B, L, C):
    """[B, L, C] fp32 -> split [B*C, L], bit-exact: Swin-B stage 1 (L = 192 * 384) and ragged L and C (tiles of 64 x 32
    cut on both axes, odd L: the last column is written alone)."""
    x = padded(B * L, C, cuda_dev)
    x.copy_(torch.randn(B * L, C, device=cuda_dev, generator=torch.Generator(device=cuda_dev).manual_seed(L)))
    out = nan_split(B * C, L, cuda_dev)
    ops.transpose_split(x, out, B=B, L=L, Cdim=C)
    torch.cuda.synchronize()
    assert_planes_bit_exact(out, x.reshape(B, L, C).transpose(1, 2).reshape(B * C, L), "transpose_split")
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
    part = sentinel((chunks, C, N), dev=dev)
    out = padded(C, N, dev)
    ops.gemm_splitk(a, w, part, out, K=K, bias=bias, chunks=chunks)
    torch.cuda.synchronize()
    want = A @ decode(w, N).t() + bias.double()
    assert torch.isfinite(out).all() and is_sentinel(pad_cols(out))
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
    chan_attention_case(ops, cuda_dev, B=B, T=T, C=C, nh=nh)


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
    assert is_sentinel(pad_cols(out))


@pytest.mark.parametrize("stage", range(3))
def test_conv3x3_s2_maps(ops, cuda_dev, stage):
    """spa_attn_ds (TP:458-460) at the three Swin-B merges: Cin = Cout = heads * T = 8 / 16 / 32 over the full-size
    logit maps stored behind T prompt columns; columns before out_offset stay untouched."""
    H, W, _, heads = SWINB[stage]
    conv3x3_s2_case(ops, cuda_dev, B=1, T=2, H=H, W=W, Cin=heads * 2, seed=stage)


@pytest.mark.parametrize("nwin", [1, 4])
def test_chan_up(ops, cuda_dev, nwin):
    """process_chan_attn (TP:463-466) at the last merge: C 1024 -> 2048 over the channel axis of raw_chan."""
    chan_up_case(ops, cuda_dev, BT=2, C=1024, nwin=nwin, seed=nwin)
