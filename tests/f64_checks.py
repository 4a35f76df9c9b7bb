"""The error model and the operands of the float64 kernel tests.

Error model. u = U = 2^-24 is the fp32 unit roundoff; each elementwise fp32 operation adds u relative. A reduction that
adds terms a_i in fp32 along a tree whose longest chain of additions is D (per-thread serial sum + warp shuffles +
shared-memory steps + atomics, counted from the kernel's launch geometry) is off by at most sum_tol(D, sum |a_i|) =
LAM sqrt(D) u sum |a_i| (the probabilistic bound of Higham & Mary 2019, with LAM = 4 covering it far beyond the
1 - 1e-6 level). Sums kept in double use U64 = 2^-53 in place of u. A value stored as split planes (hi + lo bf16)
carries a further SPLIT |x| + SPLIT_ABS (2^-17 relative, and the lo plane's spacing once it is subnormal in bf16); a
value stored as the hi plane alone (speed mode, nsplit = 1) carries HI |x| + HI_ABS (split_bound). Pure data movement
is bit-exact. Every assert states which of these it uses.

Operands. Outputs are written inside sentinels: one NaN payload per dtype (SENTINEL), so an element a kernel must not
write is checked by its bits, not by isnan."""
import math

import pytest
import torch

U = 2.0 ** -24            # fp32 unit roundoff
U64 = 2.0 ** -53          # fp64 unit roundoff (sums accumulated in double)
LAM = 4.0                 # probabilistic summation bound: |error| <= LAM sqrt(D) u sum|a_i|
SPLIT = 2.0 ** -17        # relative precision of a value stored as hi + lo bf16 planes
SPLIT_ABS = 2.0 ** -133   # ... and its absolute floor: the lo plane's spacing once it is subnormal in bf16
HI = 2.0 ** -8            # relative precision of the hi bf16 plane alone: bf16 unit roundoff (8-bit significand)
HI_ABS = 2.0 ** -133      # ... and its absolute floor: the bf16 subnormal spacing

# NaN sentinels: a kernel that leaves an output element unwritten leaves this exact bit pattern behind
_INT = {torch.float32: torch.int32, torch.bfloat16: torch.int16, torch.int64: torch.int64}
SENTINEL = {torch.float32: 0x7FC0BEEF, torch.bfloat16: 0x7FB5, torch.int64: -0x5A5A5A5A5A5A5A5B}


def sum_tol(D, abs_sum):
    """Bound of an fp32 reduction of depth D whose terms have absolute sum abs_sum (tensor or float)."""
    return LAM * math.sqrt(D) * U * abs_sum


def check(got, ref, bound, what, block=None):
    """|got - ref| <= bound elementwise (float64, on ref's device); returns the worst err / bound. On failure the report
    names the worst element, or with `block` (the number of leading dims that index a block) the worst block's error
    over that block's own max |ref|."""
    got, ref = got.double(), ref.double()
    bound = torch.as_tensor(bound, dtype=torch.float64, device=ref.device).expand_as(ref)
    assert torch.isfinite(got).all(), f"{what}: non-finite values (unwritten sentinel or NaN read)"
    err = (got - ref).abs()
    r = err / bound.clamp_min(1e-300)
    i = int(r.argmax())
    ratio = r.reshape(-1)[i].item()
    if (err <= bound).all():
        return ratio
    if block is not None:
        e = err.flatten(block).amax(-1)
        m = ref.abs().flatten(block).amax(-1).clamp_min(1e-300)
        w = int((e / m).flatten().argmax())
        raise AssertionError(f"{what}: {int((err > bound).sum())} of {err.numel()} elements over the bound; worst block "
                             f"{tuple(int(k) for k in torch.unravel_index(torch.tensor(w), e.shape))}: error / block "
                             f"max |ref| = {(e / m).flatten()[w].item():.3e}, max error / bound = {ratio:.3e}")
    idx = tuple(int(k) for k in torch.unravel_index(torch.tensor(i), ref.shape))
    raise AssertionError(f"{what}: error {ratio:.2f}x its bound at {idx}: got {got.reshape(-1)[i].item():.9e}, "
                         f"want {ref.reshape(-1)[i].item():.9e}, bound {bound.reshape(-1)[i].item():.3e} "
                         f"(max abs err {err.max().item():.3e})")


def report(name, ratios):
    print(f"{name}: worst error / bound = {max(ratios):.3f}")


def bce_rel(x):
    """Relative bound of the fp32 softplus / sigmoid of logit x in the balanced BCE (loss_terms.cuh balanced_bce_term):
    (|x| + 8) u. x is a float64 tensor."""
    return (x.abs() + 8) * U


def bce_term_bound(x):
    """Bound of one fp32 balanced BCE term at logit x (label in [0, 1], weight in [0, 1)): bce_rel(x) of a term no larger
    than |x| + 1."""
    return bce_rel(x) * (x.abs() + 1)


# ---- split planes --------------------------------------------------------------------------------------------------------
def split_planes(x, ns=2):
    """The planes the kernels write for fp32 x: hi = bf16(x) (round to nearest even), lo = bf16(x - hi)."""
    hi = x.bfloat16()
    return (hi,) if ns == 1 else (hi, (x - hi.float()).bfloat16())


def planes(sp, ns):
    """The ns planes of a Split that a mode reads: [hi] or [hi, lo], whole buffers."""
    return [sp.buf[0]] + ([sp.buf[1]] if ns == 2 else [])


def decode(sp, rows=None):
    """float64 value the planes hold (hi + lo, or hi alone): the first `rows` rows (all by default), sp.cols columns."""
    rows = sp.buf.shape[1] if rows is None else rows
    return sum(p[:rows, :sp.cols].double() for p in planes(sp, sp.nsplit))


def split_bound(ns, mag):
    """What storing a value of magnitude mag as planes adds: SPLIT |x| + SPLIT_ABS (hi + lo) or HI |x| + HI_ABS (hi)."""
    return SPLIT * mag + SPLIT_ABS if ns == 2 else HI * mag + HI_ABS


def check_planes(sp, ref, e, what):
    """|planes - ref| <= e (the fp32 computation's bound) + the split bound of the stored value."""
    return check(decode(sp), ref, e + split_bound(sp.nsplit, ref.abs() + e), f"{what} (nsplit={sp.nsplit})")


def bits(t):
    """The raw bits of a float32 / bfloat16 / int64 tensor as integers."""
    return t.detach().view(_INT[t.dtype])


def assert_bits_equal(got, want, what):
    g, w = bits(got).cpu(), bits(want).cpu()
    if not torch.equal(g, w):
        bad = (g != w).nonzero()
        i = tuple(bad[0].tolist())
        raise AssertionError(f"{what}: {bad.shape[0]} of {g.numel()} elements differ, first at {i}: "
                             f"got {got.cpu()[i].item()}, want {want.cpu()[i].item()}")


def assert_planes_bit_exact(sp, x, what):
    """The planes are the split of fp32 x [rows, sp.cols] bit for bit (hi alone when there is one plane)."""
    for i, p in enumerate(split_planes(x, sp.nsplit)):
        assert torch.equal(bits(sp.buf[i, :x.shape[0], :sp.cols]), bits(p)), f"{what}: plane {i} differs"


# ---- sentinels -----------------------------------------------------------------------------------------------------------
def round_up(x, m):
    return (x + m - 1) // m * m


def sentinel(shape, dtype=torch.float32, dev="cuda"):
    t = torch.empty(shape, dtype=dtype, device=dev)
    bits(t).fill_(SENTINEL[dtype])
    return t


def is_sentinel(t):
    """True when every element of t still holds its dtype's sentinel bits."""
    return bool((bits(t) == SENTINEL[t.dtype]).all())


def sentinel_split(rows, cols, dev="cuda", ns=2, ld=None):
    """A Split whose every element, pad columns included, holds the bf16 sentinel."""
    sp = mtt_ops().Split(rows, cols, dev, ns, ld=ld)
    bits(sp.buf).fill_(SENTINEL[torch.bfloat16])
    return sp


class Guarded:
    """A flat buffer filled with the sentinel of its dtype; `view` is the kernel's output inside it, `g` elements from
    either end. unchanged_outside(region) asserts every element outside `region` (index into `view`, or a bool mask of
    the flat buffer) still holds what it held before the call."""

    def __init__(self, shape, dtype, g=4096):
        n = math.prod(shape)
        self.flat = sentinel((n + 2 * g,), dtype)
        self.g, self.n = g, n
        self.view = self.flat[g:g + n].view(shape)

    def snapshot(self):
        self.before = self.flat.clone()

    def unchanged_outside(self, region, what):
        torch.cuda.synchronize()
        written = torch.zeros(self.flat.shape, dtype=torch.bool, device="cuda")
        if isinstance(region, torch.Tensor) and region.dtype == torch.bool and region.shape == self.flat.shape:
            written = region
        else:
            written[self.g:self.g + self.n].view(self.view.shape)[region] = True
        same = bits(self.flat)[~written] == bits(self.before)[~written]
        assert bool(same.all()), f"{what}: {int((~same).sum())} elements outside the output changed"


def guarded_split(ops, ns, rows, cols, ld=None, g=16):
    """A Split [rows, cols] of ns planes inside a 2-plane bf16 buffer with g sentinel rows around each plane, padding
    columns up to ld and (ns = 1) a whole sentinel second plane. Returns (Guarded, Split, region of the planes)."""
    ld = round_up(cols, 8) if ld is None else ld
    gb = Guarded((2, rows + 2 * g, ld), torch.bfloat16, g=64)
    sp = ops.Split.from_planes(gb.view[:ns, g:g + rows], cols)
    return gb, sp, (slice(0, ns), slice(g, g + rows), slice(0, cols))


def padded(rows, cols, dev="cuda", pad=3, fill=None):
    """A [rows, cols] fp32 view of a [rows, cols + pad] buffer whose pad columns hold `fill` (the sentinel by default:
    a read of a pad column poisons the result, a write to one changes its bits)."""
    buf = sentinel((rows, cols + pad), dev=dev) if fill is None else torch.full((rows, cols + pad), fill, device=dev)
    return buf[:, :cols]


def pad_cols(v):
    """The pad columns of a `padded` view."""
    return torch.as_strided(v, (v.shape[0], v.stride(0) - v.shape[1]), (v.stride(0), 1), v.storage_offset() + v.shape[1])


# ---- random operands and the library ---------------------------------------------------------------------------------------
def gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def randn(g, *shape, scale=1.0):
    return torch.randn(*shape, generator=g, device="cuda") * scale


def mtt_ops():
    import mtt_b200  # noqa: F401
    from mtt_b200 import ops as o
    return o


@pytest.fixture(scope="module")
def ops(cuda_dev):
    return mtt_ops()
