"""GroupNorm and LayerNorm at the edges of their launch policies, against float64.

`ladi_groupnorm_plan` and `ladi_layernorm_plan` report the grids the launches would run; they share the validation-and-policy function
with the launches and need no device.  Every GPU case first asserts, through the query at the device's SM count, the plan it means to
exercise (the expectations are those of a 132-SM H100 SXM; on another SM count only the float64 checks run).  It then runs the call the
way the workload census replays the workload's (tests/kernel_check.py): every input pitch gap is NaN, the output is NaN over its full pitch plus
TAIL rows, afterwards every owned element is finite and every other one still NaN, a second run is bit-identical, and every element is
within a float64 bound.

GroupNorm inputs make statistics mistakes visible: each (image, group) has its own mean and scale (|mean| / sigma <= 3, so the one-pass
mean^2 / var term of `norm_expect` stays small), and every chunk's first and last pixel and the last pixel of the image are sentinels at
+6 / -5 sigma.  A channel counted in the wrong group, a pixel dropped or counted twice then moves its group's statistics by more than the
bound allows near the many outputs close to zero.  One characterisation case at |mean| / sigma = 30 over 786432 values per group documents
the one-pass fp32 variance against the census bound, which prices it in.

LayerNorm computes its statistics in two passes (mean, then the sum of squared deviations), so it gets its own bound, `ln_expect`:
  d_mean = delta (|mean| + sd), delta = C_ACC sqrt(C) 2^-24    the fp32 sum of C bf16 values, divided by C (as in norm_expect);
  var:  the sum of C non-negative squares of fp32 deviations: relative error delta from the accumulation, 2^-23 from forming and
        squaring each deviation, plus (d_mean / sd)^2 because the deviations are taken from the computed mean -- no mean^2 / var term;
  d_rstd = 1.5 (delta + 2^-23 + d_mean^2 / (var + eps)) + 2^-22  (half the relative variance error through rsqrt, tripled for margin,
        plus rsqrtf's own error);
  |y - r| <= U_BF16 |r| + |gamma| (|xhat| d_rstd + d_mean rstd + 2^-23 (|x| + |mean|) rstd).
A one-pass variance (sum of squares minus mean^2) loses about 2^-24 (|mean| / sd)^2 of relative variance even when the sums are exact,
which shows against d_mean only where |xhat| |mean| / sd exceeds roughly 4 sqrt(C).  With bf16 rows the fp32 sums are nearly exact, so
at 30 sigma a one-pass kernel stays inside this bound (measured on an fp32 emulation); at 300 sigma it does not.  So every LayerNorm
width also runs on the device with row offsets up to 300 sigma, and the CPU teeth test runs both emulations on those shapes: the
two-pass one passes at 30 and 300 sigma, the one-pass one fails at 300 sigma, where the census bound (which prices the one-pass term in)
still accepts it."""
import ctypes as C
import math
import time
import zlib

import pytest
import torch

from kernel_check import (C_ACC, EPS24, TAIL, U_BF16, Replay, addr, argworst, determinism, ladi_lib, launches, layout, norm_expect, override,
                          plan_query, ratio, sms, twice)

EPS = 1e-6


GN_FIELDS = ("chunks", "gsplit", "block_channels", "lanes_v", "k", "px_per_chunk", "px_per_block", "apply_blocks", "dv", "dp", "slices")


def gn_args(c0, c1, n, hw, groups, **kw):
    """The arguments of ladi_groupnorm_apply (without the stream) on fake 256-byte aligned addresses; kw overrides by name, *_off adds
    a byte offset to a pointer."""
    return override(dict(x0=addr(1), c0=c0, pitch0=c0, x1=addr(2) if c1 else None, c1=c1, pitch1=c1, n=n, hw=hw, groups=groups,
                          ws=addr(3), gamma=addr(4), beta=addr(5), eps=EPS, silu=1, add=None, add_pitch=0, out=addr(6),
                          out_pitch=c0 + c1), kw)


_GN_ORDER = ("x0", "c0", "pitch0", "x1", "c1", "pitch1", "n", "hw", "groups", "ws", "gamma", "beta", "eps", "silu", "add", "add_pitch", "out",
             "out_pitch")


def gn_query(a, sms):
    """-> (plan dict, "") or (None, error message)."""
    return plan_query("ladi_groupnorm_plan", ladi_lib().GroupNormPlan, [a[k] for k in _GN_ORDER] + [sms], GN_FIELDS)


def gn_plan(c0, c1, n, hw, groups, sms, **kw):
    p, err = gn_query(gn_args(c0, c1, n, hw, groups, **kw), sms)
    assert p is not None, err
    return p


_LN_ORDER = ("x", "x_pitch", "rows", "c", "gamma", "beta", "eps", "out", "out_pitch")


def ln_args(rows, c, **kw):
    return override(dict(x=addr(1), x_pitch=c, rows=rows, c=c, gamma=addr(2), beta=addr(3), eps=1e-5, out=addr(4), out_pitch=c), kw)


def ln_query(a):
    return plan_query("ladi_layernorm_plan", ladi_lib().LayerNormPlan, [a[k] for k in _LN_ORDER] + [0], ("T", "vpl", "rows_per_block", "blocks"))


# ================================================================================================================ CPU: plan tables
# (c0, c1, n, hw, groups) -> plan at 132 SMs and at 114 SMs, fields in GN_FIELDS order.  The gsplit doubling stops when the stats grid
# (chunks x n x gsplit) reaches 2 x SMs, when groups are not divisible by the next split, or when a split's channels are not a multiple
# of 8; apply takes max(4096 / (C / 8), ceil(hw / ceil(3 SMs / n))) pixels per block.
GN_TABLE = [
    ("gsplit1 grid", (320, 0, 16, 3072, 32), (48, 1, 320, 40, 6, 64, 123, 25, 16, 6, 8), (48, 1, 320, 40, 6, 64, 140, 22, 16, 6, 8)),
    ("gsplit4 grid", (320, 0, 2, 3072, 32), (48, 4, 80, 10, 25, 64, 102, 31, 16, 6, 8), (48, 4, 80, 10, 25, 64, 102, 31, 16, 6, 8)),
    ("gsplit2 at 132, 1 at 114", (320, 0, 16, 960, 32), (15, 2, 160, 20, 12, 64, 102, 10, 16, 6, 8), (15, 1, 320, 40, 6, 64, 102, 10, 16, 6, 8)),
    ("gsplit16 two sources", (1280, 640, 16, 48, 32), (1, 16, 120, 15, 17, 48, 17, 3, 16, 1, 8), (1, 16, 120, 15, 17, 48, 17, 3, 16, 1, 8)),
    ("gsplit16 dp0", (2560, 0, 16, 48, 32), (1, 16, 160, 20, 12, 48, 12, 4, 256, 0, 8), (1, 16, 160, 20, 12, 48, 12, 4, 256, 0, 8)),
    ("gsplit8 groups24", (384, 0, 1, 48, 24), (1, 8, 48, 6, 42, 48, 85, 1, 16, 5, 8), (1, 8, 48, 6, 42, 48, 85, 1, 16, 5, 8)),
    ("gsplit8 channels", (320, 0, 1, 48, 32), (1, 8, 40, 5, 51, 48, 102, 1, 16, 6, 8), (1, 8, 40, 5, 51, 48, 102, 1, 16, 6, 8)),
    ("groups48 slices5", (384, 0, 2, 100, 48), (2, 16, 24, 3, 85, 50, 85, 2, 16, 5, 5), (2, 16, 24, 3, 85, 50, 85, 2, 16, 5, 5)),
    ("C8 nv1", (8, 0, 2, 200, 4), (4, 1, 8, 1, 256, 50, 4096, 1, 0, 256, 8), (4, 1, 8, 1, 256, 50, 4096, 1, 0, 256, 8)),
    ("hw 4033", (128, 0, 1, 4033, 32), (64, 8, 16, 2, 128, 64, 256, 16, 0, 16, 8), (64, 4, 32, 4, 64, 64, 256, 16, 0, 16, 8)),
    ("VAE full resolution", (128, 0, 1, 196608, 32), (64, 8, 16, 2, 128, 3072, 497, 396, 0, 16, 8), (64, 4, 32, 4, 64, 3072, 575, 342, 0, 16, 8)),
]


@pytest.mark.parametrize("name,shape,at132,at114", GN_TABLE, ids=[t[0] for t in GN_TABLE])
def test_gn_plan_table(name, shape, at132, at114):
    assert tuple(gn_plan(*shape, 132).values()) == at132
    assert tuple(gn_plan(*shape, 114).values()) == at114


def test_gn_plan_differs_between_132_and_114_sms():
    """The doubling and the apply grid both depend on the SM count: the same shape gets a different plan on a 114-SM part."""
    a, b = gn_plan(320, 0, 16, 960, 32, 132), gn_plan(320, 0, 16, 960, 32, 114)
    assert (a["gsplit"], b["gsplit"]) == (2, 1)  # 15 chunks x 16 images = 240: under 2 x 132, not under 2 x 114
    a, b = gn_plan(320, 0, 16, 3072, 32, 132), gn_plan(320, 0, 16, 3072, 32, 114)
    assert (a["px_per_block"], b["px_per_block"]) == (123, 140)  # ceil(3072 / ceil(3 sms / 16))
    a, b = gn_plan(128, 0, 1, 4033, 32, 132), gn_plan(128, 0, 1, 4033, 32, 114)
    assert (a["gsplit"], b["gsplit"]) == (8, 4)  # 64 chunks x 4 = 256: under 264, not under 228


LN_WIDTHS = [32 * v for v in range(1, 9)] + [320, 384, 448, 512, 640, 768, 896, 1024, 1280, 1536, 1792, 2048]


def _ln_shape(c):
    nv = c // 8
    for t in (4, 8, 16, 32):
        if nv % t == 0 and nv // t <= 8:
            return t, nv // t
    return None


def test_ln_plan_table():
    """All 20 (T, VPL) pairs the dispatcher reaches, and the widths between them it rejects."""
    pairs = set()
    for c in LN_WIDTHS:
        p, err = ln_query(ln_args(1000, c))
        assert p is not None, err
        want_t = 4 if c <= 256 else 8 if c <= 512 else 16 if c <= 1024 else 32
        assert (p["T"], p["vpl"]) == (want_t, c // 8 // want_t), c
        assert p["rows_per_block"] == 8 * 32 // p["T"] and p["blocks"] == -(-1000 // p["rows_per_block"])
        pairs.add((p["T"], p["vpl"]))
    assert len(pairs) == 20
    for c in (40, 264, 576, 1152, 2056):  # C / 8 = 5, 33, 72, 144: no T with VPL <= 8; 2056 > 2048
        p, err = ln_query(ln_args(10, c))
        assert p is None and "layernorm" in err, c


# ================================================================================================================ CPU: placement rules
GN_REJECT = [  # (name, overrides, word the message must contain)
    ("x0 misaligned", dict(x0_off=8), "x0"),
    ("x1 misaligned", dict(x1_off=2), "x1"),
    ("c1 negative", dict(c1=-8, x1=None), "c1"),
    ("pitch0 below c0", dict(pitch0=312), "pitch0"),
    ("pitch1 below c1", dict(pitch1=56), "pitch1"),
    ("n zero", dict(n=0), "n > 0"),
    ("hw zero", dict(hw=0), "hw > 0"),
    ("ws null", dict(ws=None), "ws"),
    ("out misaligned", dict(out_off=8), "out"),
    ("add misaligned", dict(add=addr(7, 8), add_pitch=384), "add"),
    ("add_pitch odd", dict(add=addr(7), add_pitch=385), "add_pitch"),
    ("add_pitch below C", dict(add=addr(7), add_pitch=376), "add_pitch"),
    ("gamma null", dict(gamma=None), "gamma"),
    ("beta null", dict(beta=None), "beta"),
    ("out_pitch below C", dict(out_pitch=376), "out_pitch"),
]


@pytest.mark.parametrize("name,kw,word", GN_REJECT, ids=[r[0] for r in GN_REJECT])
def test_gn_placement_rejected(name, kw, word):
    p, err = gn_query(override(gn_args(320, 64, 2, 100, 32), kw), 132)
    assert p is None, f"{name}: accepted"
    assert word in err, err


GN_ACCEPT = [
    ("x1 unaligned but unused", dict(c1=0, x1=addr(2, 2), pitch1=0)),
    ("gamma / beta 4-byte aligned (scalar loads)", dict(gamma_off=4, beta_off=12)),
    ("add aligned, wider pitch", dict(add=addr(7, 16), add_pitch=400)),
    ("pitches above the widths", dict(pitch0=328, pitch1=72, out_pitch=400)),
    ("add_pitch ignored without add", dict(add_pitch=3)),
]


@pytest.mark.parametrize("name,kw", GN_ACCEPT, ids=[r[0] for r in GN_ACCEPT])
def test_gn_placement_accepted(name, kw):
    p, err = gn_query(override(gn_args(320, 64, 2, 100, 32), kw), 132)
    assert p is not None, err


LN_REJECT = [
    ("x misaligned", dict(x_off=8), "x "),
    ("out misaligned", dict(out_off=2), "out"),
    ("gamma misaligned", dict(gamma_off=4), "gamma"),
    ("beta misaligned", dict(beta_off=8), "beta"),
    ("x_pitch below C", dict(x_pitch=312), "x_pitch"),
    ("x_pitch not a multiple of 8", dict(x_pitch=324), "x_pitch"),
    ("out_pitch not a multiple of 8", dict(out_pitch=332), "out_pitch"),
    ("out_pitch below C", dict(out_pitch=312), "out_pitch"),
    ("rows zero", dict(rows=0), "rows"),
    ("gamma null", dict(gamma=None), "gamma"),
]


@pytest.mark.parametrize("name,kw,word", LN_REJECT, ids=[r[0] for r in LN_REJECT])
def test_ln_placement_rejected(name, kw, word):
    p, err = ln_query(override(ln_args(100, 320), kw))
    assert p is None, f"{name}: accepted"
    assert word in err, err


def test_ln_placement_accepted():
    for kw in (dict(x_pitch=328, out_pitch=960), dict(x_off=16, out_off=48, gamma_off=16, beta_off=32)):
        p, err = ln_query(ln_args(100, 320, **kw))
        assert p is not None, (kw, err)


# ================================================================================================================ CPU: the checkers have teeth
def _gn_data(g, hw, C, groups, offset=3.0, sentinels=True):
    """bf16 [hw, C]: per-group mean and scale, sentinel pixels at every chunk's first (+6 sigma) and last (-5 sigma) pixel and at hw - 1."""
    cpg = C // groups
    s = torch.exp(torch.randn(groups, generator=g, dtype=torch.float64) * 0.5)
    mu = s * (torch.rand(groups, generator=g, dtype=torch.float64) * 2 - 1) * offset
    z = torch.randn((hw, C), generator=g, dtype=torch.float64)
    if sentinels:
        chunks = ladi_lib().load().ladi_groupnorm_chunks(hw)
        per = -(-hw // chunks)
        for c in range(chunks):
            p0, p1 = c * per, min(hw, (c + 1) * per)
            if p0 < hw:
                z[p0] = 6.0
                z[p1 - 1] = -5.0
        z[hw - 1] = -5.0
    gi = torch.arange(C) // cpg
    return (mu[gi] + s[gi] * z).bfloat16()


def _emulate_gn(x, groups, gamma, beta, eps, silu, add=None, fault=None):
    """fp32 emulation of gn_stats_kernel + gn_apply_kernel for one image: per-chunk {sum, sum of squares} per channel, folded per group
    and over chunks, one-pass variance, y = x a + b (a = rstd gamma, b = beta - mean a), SiLU as h (1 + tanh h), then + add."""
    hw, Cc = x.shape
    cpg = Cc // groups
    chunks = ladi_lib().load().ladi_groupnorm_chunks(hw)
    per = -(-hw // chunks)
    xf = x.float()
    grp = torch.arange(Cc) // cpg
    if fault == "straddle":  # a 16-byte vector that spans two groups counted wholly in the group of its first channel
        grp = (torch.arange(Cc) // 8 * 8) // cpg
    s = torch.zeros(groups, dtype=torch.float32)
    q = torch.zeros(groups, dtype=torch.float32)
    for c in range(chunks):
        p0, p1 = c * per, min(hw, (c + 1) * per)
        if fault == "drop_last" and c == chunks - 1:
            p1 -= 1  # the last pixel of the ragged last chunk never loaded
        if fault == "twice" and c == 0:
            p1 += 1  # the first pixel of chunk 1 also counted in chunk 0
        blk = xf[p0:p1]
        cs, cq = blk.sum(0), (blk * blk).sum(0)
        s = s + torch.zeros(groups).index_add_(0, grp, cs)
        q = q + torch.zeros(groups).index_add_(0, grp, cq)
    cnt = float(hw * cpg)
    mean = s / cnt
    var = torch.clamp(q / cnt - mean * mean, min=0.0)
    rstd = torch.rsqrt(var + eps)
    a = rstd[torch.arange(Cc) // cpg] * gamma
    b = beta - mean[torch.arange(Cc) // cpg] * a
    y = xf * a + b
    if fault == "add_first" and add is not None:
        y = y + add.float()
    if silu:
        h = 0.5 * y
        y = h * torch.tanh(h) + h
    if add is not None and fault != "add_first":
        y = y + add.float()
    return y.bfloat16()


def _gn_ref(x, groups, gamma, beta, eps, silu, add=None):
    hw, Cc = x.shape
    xd = x.double()
    xg = xd.view(hw, groups, Cc // groups)
    mean = xg.mean(dim=(0, 2), keepdim=True).expand_as(xg).reshape(hw, Cc)
    var = xg.var(dim=(0, 2), unbiased=False, keepdim=True).expand_as(xg).reshape(hw, Cc)
    return norm_expect(xd, mean, var, gamma.double(), beta.double(), eps, hw * Cc // groups, silu, add.double() if add is not None else None)


def _gn_teeth_case(seed, hw=65, Cc=48, groups=4):
    g = torch.Generator().manual_seed(seed)
    x = _gn_data(g, hw, Cc, groups)
    gamma = 1.0 + 0.25 * torch.randn(Cc, generator=g)
    beta = 0.25 * torch.randn(Cc, generator=g)
    add = torch.randn((hw, Cc), generator=g).bfloat16()
    return x, gamma, beta, add


@pytest.mark.parametrize("silu", [0, 1])
def test_gn_checker_accepts_honest_emulation(silu):
    for seed, (hw, Cc, G) in enumerate([(65, 48, 4), (4033, 64, 32), (63, 120, 2), (1, 32, 32)]):
        x, gamma, beta, add = _gn_teeth_case(seed, hw, Cc, G)
        for a in (None, add):
            r, bound = _gn_ref(x, G, gamma, beta, EPS, silu, a)
            assert float(ratio(_emulate_gn(x, G, gamma, beta, EPS, silu, a), r, bound).max()) <= 1.0, (hw, Cc, G)


@pytest.mark.parametrize("fault", ["straddle", "drop_last", "twice", "add_first"])
def test_gn_checker_rejects_faults(fault):
    """cpg = 12 (vectors straddle groups), hw = 65 (two chunks of 33 and 32 pixels: a ragged last chunk)."""
    x, gamma, beta, add = _gn_teeth_case(7)
    a = add if fault == "add_first" else None
    r, bound = _gn_ref(x, 4, gamma, beta, EPS, 1, a)
    assert float(ratio(_emulate_gn(x, 4, gamma, beta, EPS, 1, a), r, bound).max()) <= 1.0
    assert float(ratio(_emulate_gn(x, 4, gamma, beta, EPS, 1, a, fault=fault), r, bound).max()) > 1.0


def ln_expect(x, gamma, beta, eps):
    """x [rows, C] float64 -> (r, bound) for the two-pass LayerNorm (module docstring)."""
    Cc = x.shape[-1]
    mean = x.mean(-1, keepdim=True)
    var = x.var(-1, unbiased=False, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + eps)
    xhat = (x - mean) * rstd
    r = xhat * gamma + beta
    delta = C_ACC * math.sqrt(Cc) * EPS24
    d_mean = delta * (mean.abs() + var.sqrt())
    d_rstd = 1.5 * (delta + 2.0 ** -23 + d_mean * d_mean / (var + eps)) + 2.0 ** -22
    e = gamma.abs() * (xhat.abs() * d_rstd + d_mean * rstd + 2.0 ** -23 * (x.abs() + mean.abs()) * rstd)
    return r, U_BF16 * r.abs() + e


def _ln_data(g, rows, c, max_offset=30.0, dev="cpu"):
    """bf16 rows with per-row scale and offsets up to max_offset sigma (the last row at exactly max_offset)."""
    s = torch.exp(torch.randn((rows, 1), generator=g, device=dev) * 0.5)
    off = (torch.rand((rows, 1), generator=g, device=dev) * 2 - 1) * max_offset
    off[-1] = max_offset
    return (s * (off + torch.randn((rows, c), generator=g, device=dev))).bfloat16()


def _ln_affine(g, c, dev="cpu"):
    # beta of a few units: many outputs near zero at |xhat| ~ 2, where an rstd error is not hidden under the output rounding
    return 1.0 + 0.25 * torch.randn(c, generator=g, device=dev), 1.5 * torch.randn(c, generator=g, device=dev)


def _emulate_ln(x, gamma, beta, eps, one_pass=False):
    """fp32 emulation of layernorm_kernel: T lanes per row, lane tl holds vectors tl + T j, sequential per-lane sums, xor butterfly."""
    rows, c = x.shape
    T, vpl = _ln_shape(c)
    f = x.float().view(rows, vpl, T, 8).permute(0, 2, 1, 3).reshape(rows, T, vpl * 8)  # [row, lane, the lane's elements in order]

    def lane_reduce(v):
        acc = torch.zeros((rows, T))
        for i in range(v.shape[2]):
            acc = acc + v[:, :, i]
        o = T // 2
        while o:
            acc = acc + acc[:, torch.arange(T) ^ o]
            o //= 2
        return acc[:, :1]

    mean = lane_reduce(f) / c
    if one_pass:
        var = lane_reduce(f * f) / c - mean * mean
    else:
        d = f - mean[:, :, None]
        var = lane_reduce(d * d) / c
    rstd = torch.rsqrt(var + eps)
    y = (x.float() - mean) * rstd * gamma + beta
    return y.bfloat16()


@pytest.mark.parametrize("c", LN_WIDTHS)
def test_ln_checker_teeth(c):
    """On the shapes of test_layernorm_every_width (2 rows per block + 5): the two-pass emulation passes ln_expect at row offsets up to 30
    and 300 sigma; the one-pass form fails it at 300 sigma, where the census's one-pass bound still accepts it."""
    T, _ = _ln_shape(c)
    rows = 2 * (8 * 32 // T) + 5
    for off in (30.0, 300.0):
        g = torch.Generator().manual_seed(c)
        x = _ln_data(g, rows, c, max_offset=off)
        gamma, beta = _ln_affine(g, c)
        r, bound = ln_expect(x.double(), gamma.double(), beta.double(), 1e-5)
        assert float(ratio(_emulate_ln(x, gamma, beta, 1e-5), r, bound).max()) <= 1.0, off
    one = _emulate_ln(x, gamma, beta, 1e-5, one_pass=True)  # at 300 sigma
    assert float(ratio(one, r, bound).max()) > 1.0
    xd = x.double()
    mean, var = xd.mean(1, keepdim=True).expand_as(xd), xd.var(1, unbiased=False, keepdim=True).expand_as(xd)
    r1, b1 = norm_expect(xd, mean, var, gamma.double(), beta.double(), 1e-5, c, False)
    assert float(ratio(one, r1, b1).max()) <= 1.0


# ================================================================================================================ GPU: GroupNorm


def _gn_inputs(R, n, hw, c0, c1, groups, offset):
    """Per-image _gn_data on the device (the same construction), split into the two sources."""
    g = torch.Generator().manual_seed(int(torch.randint(0, 1 << 30, (1,), generator=R.g, device=R.dev)))
    x = torch.cat([_gn_data(g, hw, c0 + c1, groups, offset) for _ in range(n)]).to(R.dev)
    return x[:, :c0], x[:, c0:]


def run_gn(R, c0, c1, n, hw, groups, silu=1, add=False, offset=3.0, expect=None):
    """One GroupNorm call (stats + apply) checked as the module docstring says; -> worst err/bound."""
    lib = ladi_lib()
    L = lib.load()
    Ct = c0 + c1
    p0, p1, op, ap = c0 + 8, c1 + 24 if c1 else 0, Ct + 16, Ct + 40  # distinct pitches, all with NaN gaps
    v0, v1 = _gn_inputs(R, n, hw, c0, c1, groups, offset)
    x0 = R.poisoned(n * hw, p0, v0)
    x1 = R.poisoned(n * hw, p1, v1) if c1 else None
    gamma, beta = 1.0 + R.randn(Ct, std=0.25), R.randn(Ct, std=0.25)
    addt = R.poisoned(n * hw, ap, R.randn(n * hw, Ct)) if add else None
    P = lambda t: t.data_ptr() if t is not None else None
    chunks = L.ladi_groupnorm_chunks(hw)
    plan = None

    def call(b):
        nonlocal plan
        a = dict(x0=P(x0), c0=c0, pitch0=p0, x1=P(x1), c1=c1, pitch1=p1, n=n, hw=hw, groups=groups, ws=P(b["ws"]), gamma=P(gamma), beta=P(beta),
                 eps=EPS, silu=silu, add=P(addt), add_pitch=ap if add else 0, out=P(b["out"]), out_pitch=op)
        plan, err = gn_query(a, 0)  # what runs on this device
        assert plan is not None, err
        if expect:  # the branch the shape reaches on a 132-SM H100 SXM, asserted on any device; there, it is also what runs
            p132, _ = gn_query(a, 132)
            assert {k: p132[k] for k in expect} == expect, f"plan at 132 SMs {p132}, expected {expect}"
            if sms(R.dev) == 132:
                assert plan == p132
        lib.call("ladi_groupnorm_stats", P(x0), c0, p0, P(x1), c1, p1, n, hw, groups, P(b["ws"]), R.stream)
        lib.call("ladi_groupnorm_apply", *[a[k] for k in _GN_ORDER], R.stream)
    runs = twice(call, lambda: dict(ws=torch.full((n * chunks * groups * 2,), float("nan"), dtype=torch.float32, device=R.dev),
                                    out=R.poisoned(n * hw + TAIL, op)))
    out = runs[0]["out"]
    errs = layout(out, 0, Ct, "output", rows=n * hw)
    assert not errs, errs
    errs = determinism(runs, ["out"])
    assert not errs, errs
    worst = 0.0
    for b in range(n) if n * hw * Ct <= 1 << 26 else (0, n - 1):
        xb = torch.cat([v0[b * hw:(b + 1) * hw], v1[b * hw:(b + 1) * hw]], dim=1) if c1 else v0[b * hw:(b + 1) * hw]
        ab = addt[b * hw:(b + 1) * hw, :Ct] if add else None
        r, bound = _gn_ref(xb, groups, gamma, beta, EPS, silu, ab)
        qm, (p, c) = argworst(ratio(out[b * hw:(b + 1) * hw, :Ct], r, bound))
        if qm > 1.0:
            pytest.fail(f"image {b}: err/bound {qm:.3g} at pixel {p}, channel {c} (group {c // (Ct // groups)}); plan {plan}")
        worst = max(worst, qm)
    return worst


# (name, (c0, c1, n, hw, groups), options, plan fields expected at 132 SMs)
GN_CASES = [
    # the group split: each value, and each reason the doubling stops
    ("gsplit1", (320, 0, 16, 3072, 32), {}, dict(gsplit=1, px_per_block=123)),
    ("gsplit2", (320, 0, 16, 960, 32), {}, dict(gsplit=2, chunks=15)),
    ("gsplit4 grid full", (320, 0, 2, 3072, 32), {}, dict(gsplit=4, px_per_block=102, apply_blocks=31)),
    ("gsplit8 groups24", (384, 0, 1, 48, 24), {}, dict(gsplit=8, block_channels=48)),
    ("gsplit8 channels not x8", (320, 0, 1, 48, 32), {}, dict(gsplit=8, block_channels=40)),
    ("gsplit16 crosses x0/x1", (1280, 640, 16, 48, 32), {}, dict(gsplit=16, block_channels=120, dv=16, dp=1)),
    ("gsplit16 dp0", (2560, 0, 16, 48, 32), {}, dict(gsplit=16, dp=0, dv=256)),
    # channels per group: straddling vectors, fewer than 8, groups across the x0 / x1 boundary
    ("cpg60 straddles x0/x1", (1280, 640, 2, 96, 32), {}, dict(block_channels=120)),
    ("cpg30 straddles x0/x1", (640, 320, 2, 96, 32), {}, dict(gsplit=8, block_channels=120)),  # 960 / 16 = 60: not whole vectors
    ("cpg20", (640, 0, 2, 96, 32), {}, dict(gsplit=16, block_channels=40)),
    ("cpg12 straddles x0/x1", (256, 128, 2, 96, 32), {}, dict(gsplit=16, block_channels=24)),
    ("cpg4", (128, 0, 2, 200, 32), {}, dict(gsplit=16, block_channels=8, lanes_v=1, k=256)),
    ("cpg2", (64, 0, 2, 200, 32), {}, dict(gsplit=8, block_channels=8)),
    ("cpg1", (32, 0, 2, 200, 32), {}, dict(gsplit=4, block_channels=8)),
    ("groups1", (64, 0, 2, 200, 1), {}, dict(gsplit=1, slices=8)),
    ("groups64", (128, 0, 2, 200, 64), {}, dict(gsplit=16, slices=4)),
    ("groups48 slices5", (384, 0, 2, 100, 48), {}, dict(slices=5)),
    # pixel chunks
    ("hw1", (320, 0, 2, 1, 32), {}, dict(chunks=1, px_per_chunk=1, apply_blocks=1)),
    ("hw63", (320, 0, 2, 63, 32), {}, dict(chunks=1, px_per_chunk=63)),
    ("hw64", (320, 0, 2, 64, 32), {}, dict(chunks=1, px_per_chunk=64)),
    ("hw65", (320, 0, 2, 65, 32), {}, dict(chunks=2, px_per_chunk=33)),
    ("hw4032", (128, 0, 2, 4032, 32), {}, dict(chunks=63, px_per_chunk=64)),
    ("hw4033 last chunk 1 pixel", (128, 0, 2, 4033, 32), {}, dict(chunks=64, px_per_chunk=64)),
    ("VAE full resolution", (128, 0, 1, 196608, 32), {}, dict(chunks=64, px_per_chunk=3072)),
    # pixels per stats thread (k = 1 pixel lane): counts 64..71, i.e. 0 mod 8, the predicated batch of 4 alone (1-3), and 4 + 1-3
    *[(f"per-thread count {c}", (1280, 0, 5, 64 * c, 32), {}, dict(gsplit=1, k=1, px_per_chunk=c)) for c in (64, 65, 66, 67, 69, 70, 71)],
    # apply grid
    ("apply single block", (320, 0, 1, 48, 32), {}, dict(apply_blocks=1, px_per_block=102)),
    ("apply ragged last block", (320, 0, 2, 3100, 32), {}, dict(px_per_block=102, apply_blocks=31)),
    ("apply C8 nv1", (8, 0, 2, 200, 4), {}, dict(dv=0, dp=256, px_per_block=4096, apply_blocks=1)),
    ("apply nv 240", (1920, 0, 2, 500, 32), {}, dict(dv=16, dp=1)),
    ("apply nv 320", (2560, 0, 2, 300, 32), {}, dict(dv=256, dp=0)),
    # the add operand (its own pitch), with and without SiLU, two sources with three distinct pitches
    ("add silu", (512, 0, 2, 300, 32), dict(add=True, silu=1), {}),
    ("add no silu", (512, 0, 2, 300, 32), dict(add=True, silu=0), {}),
    ("add two sources", (256, 256, 2, 300, 32), dict(add=True, silu=1), dict(gsplit=16)),
    ("no silu", (1280, 640, 3, 96, 32), dict(silu=0), {}),
]


@pytest.mark.gpu
@pytest.mark.parametrize("name,shape,opt,expect", GN_CASES, ids=[c[0] for c in GN_CASES])
def test_groupnorm_schedule(cuda, name, shape, opt, expect):
    t0 = time.time()
    worst = run_gn(Replay(cuda, zlib.crc32(name.encode()) & 0xFFFF), *shape, expect=expect, **opt)
    print(f"\n{name}: worst err/bound {worst:.3g} ({time.time() - t0:.2f} s)")


@pytest.mark.gpu
def test_groupnorm_one_pass_characterisation(cuda):
    """|mean| / sigma = 30 over 786432 values per group (C 128, 32 groups, the VAE's full resolution): the one-pass fp32 variance
    against the census bound, whose mean^2 / var term prices it in."""
    worst = run_gn(Replay(cuda, 30), 128, 0, 1, 196608, 32, offset=30.0)
    print(f"\nGroupNorm at |mean|/sigma 30, 786432 values per group: worst err/bound {worst:.3g}")


# ================================================================================================================ GPU: LayerNorm
def run_ln(R, rows, c, expect=None, max_offset=30.0):
    lib = ladi_lib()
    xp, op = c + 24, c + 8
    g = torch.Generator(device=R.dev).manual_seed(rows * 4099 + c)
    xv = _ln_data(g, rows, c, max_offset=max_offset, dev=R.dev)
    gamma, beta = _ln_affine(g, c, dev=R.dev)
    x = R.poisoned(rows, xp, xv)
    plan = None

    def call(b):
        nonlocal plan
        a = ln_args(rows, c, x=x.data_ptr(), x_pitch=xp, gamma=gamma.data_ptr(), beta=beta.data_ptr(), out=b["out"].data_ptr(), out_pitch=op)
        plan, err = ln_query(a)
        assert plan is not None, err
        if expect:
            assert {k: plan[k] for k in expect} == expect, f"plan {plan}, expected {expect}"
        lib.call("ladi_layernorm", a["x"], xp, rows, c, a["gamma"], a["beta"], a["eps"], a["out"], op, R.stream)
    runs = twice(call, lambda: dict(out=R.poisoned(rows + TAIL, op)))
    errs = layout(runs[0]["out"], 0, c, "output", rows=rows)
    assert not errs, errs
    errs = determinism(runs, ["out"])
    assert not errs, errs
    r, bound = ln_expect(xv.double(), gamma.double(), beta.double(), 1e-5)
    worst, (i, j) = argworst(ratio(runs[0]["out"][:rows, :c], r, bound))
    if worst > 1.0:
        pytest.fail(f"err/bound {worst:.3g} at row {i}, column {j}; plan {plan}")
    return worst


@pytest.mark.gpu
@pytest.mark.parametrize("offset", [30.0, 300.0])
@pytest.mark.parametrize("c", LN_WIDTHS)
def test_layernorm_every_width(cuda, c, offset):
    """Row offsets up to 30 sigma, and up to 300 sigma, where a one-pass variance would leave ln_expect at every width (the CPU test
    test_ln_checker_teeth runs the one-pass emulation on these shapes)."""
    T, vpl = _ln_shape(c)
    rpb = 8 * 32 // T
    worst = run_ln(Replay(cuda, c), 2 * rpb + 5, c, expect=dict(T=T, vpl=vpl, rows_per_block=rpb), max_offset=offset)
    print(f"\nLayerNorm C {c} (T {T}, VPL {vpl}), offsets up to {offset:g} sigma: worst err/bound {worst:.3g}")


LN_ROWS = {"1": lambda rpw, rpb, s: 1, "rpw-1": lambda rpw, rpb, s: max(1, rpw - 1), "rpw+1": lambda rpw, rpb, s: rpw + 1,
           "rpb-1": lambda rpw, rpb, s: rpb - 1, "rpb+1": lambda rpw, rpb, s: rpb + 1, "waves": lambda rpw, rpb, s: rpb * 9 * s + 7}


@pytest.mark.gpu
@pytest.mark.parametrize("rows", list(LN_ROWS))
@pytest.mark.parametrize("c", [96, 448, 640, 2048])  # T = 4, 8, 16, 32
def test_layernorm_row_counts(cuda, c, rows):
    T, _ = _ln_shape(c)
    rpw, rpb = 32 // T, 8 * 32 // T
    n = LN_ROWS[rows](rpw, rpb, sms(cuda))
    worst = run_ln(Replay(cuda, n), n, c, expect=dict(T=T, blocks=-(-n // rpb)))
    print(f"\nLayerNorm C {c}, {n} rows: worst err/bound {worst:.3g}")


# ================================================================================================================ GPU: placement


GN_GPU_REJECT = [("x0 misaligned", "x0", 8), ("x1 misaligned", "x1", 8), ("out misaligned", "out", 8), ("add misaligned", "add", 8),
                 ("pitch0 below c0", "pitch0", None)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,what,off", GN_GPU_REJECT, ids=[r[0] for r in GN_GPU_REJECT])
def test_groupnorm_placement_rejected_on_device(cuda, name, what, off):
    """The query rejects the placement first; only then do the launching calls see it, and they return the same error, launch nothing
    and leave the output NaN."""
    L = ladi_lib().load()
    n, hw, c0, c1, G = 2, 100, 256, 64, 32
    R = Replay(cuda, 5)
    x0 = R.poisoned(n * hw + 1, c0 + 8, R.randn(n * hw + 1, c0))
    x1 = R.poisoned(n * hw + 1, c1 + 8, R.randn(n * hw + 1, c1))
    addt = R.poisoned(n * hw + 1, c0 + c1, R.randn(n * hw + 1, c0 + c1))
    ws = torch.full((n * 2 * G * 2,), float("nan"), device=cuda)
    gamma, beta = torch.ones(c0 + c1, device=cuda), torch.zeros(c0 + c1, device=cuda)
    o = R.poisoned(n * hw + 1, c0 + c1)
    a = dict(x0=x0.data_ptr(), c0=c0, pitch0=c0 + 8, x1=x1.data_ptr(), c1=c1, pitch1=c1 + 8, n=n, hw=hw, groups=G, ws=ws.data_ptr(),
             gamma=gamma.data_ptr(), beta=beta.data_ptr(), eps=EPS, silu=1, add=addt.data_ptr(), add_pitch=c0 + c1, out=o.data_ptr(),
             out_pitch=c0 + c1)
    if off is None:
        a["pitch0"] = c0 - 8
    else:
        a[what] += off
    plan, err = gn_query(a, 0)
    assert plan is None and what in err, (plan, err)
    before = launches()
    if what in ("x0", "x1", "pitch0"):
        assert L.ladi_groupnorm_stats(a["x0"], c0, a["pitch0"], a["x1"], c1, a["pitch1"], n, hw, G, a["ws"], None) == 1
        assert L.ladi_last_error().decode() == err
    assert L.ladi_groupnorm_apply(*[a[k] for k in _GN_ORDER], None) == 1
    assert L.ladi_last_error().decode() == err
    torch.cuda.synchronize()
    assert launches() == before
    assert bool(torch.isnan(o.float()).all())


LN_GPU_REJECT = [("x misaligned", "x"), ("out misaligned", "out"), ("gamma misaligned", "gamma"), ("beta misaligned", "beta")]


@pytest.mark.gpu
@pytest.mark.parametrize("name,what", LN_GPU_REJECT, ids=[r[0] for r in LN_GPU_REJECT])
def test_layernorm_placement_rejected_on_device(cuda, name, what):
    L = ladi_lib().load()
    rows, c = 100, 320
    R = Replay(cuda, 6)
    x = R.poisoned(rows + 1, c, R.randn(rows + 1, c))
    gamma, beta = torch.ones(c + 4, device=cuda), torch.zeros(c + 4, device=cuda)
    o = R.poisoned(rows + 1, c)
    a = ln_args(rows, c, x=x.data_ptr(), gamma=gamma.data_ptr(), beta=beta.data_ptr(), out=o.data_ptr())
    a[what] += 4 if what in ("gamma", "beta") else 8
    plan, err = ln_query(a)
    assert plan is None and what in err, (plan, err)
    before = launches()
    assert L.ladi_layernorm(a["x"], c, rows, c, a["gamma"], a["beta"], a["eps"], a["out"], c, None) == 1
    assert L.ladi_last_error().decode() == err
    torch.cuda.synchronize()
    assert launches() == before
    assert bool(torch.isnan(o.float()).all())
