"""The conv/GEMM kernel's schedule, store paths and placement rules, each case asserting which path it runs and checked against float64.

`ladi_conv2d_plan` reports the plan `ladi_conv2d_bf16` runs for a descriptor (N tile, split-K factor, CTA pairs, staged or fragment
epilogue, pipeline stages, tile grid), from the same code that launches it.  Every GPU case below first asserts the plan it means to
exercise -- N tile, splits, pair, store path, and the work-item count relative to the device's SM count -- and then runs the call the way
the workload census replays the workloads (tests/kernel_check.py): input pitch gaps NaN, the output NaN over its full pitch plus tail rows, every
owned element finite and every other still NaN afterwards, a second run bit-identical, and every element within the census's per-element
float64 bound (conv_expect / ratio).

The schedule edges: each CTA is persistent and carries its ring stage and phase from one work item to the next, and the ring depth is
whatever fits in shared memory (BN 32 / 64: 8 stages, 128: 6 staged / 7 fragment, 160: 6, 192: 5, 256: 4).  So the cases put the work-item
count at 1, 2, sms - 1, sms, sms + 1 and 2 sms + 1, and the K-block count at 1, 2, stages - 1, stages, stages + 1 and 2 stages + 1 at one
item and at sms + 1 items (where a CTA's second item starts mid-ring).  Split-K runs at S = 2, at a middle S with a ragged last split and
at the 16-split cap, through every form of the reduce pass; its bound is the census's: the fp32 sum of S <= 16 partials adds at most
S * 2^-24 * sum |partials|, far inside C_ACC * sqrt(K) * 2^-24 * m.

The LayerNorm fold (the producer's per-row, per-32-column statistics and the consumer's rstd * (acc - mean * colsum) + bias) has its own
float64 bounds here, built like the census's: see rowstat_expect and ln_fold_expect.

The CPU tests pin the plan table at 132 and 114 SMs (no device needed: the query dereferences nothing), the placement rules, and show that
the checkers reject six simulated schedule faults and accept an honest fp32 emulation."""
import ctypes as C
import math
import os

import pytest
import torch
import torch.nn.functional as F

from kernel_check import (C_ACC, EPS24, TAIL, addr, attn_expect, attn_ref, conv_expect, cpu_gen, determinism, ladi_lib, layout, max_ratio, nan_buf,
                          plan_query, same, sms, twice)

FORMS = ["bias", "nobias", "stepbias", "rowbias", "silu", "gelu", "relu", "geglu", "residual", "inplace", "rowscale", "fp32"]
SPLIT_FORMS = ["nobias", "bias", "stepbias", "silu", "gelu", "relu", "residual", "inplace"]


# ================================================================================================================ float64 expectations
def gemm_expect(acc, m, K, bcol=None, brow=None, res=None, rs=None, act=0, out_fp32=False):
    """acc = A W^T and m = |A| |W|^T (float64 [rows, c_out]) plus the epilogue operands -> (r, bound) [rows, c_eff] (conv_expect)."""
    pre, mm = acc.clone(), m.clone()
    if bcol is not None:
        pre += bcol
        mm += bcol.abs()
    if brow is not None:
        pre += brow[:, None]
        mm += brow.abs()[:, None]
    if res is not None:
        mm += res.abs()
    return conv_expect(pre, mm, K, act, res, None if rs is None else rs[:, None], out_fp32)


def rowstat_expect(r, e):
    """The producer's row statistics: r float64 [rows, c] (unrounded output, before any bf16 rounding) with per-element error e (the
    kernel's fp32 value differs from r by at most e) -> (sums, sums of squares, their bounds) [rows, c / 32].  The kernel adds the 32
    values of a chunk in fp32 (pairs, then 4 partial sums, then a lane shuffle): at most 32 * 2^-24 * sum |x| on top of the inputs'
    errors, doubled; each value's fp32 epilogue adds (bias, residual) add 2^-22 |x|."""
    rows, c = r.shape
    rc, ec = r.view(rows, c // 32, 32), (e + 2.0 ** -22 * r.abs()).view(rows, c // 32, 32)
    s, q = rc.sum(-1), (rc * rc).sum(-1)
    gam = 2 * 32 * EPS24
    bs = ec.sum(-1) + gam * rc.abs().sum(-1)
    bq = (2 * rc.abs() * ec + ec * ec).sum(-1) + gam * (rc * rc).sum(-1)
    return s, q, bs, bq


def ln_fold_expect(t, wp, colsum, bp, eps, act=0):
    """The LayerNorm-folded GEMM out = rstd * (t Wp^T - mean * colsum) + bp on the folded operands (weights.fold_layernorm):
    t bf16 [rows, C], wp bf16 [N, C], colsum / bp fp32 [N] -> (r, bound) [rows, c_eff].  The pre-activation error carries
      the GEMM's accumulation error             rstd * C_ACC sqrt(C) 2^-24 |t| |Wp|,
      the statistics' error (norm_expect's model of the one-pass fp32 E[x^2] - mean^2: d_mean absolute, d_rstd relative)
                                                rstd |colsum| d_mean + d_rstd |rstd (acc - mean colsum)|,
      the cancellation in fma(-rstd mean, colsum, rstd acc) and the bias add, each an fp32 rounding of its operands
                                                2^-22 rstd (|acc| + |mean colsum|) + 2^-23 |bp|;
    the activation and the output rounding are conv_expect's."""
    C_ = t.shape[1]
    x = t.double()
    mean = x.mean(1, keepdim=True)
    var = (x * x).mean(1, keepdim=True) - mean * mean
    rstd = 1.0 / torch.sqrt(var + eps)
    w64, cs, b64 = wp[:, :C_].double(), colsum.double(), bp.double()
    acc = x @ w64.t()
    core = rstd * (acc - mean * cs)
    pre = core + b64
    delta = C_ACC * math.sqrt(C_) * EPS24
    d_mean = delta * (mean.abs() + var.sqrt())
    d_rstd = 1.5 * delta * (mean * mean + var) / (var + eps) + 2.0 ** -22
    e = (rstd * C_ACC * math.sqrt(C_) * EPS24 * (x.abs() @ w64.abs().t()) + rstd * cs.abs() * d_mean + d_rstd * core.abs()
         + 2.0 ** -22 * rstd * (acc.abs() + (mean * cs).abs()) + 2.0 ** -23 * b64.abs())
    return conv_expect(pre, e / (C_ACC * math.sqrt(C_) * EPS24), C_, act)


# ================================================================================================================ CPU: the plan table


def gemm_desc(M, K, N, **kw):
    """A GEMM descriptor on fake, 256-byte aligned addresses; kw overrides fields (pointer fields take byte offsets via *_off)."""
    lib = ladi_lib()
    d = lib.ConvDesc()
    d.n, d.h_out, d.w_out, d.c_out = 1, 1, M, N
    d.ksize, d.stride, d.pad_lo = 1, 1, 0
    d.n_src, d.src[0], d.src_c[0], d.src_pitch[0] = 1, addr(1), K, (K + 7) // 8 * 8
    kt = (K + 63) // 64 * 64
    d.weight, d.k_total, d.weight_pitch = addr(2), kt, kt
    d.out, d.out_pitch = addr(3), N
    return _fill(d, kw)


def conv_desc(n, h, w, cin, cout, k=3, s=1, **kw):
    lib = ladi_lib()
    d = lib.ConvDesc()
    d.n, d.h_out, d.w_out, d.c_out = n, h, w, cout
    d.h_in, d.w_in = h * s, w * s
    d.ksize, d.stride, d.pad_lo = k, s, 1 if k == 3 else 0
    d.n_src, d.src[0], d.src_c[0], d.src_pitch[0] = 1, addr(1), cin, (cin + 7) // 8 * 8
    kt = k * k * ((cin + 63) // 64 * 64)
    d.weight, d.k_total, d.weight_pitch = addr(2), kt, kt
    d.out, d.out_pitch = addr(3), cout
    return _fill(d, kw)


def _fill(d, kw):
    slots = {"bias": 4, "residual": 5, "splitk_ws": 6, "rowstat_out": 7, "ln_stats": 8, "ln_colsum": 9, "row_scale": 10, "step_ptr": 11}
    for key, v in kw.items():
        if key.endswith("_off"):
            name = key[:-4]
            setattr(d, name, (getattr(d, name) or addr(slots[name])) + v)
        elif key in slots and v is True:
            setattr(d, key, addr(slots[key]))
        else:
            setattr(d, key, v)
    if d.splitk_ws and not d.splitk_ws_bytes:
        d.splitk_ws_bytes = 64 << 20
    if d.residual and not d.residual_pitch:
        d.residual_pitch = d.out_pitch
    return d


def plan_of(d, sms):
    p = ladi_lib().conv_plan(d, sms)
    return dict(bn=p.bn, splits=p.splits, per=p.kb_per_split, pair=bool(p.pair), staged=bool(p.staged), stages=p.stages,
                tiles_m=p.tiles_m, tiles_n=p.tiles_n, kb=p.total_kb, items=p.items())


def rejected(d, sms=132):
    p, err = plan_query("ladi_conv2d_plan", ladi_lib().ConvPlan, [C.byref(d), sms], ())
    return (0, "") if p is not None else (1, err)


no_env_pairs = pytest.mark.skipif(os.environ.get("LADI_CONV_2CTA") == "1", reason="LADI_CONV_2CTA=1 changes the library default")

# (descriptor, sms) -> the plan fields pinned; the N tile / split choices follow choose_plan's cost rule, the stage counts the shared
# memory budget (227 KiB less the staging tile)
PLAN_TABLE = [
    ("gemm 4096x320x320 aligned: BN 128 staged", lambda: gemm_desc(4096, 320, 320), 132,
     dict(bn=128, splits=1, pair=False, staged=True, stages=6, tiles_m=32, tiles_n=3, kb=5)),
    ("same, out_pitch 324: fragment", lambda: gemm_desc(4096, 320, 320, out_pitch=324), 132,
     dict(bn=128, staged=False, stages=7)),
    ("same, fp32 out: fragment", lambda: gemm_desc(4096, 320, 320, out_fp32=1), 132, dict(bn=128, staged=False, stages=7)),
    ("same at 114 SMs", lambda: gemm_desc(4096, 320, 320), 114, dict(bn=128, staged=True, stages=6)),
    ("gemm 1000x320x320: 8 M tiles, BN 32 fills the SMs", lambda: gemm_desc(1000, 1024, 320), 132,
     dict(bn=32, staged=True, stages=8, tiles_m=8, tiles_n=10)),
    ("short K with c_out >= 128: BN 128", lambda: gemm_desc(1000, 512, 320), 132, dict(bn=128, staged=True, tiles_n=3)),
    ("force_bn 32", lambda: gemm_desc(1000, 320, 320, force_bn=32), 132, dict(bn=32, staged=True, stages=8)),
    ("force_bn 64", lambda: gemm_desc(1000, 320, 320, force_bn=64), 132, dict(bn=64, staged=True, stages=8)),
    ("force_bn 64 fragment", lambda: gemm_desc(1000, 320, 320, force_bn=64, out_pitch=324), 132, dict(bn=64, staged=False, stages=8)),
    ("force_bn 160", lambda: gemm_desc(1000, 320, 320, force_bn=160), 132, dict(bn=160, staged=False, stages=6, tiles_n=2)),
    ("force_bn 192", lambda: gemm_desc(1000, 320, 320, force_bn=192), 132, dict(bn=192, staged=False, stages=5, tiles_n=2)),
    ("force_bn 256", lambda: gemm_desc(1000, 320, 320, force_bn=256), 132, dict(bn=256, staged=False, stages=4, tiles_n=2)),
    ("pair forced", lambda: gemm_desc(1000, 320, 320, pair_mode=1, force_bn=128), 132,
     dict(bn=128, pair=True, staged=False, stages=7, tiles_m=8, items=12)),
    ("pair forced, 3 M tiles (a phantom)", lambda: gemm_desc(300, 320, 256, pair_mode=1, force_bn=256), 132,
     dict(bn=256, pair=True, staged=False, stages=4, tiles_m=3, items=2)),
    ("pair forced, library chooses the tile", lambda: gemm_desc(4096, 320, 320, pair_mode=1), 132, dict(bn=128, pair=True)),
    ("pair never", lambda: gemm_desc(4096, 320, 320, pair_mode=2), 132, dict(pair=False, staged=True)),
    ("split-K: 16x8x6 3x3 1280 -> 1280", lambda: conv_desc(16, 8, 6, 1280, 1280, splitk_ws=True), 132,
     dict(bn=256, splits=4, per=45, staged=False, stages=4, tiles_m=6, tiles_n=5, kb=180)),
    ("split-K at 114 SMs", lambda: conv_desc(16, 8, 6, 1280, 1280, splitk_ws=True), 114,
     dict(bn=256, splits=3, per=60, tiles_m=6, tiles_n=5)),
    ("split-K 16-split cap, ragged", lambda: gemm_desc(100, 156 * 64, 256, splitk_ws=True), 132,
     dict(bn=256, splits=16, per=10, kb=156, tiles_m=1, tiles_n=1)),
    ("split-K middle S, ragged", lambda: gemm_desc(2048, 60 * 64, 128, splitk_ws=True), 132, dict(bn=128, splits=7, per=9, kb=60)),
    ("split-K S = 2", lambda: gemm_desc(66 * 128, 33 * 64, 256, splitk_ws=True), 132, dict(bn=256, splits=2, per=17)),
    ("split-K needs total_kb >= 32", lambda: gemm_desc(100, 31 * 64, 256, splitk_ws=True), 132, dict(splits=1)),
    ("split-K not with force_bn", lambda: gemm_desc(100, 156 * 64, 256, splitk_ws=True, force_bn=256), 132, dict(splits=1, bn=256)),
    ("split-K not with a too small workspace", lambda: gemm_desc(100, 156 * 64, 256, splitk_ws=True, splitk_ws_bytes=1 << 20), 132,
     dict(splits=1)),
    ("split-K not for fp32 out", lambda: gemm_desc(100, 156 * 64, 256, splitk_ws=True, out_fp32=1), 132, dict(splits=1)),
    ("up2x 16x12 -> 32x24", lambda: conv_desc(2, 32, 24, 320, 320, up2x=1, k_total=4 * 320), 132,
     dict(bn=32, staged=True, tiles_m=4 * 3, kb=20)),
    ("3x3 at odd W: 128 images per tile", lambda: conv_desc(3, 5, 7, 64, 64), 132, dict(tiles_m=35, kb=9)),
    ("LN-fold consumer: fragment", lambda: gemm_desc(1024, 320, 320, ln_stats=True, ln_colsum=True), 132, dict(staged=False)),
    ("row-statistics producer: fragment", lambda: gemm_desc(1024, 320, 320, rowstat_out=True), 132, dict(staged=False)),
]


@no_env_pairs
@pytest.mark.parametrize("name,make,sms,want", PLAN_TABLE, ids=[p[0] for p in PLAN_TABLE])
def test_plan_table(name, make, sms, want):
    got = plan_of(make(), sms)
    assert {k: got[k] for k in want} == want, got


# alignment rules: (descriptor, expected: None = rejected naming `operand`, else the plan fields)
PLACEMENT_TABLE = [
    # split-K's reduce moves 4 columns at a time: any placement it cannot serve runs unsplit (not an error)
    ("split: out 8-byte aligned", dict(out_off=8), dict(splits=16)),
    ("split: out 4-byte aligned -> unsplit", dict(out_off=4), dict(splits=1)),
    ("split: residual 4-byte aligned -> unsplit", dict(residual=True, residual_off=4), dict(splits=1)),
    ("split: residual 8-byte aligned", dict(residual=True, residual_off=8), dict(splits=16)),
    ("split: bias 8-byte aligned -> unsplit", dict(bias=True, bias_off=8), dict(splits=1)),
    ("split: bias 16-byte aligned", dict(bias=True, bias_off=16), dict(splits=16)),
    ("split: bias_step_stride % 4 != 0 -> unsplit", dict(bias=True, bias_step_stride=258, step_ptr=True), dict(splits=1)),
    ("split: bias_step_stride % 4 == 0", dict(bias=True, bias_step_stride=260, step_ptr=True), dict(splits=16)),
    ("split: workspace 8-byte aligned -> unsplit", dict(splitk_ws_off=8), dict(splits=1)),
    ("split: out_pitch % 4 != 0 -> unsplit", dict(out_pitch=258), dict(splits=1)),
    # what no store path can serve: rejected
    ("bf16 out 2-byte aligned", dict(out_off=2), "out"),
    ("fp32 out 4-byte aligned", dict(out_fp32=1, out_off=4), "out"),
    ("fp32 out 8-byte aligned", dict(out_fp32=1, out_off=8), dict(splits=1, staged=False)),
    ("residual 2-byte aligned", dict(residual=True, residual_off=2), "residual"),
    ("out_pitch below c_out", dict(out_pitch=248), "out_pitch"),
    ("residual_pitch below c_out", dict(residual=True, residual_pitch=252), "residual_pitch"),
    ("source 8-byte aligned", dict(src_off=8), "source 0"),
]


@pytest.mark.parametrize("name,kw,want", PLACEMENT_TABLE, ids=[p[0] for p in PLACEMENT_TABLE])
def test_placement_rules_split(name, kw, want):
    """On the 16-split shape (M 100, K 9984, N 256) at 132 SMs."""
    kw = dict(kw)
    if "src_off" in kw:
        off = kw.pop("src_off")
        d = gemm_desc(100, 156 * 64, 256, splitk_ws=True, **kw)
        d.src[0] += off
    else:
        d = gemm_desc(100, 156 * 64, 256, splitk_ws=True, **kw)
    if isinstance(want, str):
        rc, msg = rejected(d)
        assert rc == 1 and msg.startswith(want), (rc, msg)
    else:
        got = plan_of(d, 132)
        assert {k: got[k] for k in want} == want, got


STAGED_PLACEMENT = [
    ("out 16-byte aligned", dict(out_off=16), True),
    ("out 8-byte aligned -> fragment", dict(out_off=8), False),
    ("out 4-byte aligned -> fragment", dict(out_off=4), False),
    ("out_pitch % 8 == 4 -> fragment", dict(out_pitch=324), False),
    ("odd out_pitch -> fragment", dict(out_pitch=321), False),
    ("residual 16-byte aligned", dict(residual=True, residual_off=16), True),
    ("residual 8-byte aligned -> fragment", dict(residual=True, residual_off=8), False),
    ("residual_pitch % 8 == 4 -> fragment", dict(residual=True, residual_pitch=324), False),
    ("bias 8-byte aligned", dict(bias=True, bias_off=8), True),
    ("bias 4-byte aligned -> fragment", dict(bias=True, bias_off=4), False),
    ("odd bias_step_stride -> fragment", dict(bias=True, bias_step_stride=321, step_ptr=True), False),
    ("row statistics -> fragment", dict(rowstat_out=True), False),
]


@pytest.mark.parametrize("name,kw,staged", STAGED_PLACEMENT, ids=[p[0] for p in STAGED_PLACEMENT])
def test_placement_rules_staged(name, kw, staged):
    """On the staged shape (M 4096, K 320, N 320: BN 128) at 132 SMs; every placement here is valid."""
    got = plan_of(gemm_desc(4096, 320, 320, **kw), 132)
    assert (got["bn"], got["staged"], got["stages"]) == (128, staged, 6 if staged else 7), got


@pytest.mark.parametrize("what", ["ln_stats", "rowstat_out"])
def test_placement_rules_statistics(what):
    ok = dict(ln_stats=16, rowstat_out=8)[what]
    extra = dict(ln_colsum=True) if what == "ln_stats" else {}
    plan_of(gemm_desc(1024, 320, 320, **{what: True, what + "_off": ok}, **extra), 132)
    rc, msg = rejected(gemm_desc(1024, 320, 320, **{what: True, what + "_off": ok // 2}, **extra))
    assert rc == 1 and msg.startswith(what), msg


def _attn_desc(**kw):
    lib = ladi_lib()
    d = lib.AttnDesc()
    d.batch, d.heads, d.nq, d.nkv = 2, 2, 100, 77
    d.q, d.q_pitch, d.q_batch_stride = addr(1), 128, 128 * 100
    d.k, d.k_pitch, d.k_batch_stride = addr(2), 128, 128 * 77
    d.v, d.v_pitch, d.v_batch_stride = addr(3), 128, 128 * 77
    d.out, d.out_pitch, d.out_batch_stride = addr(4), 128, 128 * 100
    d.scale = 0.125
    for k, v in kw.items():
        setattr(d, k, v)
    return d


ATTN_REJECT = {"out 2-byte aligned": ("out", "out"), "odd out_batch_stride": ("out_batch_stride", "out_batch_stride"),
               "out_pitch below the head columns": ("out_pitch", "pitch"), "q 8-byte aligned": ("q", "q 0x"),
               "k_batch_stride not a multiple of 8": ("k_batch_stride", "k_batch_stride")}


@pytest.mark.parametrize("entry", ["ladi_attention_bf16", "ladi_attention_d512_bf16", "plan", "plan wide"])
@pytest.mark.parametrize("name", list(ATTN_REJECT))
def test_attention_placement_rejected(entry, name):
    """Both entry points and their plan query validate before they touch a device, so the rejection is visible here."""
    lib = ladi_lib().load()
    field, word = ATTN_REJECT[name]
    if entry in ("ladi_attention_d512_bf16", "plan wide"):
        cols = 512
        d = _attn_desc(heads=1, head_dim=512, q_pitch=cols, k_pitch=cols, v_pitch=cols, out_pitch=cols, q_batch_stride=cols * 100,
                       k_batch_stride=cols * 77, v_batch_stride=cols * 77, out_batch_stride=cols * 100)
    else:
        cols = 128
        d = _attn_desc()
    if field == "out":
        d.out += 2
    elif field == "q":
        d.q += 8
    elif field == "out_batch_stride":
        d.out_batch_stride += 1
    elif field == "k_batch_stride":
        d.k_batch_stride += 4
    else:
        d.out_pitch = cols // 2
    before = lib.ladi_launch_count()
    if entry.startswith("plan"):
        assert lib.ladi_attention_plan(C.byref(d), int(entry == "plan wide"), 132, C.byref(ladi_lib().AttnPlan())) == 1
    else:
        assert getattr(lib, entry)(C.byref(d), None) == 1
    assert word in lib.ladi_last_error().decode()
    assert lib.ladi_launch_count() == before


# ================================================================================================================ CPU: the checkers have teeth
def _tile_case(seed, M=300, K=640, N=192):
    g = torch.Generator().manual_seed(seed)
    a = torch.randn((M, K), generator=g).bfloat16()
    w = (torch.randn((N, K), generator=g) * K ** -0.5).bfloat16()
    b = torch.randn((N,), generator=g) * 0.5
    acc = a.double() @ w.double().t()
    m = a.double().abs() @ w.double().abs().t()
    return a, w, b, acc, m


def _emulate_tiles(a, w, b, bn=64, splits=1, fault=None):
    """The kernel's schedule in fp32 on the CPU: 128 x bn tiles, each reducing its 64-wide K blocks (in reverse order, an order no float64
    reference uses) into fp32, split-K partials summed in split order, then + bias and one bf16 rounding.  `fault` simulates one mistake."""
    M, K = a.shape
    N, nb = w.shape[0], K // 64
    per = -(-nb // splits)
    y = torch.empty((M, N), dtype=torch.float32)
    for m0 in range(0, M, 128):
        for n0 in range(0, N, bn):
            parts = []
            for sp in range(splits):
                acc = torch.zeros((min(128, M - m0), min(bn, N - n0)))
                kbs = list(range(sp * per, min(nb, (sp + 1) * per)))
                if fault == "drop_last_kb" and (m0, n0) == (128, 64):
                    kbs = kbs[:-1]
                for kb in reversed(kbs):
                    acc += a[m0:m0 + 128, kb * 64:(kb + 1) * 64].float() @ w[n0:n0 + bn, kb * 64:(kb + 1) * 64].float().t()
                parts.append(acc)
            tot = parts[0]
            for p in parts[1:]:
                tot = tot + p
            if fault == "split_twice" and (m0, n0) == (0, 0):
                tot = tot + parts[1]
            y[m0:m0 + 128, n0:n0 + bn] = tot + b[n0:n0 + bn]
    y = y.bfloat16()
    if fault == "tile_shift":  # M tile 1 stored at M tile 2's rows (the last, ragged one)
        y[256:] = y[128:128 + M - 256].clone()
    if fault == "phantom":  # the phantom tile of an odd M-tile count (zero-filled A: bias only) stored into the last real tile
        y[256:] = b.bfloat16()
    return y


def test_gemm_checker_accepts_honest_schedule():
    a, w, b, acc, m = _tile_case(5)
    r, bound = gemm_expect(acc, m, a.shape[1], bcol=b.double())
    for splits in (1, 3, 10):
        assert max_ratio(_emulate_tiles(a, w, b, splits=splits), r, bound) <= 1.0


@pytest.mark.parametrize("fault,splits", [("drop_last_kb", 1), ("tile_shift", 1), ("split_twice", 3), ("phantom", 1)])
def test_gemm_checker_rejects_schedule_faults(fault, splits):
    """1. the last K block dropped from one tile; 2. one tile written at the neighbouring tile's rows; 3. one split's partial counted
    twice; 4. the phantom pair row stored into the last real tile."""
    a, w, b, acc, m = _tile_case(6)
    r, bound = gemm_expect(acc, m, a.shape[1], bcol=b.double())
    assert max_ratio(_emulate_tiles(a, w, b, splits=splits), r, bound) <= 1.0
    assert max_ratio(_emulate_tiles(a, w, b, splits=splits, fault=fault), r, bound) > 1.0


def _ln_case(seed, M=96, Cin=320, N=192, mean=8.0):
    from ladi_vton_b200 import weights
    g = torch.Generator().manual_seed(seed)
    t = (torch.randn((M, Cin), generator=g) + mean + torch.randn((M, 1), generator=g)).bfloat16()
    w = torch.randn((N, Cin), generator=g) * Cin ** -0.5
    gamma, beta, bias = 1 + 0.1 * torch.randn(Cin, generator=g), 0.1 * torch.randn(Cin, generator=g), torch.randn(N, generator=g)
    wp, colsum, bp = weights.fold_layernorm(w, gamma, beta, bias)
    return t, wp, colsum, bp


def _stats_table(t):
    """fp32 {sum, sum of squares} per row and 32-column chunk, as a producer writes it."""
    x = t.float().view(t.shape[0], -1, 32)
    return torch.stack([x.sum(-1), (x * x).sum(-1)], dim=-1).contiguous()


def _emulate_ln_consumer(t, wp, colsum, bp, eps, drop_mean_row=None):
    st = _stats_table(t)
    C_ = t.shape[1]
    s, q = st[..., 0].sum(1, keepdim=True), st[..., 1].sum(1, keepdim=True)
    mean = s / C_
    rstd = torch.rsqrt((q / C_ - mean * mean).clamp_min(0) + eps)
    acc = torch.zeros((t.shape[0], wp.shape[0]))
    for kb in reversed(range(C_ // 64)):
        acc += t[:, kb * 64:(kb + 1) * 64].float() @ wp[:, kb * 64:(kb + 1) * 64].float().t()
    mterm = -rstd * mean * colsum
    if drop_mean_row is not None:
        mterm[drop_mean_row] = 0
    return (rstd * acc + mterm + bp).bfloat16()


def test_ln_checker_teeth():
    """5. the LayerNorm mean term dropped for one row: rejected; the honest fp32 emulation (mean 8 >> std 1): accepted."""
    t, wp, colsum, bp = _ln_case(7)
    r, bound = ln_fold_expect(t, wp, colsum, bp, 1e-5)
    assert max_ratio(_emulate_ln_consumer(t, wp, colsum, bp, 1e-5), r, bound) <= 1.0
    assert max_ratio(_emulate_ln_consumer(t, wp, colsum, bp, 1e-5, drop_mean_row=17), r, bound) > 1.0


def test_rowstat_checker_teeth():
    """6. a row statistic taken from the wrong 32-column chunk: rejected; the honest fp32 sums of the fp32 values: accepted."""
    a, w, b, acc, m = _tile_case(8, K=320, N=256)
    res = (torch.randn(acc.shape, generator=torch.Generator().manual_seed(9)) + 8).bfloat16().double()
    pre = acc + b.double()
    r, bound = gemm_expect(acc, m, a.shape[1], bcol=b.double(), res=res)
    e = bound - 2.0 ** -7 * r.abs()  # the value's error before the output rounding
    s, q, bs, bq = rowstat_expect(pre + res, e)
    y32 = (a.float() @ w.float().t() + b) + res.float()
    honest = _stats_table(y32)
    assert max_ratio(honest[..., 0], s, bs) <= 1.0 and max_ratio(honest[..., 1], q, bq) <= 1.0
    bad = honest.clone()
    bad[5, 2] = honest[5, 3]
    assert max_ratio(bad[..., 0], s, bs) > 1.0 or max_ratio(bad[..., 1], q, bq) > 1.0


# ================================================================================================================ GPU


def _operands(form, rows, c_out, c_eff, dev, seed):
    """(ops kwargs, column bias, row bias, residual bf16 [rows, c_eff], row scale, act, fp32 out) of one epilogue form; float64 copies."""
    from ladi_vton_b200 import ops
    g = cpu_gen(seed)
    act = {"silu": ops.ACT_SILU, "gelu": ops.ACT_GELU, "relu": ops.ACT_RELU, "geglu": ops.ACT_GEGLU}.get(form, ops.ACT_NONE)
    kw, bcol, brow, res, rs = {"act": act}, None, None, None, None
    if form == "stepbias":  # the engine's per-step tables: the row of step 2, at an offset into the table
        table = torch.randn((3 * c_out + 8,), generator=g).to(dev)
        kw.update(bias=table[4:], bias_step_stride=c_out, step_ptr=torch.tensor([2, 0], dtype=torch.int32, device=dev))
        bcol = table[4 + 2 * c_out:4 + 3 * c_out].double()
    elif form == "rowbias":
        brow = torch.randn((rows,), generator=g).to(dev)
        kw.update(bias=brow, bias_per_row=True)
        brow = brow.double()
    elif form != "nobias":
        bcol = (torch.randn((c_out,), generator=g) * 0.5).to(dev)
        kw.update(bias=bcol)
        bcol = bcol.double()
    if form in ("residual", "inplace"):
        res = torch.randn((rows, c_eff), generator=g).to(dev).bfloat16()
    if form == "rowscale":
        rs = torch.rand((rows,), generator=g).to(dev)
        kw.update(row_scale=rs)
        rs = rs.double()
    return kw, bcol, brow, res, rs, act, form == "fp32"


def run_gemm(dev, M, K, N, form="bias", out_pitch=None, expect=None, seed=0, **kw):
    """One GEMM through ops.gemm as described in the module docstring; `expect(plan)` asserts the plan first.  -> (plan, output)."""
    from ladi_vton_b200 import ops, weights
    g = cpu_gen(seed)
    c_eff = N // 2 if form == "geglu" else N
    abuf = nan_buf((M, K + 8), torch.bfloat16, dev)
    abuf[:, :K] = torch.randn((M, K), generator=g).to(dev).bfloat16()
    a = abuf[:, :K]
    w = (torch.randn((N, K), generator=g) * K ** -0.5).bfloat16()
    wp = weights.pack_linear(w.float()).to(dev)
    okw, bcol, brow, res, rs, act, f32 = _operands(form, M, N, c_eff, dev, seed + 1)
    okw.update(kw)
    odt = torch.float32 if f32 else torch.bfloat16
    pitch = out_pitch or c_eff + 8
    rbuf = None
    if res is not None and form != "inplace":
        rbuf = nan_buf((M, pitch), torch.bfloat16, dev)
        rbuf[:, :c_eff] = res

    def fresh():
        buf = nan_buf((M + TAIL, pitch), odt, dev)
        if form == "inplace":
            buf[:M, :c_eff] = res
            return buf, buf[:M, :c_eff]
        return buf, None if rbuf is None else rbuf[:, :c_eff]

    buf, resid = fresh()
    plan = ops.gemm_plan(a, wp, N, out=buf[:M, :c_eff], residual=resid, out_fp32=f32, **okw)
    if expect is not None:
        expect(plan)
    runs = twice(lambda b: ops.gemm(a, wp, N, out=b["out"][:M, :c_eff], residual=b["res"], out_fp32=f32, **okw),
                 lambda: dict(zip(("out", "res"), fresh())))
    outs = [r["out"] for r in runs]
    errs = layout(outs[0], 0, c_eff, "output", rows=M)
    assert not errs, errs
    assert not determinism(runs, ["out"]), "two runs differ bitwise"
    acc = a.double() @ w.to(dev).double().t()
    m = a.double().abs() @ w.to(dev).double().abs().t()
    r, bound = gemm_expect(acc, m, K, bcol, brow, None if res is None else res.double(), rs, act, f32)
    q = max_ratio(outs[0][:M, :c_eff], r, bound)
    assert q <= 1.0, f"err/bound {q:.3g} (plan bn {plan.bn} splits {plan.splits} pair {plan.pair} staged {plan.staged})"
    return plan, outs[0][:M, :c_eff]


def _want(**fields):
    def check(plan):
        got = {k: (plan.items() if k == "items" else getattr(plan, k)) for k in fields}
        assert got == fields, f"plan {got}, want {fields}"
    return check


# ---------------------------------------------------------------------------------------------------------------- items vs SMs
ITEM_COUNTS = {"1": lambda s: 1, "2": lambda s: 2, "sms-1": lambda s: s - 1, "sms": lambda s: s, "sms+1": lambda s: s + 1,
               "2sms+1": lambda s: 2 * s + 1}


@pytest.mark.gpu
@pytest.mark.parametrize("items", list(ITEM_COUNTS))
@pytest.mark.parametrize("path", ["staged128", "fragment256", "pair128"])
def test_items_vs_sms(cuda, path, items):
    """Work items around the persistent grid: a CTA's last item, one item per CTA, one CTA taking a second item, and (pairs) more pairs
    than co-resident clusters.  The last M tile is ragged; pairs run an odd M-tile count (a phantom tile) except at 1 item."""
    T = ITEM_COUNTS[items](sms(cuda))
    if path == "pair128":
        tiles_m = 2 if T == 1 else 2 * T - 1
        M, N, kw = 128 * tiles_m - 40, 128, dict(force_bn=128, pair=True)
        want = _want(bn=128, pair=1, staged=0, splits=1, tiles_m=tiles_m, items=T)
    else:
        bn = 128 if path == "staged128" else 256
        M, N, kw = 128 * T - 40, bn, dict(force_bn=bn)
        want = _want(bn=bn, pair=0, staged=int(bn == 128), splits=1, items=T)
    run_gemm(cuda, M, 5 * 64, N, form="silu", expect=want, seed=T, **kw)


# ---------------------------------------------------------------------------------------------------------------- K depth vs ring depth
DEPTHS = {"1": lambda s: 1, "2": lambda s: 2, "st-1": lambda s: s - 1, "st": lambda s: s, "st+1": lambda s: s + 1, "2st+1": lambda s: 2 * s + 1}
PATHS = {"bn32": (32, True), "bn64": (64, True), "bn128_staged": (128, True), "bn128_fragment": (128, False), "bn160": (160, False),
         "bn192": (192, False), "bn256": (256, False)}


@pytest.mark.gpu
@pytest.mark.parametrize("depth", list(DEPTHS))
@pytest.mark.parametrize("items", ["1", "sms+1"])
@pytest.mark.parametrize("path", list(PATHS))
def test_k_depth(cuda, path, items, depth):
    """K-block counts around the ring depth the query reports, at one work item and at sms + 1 (a CTA's second item starts where the
    first left the ring's stage and phase)."""
    from ladi_vton_b200 import lib
    bn, staged = PATHS[path]
    pitch = bn + 8 if staged else bn + 4  # c_out + 4: rows are not whole 16-byte chunks -> fragment stores
    stages = lib.conv_plan(gemm_desc(1000, 64, bn, force_bn=bn, out_pitch=pitch), sms(cuda)).stages
    assert stages == {32: 8, 64: 8, 128: 6 if staged else 7, 160: 6, 192: 5, 256: 4}[bn]
    kb = DEPTHS[depth](stages)
    T = 1 if items == "1" else sms(cuda) + 1
    run_gemm(cuda, 128 * T - 24, 64 * kb, bn, form="bias", out_pitch=pitch, force_bn=bn, seed=kb,
             expect=_want(bn=bn, staged=int(staged), stages=stages, total_kb=kb, splits=1, pair=0, items=T))


# ---------------------------------------------------------------------------------------------------------------- split-K
def _split_shape(plan_name, sms):
    """(M, K, N) giving S = 2, a middle S with a ragged last split, or the 16-split cap on this device."""
    if plan_name == "S2":
        return (sms // 2) * 128, 33 * 64, 256
    if plan_name == "ragged":
        return 16 * 128, 60 * 64, 128
    return 100, 156 * 64, 256


@pytest.mark.gpu
@pytest.mark.parametrize("form", SPLIT_FORMS)
@pytest.mark.parametrize("plan_name", ["S2", "ragged", "S16"])
def test_split_k(cuda, plan_name, form):
    M, K, N = _split_shape(plan_name, sms(cuda))

    def expect(plan):
        S, per, kb = plan.splits, plan.kb_per_split, plan.total_kb
        assert plan.pair == 0 and plan.staged == 0 and S > 1
        if plan_name == "S2":
            assert S == 2
        elif plan_name == "ragged":
            assert 2 < S < 16 and kb % per != 0, (S, per, kb)
        else:
            assert S == 16 and kb % per != 0, (S, per, kb)
        assert (S - 1) * per < kb <= S * per
    run_gemm(cuda, M, K, N, form=form, split_k=True, expect=expect, seed=len(form))


# ---------------------------------------------------------------------------------------------------------------- wide tiles and pairs
@pytest.mark.gpu
@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("bn", [160, 192, 256])
def test_wide_tiles(cuda, bn, form):
    """M 1000 (a ragged M tile), c_out 448 (not a multiple of any N tile; 896 interleaved columns for GEGLU)."""
    N = 896 if form == "geglu" else 448
    run_gemm(cuda, 1000, 320, N, form=form, force_bn=bn, seed=bn, expect=_want(bn=bn, staged=0, splits=1, pair=0))


@pytest.mark.gpu
@pytest.mark.parametrize("bn", [128, 160, 192, 256])
def test_pair_matches_single(cuda, bn):
    """CTA pairs (B tile halves multicast) against single CTAs: bit-identical, and both within the float64 bound.  7 M tiles: a phantom."""
    M, K, N = 7 * 128 - 5, 9 * 64, 2 * bn + 64
    _, y2 = run_gemm(cuda, M, K, N, form="residual", force_bn=bn, pair=True, seed=3, expect=_want(bn=bn, pair=1, tiles_m=7, items=4 * 3))
    _, y1 = run_gemm(cuda, M, K, N, form="residual", force_bn=bn, pair=False, seed=3, expect=_want(bn=bn, pair=0))
    assert same(y1, y2), "paired and single CTAs differ"


# ---------------------------------------------------------------------------------------------------------------- convolutions
def run_conv(dev, n, hin, win, cins, cout, *, k=3, s=1, pad_lo=1, scs=(), form="bias", up2x=False, expect=None, seed=0, **kw):
    """One convolution through ops.conv2d: sources (and shortcut sources) with NaN channel-pitch gaps, NaN-poisoned output; the float64
    reference is the convolution of the concatenated sources (zero padding pad_lo before, whatever the output extent needs after).
    up2x: weights are multiples of 1/64 below 1/8, so the merged sub-pixel taps are exact and the reference is the convolution of the
    nearest-upsampled input."""
    from ladi_vton_b200 import ops, weights
    g = cpu_gen(seed)
    xs = []
    for c in cins:
        b = nan_buf((n, hin, win, c + 8), torch.bfloat16, dev)
        b[..., :c] = torch.randn((n, hin, win, c), generator=g).to(dev).bfloat16()
        xs.append(b[..., :c])
    if up2x:
        h, w = 2 * hin, 2 * win
    elif s == 2:
        pads = (2 if pad_lo == 1 else 1) if k == 3 else 0
        h, w = (hin + pads - k) // 2 + 1, (win + pads - k) // 2 + 1
    else:
        h, w = hin, win
    sc = []
    for c in scs:
        b = nan_buf((n, h, w, c + 8), torch.bfloat16, dev)
        b[..., :c] = torch.randn((n, h, w, c), generator=g).to(dev).bfloat16()
        sc.append(b[..., :c])
    cin, csc = sum(cins), sum(scs)
    fan = k * k * cin + csc
    if up2x:
        wt = (torch.randint(-7, 8, (cout, cin, 3, 3), generator=g).float() / 64)
        wp = weights.pack_conv_up2x(wt, list(cins))
    else:
        wt = (torch.randn((cout, cin, k, k), generator=g) * fan ** -0.5).bfloat16().float()
    wsc = (torch.randn((cout, csc), generator=g) * fan ** -0.5).bfloat16().float() if scs else None
    if not up2x:
        wp = weights.pack_conv(wt, list(cins), wsc[:, :, None, None] if scs else None, list(scs))
    rows = n * h * w
    okw, bcol, brow, res, rs, act, f32 = _operands(form, rows, cout, cout, dev, seed + 1)
    okw.update(kw)
    odt = torch.float32 if f32 else torch.bfloat16
    pitch = cout + 8
    rbuf = None
    if res is not None:
        rbuf = nan_buf((rows, pitch), torch.bfloat16, dev)
        rbuf[:, :cout] = res
    common = dict(ksize=k, stride=s, pad_lo=pad_lo, shortcut=sc, up2x=up2x, out_fp32=f32, **okw)

    def views(buf):
        return buf[:rows].view(n, h, w, pitch)[..., :cout], None if rbuf is None else rbuf.view(n, h, w, pitch)[..., :cout]

    buf = nan_buf((rows + TAIL, pitch), odt, dev)
    o4, r4 = views(buf)
    plan = ops.conv_plan(xs, wp.to(dev), cout, out=o4, residual=r4, **common)
    if expect is not None:
        expect(plan)
    runs = twice(lambda b: ops.conv2d(xs, wp.to(dev), cout, out=views(b["out"])[0], residual=views(b["out"])[1], **common),
                 lambda: dict(out=nan_buf((rows + TAIL, pitch), odt, dev)))
    outs = [r["out"] for r in runs]
    errs = layout(outs[0], 0, cout, "output", rows=rows)
    assert not errs, errs
    assert not determinism(runs, ["out"]), "two runs differ bitwise"
    X = torch.cat([x.double() for x in xs], dim=3).permute(0, 3, 1, 2)
    if up2x:
        X = F.interpolate(X, scale_factor=2, mode="nearest")
        pe, hin_e, win_e, s_e = 1, h, w, 1
    else:
        pe, hin_e, win_e, s_e = (pad_lo if k == 3 else 0), hin, win, s
    Xp = F.pad(X, (pe, max(0, (w - 1) * s_e + k - pe - win_e), pe, max(0, (h - 1) * s_e + k - pe - hin_e)))
    w64 = wt.to(dev).double()
    acc = F.conv2d(Xp, w64, stride=s_e)[:, :, :h, :w].permute(0, 2, 3, 1).reshape(rows, cout)
    m = F.conv2d(Xp.abs(), w64.abs(), stride=s_e)[:, :, :h, :w].permute(0, 2, 3, 1).reshape(rows, cout)
    if scs:
        S_ = torch.cat([t.double() for t in sc], dim=3).reshape(rows, csc)
        acc += S_ @ wsc.to(dev).double().t()
        m += S_.abs() @ wsc.to(dev).double().abs().t()
    K = wp.shape[1]
    r, bound = gemm_expect(acc, m, K, bcol, brow, None if res is None else res.double(), rs, act, f32)
    q = max_ratio(outs[0][:rows, :cout], r, bound)
    assert q <= 1.0, f"err/bound {q:.3g}"
    return plan


GEOMETRY = {
    "3x3 odd W and H, n 3": dict(n=3, hin=5, win=7, cins=(64,), cout=64, want=dict(tiles_m=35)),
    "3x3 8x6 batch 16": dict(n=16, hin=8, win=6, cins=(64,), cout=320, form="silu", want=dict(tiles_m=6)),
    "3x3 stride 2 pad_lo 0, odd input": dict(n=2, hin=13, win=11, cins=(64,), cout=128, s=2, pad_lo=0),
    "3x3 stride 2 pad_lo 1, odd input": dict(n=2, hin=13, win=11, cins=(96,), cout=128, s=2, pad_lo=1),
    "1x1 stride 2": dict(n=2, hin=14, win=10, cins=(64,), cout=96, k=1, s=2),
    "two sources and a shortcut, ragged channels": dict(n=2, hin=12, win=10, cins=(40, 72), cout=200, scs=(24,), form="residual"),
    "up2x, odd tiles per parity": dict(n=1, hin=8, win=6, cins=(64,), cout=192, up2x=True, want=dict(tiles_m=4 * 3)),
    "up2x pairs": dict(n=16, hin=8, win=6, cins=(64,), cout=256, up2x=True, pair=True, force_bn=128, want=dict(pair=1, tiles_m=4 * 6)),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(GEOMETRY))
def test_conv_geometry(cuda, name):
    kw = dict(GEOMETRY[name])
    want = kw.pop("want", {})
    run_conv(cuda, seed=7, expect=_want(**want) if want else None, **kw)


# ---------------------------------------------------------------------------------------------------------------- LayerNorm fold
@pytest.mark.gpu
@pytest.mark.parametrize("form", ["residual", "silu"])
def test_rowstat_producer(cuda, form):
    """The producer's {sum, sum of squares} per row and 32-column chunk against float64 sums of its unrounded float64 output (residual
    rows of mean 8: the statistics of a tensor whose mean dwarfs its spread)."""
    from ladi_vton_b200 import ops, weights
    M, K, N = 1000, 320, 320
    g = cpu_gen(31)
    a = torch.randn((M, K), generator=g).to(cuda).bfloat16()
    w = (torch.randn((N, K), generator=g) * K ** -0.5).bfloat16()
    wp = weights.pack_linear(w.float()).to(cuda)
    b = (torch.randn((N,), generator=g) * 0.5).to(cuda)
    res = (torch.randn((M, N), generator=g) + 8).to(cuda).bfloat16() if form == "residual" else None
    act = ops.ACT_SILU if form == "silu" else ops.ACT_NONE
    stats = torch.full((M, N // 32, 2), float("nan"), device=cuda)
    out = nan_buf((M, N + 8), torch.bfloat16, cuda)
    plan = ops.gemm_plan(a, wp, N, bias=b, residual=res, act=act, out=out[:, :N], rowstat=stats, split_k=False)
    assert plan.staged == 0 and plan.splits == 1
    ops.gemm(a, wp, N, bias=b, residual=res, act=act, out=out[:, :N], rowstat=stats, split_k=False)
    torch.cuda.synchronize()
    acc = a.double() @ w.to(cuda).double().t()
    m = a.double().abs() @ w.to(cuda).double().abs().t()
    r64 = None if res is None else res.double()
    r, bound = gemm_expect(acc, m, K, bcol=b.double(), res=r64, act=act)
    assert max_ratio(out[:, :N], r, bound) <= 1.0
    s, q, bs, bq = rowstat_expect(r, bound - 2.0 ** -7 * r.abs())
    assert max_ratio(stats[..., 0], s, bs) <= 1.0, "row sums"
    assert max_ratio(stats[..., 1], q, bq) <= 1.0, "row sums of squares"


@pytest.mark.gpu
@pytest.mark.parametrize("bn", [0, 256])
@pytest.mark.parametrize("act", ["none", "gelu", "geglu"])
def test_ln_fold_consumer(cuda, act, bn):
    """The consumer against rstd64 (t Wp - mean64 colsum) + bp on the folded operands; rows of mean 8 (plus a per-row offset), std 1."""
    from ladi_vton_b200 import ops
    M, Cin, N = 1000, 320, 384
    t, wp, colsum, bp = _ln_case(41, M=M, Cin=Cin, N=N)
    t, wp, colsum, bp = t.to(cuda), wp.to(cuda), colsum.to(cuda), bp.to(cuda)
    a_code = {"none": ops.ACT_NONE, "gelu": ops.ACT_GELU, "geglu": ops.ACT_GEGLU}[act]
    c_eff = N // 2 if act == "geglu" else N
    stats = _stats_table(t.float()).to(cuda)
    eps = 1e-5
    tbuf = nan_buf((M, Cin + 8), torch.bfloat16, cuda)
    tbuf[:, :Cin] = t
    out = nan_buf((M + TAIL, c_eff + 8), torch.bfloat16, cuda)
    kw = dict(bias=bp, act=a_code, ln=(stats, colsum, eps), force_bn=bn, split_k=False)
    plan = ops.gemm_plan(tbuf[:, :Cin], wp, N, out=out[:M, :c_eff], **kw)
    assert plan.staged == 0 and plan.splits == 1 and (bn == 0 or plan.bn == bn)
    ops.gemm(tbuf[:, :Cin], wp, N, out=out[:M, :c_eff], **kw)
    torch.cuda.synchronize()
    errs = layout(out, 0, c_eff, "output", rows=M)
    assert not errs, errs
    r, bound = ln_fold_expect(t, wp, colsum, bp, eps, a_code)
    q = max_ratio(out[:M, :c_eff], r, bound)
    assert q <= 1.0, f"err/bound {q:.3g}"


# ---------------------------------------------------------------------------------------------------------------- placement
PLACE_PATHS = {"staged": (1000, 320, 256, {}), "fragment": (1000, 320, 256, dict(force_bn=256)), "split": (100, 156 * 64, 256, {})}


def _expected_plan(path, out_b, res_b, bias_b, pitch):
    """The header's rules for this test's placements: None (rejected), else (split, staged).  Byte offsets of out / residual / bias."""
    if out_b % 4 or res_b % 4:
        return None
    split = path == "split" and pitch % 4 == 0 and out_b % 8 == 0 and res_b % 8 == 0 and bias_b % 16 == 0
    staged = path != "fragment" and not split and pitch % 8 == 0 and out_b % 16 == 0 and res_b % 16 == 0 and bias_b % 8 == 0
    return split, staged


@pytest.mark.gpu
@pytest.mark.parametrize("parity", ["even", "odd"])
@pytest.mark.parametrize("offset", [0, 1, 2, 4])
@pytest.mark.parametrize("operand", ["out", "residual", "bias"])
@pytest.mark.parametrize("path", list(PLACE_PATHS))
def test_placement(cuda, path, operand, offset, parity):
    """out, residual and bias at element offsets 0 / 1 / 2 / 4 with an even (c + 8) or odd (c + 3) output and residual pitch.  An accepted
    placement takes the plan the header's rules give and is within the float64 bound; a rejected one raises naming the operand, launches
    nothing and leaves the output NaN."""
    from ladi_vton_b200 import lib, ops, weights
    M, K, N, kw = PLACE_PATHS[path]
    pitch = N + 8 if parity == "even" else N + 3
    g = cpu_gen(offset * 7 + len(operand))
    abuf = nan_buf((M, K + 8), torch.bfloat16, cuda)
    abuf[:, :K] = torch.randn((M, K), generator=g).to(cuda).bfloat16()
    a = abuf[:, :K]
    w = (torch.randn((N, K), generator=g) * K ** -0.5).bfloat16()
    wp = weights.pack_linear(w.float()).to(cuda)
    o_off, r_off, b_off = (offset if operand == x else 0 for x in ("out", "residual", "bias"))
    bstore = torch.full((N + 16,), float("nan"), device=cuda)
    bstore[b_off:b_off + N] = (torch.randn((N,), generator=g) * 0.5).to(cuda)
    bias = bstore[b_off:b_off + N]
    res = torch.randn((M, N), generator=g).to(cuda).bfloat16()
    rstore = nan_buf((M * pitch + 16,), torch.bfloat16, cuda)
    resid = rstore[r_off:r_off + M * pitch].view(M, pitch)[:, :N]
    resid.copy_(res)
    ostore = nan_buf(((M + TAIL) * pitch + 16,), torch.bfloat16, cuda)
    out = ostore[o_off:o_off + M * pitch].view(M, pitch)[:, :N]
    want = _expected_plan(path, 2 * o_off, 2 * r_off, 4 * b_off, pitch)
    args = dict(bias=bias, residual=resid, out=out, **kw)
    if want is None:
        before, before_py = lib.load().ladi_launch_count(), lib.launches
        with pytest.raises(RuntimeError, match=operand):
            ops.gemm_plan(a, wp, N, **args)
        with pytest.raises(RuntimeError, match=operand):
            ops.gemm(a, wp, N, **args)
        torch.cuda.synchronize()
        assert lib.load().ladi_launch_count() == before and lib.launches == before_py
        assert bool(torch.isnan(ostore.float()).all()), "a rejected call wrote its output"
        return
    plan = ops.gemm_plan(a, wp, N, **args)
    assert (plan.splits > 1, bool(plan.staged)) == want, (plan.splits, plan.staged, want)
    ops.gemm(a, wp, N, **args)
    torch.cuda.synchronize()
    y = ostore[o_off:o_off + (M + TAIL) * pitch].view(M + TAIL, pitch)
    errs = layout(y, 0, N, "output", rows=M)
    assert not errs, errs
    assert bool(torch.isnan(ostore[:o_off].float()).all()) and bool(torch.isnan(ostore[o_off + (M + TAIL) * pitch:].float()).all())
    acc = a.double() @ w.to(cuda).double().t()
    m = a.double().abs() @ w.to(cuda).double().abs().t()
    r, bound = gemm_expect(acc, m, K, bcol=bias.double(), res=res.double())
    q = max_ratio(y[:M, :N], r, bound)
    assert q <= 1.0, f"err/bound {q:.3g}"


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["d64 out +2", "d64 out +1", "d64 odd batch stride", "d512 out +2", "d512 out +1", "d512 odd batch stride"])
def test_attention_out_placement(cuda, case):
    """Both attention kernels store bf16 pairs: out 4-byte aligned with an even batch stride runs (and is right against float64), anything
    else is rejected before a launch."""
    from ladi_vton_b200 import lib, ops
    D = 512 if case.startswith("d512") else 64
    heads = 1 if D == 512 else 2
    B, nq, nkv, cols = 2, 100, 77, heads * D
    g = cpu_gen(51)
    q = (torch.randn((B, nq, cols), generator=g) * 2 ** 0.5).to(cuda).bfloat16()
    k = (torch.randn((B, nkv, cols), generator=g) * 2 ** 0.5).to(cuda).bfloat16()
    v = torch.randn((B, nkv, cols), generator=g).to(cuda).bfloat16()
    off = 1 if case.endswith("+1") else (2 if case.endswith("+2") else 0)
    bstride = nq * cols + (1 if "odd" in case else 0)
    store = nan_buf((B * bstride + cols + 16,), torch.bfloat16, cuda)
    out = store[off:].as_strided((B, nq, cols), (bstride, cols, 1))
    call = (lambda: ops.attention(q, k, v, heads, D ** -0.5, out=out)) if D == 64 else (lambda: ops.attention_d512(q, k, v, D ** -0.5, out=out))
    if off == 1 or "odd" in case:
        before, before_py = lib.load().ladi_launch_count(), lib.launches
        with pytest.raises(RuntimeError, match="out"):
            call()
        torch.cuda.synchronize()
        assert lib.load().ladi_launch_count() == before and lib.launches == before_py
        assert bool(torch.isnan(store.float()).all())
        return
    call()
    torch.cuda.synchronize()
    assert bool(torch.isnan(store[:off].float()).all())
    for b in range(B):
        o, sv = attn_ref(q[b].double(), k[b].double(), v[b].double(), heads, D, D ** -0.5)
        assert max_ratio(out[b], o, attn_expect(o, sv, nkv)) <= 1.0
