"""GPU tests of the metric networks' tf32 precision on an H100: `ladi_gemm_tf32` and the fp32 im2col / pool / LPIPS kernels against float64
at their edges and on every distinct call the tf32 networks make, the networks end to end against the fp32 oracle, the FID / KID / IS
statistics, and the CLI's --precision with its statistics cache.

References and bounds (per element; u = 2^-24):
  ladi_gemm_tf32  the float64 product of the fp32 operands as stored, + bias, ReLU.  The kernel rounds both operands to nearest TF32
            (10 explicit mantissa bits): each product is within E_TF32 = 2 * 2^-11 = 2^-10 relative of the exact one; the fp32 sum of K
            terms adds C_ACC sqrt(K) u (tests/kernel_check.py); the fp32 bias add and output U_F32:
            U_F32 |r| + (E_TF32 + C_ACC sqrt(K) u) m,  m = |A| |W|^T + |bias|.  ReLU is 1-Lipschitz and leaves the bound as it is.
  the fp32 forms of tests/test_gpu_metrics_census.py's kernels, with its bf16 rounding term removed:
            im2col NHWC and max pool exact; im2col pixels bit-equal to torch's fp32 (x - shift) / scale and within 2^-22 (|x| + |shift|) /
            scale of float64; average pools (k*k + 2) u mean|x| (the clipped window's count as torch takes it); global average 2u |r| +
            (hw + 1) u mean|x|; lpips_layer the census's bound on the same fp32 features.
Every replay also checks that the call wrote exactly its columns (NaN-poisoned pitch gaps, output slices and tails stay NaN, poisoned input
gaps are never read) and that two runs give the same bits.

End to end (random weights, BatchNorm calibrated on the test batch as in tests/test_gpu_metrics.py): the error against the fp32 oracle with
TF32 off must be at most TF32_VS_CUDNN times the error of the same oracle with `torch.backends.cudnn.allow_tf32 = True` (what clean-fid and
torchmetrics compute in by default), and at most TF32_VS_BF16 times the engine's own bf16 error on the same batch -- per Inception stage
and for LPIPS.  End to end through the Inception the bf16 error of the random network has grown to 0.2 rel-L2 and grows no further at the
rate a small error does (each block amplifies a small error about 1.5x), so there the ratio is larger and its gate is TF32_VS_BF16_E2E.
KID between two halves of one image distribution is the unbiased estimate of a value near zero (3e-4 here), so its relative error is
large for both precisions."""
import json
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from kernel_check import C_ACC, EPS24, U_F32, Replay, cpu_pack, determinism, flat_buf, layout, ptr, recorded, tail_nan, twice, worst_at

pytestmark = pytest.mark.gpu

E_TF32 = 2.0 ** -10       # both operands rounded to nearest TF32 inside ladi_gemm_tf32
# Gates set from values measured on an H100 80GB HBM3 (700 W power limit), recorded in DESIGN.md section 7, with headroom.
TF32_VS_CUDNN = 1.5       # engine tf32 error <= 1.5 x cuDNN TF32's error, both against the fp32 oracle (SURVEY section 8(c))
TF32_VS_BF16 = 0.25       # ... and <= a quarter of the engine's bf16 error: per Inception stage, and LPIPS per pair (measured 0.065)
TF32_VS_BF16_E2E = 0.35   # ... pool3 features and logits end to end (measured 0.265)
STAGE_REL_L2 = 2e-3       # each Inception stage fed the oracle's fp32 input (measured <= 9.7e-4)
STAT_REL = {"fid": 1e-2, "kid": 0.6, "is": 5e-5}  # tf32 engine vs oracle features of 16 + 16 images (measured 3.3e-3, 0.41, 4.1e-6)
POOL_MAX, POOL_AVG, POOL_EXCL, POOL_GLOBAL = 0, 1, 2, 3


@pytest.fixture(autouse=True)
def _fp32_reference():
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def rel_l2(a, b):
    a, b = a.double().flatten().cpu(), b.double().flatten().cpu()
    return float((a - b).norm() / b.norm())


def _lib():
    from ladi_vton_b200 import lib
    return lib


def _f32(R, rows, pitch, values):
    return R.poisoned(rows, pitch, values, dtype=torch.float32)


# ================================================================================================================ ladi_gemm_tf32
def replay_gemm(R, f, chunk=1 << 18):
    m, k, ap, n, wp, op, c_off = (f[q] for q in ("m", "k", "a_pitch", "n", "w_pitch", "out_pitch", "c_off"))
    a = _f32(R, m, ap, R.randn(m, k) * 2.0)
    w = _f32(R, n, wp, R.randn(n, k) / math.sqrt(k))
    b = R.randn(n) * 0.5

    def fresh():
        flat, o = flat_buf(R, m * op, torch.float32)
        return dict(flat=flat, out=o)
    runs = twice(lambda bf: _lib().call("ladi_gemm_tf32", ptr(a), m, k, ap, ptr(w), n, wp, ptr(b), 1, ptr(bf["out"]), op, c_off, R.stream), fresh)
    out = runs[0]["out"].view(m, op)
    errs = layout(out, c_off, c_off + n, "out") + tail_nan(runs[0]["flat"], m * op, "out") + determinism(runs, ["flat"])
    W, B = w[:, :k].double(), b.double()
    worst = (0.0, "")
    for r0 in range(0, m, chunk):
        A = a[r0:r0 + chunk, :k].double()
        pre = A @ W.T + B
        mag = A.abs() @ W.abs().T + B.abs()
        r = pre.clamp_min(0)
        bound = U_F32 * r.abs() + (E_TF32 + C_ACC * math.sqrt(k) * EPS24) * mag
        q = torch.nan_to_num((out[r0:r0 + chunk, c_off:c_off + n].double() - r).abs() / bound.clamp_min(1e-300), nan=float("inf"))
        e, res = worst_at(q, ("row", "column"), f" (rows from {r0}; m {m} n {n} k {k})")
        errs += e
        worst = max(worst, res)
    return errs, worst


def _gemm(m, n, k, c_off=0, gap=0, a_gap=4, w_gap=8):
    return dict(m=m, k=k, a_pitch=k + a_gap, n=n, w_pitch=k + w_gap, out_pitch=c_off + n + gap, c_off=c_off)


WIDTHS = [32, 48, 64, 80, 96, 128, 160, 192, 256, 320, 384, 448]
GEMM_EDGES = ([(f"width {n}", _gemm(129, n, 100)) for n in WIDTHS]
              + [("one row", _gemm(1, 64, 64)), ("a tile minus one row", _gemm(127, 96, 36)), ("a tile plus one row", _gemm(129, 256, 36)),
                 ("K = 4", _gemm(200, 64, 4)), ("K = 28 (the Inception stem)", _gemm(300, 32, 28, a_gap=0, w_gap=0)),
                 ("K = 2052", _gemm(257, 320, 2052)), ("K = 3456 (Mixed_7b 3x3dbl_2)", _gemm(130, 384, 3456)),
                 ("slice at c_off 4 with a pitch gap", _gemm(131, 48, 68, c_off=4, gap=12)),
                 ("slice at c_off 1856 of 2048", _gemm(128 * 3 + 5, 192, 1280, c_off=1856)),
                 ("slice at c_off 64, 128-wide tile", _gemm(70, 384, 40, c_off=64, gap=4)),
                 ("many row tiles", _gemm(128 * 600 + 77, 64, 32))])


@pytest.mark.parametrize("case", [c for _, c in GEMM_EDGES], ids=[i for i, _ in GEMM_EDGES])
def test_gemm_tf32_edges_against_float64(cuda, case):
    errs, (w, where) = replay_gemm(Replay(cuda, 4321), case)
    print(f"\n[tf32] gemm worst err/bound {w:.3f} at {where}")
    assert not errs, errs[:5]


def test_gemm_tf32_rounds_to_nearest(cuda):
    """Operands one TF32 half-ulp step away from a TF32 value: rounding to nearest reproduces them exactly, truncation would not."""
    a = torch.full((1, 8), 1.0 + 2.0 ** -10 + 2.0 ** -11 + 2.0 ** -13, device=cuda)  # 1 + 3 half-ulps + a bit: nearest is 1 + 2^-9
    w = torch.ones((4, 8), device=cuda)
    out = torch.zeros((1, 4), device=cuda)
    from ladi_vton_b200 import ops
    ops.gemm_tf32(a, w, 4, out)
    torch.cuda.synchronize()
    assert torch.equal(out, torch.full((1, 4), 8 * (1.0 + 2.0 ** -9), device=cuda)), out


# ================================================================================================================ fp32 glue kernels
def im2col_ref(x, kh, kw, sh, sw, ph, pw, k_pad):
    """x NHWC [n, h, w, c] -> rows [n*oh*ow, k_pad], column (ky*kw + kx)*c + ch, zeros in the padding and in columns >= kh*kw*c."""
    n, h, w, c = x.shape
    oh, ow = (h + 2 * ph - kh) // sh + 1, (w + 2 * pw - kw) // sw + 1
    xp = F.pad(x, (0, 0, pw, pw, ph, ph))
    taps = [xp[:, ky:ky + sh * (oh - 1) + 1:sh, kx:kx + sw * (ow - 1) + 1:sw, :] for ky in range(kh) for kx in range(kw)]
    return F.pad(torch.stack(taps, dim=3).reshape(n * oh * ow, kh * kw * c), (0, k_pad - kh * kw * c))


def replay_im2col(R, f):
    n, c, h, w, pitch, kh, kw, sh, sw, ph, pw, kp = (f[q] for q in ("n", "c", "h", "w", "pitch", "kh", "kw", "sh", "sw", "ph", "pw", "kpad"))
    oh, ow = (h + 2 * ph - kh) // sh + 1, (w + 2 * pw - kw) // sw + 1
    rows = n * oh * ow
    geo = (kh, kw, sh, sw, ph, pw, kp)
    if f["pixels"]:
        x = R.rand(n, c, h, w) * 255.0
        shift, scale = torch.full((c,), 128.0, device=R.dev), torch.full((c,), 128.0, device=R.dev)
        if kh == 11:  # the LPIPS scaling layer of AlexNet's stem
            x = x / 255.0
            shift = torch.tensor([0.485, 0.456, 0.406][:c], device=R.dev)
            scale = torch.tensor([0.229, 0.224, 0.225][:c], device=R.dev)
    else:
        x, shift, scale = _f32(R, n * h * w, pitch, R.randn(n * h * w, c) * 2.0), None, None

    def fresh():
        flat, o = flat_buf(R, rows * kp, torch.float32)
        return dict(flat=flat, out=o)
    runs = twice(lambda b: _lib().call("ladi_im2col_f32", ptr(x), int(f["pixels"]), n, c, h, w, pitch, kh, kw, sh, sw, ph, pw, ptr(shift),
                                       ptr(scale), ptr(b["out"]), kp, R.stream), fresh)
    out = runs[0]["out"].view(rows, kp)
    errs = layout(out, 0, kp, "rows") + tail_nan(runs[0]["flat"], rows * kp, "rows") + determinism(runs, ["flat"])
    if f["pixels"]:
        q = (x - shift.view(-1, 1, 1)) / scale.view(-1, 1, 1)  # torch fp32, IEEE division
        if not torch.equal(out, im2col_ref(q.permute(0, 2, 3, 1), *geo)):
            errs.append("pixel im2col differs from torch's fp32 affine")
        s64, c64 = shift.double().view(-1, 1, 1), scale.double().view(-1, 1, 1)
        r = im2col_ref(((x.double() - s64) / c64).permute(0, 2, 3, 1), *geo)
        mag = im2col_ref(((x.double().abs() + s64.abs()) / c64.abs()).permute(0, 2, 3, 1), *geo)
        q = torch.nan_to_num((out.double() - r).abs() / (2.0 ** -22 * mag).clamp_min(1e-300), nan=float("inf"))
        e, res = worst_at(q, ("row", "column"))
        return errs + e, res
    if not torch.equal(out, im2col_ref(x.view(n, h, w, pitch)[..., :c], *geo)):
        errs.append("NHWC im2col is not an exact copy")
    return errs, (0.0, "exact")


def replay_pool2d(R, f):
    n, h, w, c, xp, k, s, p, mode, op, c_off = (f[q] for q in ("n", "h", "w", "c", "xp", "k", "s", "p", "mode", "op", "c_off"))
    x = _f32(R, n * h * w, xp, R.randn(n * h * w, c) * 2.0)
    X = x[:, :c].reshape(n, h, w, c).permute(0, 3, 1, 2).double()
    oh, ow = (1, 1) if mode == POOL_GLOBAL else ((h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1)
    rows = n * oh * ow

    def fresh():
        flat, o = flat_buf(R, rows * op, torch.float32)
        return dict(flat=flat, out=o)
    runs = twice(lambda b: _lib().call("ladi_pool2d_f32", ptr(x), n, h, w, c, xp, k, s, p, mode, ptr(b["out"]), op, c_off, R.stream), fresh)
    out = runs[0]["out"].view(rows, op)
    errs = layout(out, c_off, c_off + c, "output") + tail_nan(runs[0]["flat"], rows * op, "output") + determinism(runs, ["flat"])
    y = out[:, c_off:c_off + c].double()
    if mode == POOL_GLOBAL:
        r = X.mean((2, 3))
        bound = 2 * EPS24 * r.abs() + (h * w + 1) * EPS24 * X.abs().mean((2, 3))
    elif mode == POOL_MAX:
        r = F.max_pool2d(X, k, s, p).permute(0, 2, 3, 1).reshape(rows, c)
        return errs + ([] if torch.equal(y, r) else ["max pool is not exact"]), (0.0, "exact")
    else:
        r = F.avg_pool2d(X, k, s, p, count_include_pad=mode == POOL_AVG)
        ma = F.avg_pool2d(X.abs(), k, s, p, count_include_pad=mode == POOL_AVG)
        r, bound = r.permute(0, 2, 3, 1).reshape(rows, c), ((k * k + 2) * EPS24 * ma).permute(0, 2, 3, 1).reshape(rows, c)
    e, res = worst_at(torch.nan_to_num((y - r).abs() / bound.clamp_min(1e-300), nan=float("inf")), ("output pixel", "channel"))
    return errs + e, res


def lpips_expect(a, b, lin):
    """tests/test_gpu_metrics_census.py's bound: a, b [n, hw, c] float64, lin [c] -> (D, E) [n] without the final `acc +=` rounding."""
    n, hw, c = a.shape
    ra = 1.0 / ((a * a).sum(-1, keepdim=True).sqrt() + 1e-10)
    rb = 1.0 / ((b * b).sum(-1, keepdim=True).sqrt() + 1e-10)
    t = a * ra - b * rb
    dpx = (lin * t * t).sum(-1)
    g = math.ceil(c / 32) + 5
    dr = (g / 2 + 3) * EPS24
    Et = (dr + 2 * EPS24) * (a.abs() * ra + b.abs() * rb)
    Ed = (lin * (2 * t.abs() * Et + Et * Et + 2 * EPS24 * t * t)).sum(-1) + g * EPS24 * dpx
    D = dpx.mean(-1)
    return D, Ed.mean(-1) + (math.ceil(hw / 16) + 17) * EPS24 * D


def replay_lpips(R, f):
    n, h, w, c, pitch = (f[q] for q in ("n", "h", "w", "c", "pitch"))
    hw = h * w
    a = R.randn(n, hw, c).clamp_min(0.0)
    b = R.randn(n, hw, c).clamp_min(0.0)
    near = (a + 0.02 * R.randn(n, hw, c)).clamp_min(0.0)
    b[1::2] = near[1::2]  # near-identical pairs, where unit(a) - unit(b) cancels
    feats = _f32(R, 2 * n * hw, pitch, torch.cat([a, b]).view(2 * n * hw, c))
    fa, fb = feats[:n * hw], feats[n * hw:]
    lin_flat, lin = flat_buf(R, c, torch.float32)
    lin.copy_(R.rand(c) * 0.1)
    acc0 = R.rand(n) + 0.25

    def fresh():
        flat, acc = flat_buf(R, n, torch.float32)
        acc.copy_(acc0)
        return dict(flat=flat, acc=acc)
    runs = twice(lambda bf: _lib().call("ladi_lpips_layer_f32", ptr(fa), ptr(fb), n, h, w, c, pitch, ptr(lin), ptr(bf["acc"]), R.stream), fresh)
    errs = tail_nan(runs[0]["flat"], n, "acc") + tail_nan(lin_flat, c, "lin") + determinism(runs, ["flat"])
    D, E = lpips_expect(fa[:, :c].double().reshape(n, hw, c), fb[:, :c].double().reshape(n, hw, c), lin.double())
    r = acc0.double() + D
    q = torch.nan_to_num((runs[0]["acc"].double() - r).abs() / (E + EPS24 * r.abs()), nan=float("inf"))
    e, res = worst_at(q, ("image",), f" (hw {hw}, c {c})")
    return errs + e, res


def _im(n, c, h, w, pitch, k, s, p, kpad, pixels=0):
    kh, kw = k if isinstance(k, tuple) else (k, k)
    ph, pw = p if isinstance(p, tuple) else (p, p)
    return dict(n=n, c=c, h=h, w=w, pitch=pitch, kh=kh, kw=kw, sh=s, sw=s, ph=ph, pw=pw, kpad=kpad, pixels=pixels)


def _pool(n, h, w, c, xp, k, s, p, mode, op, c_off):
    return dict(n=n, h=h, w=w, c=c, xp=xp, k=k, s=s, p=p, mode=mode, op=op, c_off=c_off)


GLUE_EDGES = [
    ("im2col c 4 with a pitch gap, 3x3 same", "im2col", _im(2, 4, 9, 7, 12, 3, 1, 1, 40)),
    ("im2col 1x7, K tail", "im2col", _im(2, 12, 5, 9, 12, (1, 7), 1, (0, 3), 88)),
    ("im2col 7x1 into a channel slice view", "im2col", _im(1, 20, 11, 3, 32, (7, 1), 1, (3, 0), 140)),
    ("im2col 5x5", "im2col", _im(3, 8, 6, 6, 8, 5, 1, 2, 200)),
    ("im2col 3x3/2 valid", "im2col", _im(2, 36, 10, 9, 40, 3, 2, 0, 324)),
    ("pixel im2col 3x3/2 stem", "im2col", _im(2, 3, 31, 29, 0, 3, 2, 0, 28, pixels=1)),
    ("pixel im2col 11x11/4 stem", "im2col", _im(2, 3, 45, 37, 0, 11, 4, 2, 364, pixels=1)),
    ("max pool 3/2 into c_off 4 of a pitch gap", "pool2d", _pool(2, 9, 8, 12, 16, 3, 2, 0, POOL_MAX, 24, 4)),
    ("average pool 3/1/1", "pool2d", _pool(2, 7, 5, 8, 8, 3, 1, 1, POOL_AVG, 8, 0)),
    ("exclude-pad average pool 3/1/1 at c_off 20", "pool2d", _pool(3, 5, 6, 4, 12, 3, 1, 1, POOL_EXCL, 28, 20)),
    ("global average, c 4, pitch gap", "pool2d", _pool(3, 5, 3, 4, 8, 0, 0, 0, POOL_GLOBAL, 12, 4)),
    ("global average 8x8x2048", "pool2d", _pool(2, 8, 8, 2048, 2048, 0, 0, 0, POOL_GLOBAL, 2048, 0)),
    ("lpips c 4, 17 pixels", "lpips", dict(n=3, h=17, w=1, c=4, pitch=8)),
    ("lpips c 36 (a lane remainder), one pair", "lpips", dict(n=1, h=5, w=7, c=36, pitch=36)),
    ("lpips c 384 at 13x11", "lpips", dict(n=4, h=13, w=11, c=384, pitch=392)),
]
REPLAY = {"gemm": replay_gemm, "im2col": replay_im2col, "pool2d": replay_pool2d, "lpips": replay_lpips}


@pytest.mark.parametrize("kind,case", [(k, c) for _, k, c in GLUE_EDGES], ids=[i for i, _, _ in GLUE_EDGES])
def test_fp32_glue_edges_against_float64(cuda, kind, case):
    errs, (w, where) = REPLAY[kind](Replay(cuda, 8642), case)
    print(f"\n[tf32] {kind} worst err/bound {w:.3f} {where}")
    assert not errs, errs[:5]


# ================================================================================================================ census replay
ARGS = {"ladi_gemm_tf32": ("gemm", "a m k a_pitch wt n w_pitch bias relu out out_pitch c_off stream"),
        "ladi_im2col_f32": ("im2col", "x pixels n c h w pitch kh kw sh sw ph pw shift scale out kpad stream"),
        "ladi_pool2d_f32": ("pool2d", "x n h w c xp k s p mode out op c_off stream"),
        "ladi_lpips_layer_f32": ("lpips", "fa fb n h w c pitch lin acc stream")}
POINTERS = {"a", "wt", "bias", "out", "stream", "x", "shift", "scale", "fa", "fb", "lin", "acc"}
BATCHES = (1, 8, 16, 32, 64)


def tf32_census():
    """Distinct (kind, fields) of the kernel calls of FIDInceptionV3 (FID features and is_features) and LPIPSAlex in tf32 at BATCHES,
    recorded on the CPU -> {key: (kind, fields, first batch)}."""
    from ladi_vton_b200.metrics import FIDInceptionV3, LPIPSAlex, random_state_dict
    inc = cpu_pack(FIDInceptionV3("tf32"), random_state_dict(FIDInceptionV3().param_shapes(), 0))
    lp = cpu_pack(LPIPSAlex("tf32"), random_state_dict(LPIPSAlex().param_shapes(), 1))
    desc = {}
    for B in BATCHES:
        def run():
            inc(torch.zeros((B, 3, 299, 299)))
            inc.is_features(torch.zeros((B, 3, 512, 384)))
            lp(torch.zeros((B, 3, 512, 384)), torch.zeros((B, 3, 512, 384)))
        for name, args in recorded(run):
            if name not in ARGS:
                assert name == "ladi_resize_tf1_u8", name  # fp32 already, replayed by the metrics census
                continue
            kind, spec = ARGS[name]
            f = {k: int(v) for k, v in zip(spec.split(), args) if k not in POINTERS}
            desc.setdefault(kind + " " + " ".join(f"{k}={v}" for k, v in f.items()), (kind, f, B))
    return desc


def test_tf32_census_replay_against_float64(cuda):
    desc = tf32_census()
    R = Replay(cuda, 97531)
    bad, worst = [], {}
    for key, (kind, f, B) in desc.items():
        errs, res = REPLAY[kind](R, f)
        bad += [f"{key} (batch {B}): {e}" for e in errs[:2]]
        worst[kind] = max(worst.get(kind, (0.0, "")), (res[0], f"{key}: {res[1]}"))
    per = {k: sum(1 for d in desc.values() if d[0] == k) for k in REPLAY}
    print(f"\n[tf32] census: {len(desc)} distinct calls over batches {BATCHES}: {per}")
    for k, (w, where) in worst.items():
        print(f"  {k}: worst err/bound {w:.3f} at {where}")
    assert not bad, "\n".join(bad[:10])


# ================================================================================================================ networks end to end
def _oracle(fn, tf32):
    """fn() with cuDNN's TF32 convolutions on or off (matmuls stay fp32, PyTorch's default)."""
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = tf32
    try:
        with torch.no_grad():
            return fn()
    finally:
        torch.backends.cudnn.allow_tf32 = old


def _inception_pair(cuda, n=8, seed=11):
    """tf32 and bf16 engine FIDInceptionV3 and the oracle state dict, sharing random weights with BatchNorm calibrated on the batch."""
    from ladi_oracle import metrics as OM
    from ladi_vton_b200.metrics import FIDInceptionV3, random_state_dict
    sd = {k: v.to(cuda) for k, v in random_state_dict(FIDInceptionV3().param_shapes(), seed).items()}
    g = torch.Generator(device=cuda).manual_seed(seed)
    x = F.interpolate(torch.rand(n, 3, 75, 75, generator=g, device=cuda), size=(299, 299), mode="bilinear") * 255
    with torch.no_grad():
        OM.calibrate_batchnorm(sd, x)
    cpu = {k: v.cpu() for k, v in sd.items()}
    return FIDInceptionV3("tf32").load_state_dict(cpu).to(cuda), FIDInceptionV3().load_state_dict(cpu).to(cuda), sd, x


def test_cudnn_runs_tf32(cuda):
    """The comparison below means something only if cuDNN's TF32 setting changes its convolutions on this card: report both errors."""
    g = torch.Generator(device=cuda).manual_seed(3)
    x = torch.randn(8, 192, 35, 35, generator=g, device=cuda)
    w = torch.randn(64, 192, 3, 3, generator=g, device=cuda) / 40
    ref = F.conv2d(x.double(), w.double(), padding=1)
    e = {t: rel_l2(_oracle(lambda: F.conv2d(x, w, padding=1), t), ref) for t in (False, True)}
    print(f"\n[tf32] cuDNN 3x3 conv rel-L2 against float64: allow_tf32=False {e[False]:.2e}, True {e[True]:.2e}")
    assert e[True] > 10 * e[False], e


def test_inception_stages_vs_oracle(cuda):
    """Every stage fed the oracle's own fp32 input: the error one stage adds in tf32, and in bf16 (fed the input rounded to bf16)."""
    from ladi_oracle import metrics as OM
    from ladi_vton_b200 import ops
    net_tf, net_bf, sd, x = _inception_pair(cuda)
    nets = {"tf32": net_tf, "bf16": net_bf}
    with torch.no_grad():
        o = OM._bconv(sd, "Conv2d_1a_3x3", (x - 128) / 128, stride=2)
    errs = {p: {"Conv2d_1a_3x3": rel_l2(n.layers["Conv2d_1a_3x3"](x, shift=n.shift, scale=n.scale).permute(0, 3, 1, 2), o)}
            for p, n in nets.items()}

    def stage(name, net):
        L = net.layers
        if name in ("maxpool1", "maxpool2"):
            return lambda t: ops.pool2d(t, 3, 2, 0, ops.POOL_MAX)
        if name.startswith("Conv2d"):
            return L[name]
        if name in ("Mixed_5b", "Mixed_5c", "Mixed_5d"):
            return lambda t: net._block_a(t, name)
        if name == "Mixed_6a":
            return lambda t: net._block_b(t, name)
        if name == "Mixed_7a":
            return lambda t: net._block_d(t, name)
        if name in ("Mixed_7b", "Mixed_7c"):
            return lambda t: net._block_e(t, name, ops.POOL_AVG_EXCLUDE_PAD if name == "Mixed_7b" else ops.POOL_MAX)
        return lambda t: net._block_c(t, name)

    oracle = [("Conv2d_2a_3x3", lambda t: OM._bconv(sd, "Conv2d_2a_3x3", t)),
              ("Conv2d_2b_3x3", lambda t: OM._bconv(sd, "Conv2d_2b_3x3", t, padding=1)), ("maxpool1", lambda t: F.max_pool2d(t, 3, 2)),
              ("Conv2d_3b_1x1", lambda t: OM._bconv(sd, "Conv2d_3b_1x1", t)), ("Conv2d_4a_3x3", lambda t: OM._bconv(sd, "Conv2d_4a_3x3", t)),
              ("maxpool2", lambda t: F.max_pool2d(t, 3, 2))]
    oracle += [(m, lambda t, m=m: OM._a(sd, m, t)) for m in ("Mixed_5b", "Mixed_5c", "Mixed_5d")]
    oracle += [("Mixed_6a", lambda t: OM._b(sd, "Mixed_6a", t))]
    oracle += [(m, lambda t, m=m: OM._c(sd, m, t)) for m in ("Mixed_6b", "Mixed_6c", "Mixed_6d", "Mixed_6e")]
    oracle += [("Mixed_7a", lambda t: OM._d(sd, "Mixed_7a", t)), ("Mixed_7b", lambda t: OM._e(sd, "Mixed_7b", t, False)),
               ("Mixed_7c", lambda t: OM._e(sd, "Mixed_7c", t, True))]
    with torch.no_grad():
        for name, orc in oracle:
            t = o.permute(0, 2, 3, 1).contiguous()
            e_tf, e_bf = stage(name, nets["tf32"])(t), stage(name, nets["bf16"])(t.to(torch.bfloat16))
            assert e_tf.dtype == torch.float32
            o = orc(o)
            errs["tf32"][name] = rel_l2(e_tf.permute(0, 3, 1, 2), o)
            errs["bf16"][name] = rel_l2(e_bf.permute(0, 3, 1, 2), o)
    for p in ("tf32", "bf16"):
        print(f"\n[tf32] inception stage rel-L2 {p}: " + ", ".join(f"{k} {v:.2e}" for k, v in errs[p].items()))
    assert max(errs["tf32"].values()) < STAGE_REL_L2, errs["tf32"]
    ratios = {k: errs["tf32"][k] / errs["bf16"][k] for k in errs["tf32"] if errs["bf16"][k] > 0}
    print("[tf32] stage error ratio tf32 / bf16: " + ", ".join(f"{k} {v:.3f}" for k, v in ratios.items()))
    assert max(ratios.values()) <= TF32_VS_BF16, ratios


def _gate(what, e_tf, e_cu, e_bf, vs_bf16=TF32_VS_BF16):
    print(f"\n[tf32] {what}: engine tf32 {e_tf:.3e}, cuDNN TF32 {e_cu:.3e} (ratio {e_tf / e_cu:.2f}), engine bf16 {e_bf:.3e} "
          f"(ratio {e_tf / e_bf:.3f})")
    assert e_tf <= TF32_VS_CUDNN * e_cu, (what, e_tf, e_cu)
    assert e_tf <= vs_bf16 * e_bf, (what, e_tf, e_bf)


def test_inception_vs_oracle(cuda):
    from ladi_oracle import metrics as OM
    net, net_bf, sd, x = _inception_pair(cuda)
    feats = net(x)
    of, ol = _oracle(lambda: OM.inception_features(sd, x), False)
    cf, cl = _oracle(lambda: OM.inception_features(sd, x), True)
    bf = net_bf(x)
    assert feats.shape == (8, 2048) and feats.dtype == torch.float32
    _gate("pool3 features rel-L2", rel_l2(feats, of), rel_l2(cf, of), rel_l2(bf, of), TF32_VS_BF16_E2E)
    _gate("unbiased logits rel-L2", rel_l2(net.unbiased_logits(feats), ol), rel_l2(cl, ol), rel_l2(net_bf.unbiased_logits(bf), ol), TF32_VS_BF16_E2E)
    assert torch.equal(net(x), feats)
    # the IS path: TF1 resize of [0, 1] images, then the same network
    imgs = F.interpolate(x / 255, size=(512, 384), mode="bilinear").clamp(0, 1)
    ref_is = _oracle(lambda: OM.inception_features(sd, OM.resize_tf1_u8(imgs, 299, 299))[1], False)
    cud_is = _oracle(lambda: OM.inception_features(sd, OM.resize_tf1_u8(imgs, 299, 299))[1], True)
    _gate("is_features logits rel-L2", rel_l2(net.is_features(imgs), ref_is), rel_l2(cud_is, ref_is), rel_l2(net_bf.is_features(imgs), ref_is), TF32_VS_BF16_E2E)


def test_lpips_vs_oracle(cuda):
    from ladi_oracle import metrics as OM
    from ladi_vton_b200.metrics import LPIPSAlex, random_state_dict
    sd = random_state_dict(LPIPSAlex().param_shapes(), 12)
    net, net_bf = LPIPSAlex("tf32").load_state_dict(sd).to(cuda), LPIPSAlex().load_state_dict(sd).to(cuda)
    g = torch.Generator(device=cuda).manual_seed(12)
    a = F.interpolate(torch.rand(4, 3, 64, 48, generator=g, device=cuda), size=(512, 384), mode="bilinear")
    b = (a + 0.1 * torch.randn(a.shape, generator=g, device=cuda)).clamp(0, 1)
    sdc = {k: v.to(cuda) for k, v in sd.items()}
    want = _oracle(lambda: OM.lpips(sdc, a, b), False).double()
    cud = _oracle(lambda: OM.lpips(sdc, a, b), True).double()
    got = net(a, b)
    rel = lambda y: float(((y.double() - want).abs() / want.abs()).max())  # noqa: E731
    _gate("lpips per-pair max rel", rel(got), rel(cud), rel(net_bf(a, b)))
    assert [t.dtype for t in net.taps(a)] == [torch.float32] * 5
    assert torch.equal(net(a, b), got)


def test_statistics_from_engine_vs_oracle_features(cuda):
    """FID / KID / IS from tf32 and bf16 engine features against the same statistics from fp32 oracle features of the same images."""
    from ladi_oracle import metrics as OM
    from ladi_vton_b200.metrics import feature_stats, frechet_distance, inception_score, kernel_distance
    net, net_bf, sd, x = _inception_pair(cuda, n=32, seed=13)
    gen, ref = x[:16], x[16:]
    of_gen, ol_gen = _oracle(lambda: OM.inception_features(sd, gen), False)
    of_ref, _ = _oracle(lambda: OM.inception_features(sd, ref), False)
    f = lambda a, b: frechet_distance(*feature_stats(a), *feature_stats(b))  # noqa: E731
    np_ = lambda t: t.double().cpu().numpy()  # noqa: E731
    o = {"fid": f(np_(of_gen), np_(of_ref)), "kid": kernel_distance(np_(of_ref), np_(of_gen), seed=3),
         "is": inception_score(ol_gen.cpu().numpy(), seed=3)[0]}
    rels = {}
    for prec, m in (("tf32", net), ("bf16", net_bf)):
        eg, er = m(gen), m(ref)
        e = {"fid": f(np_(eg), np_(er)), "kid": kernel_distance(np_(er), np_(eg), seed=3), "is": inception_score(m.unbiased_logits(eg).numpy(), seed=3)[0]}
        rels[prec] = {k: abs(e[k] - o[k]) / abs(o[k]) for k in o}
    for k in o:
        print(f"\n[tf32] {k}: oracle {o[k]:.6g}; rel error tf32 {rels['tf32'][k]:.3e}, bf16 {rels['bf16'][k]:.3e}")
    for k in o:
        assert rels["tf32"][k] <= STAT_REL[k], (k, rels)


# ================================================================================================================ CLI
def _write_tree(root, gen, n=6, seed=15):
    from PIL import Image
    rs = np.random.RandomState(seed)
    names = [f"{i:05d}_00.jpg" for i in range(n)]
    os.makedirs(os.path.join(root, "test", "image"))
    os.makedirs(os.path.join(gen, "upper_body"))
    with open(os.path.join(root, "test_pairs.txt"), "w") as f:
        f.write("".join(f"{a} {b}\n" for a, b in zip(names, reversed(names))))
    for nm in names:
        gt = Image.fromarray(rs.randint(0, 256, size=(8, 6, 3)).astype(np.uint8)).resize((384, 512), Image.BILINEAR)
        gt.save(os.path.join(root, "test", "image", nm), quality=95)
        noisy = np.clip(np.asarray(gt, dtype=np.int16) + rs.randint(-20, 21, size=(512, 384, 3)), 0, 255).astype(np.uint8)
        Image.fromarray(noisy).save(os.path.join(gen, "upper_body", nm.replace(".jpg", ".png")))


def test_main_precision_tf32(cuda, tmp_path):
    from ladi_vton_b200.val_metrics import main
    root, gen, cache = str(tmp_path / "vitonhd"), str(tmp_path / "gen"), str(tmp_path / "cache")
    _write_tree(root, gen)
    argv = ["--gen_folder", gen, "--test_order", "paired", "--dataset", "vitonhd", "--vitonhd_dataroot", root, "--batch_size", "4",
            "--workers", "0", "--random_init", "--cache_dir", cache]
    m_bf = main(argv)
    assert sorted(os.listdir(cache)) == ["vitonhd_all_random0.npz"]
    m = main(argv + ["--precision", "tf32"])
    out = json.load(open(os.path.join(gen, "metrics_paired_all.json")))
    assert list(out) == ['ssim_score', 'lpips_score', 'fid_score', 'kid_score', 'is_score'] and out == m
    assert all(np.isfinite(v) for v in out.values()), out
    # its own statistics: the bf16 file was not reused
    assert sorted(os.listdir(cache)) == ["vitonhd_all_random0-tf32.npz", "vitonhd_all_random0.npz"]
    bf_feats = np.load(os.path.join(cache, "vitonhd_all_random0.npz"))["feats"]
    tf_feats = np.load(os.path.join(cache, "vitonhd_all_random0-tf32.npz"))["feats"]
    assert not np.array_equal(bf_feats, tf_feats)
    assert main(argv + ["--precision", "tf32"]) == m  # its own cache, fixed seeds: the same numbers
    assert sorted(os.listdir(cache)) == ["vitonhd_all_random0-tf32.npz", "vitonhd_all_random0.npz"]
    assert m["ssim_score"] == m_bf["ssim_score"]  # SSIM is fp32 in both
    print(f"\n[tf32] main(): tf32 {m}\n             bf16 {m_bf}")
