"""The kernel calls of the evaluation metrics (`val_metrics.compute_metrics`, `tools/bench_metrics.py`), replayed one by one against a
float64 reference with per-element error bounds, and the metrics kernels tested at their edges with the same checkers.

The census (CPU).  The metrics networks are packed on the CPU from `random_state_dict` and their Python sequencing runs on CPU tensors
with the ABI calls recorded instead of launched (`lib.RECORD`): `FIDInceptionV3.__call__` on 299x299 pixels, `is_features` (the TF1
resize of 512x384 images to 299x299, then the Inception), `LPIPSAlex.__call__` on B pairs (2B images through AlexNet) and `metrics.ssim`
at 512x384.  Batches: 32 (`compute_metrics`' default), 64 (`bench_metrics.py`), 1, and the ragged last batches at batch 32 of the
standard test splits (VITON-HD's 2032 pairs leave 16, a Dress Code category's 1800 leave 8).  Convolutions / GEMMs go through
python_trace in the workload census's fields (those either other census replays are skipped); their plans are queried
with the production split-K workspace (ops.SPLITK_WS_BYTES), because under `lib.RECORD` `ops.splitk_workspace` hands out a 4 KB stub
that would rule split-K out.  Every other entry point needs a row in this file's SCHEMA, or test_metrics_census_integrity fails.
Every recorded GEMM output starts at a multiple of 8 columns of its concatenation (asserted), so replaying it at column 0 of a
buffer of the same pitch takes the same plan.

The replay (GPU).  Conv / GEMM through the workload census's replay_conv (tests/kernel_check.py).  Every other kind on fresh buffers: NaN input pitch gaps, a
NaN-poisoned output with a tail, the call's columns finite afterwards and everything else NaN (a pool into a concatenation slice leaves
the other channels NaN; `lpips_layer` adds to a non-zero `acc` and touches nothing else), and a second run bit-identical.

References and bounds (per element; u = 2^-24; ROUND1 = 2^-8, one bf16 rounding):
  im2col NHWC, max pool   exact (a copy, zeros in the padding and in the columns >= kh*kw*c; the maximum of bf16 values).
  im2col pixels   bit-equal to torch's fp32 (x - shift) / scale rounded to bf16 (the Makefile has no fast-math: the division is IEEE),
            and within ROUND1 |r| + (1 + ROUND1) 2^-22 (|x| + |shift|) / scale of float64 (the fp32 difference and quotient: 2u each).
  average pools   float64 mean over the window with torch's count for the mode (AVG: the window clipped to the padded image; EXCLUDE_PAD:
            clipped to the image).  The kernel sums the m <= k*k values in fp32 in order ((m - 1) u sum|x|), multiplies by the fp32
            reciprocal of the count (2u), then rounds to bf16: ROUND1 |r| + (1 + ROUND1)(k*k + 2) u mean|x|.
  global average  fp32 out: a sequential sum of hw terms and one division: 2u |r| + (hw + 1) u mean|x|.
  lpips_layer   the same formula in float64 on the same bf16 features, per image.  With g = ceil(c / 32) + 5 (the lanes' FMA chains and
            the 5-level butterfly), the fp32 sum of squares is off by g u relative, so ra = 1 / (sqrt(sa) + 1e-10) by
            dr = (g / 2 + 3) u (sqrt, add, divide); t = a ra - b rb by E_t = (dr + 2u)(|a| ra + |b| rb), an absolute bound that holds
            for near-identical pairs where t cancels; d = sum lin t^2 by sum lin (2|t| E_t + E_t^2 + 2u t^2) + g u d.  The pixel mean:
            each warp sums ceil(hw / 16) values, the 16 warps are combined in order, then / hw and acc +=:
            (ceil(hw / 16) + 17) u D + u |acc + D|.
  ssim      float64 reference with float64 Gaussian weights.  Each of the five filtered moments m0 = G*x, m1 = G*y, m2 = G*x^2,
            m3 = G*y^2, m4 = G*xy is off by E_MOM G*|source|: the kernel's fp32 weights (expf and the normalisation, measured on an fp32
            emulation plus 4u for expf's 2 ulp, twice for the two passes) and two 11-tap FMA chains with the product (24u).  These go
            through mu^2, mu_x mu_y, the one-pass variances E[x^2] - mu^2 (their cancellation is where the bound grows) and the ratio
            S = A1 A2 / (B1 B2) by its float64 partial derivatives, with the denominators' errors taken against B - eB.  The image value
            adds the per-thread channel sum, the 8-level block tree, the reduce's ceil(tiles / 256) strided terms and its 8-level tree,
            and the two fp32 operations of the scale.
  resize_tf1_u8   texels quantised from the fp32 product x * 255 by truncation, as torch's fp32 `.byte()` does; float64 lerp at the
            float64 source position o * in / out.  Bound: 8 u 255 for the fp32 lerps, plus the fp32 position's error (2^-22 pos + u)
            times the largest texel step within one texel of the sample on that axis: bilinear interpolation is continuous, so a floor
            that lands on the other side of an integer stays inside this bound.
The CPU tests show the bounds have teeth: the same checkers reject simulated faults and accept honest fp32 emulations.

Placement rules of the metrics entry points are tested on the CPU in a child process without a visible device: the entry point must
return the named error; a call that passes its checks fails for lack of a device instead, so these tests never launch a kernel."""
import ctypes as C
import functools
import math
import time
from collections import defaultdict

import pytest
import torch
import torch.nn.functional as F

from kernel_check import (A, EPS24, ROUND1, SMS, Replay, assert_all_known, census, check_library_defaults, check_placement, collect, cpu_pack,
                          describe, determinism, exact, flat_buf, glue_census, key_of, layout, max_ratio, parse, pick, ptr, python_trace, ratio,
                          recorded, replay_conv, tail_nan, twice, worst_at)

POOL_MAX, POOL_AVG, POOL_EXCL, POOL_GLOBAL = 0, 1, 2, 3
SSIM_C1, SSIM_C2 = 0.01 ** 2, 0.03 ** 2

# ================================================================================================================ the census (CPU)
# entry point -> (kind, its arguments in order: pointers are "name:role" with role in / out / io; "stream" is dropped)
SCHEMA = {
    "ladi_im2col_bf16": ("im2col", "x:in f32 n c h w pitch kh kw sh sw ph pw shift:in scale:in out:out kpad stream"),
    "ladi_pool2d_bf16": ("pool2d", "x:in n h w c xp k s p mode out:out op c_off stream"),
    "ladi_lpips_layer": ("lpips_layer", "fa:in fb:in n h w c pitch lin:in acc:io stream"),
    "ladi_ssim_f32": ("ssim", "x:in y:in n c h w ws:out out:out stream"),
    "ladi_resize_tf1_u8": ("resize_tf1", "x:in n c h w oh ow out:out stream"),
}
KINDS = ["conv"] + sorted({k for k, _ in SCHEMA.values()})
# (label, batch): compute_metrics' default, bench_metrics.py's second size, one image, and the ragged last batches at batch 32
BATCHES = [("batch 32 (compute_metrics default)", 32), ("batch 64 (tools/bench_metrics.py)", 64), ("batch 1", 1),
           ("batch 16 (VITON-HD: 2032 test pairs at batch 32)", 16), ("batch 8 (Dress Code: 1800 pairs per category at batch 32)", 8)]


@functools.lru_cache(maxsize=None)
def _nets():
    from ladi_vton_b200.metrics import FIDInceptionV3, LPIPSAlex, random_state_dict
    inc, lp = FIDInceptionV3(), LPIPSAlex()
    return cpu_pack(inc, random_state_dict(inc.param_shapes(), 0)), cpu_pack(lp, random_state_dict(lp.param_shapes(), 1))


def _metrics_calls(B, H=512, W=384):
    from ladi_vton_b200 import metrics as M
    inc, lp = _nets()

    def run():
        inc(torch.zeros((B, 3, 299, 299)))  # FID / KID features of clean-resized images
        inc.is_features(torch.zeros((B, 3, H, W)))  # IS: TF1 resize, then the same network
        lp(torch.zeros((B, 3, H, W)), torch.zeros((B, 3, H, W)))
        M.ssim(torch.zeros((B, 3, H, W)), torch.zeros((B, 3, H, W)))
    return recorded(run)


def conv_plan_at_production_ws(desc):
    """The plan of a recorded ConvDesc with the production split-K workspace (never dereferenced) on SMS SMs."""
    from ladi_vton_b200 import lib, ops
    q = lib.ConvDesc.from_buffer_copy(desc)
    q.splitk_ws, q.splitk_ws_bytes = 1 << 40, ops.SPLITK_WS_BYTES
    return lib.conv_plan(q, SMS)


def metrics_collect(work):
    """work = [(label, () -> recorded calls)] -> (desc, calls, unknown, misplaced): desc = OrderedDict key -> {kind, f, first, n, plan}
    of the descriptors neither other census replays; calls = {label: {kind: [calls, set of keys]}}; unknown = entry points recorded
    without a SCHEMA row; misplaced = GEMM outputs that do not start at a multiple of 8 columns."""
    known = set(census()[0]) | {k for k, d in glue_census()[0].items() if d["kind"] == "conv"}
    unknown, misplaced = [], []

    def classify(call):
        name, args = call
        if name == "ladi_conv2d_bf16":
            d = args[0]._obj
            if d.out % 16:  # bf16 columns: the CPU allocator's blocks are 64-byte aligned, so this is the column offset mod 8
                misplaced.append(f"out column offset {d.out % 16 // 2} mod 8")
            op, f = parse(python_trace([call])[0])
            if key_of(op, f) in known:
                return op, key_of(op, f), None, None
            plan = conv_plan_at_production_ws(d)
            return op, key_of(op, f), {k: int(v) for k, v in f.items()}, dict(plan=dict(bn=plan.bn, splits=plan.splits, staged=plan.staged))
        if name in SCHEMA:
            kind, f = describe(name, args, SCHEMA)
            return kind, key_of(kind, f), f, dict(plan=None)
        unknown.append(name)
        return None
    desc, calls = collect([(wl, wl, rec) for wl, rec in work], classify)
    return desc, calls, unknown, misplaced


@functools.lru_cache(maxsize=None)
def metrics_census():
    check_library_defaults()
    return metrics_collect([(wl, functools.partial(_metrics_calls, B)) for wl, B in BATCHES])


# ================================================================================================================ references and bounds
def im2col_ref(x, kh, kw, sh, sw, ph, pw, k_pad):
    """x NHWC [n, h, w, c] -> rows [n*oh*ow, k_pad], column (ky*kw + kx)*c + ch, zeros in the padding and in columns >= kh*kw*c."""
    n, h, w, c = x.shape
    oh, ow = (h + 2 * ph - kh) // sh + 1, (w + 2 * pw - kw) // sw + 1
    xp = F.pad(x, (0, 0, pw, pw, ph, ph))
    taps = [xp[:, ky:ky + sh * (oh - 1) + 1:sh, kx:kx + sw * (ow - 1) + 1:sw, :] for ky in range(kh) for kx in range(kw)]
    return F.pad(torch.stack(taps, dim=3).reshape(n * oh * ow, kh * kw * c), (0, k_pad - kh * kw * c))


def im2col_pixel_expect(x, shift, scale, geo):
    """x NCHW fp32 pixels (one or more images), shift / scale fp32 [c] -> (r, bound) float64 rows of the pixel im2col."""
    s64, c64 = shift.double().view(-1, 1, 1), scale.double().view(-1, 1, 1)
    r = im2col_ref(((x.double() - s64) / c64).permute(0, 2, 3, 1), *geo)
    mag = im2col_ref(((x.double().abs() + s64.abs()) / c64.abs()).permute(0, 2, 3, 1), *geo)
    return r, ROUND1 * r.abs() + (1 + ROUND1) * 2.0 ** -22 * mag


def pool_expect(X, k, s, p, mode):
    """X NCHW float64 -> (r, bound) of max / average pooling (bound 0: exact for max)."""
    if mode == POOL_MAX:
        r = F.max_pool2d(X, k, s, p)
        return r, torch.zeros_like(r)
    r = F.avg_pool2d(X, k, s, p, count_include_pad=mode == POOL_AVG)
    ma = F.avg_pool2d(X.abs(), k, s, p, count_include_pad=mode == POOL_AVG)
    return r, ROUND1 * r.abs() + (1 + ROUND1) * (k * k + 2) * EPS24 * ma


def global_avg_expect(X):
    """X NCHW float64 -> (r, bound) [n, c]."""
    r = X.mean((2, 3))
    return r, 2 * EPS24 * r.abs() + (X.shape[2] * X.shape[3] + 1) * EPS24 * X.abs().mean((2, 3))


def lpips_expect(a, b, lin):
    """a, b [n, hw, c] float64 features, lin [c] -> (D, E) [n]: the spatial mean of sum_c lin (unit(a) - unit(b))^2 and its bound without
    the final `acc +=` rounding."""
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


@functools.lru_cache(maxsize=None)
def ssim_weights():
    """-> (float64 Gaussian weights, E_MOM): the relative error bound of a filtered moment (module docstring)."""
    k = torch.arange(11, dtype=torch.float64)
    g64 = torch.exp(-0.5 * ((k - 5) / 1.5) ** 2)
    g64 = g64 / g64.sum()
    d = (torch.arange(11, dtype=torch.float32) - 5.0) / 1.5  # the kernel's fp32 computation
    g32 = torch.exp(-0.5 * d * d)
    g32 = g32 / g32.sum()
    ew = float((g32.double() / g64 - 1).abs().max()) + 4 * EPS24
    return [float(v) for v in g64], 2 * ew + 24 * EPS24


def _gfilt(t, g):
    """Valid 11 x 11 separable filter of t [..., H, W] with the weights g -> [..., H - 10, W - 10]."""
    W, H = t.shape[-1] - 10, t.shape[-2] - 10
    hs = sum(g[k] * t[..., :, k:k + W] for k in range(11))
    return sum(g[k] * hs[..., k:k + H, :] for k in range(11))


def ssim_expect(x, y):
    """x, y NCHW float64 -> (r, bound) [n] per the module docstring."""
    n, c, h, w = x.shape
    g, em = ssim_weights()
    u = EPS24
    m0, m1, m2, m3, m4 = (_gfilt(t, g) for t in (x, y, x * x, y * y, x * y))
    e0, e1, e2, e3, e4 = (em * _gfilt(t, g) for t in (x.abs(), y.abs(), x * x, y * y, (x * y).abs()))
    mxx, myy, mxy = m0 * m0, m1 * m1, m0 * m1
    exx, eyy = 2 * m0.abs() * e0 + e0 * e0 + u * mxx, 2 * m1.abs() * e1 + e1 * e1 + u * myy
    exy = m1.abs() * e0 + m0.abs() * e1 + e0 * e1 + u * mxy.abs()
    vx, vy, cxy = m2 - mxx, m3 - myy, m4 - mxy
    evx, evy = e2 + exx + u * (m2 + mxx), e3 + eyy + u * (m3 + myy)
    ecxy = e4 + exy + u * (m4.abs() + mxy.abs())
    A1, A2, B1, B2 = 2 * mxy + SSIM_C1, 2 * cxy + SSIM_C2, mxx + myy + SSIM_C1, vx + vy + SSIM_C2
    eA1, eA2 = 2 * exy + 2 * u * A1.abs(), 2 * ecxy + 2 * u * A2.abs()
    eB1, eB2 = exx + eyy + 2 * u * B1, evx + evy + 2 * u * B2.abs()
    S = A1 * A2 / (B1 * B2)
    low = lambda B, e: torch.maximum(B - e, 0.5 * B)  # noqa: E731
    eS = (eA1 * A2.abs() + A1.abs() * eA2) / (B1 * B2).abs() + S.abs() * (eB1 / low(B1, eB1) + eB2 / low(B2, eB2) + 4 * u)
    vh, vw = h - 10, w - 10
    tiles = -(-vh // 16) * -(-vw // 16)
    cnt = c * vh * vw
    depth = c + 8 + math.ceil(tiles / 256) + 8
    r = S.sum((1, 2, 3)) / cnt
    return r, (eS.sum((1, 2, 3)) + depth * u * S.abs().sum((1, 2, 3))) / cnt + 2 * u * r.abs()


def resize_texels(x):
    """torch's fp32 (x * 255).byte() for x in [0, 1] (clamped as the kernel does), as float64."""
    return (x.float() * 255.0).clamp(0.0, 255.0).trunc().double()


def _tf1_axis(n_in, n_out, dev):
    pos = torch.arange(n_out, dtype=torch.float64, device=dev) * (n_in / n_out)
    i0 = pos.floor().long().clamp_max(n_in - 1)
    return i0, (i0 + 1).clamp_max(n_in - 1), pos - i0, 2.0 ** -22 * pos + EPS24


def resize_expect(x, oh, ow):
    """x NCHW fp32 in [0, 1] -> (r, bound) float64 [n, c, oh, ow] of the TF1 resize of the truncated texels."""
    q = resize_texels(x)
    h, w = q.shape[-2:]
    y0, y1, ly, dy = _tf1_axis(h, oh, q.device)
    x0, x1, lx, dx = _tf1_axis(w, ow, q.device)
    at = lambda yy, xx: q[:, :, yy[:, None], xx[None, :]]  # noqa: E731
    ly, lx = ly.view(-1, 1), lx.view(1, -1)
    tl, tr, bl, br = at(y0, x0), at(y0, x1), at(y1, x0), at(y1, x1)
    r = (1 - ly) * ((1 - lx) * tl + lx * tr) + ly * ((1 - lx) * bl + lx * br)
    # the largest texel step within one texel of the sample, per axis
    dX = F.max_pool2d(F.pad((q[..., 1:] - q[..., :-1]).abs(), (0, 1)), (1, 3), 1, (0, 1))
    dY = F.max_pool2d(F.pad((q[..., 1:, :] - q[..., :-1, :]).abs(), (0, 0, 0, 1)), (3, 1), 1, (1, 0))
    sx = torch.maximum(dX[:, :, y0[:, None], x0[None, :]], dX[:, :, y1[:, None], x0[None, :]])
    sy = torch.maximum(dY[:, :, y0[:, None], x0[None, :]], dY[:, :, y0[:, None], x1[None, :]])
    return r, 8 * EPS24 * 255.0 + dx.view(1, -1) * sx + dy.view(-1, 1) * sy


# ================================================================================================================ replay (GPU)


def _features(R, rows, c):
    """Post-ReLU-like activations with a sign: max pools must not let the padding win over negative values."""
    return R.randn(rows, c) * 2.0


def _pixel_affine(R, kh, c):
    """shift / scale of the pixel im2col: the LPIPS scaling layer for AlexNet's 11x11 stem, (x - 128) / 128 for the Inception's."""
    from ladi_vton_b200.metrics import LPIPS_SCALE, LPIPS_SHIFT
    if kh == 11:
        sh = torch.tensor([(1.0 + s) / 2 for s in LPIPS_SHIFT][:c], dtype=torch.float32, device=R.dev)
        sc = torch.tensor([s / 2 for s in LPIPS_SCALE][:c], dtype=torch.float32, device=R.dev)
        return R.rand, sh, sc
    return (lambda *s: R.rand(*s) * 255.0), torch.full((c,), 128.0, device=R.dev), torch.full((c,), 128.0, device=R.dev)


def replay_im2col(R, f):
    from ladi_vton_b200 import lib
    n, c, h, w, pitch, kh, kw, sh, sw, ph, pw, kp = (f[k] for k in ("n", "c", "h", "w", "pitch", "kh", "kw", "sh", "sw", "ph", "pw", "kpad"))
    oh, ow = (h + 2 * ph - kh) // sh + 1, (w + 2 * pw - kw) // sw + 1
    rows = n * oh * ow
    geo = (kh, kw, sh, sw, ph, pw, kp)
    if f["f32"]:
        draw, shift, scale = _pixel_affine(R, kh, c)
        x = draw(n, c, h, w)
    else:
        x, shift, scale = R.poisoned(n * h * w, pitch, _features(R, n * h * w, c)), None, None

    def fresh():
        flat, o = flat_buf(R, rows * kp, torch.bfloat16)
        return dict(flat=flat, out=o)
    runs = twice(lambda b: lib.call("ladi_im2col_bf16", ptr(x), f["f32"], n, c, h, w, pitch, kh, kw, sh, sw, ph, pw, ptr(shift), ptr(scale),
                                     ptr(b["out"]), kp, R.stream), fresh)
    out = runs[0]["out"].view(n, oh * ow, kp)
    errs = layout(out.view(rows, kp), 0, kp, "rows") + tail_nan(runs[0]["flat"], rows * kp, "rows") + determinism(runs, ["flat"])
    worst = (0.0, "bit-exact")
    for b in pick(n, rows * kp, 1 << 28):
        y = out[b]
        if f["f32"]:
            q = ((x[b:b + 1] - shift.view(-1, 1, 1)) / scale.view(-1, 1, 1)).bfloat16()  # torch fp32, IEEE division
            e, _ = exact(y, im2col_ref(q.permute(0, 2, 3, 1), *geo), f"image {b}: against bf16 of torch's fp32 affine")
            r, bound = im2col_pixel_expect(x[b:b + 1], shift, scale, geo)
            e2, res = worst_at(ratio(y, r, bound), ("row", "column"), f" of image {b}")
            errs += e + e2
            worst = max(worst, res)
        else:
            e, _ = exact(y, im2col_ref(x.view(n, h, w, pitch)[b:b + 1, ..., :c], *geo), f"image {b}")
            errs += e
    return errs, worst


def replay_pool2d(R, f, values=None):
    from ladi_vton_b200 import lib
    n, h, w, c, xp, k, s, p, mode, op, c_off = (f[q] for q in ("n", "h", "w", "c", "xp", "k", "s", "p", "mode", "op", "c_off"))
    x = R.poisoned(n * h * w, xp, _features(R, n * h * w, c) if values is None else values)
    X = x[:, :c].reshape(n, h, w, c).permute(0, 3, 1, 2).double()
    if mode == POOL_GLOBAL:
        oh = ow = 1
        dt = torch.float32
    else:
        oh, ow = (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1
        dt = torch.bfloat16
    rows = n * oh * ow

    def fresh():
        flat, o = flat_buf(R, rows * op, dt)
        return dict(flat=flat, out=o)
    runs = twice(lambda b: lib.call("ladi_pool2d_bf16", ptr(x), n, h, w, c, xp, k, s, p, mode, ptr(b["out"]), op, c_off, R.stream), fresh)
    out = runs[0]["out"].view(rows, op)
    errs = layout(out, c_off, c_off + c, "output") + tail_nan(runs[0]["flat"], rows * op, "output") + determinism(runs, ["flat"])
    y = out[:, c_off:c_off + c]
    if mode == POOL_GLOBAL:
        r, bound = global_avg_expect(X)
        e, res = worst_at(ratio(y, r, bound), ("image", "channel"))
        return errs + e, res
    r, bound = pool_expect(X, k, s, p, mode)
    r, bound = (t.permute(0, 2, 3, 1).reshape(rows, c) for t in (r, bound))
    if mode == POOL_MAX:
        e, res = exact(y.contiguous(), r.bfloat16(), "max pool")
        return errs + e, res
    e, res = worst_at(ratio(y, r, bound), ("output pixel", "channel"))
    return errs + e, res


def _lpips_features(R, n, hw, c):
    """Post-ReLU features of n image pairs [2n * hw, c]: odd pairs are near-identical (b = relu(a + small noise)), where t cancels."""
    a = R.randn(n, hw, c).clamp_min(0.0)
    b = R.randn(n, hw, c).clamp_min(0.0)
    near = (a + 0.02 * R.randn(n, hw, c)).clamp_min(0.0)
    b[1::2] = near[1::2]
    return torch.cat([a, b]).view(2 * n * hw, c)


def replay_lpips_layer(R, f, self_pair=False, calls=1):
    from ladi_vton_b200 import lib
    n, h, w, c, pitch = (f[k] for k in ("n", "h", "w", "c", "pitch"))
    hw = h * w
    feats = R.poisoned(2 * n * hw, pitch, _lpips_features(R, n, hw, c))
    fa, fb = feats[:n * hw], (feats[:n * hw] if self_pair else feats[n * hw:])
    lin_flat, lin = flat_buf(R, c, torch.float32)
    lin.copy_(R.rand(c) * 0.1)
    acc0 = R.rand(n) + 0.25

    def fresh():
        flat, a = flat_buf(R, n, torch.float32)
        a.copy_(acc0)
        return dict(flat=flat, acc=a)

    def call(b):
        for _ in range(calls):
            lib.call("ladi_lpips_layer", ptr(fa), ptr(fb), n, h, w, c, pitch, ptr(lin), ptr(b["acc"]), R.stream)
    runs = twice(call, fresh)
    acc = runs[0]["acc"]
    errs = tail_nan(runs[0]["flat"], n, "acc") + tail_nan(lin_flat, c, "lin") + determinism(runs, ["flat"])
    if self_pair:
        e, res = exact(acc, acc0, "acc after comparing each image with itself")
        return errs + e, res
    A = fa[:, :c].double().reshape(n, hw, c)
    B = fb[:, :c].double().reshape(n, hw, c)
    D, E = lpips_expect(A, B, lin.double())
    r, bound = acc0.double(), torch.zeros_like(D)
    for _ in range(calls):
        r = r + D
        bound = bound + E + EPS24 * r.abs()
    e, res = worst_at(ratio(acc, r, bound), ("image",), f" (hw {hw}, c {c}, {calls} call(s))")
    return errs + e, res


def _ssim_images(R, n, c, h, w, inputs):
    if inputs == "const":  # zero variance: S = 1 where the two constants agree
        x = torch.full((n, c, h, w), 0.5, device=R.dev)
        y = x.clone()
        y[1::2] = 0.75
        return x, y
    if inputs == "white":  # near-white backgrounds: tiny variance under a large mean, the one-pass cancellation regime
        x = 0.985 + 0.01 * R.rand(n, c, h, w)
        return x, (x + 0.002 * R.randn(n, c, h, w)).clamp(0.0, 1.0)
    x = R.rand(n, c, h, w)
    return x, (x + 0.15 * R.randn(n, c, h, w)).clamp(0.0, 1.0)


def replay_ssim(R, f, inputs="noise"):
    from ladi_vton_b200 import lib
    n, c, h, w = (f[k] for k in ("n", "c", "h", "w"))
    tiles = lib.load().ladi_ssim_partials(h, w)
    x, y = _ssim_images(R, n, c, h, w, inputs)

    def fresh():
        wf, ws = flat_buf(R, n * tiles, torch.float32)
        of, o = flat_buf(R, n, torch.float32)
        return dict(wf=wf, ws=ws, of=of, out=o)
    runs = twice(lambda b: lib.call("ladi_ssim_f32", ptr(x), ptr(y), n, c, h, w, ptr(b["ws"]), ptr(b["out"]), R.stream), fresh)
    errs = tail_nan(runs[0]["wf"], n * tiles, "ws") + tail_nan(runs[0]["of"], n, "out") + determinism(runs, ["wf", "of"])
    r, bound = ssim_expect(x.double(), y.double())
    e, res = worst_at(ratio(runs[0]["out"], r, bound), ("image",), f" ({h}x{w}, c {c}, {tiles} partials, {inputs})")
    return errs + e, res


def _tie_inputs(R, n, c, h, w):
    """fp32(k / 255) and one ulp either side: the values whose product with 255 lands on an integer or next to it."""
    k = torch.randint(0, 256, (n, c, h, w), device=R.dev, generator=R.g).float()
    v = k / 255.0
    side = torch.randint(0, 3, (n, c, h, w), device=R.dev, generator=R.g)
    v = torch.where(side == 0, torch.nextafter(v, torch.zeros_like(v)), torch.where(side == 2, torch.nextafter(v, torch.ones_like(v)), v))
    return v.clamp(0.0, 1.0)


def replay_resize_tf1(R, f, inputs="noise"):
    from ladi_vton_b200 import lib
    n, c, h, w, oh, ow = (f[k] for k in ("n", "c", "h", "w", "oh", "ow"))
    x = _tie_inputs(R, n, c, h, w) if inputs == "ties" else R.rand(n, c, h, w)
    cnt = n * c * oh * ow

    def fresh():
        flat, o = flat_buf(R, cnt, torch.float32)
        return dict(flat=flat, out=o)
    runs = twice(lambda b: lib.call("ladi_resize_tf1_u8", ptr(x), n, c, h, w, oh, ow, ptr(b["out"]), R.stream), fresh)
    errs = tail_nan(runs[0]["flat"], cnt, "output") + determinism(runs, ["flat"])
    y = runs[0]["out"].view(n, c, oh, ow)
    if (oh, ow) == (h, w):  # identity: sample positions are integers, the output is the texels themselves
        e, res = exact(y, resize_texels(x).float(), "identity resize against torch's fp32 (x * 255).byte()")
        return errs + e, res
    worst = (0.0, "")
    for b in pick(n, cnt * 16, 1 << 28):
        r, bound = resize_expect(x[b:b + 1], oh, ow)
        e, res = worst_at(ratio(y[b:b + 1], r, bound)[0], ("channel", "y", "x"), f" of image {b}")
        errs += e
        worst = max(worst, res)
    return errs, worst


REPLAY = {"conv": replay_conv, "im2col": replay_im2col, "pool2d": replay_pool2d, "lpips_layer": replay_lpips_layer, "ssim": replay_ssim,
          "resize_tf1": replay_resize_tf1}


# ================================================================================================================ CPU: census integrity
def _threads(kind, f):
    """Threads the grid-stride loop of the call covers (one per 8 channels / 8 columns, one per element for the pixel form)."""
    if kind == "pool2d":
        oh, ow = (f["h"] + 2 * f["p"] - f["k"]) // f["s"] + 1, (f["w"] + 2 * f["p"] - f["k"]) // f["s"] + 1
        return f["n"] * oh * ow * f["c"] // 8
    oh = (f["h"] + 2 * f["ph"] - f["kh"]) // f["sh"] + 1
    ow = (f["w"] + 2 * f["pw"] - f["kw"]) // f["sw"] + 1
    return f["n"] * oh * ow * (f["kpad"] if f["f32"] else f["kpad"] // 8)


def print_metrics_census(desc, calls):
    print("\nmetrics census: calls (distinct descriptors neither other census replays) per kind")
    for wl, cnt in calls.items():
        print(f"  {wl}: {sum(v[0] for v in cnt.values())} calls; " + ", ".join(f"{k} {v[0]} ({len(v[1])})" for k, v in sorted(cnt.items())))
    per = defaultdict(int)
    for d in desc.values():
        per[d["kind"]] += 1
    print("  distinct over all batches: " + ", ".join(f"{k} {per[k]}" for k in KINDS if per[k]) + f"; {len(desc)} in all")
    plans = defaultdict(int)
    for d in desc.values():
        if d["plan"]:
            p = d["plan"]
            plans[("split-K" if p["splits"] > 1 else "staged" if p["staged"] else "direct", p["bn"])] += 1
    print(f"  conv / GEMM plans at {SMS} SMs with the production split-K workspace: "
          + ", ".join(f"{path} BN {bn}: {v}" for (path, bn), v in sorted(plans.items())))


def test_metrics_census_integrity():
    from ladi_vton_b200 import lib
    desc, calls, unknown, misplaced = metrics_census()
    print_metrics_census(desc, calls)
    assert_all_known(unknown)
    assert not misplaced, f"GEMM outputs off the 8-column grid: {misplaced[:5]}"
    assert set(REPLAY) == set(KINDS) and {d["kind"] for d in desc.values()} <= set(REPLAY)
    for name, (kind, spec) in SCHEMA.items():
        assert name in lib.SIGNATURES and len(spec.split()) == len(lib.SIGNATURES[name][0]), f"SCHEMA row of {name} does not match its signature"
    for wl, cnt in calls.items():
        assert cnt["lpips_layer"][0] == 5 and cnt["ssim"][0] == 1 and cnt["resize_tf1"][0] == 1, wl
    by = defaultdict(list)
    for d in desc.values():
        by[d["kind"]].append(d["f"])
    cap = SMS * 16 * 256
    im = by["im2col"]
    assert any(f["f32"] and f["shift"] and f["scale"] and (f["kh"], f["sh"]) == (11, 4) for f in im), "pixel im2col of AlexNet's 11x11/4 stem"
    assert any(f["f32"] and f["shift"] and f["scale"] and (f["kh"], f["sh"]) == (3, 2) for f in im), "pixel im2col of the Inception's 3x3/2 stem"
    assert any(_threads("im2col", f) > cap for f in im), "im2col past the grid-stride cap"
    pools = by["pool2d"]
    assert {(f["c_off"], f["op"]) for f in pools if f["mode"] == POOL_MAX and f["c_off"]} >= {(480, 768), (512, 1280)}, \
        "max pool into the concatenation of Mixed_6a and Mixed_7a"
    assert {f["h"] for f in pools if f["mode"] == POOL_EXCL} >= {35, 17, 8}, "exclude-pad average pool at 35x35, 17x17 and 8x8"
    assert any(f["mode"] == POOL_GLOBAL for f in pools), "fp32 global average"
    assert any(_threads("pool2d", f) > cap for f in pools if f["mode"] != POOL_GLOBAL), "pool2d past the grid-stride cap"
    assert all(f["c_off"] % 8 == 0 for f in pools)
    convs = [d for d in desc.values() if d["kind"] == "conv"]
    split = [d["f"] for d in convs if d["plan"]["splits"] > 1]
    assert any(f["K"] == 2048 and f["cout"] == 320 and f["op"] == 2048 for f in split), "split-K Mixed_7c branch1x1 into its concatenation"
    assert any(f["K"] == 2048 and f["cout"] == 192 and f["op"] == 2048 for f in split), "split-K Mixed_7c branch_pool into its concatenation"
    assert any(f["n"] == 1 and f["cout"] == 384 and f["op"] == 768 for f in split), "split-K Mixed_6a branch3x3 into its concatenation at batch 1"
    assert any(d["f"]["k"] == 3 and d["f"]["h"] == d["f"]["w"] == 8 for d in convs), "implicit 3x3 at 8x8"
    assert any(lib.load().ladi_ssim_partials(f["h"], f["w"]) > 256 for f in by["ssim"]), "SSIM with more than 256 partials"
    # taps 4 and 5 (256 channels at 31x23) share one descriptor
    assert {(f["c"], f["h"], f["w"]) for f in by["lpips_layer"]} >= {(64, 127, 95), (192, 63, 47), (384, 31, 23), (256, 31, 23)}, "all LPIPS taps"
    assert any((f["h"], f["w"], f["oh"], f["ow"]) == (512, 384, 299, 299) for f in by["resize_tf1"])


def test_metrics_census_rejects_unknown_entry_point():
    """A workload that records an entry point without a SCHEMA row next to a known one: the census reports it, the integrity check fails."""
    known = ("ladi_resize_tf1_u8", (C.c_void_p(16), 1, 3, 8, 8, 4, 4, C.c_void_p(32), C.c_void_p(0)))
    desc, calls, unknown, _ = metrics_collect([("fake workload", lambda: [known, ("ladi_not_in_the_schema", (C.c_void_p(16), 3, C.c_void_p(0)))])])
    assert unknown == ["ladi_not_in_the_schema"] and [d["kind"] for d in desc.values()] == ["resize_tf1"]
    with pytest.raises(AssertionError, match="ladi_not_in_the_schema"):
        assert_all_known(unknown)


# ================================================================================================================ CPU: the bounds have teeth


def test_teeth_exclude_pad_counts_padding():
    g = torch.Generator().manual_seed(11)
    x = (torch.randn((2, 16, 9, 7), generator=g) * 2).bfloat16().float()
    r, bound = pool_expect(x.double(), 3, 1, 1, POOL_EXCL)
    assert max_ratio(F.avg_pool2d(x, 3, 1, 1, count_include_pad=False).bfloat16(), r, bound) <= 1
    assert max_ratio(F.avg_pool2d(x, 3, 1, 1, count_include_pad=True).bfloat16(), r, bound) > 1  # 1. padding counted at the border


@pytest.mark.parametrize("kh,sh,ph", [(11, 4, 2), (3, 2, 1)])
def test_teeth_pixel_affine_on_padding(kh, sh, ph):
    g = torch.Generator().manual_seed(12)
    lpips = kh == 11
    x = torch.rand((1, 3, 24, 20), generator=g) * (1.0 if lpips else 255.0)
    from ladi_vton_b200.metrics import LPIPS_SCALE, LPIPS_SHIFT
    shift = torch.tensor([(1.0 + s) / 2 for s in LPIPS_SHIFT]) if lpips else torch.full((3,), 128.0)
    scale = torch.tensor([s / 2 for s in LPIPS_SCALE]) if lpips else torch.full((3,), 128.0)
    geo = (kh, kh, sh, sh, ph, ph, (kh * kh * 3 + 63) // 64 * 64)
    r, bound = im2col_pixel_expect(x, shift, scale, geo)
    honest = im2col_ref(((x - shift.view(-1, 1, 1)) / scale.view(-1, 1, 1)).bfloat16().permute(0, 2, 3, 1), *geo)
    xp = F.pad(x, (ph, ph, ph, ph))  # 2. zero padding first, then the affine: the padding becomes -shift / scale
    faulty = im2col_ref(((xp - shift.view(-1, 1, 1)) / scale.view(-1, 1, 1)).bfloat16().permute(0, 2, 3, 1), kh, kh, sh, sh, 0, 0, geo[6])
    assert max_ratio(honest, r, bound) <= 1
    assert max_ratio(faulty, r, bound) > 1


def _ssim_emulate(x, y, extent=0, drop_last_tile=False):
    """fp32 SSIM per image as the kernel computes it (fp32 weights from exp and the normalisation, separable fp32 filtering, one-pass
    variances); faults: `extent` more valid positions per axis (the window hangs off the zero-filled image), the last tile's sum dropped."""
    n, c, h, w = x.shape
    d = (torch.arange(11, dtype=torch.float32) - 5.0) / 1.5
    g = torch.exp(-0.5 * d * d)
    g = g / g.sum()

    def filt(t):
        t = F.pad(t, (0, extent, 0, extent)).reshape(n * c, 1, h + extent, w + extent)
        return F.conv2d(F.conv2d(t, g.view(1, 1, 1, 11)), g.view(1, 1, 11, 1)).view(n, c, h + extent - 10, w + extent - 10)
    m0, m1, m2, m3, m4 = (filt(t) for t in (x, y, x * x, y * y, x * y))
    mxx, myy, mxy = m0 * m0, m1 * m1, m0 * m1
    S = ((2 * mxy + SSIM_C1) * (2 * (m4 - mxy) + SSIM_C2)) / ((mxx + myy + SSIM_C1) * ((m2 - mxx) + (m3 - myy) + SSIM_C2))
    vh, vw = h - 10, w - 10
    if drop_last_tile:
        S = S.clone()
        S[:, :, (vh - 1) // 16 * 16:, (vw - 1) // 16 * 16:] = 0.0
    return S.sum((1, 2, 3)) / (c * vh * vw)


def test_teeth_ssim():
    g = torch.Generator().manual_seed(13)
    x = torch.rand((2, 3, 64, 48), generator=g)
    y = (x + 0.15 * torch.randn(x.shape, generator=g)).clamp(0.0, 1.0)
    r, bound = ssim_expect(x.double(), y.double())
    assert max_ratio(_ssim_emulate(x, y), r, bound) <= 1
    assert max_ratio(_ssim_emulate(x, y, extent=1), r, bound) > 1  # 3. valid extent one too large
    assert max_ratio(_ssim_emulate(x, y, drop_last_tile=True), r, bound) > 1  # 4. the last partial tile dropped


def test_teeth_lpips_remainder_pixels():
    g = torch.Generator().manual_seed(14)
    n, hw, c = 3, 31 * 23, 256  # taps 4 / 5 at 512x384: hw % 16 = 9
    a = torch.randn((n, hw, c), generator=g).clamp_min(0).bfloat16().float()
    b = torch.randn((n, hw, c), generator=g).clamp_min(0).bfloat16().float()
    lin = torch.rand(c, generator=g) * 0.1
    D, E = lpips_expect(a.double(), b.double(), lin.double())

    def emulate(drop):
        ra = 1.0 / ((a * a).sum(-1, keepdim=True).sqrt() + 1e-10)
        rb = 1.0 / ((b * b).sum(-1, keepdim=True).sqrt() + 1e-10)
        d = (lin * (a * ra - b * rb) ** 2).sum(-1)
        return (d[:, :hw - hw % 16] if drop else d).sum(1) / hw
    assert max_ratio(emulate(False), D, E) <= 1
    assert max_ratio(emulate(True), D, E) > 1  # 5. the hw % 16 remainder pixels dropped


@pytest.mark.parametrize("fault", ["round", "half_pixel"])
def test_teeth_resize_tf1(fault):
    g = torch.Generator().manual_seed(15)
    x = torch.rand((1, 3, 64, 48), generator=g)
    oh, ow = 37, 37
    r, bound = resize_expect(x, oh, ow)

    def emulate(fault=None):
        q = x * 255.0
        q = q.round() if fault == "round" else q.trunc()

        def axis(n_in, n_out):
            s = torch.tensor(n_in / n_out, dtype=torch.float32)
            pos = torch.arange(n_out, dtype=torch.float32) * s
            if fault == "half_pixel":
                pos = ((torch.arange(n_out, dtype=torch.float32) + 0.5) * s - 0.5).clamp_min(0.0)
            i0 = pos.floor().long().clamp_max(n_in - 1)
            return i0, (i0 + 1).clamp_max(n_in - 1), pos - i0
        y0, y1, ly = axis(64, oh)
        x0, x1, lx = axis(48, ow)
        at = lambda yy, xx: q[:, :, yy[:, None], xx[None, :]]  # noqa: E731
        top = at(y0, x0) + (at(y0, x1) - at(y0, x0)) * lx
        bot = at(y1, x0) + (at(y1, x1) - at(y1, x0)) * lx
        return top + (bot - top) * ly.view(-1, 1)
    assert max_ratio(emulate(), r, bound) <= 1
    assert max_ratio(emulate(fault), r, bound) > 1  # 6. rounding instead of truncating / 7. half-pixel centres


# ================================================================================================================ CPU: placement rules
# (id, entry point, arguments with pointers as ints, expected message or None = the checks pass and the launch fails for lack of a device)
_IM2COL_NHWC = lambda x=A, out=A: ("ladi_im2col_bf16", [x, 0, 1, 8, 4, 4, 8, 3, 3, 1, 1, 1, 1, 0, 0, out, 72])  # noqa: E731
_IM2COL_PX = lambda x=A, sh=A, sc=A + 64, out=A: ("ladi_im2col_bf16", [x, 1, 1, 3, 8, 8, 0, 3, 3, 2, 2, 0, 0, sh, sc, out, 64])  # noqa: E731
_POOL = lambda x=A, out=A, mode=POOL_MAX: ("ladi_pool2d_bf16", [x, 1, 4, 4, 8, 8, 3, 1, 1, mode, out, 8, 0])  # noqa: E731
_LPIPS = lambda fa=A, fb=A, lin=A, acc=A: ("ladi_lpips_layer", [fa, fb, 2, 4, 4, 8, 8, lin, acc])  # noqa: E731
_SSIM = lambda x=A, y=A, ws=A, out=A, n=2: ("ladi_ssim_f32", [x, y, n, 3, 16, 16, ws, out])  # noqa: E731
_RESIZE = lambda x=A, out=A: ("ladi_resize_tf1_u8", [x, 1, 3, 8, 8, 4, 4, out])  # noqa: E731
PLACEMENT = [
    ("im2col nhwc x", *_IM2COL_NHWC(x=A + 8), "x 0x100008 must be 16-byte aligned"),
    ("im2col nhwc out", *_IM2COL_NHWC(out=A + 8), "out 0x100008 must be 16-byte aligned"),
    ("im2col nhwc ok", *_IM2COL_NHWC(), None),
    ("im2col pixels x", *_IM2COL_PX(x=A + 2), "x 0x100002 must be 4-byte aligned"),
    ("im2col pixels shift", *_IM2COL_PX(sh=A + 2), "shift 0x100002 must be 4-byte aligned"),
    ("im2col pixels scale", *_IM2COL_PX(sc=A + 66), "scale 0x100042 must be 4-byte aligned"),
    ("im2col pixels out", *_IM2COL_PX(out=A + 1), "out 0x100001 must be 2-byte aligned"),
    ("im2col pixels ok (out at a 2-byte offset)", *_IM2COL_PX(x=A + 4, out=A + 2), None),
    ("pool2d window x", *_POOL(x=A + 8), "x 0x100008 must be 16-byte aligned"),
    ("pool2d window out", *_POOL(out=A + 8, mode=POOL_EXCL), "out 0x100008 must be 16-byte aligned"),
    ("pool2d window ok", *_POOL(mode=POOL_AVG), None),
    ("pool2d global out", *_POOL(out=A + 2, mode=POOL_GLOBAL), "out 0x100002 must be 4-byte aligned"),
    ("pool2d global x", *_POOL(x=A + 1, mode=POOL_GLOBAL), "x 0x100001 must be 2-byte aligned"),
    ("pool2d global ok (x at a 2-byte offset)", *_POOL(x=A + 2, out=A + 4, mode=POOL_GLOBAL), None),
    ("lpips fa", *_LPIPS(fa=A + 1), "fa 0x100001 must be 2-byte aligned"),
    ("lpips fb", *_LPIPS(fb=A + 1), "fb 0x100001 must be 2-byte aligned"),
    ("lpips lin", *_LPIPS(lin=A + 2), "lin 0x100002 must be 4-byte aligned"),
    ("lpips acc", *_LPIPS(acc=A + 2), "acc 0x100002 must be 4-byte aligned"),
    ("lpips ok", *_LPIPS(fa=A + 2, fb=A + 6, lin=A + 4, acc=A + 12), None),
    ("ssim x", *_SSIM(x=A + 2), "x 0x100002 must be 4-byte aligned"),
    ("ssim y", *_SSIM(y=A + 2), "y 0x100002 must be 4-byte aligned"),
    ("ssim ws", *_SSIM(ws=A + 2), "ws 0x100002 must be 4-byte aligned"),
    ("ssim out", *_SSIM(out=A + 2), "out 0x100002 must be 4-byte aligned"),
    ("ssim n", *_SSIM(n=65536), "n 65536 exceeds 65535"),
    ("ssim ok at n = 65535", *_SSIM(n=65535), None),
    ("resize x", *_RESIZE(x=A + 2), "x 0x100002 must be 4-byte aligned"),
    ("resize out", *_RESIZE(out=A + 2), "out 0x100002 must be 4-byte aligned"),
    ("resize ok", *_RESIZE(x=A + 4, out=A + 4), None),
]


def test_placement_rules_without_a_device():
    """The placement rules of the metrics entry points (PLACEMENT), checked in a process that sees no device."""
    check_placement(PLACEMENT)


# ================================================================================================================ GPU: replay
@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_metrics_replay_against_float64(cuda, kind):
    desc = metrics_census()[0]
    todo = [(key, d) for key, d in desc.items() if d["kind"] == kind]
    assert todo, f"no {kind} descriptor in the metrics census"
    R = Replay(cuda, 5678)
    failures, worst, t0 = [], (0.0, "", ""), time.time()
    for key, d in todo:
        errs, res = REPLAY[kind](R, d["f"])
        if errs:
            failures.append(f"{key}\n    first issued by {d['first']}\n    " + "\n    ".join(errs))
        if res is not None and res[0] >= worst[0]:
            worst = (res[0], key, res[1])
        torch.cuda.empty_cache()
    print(f"\n{kind}: {len(todo)} distinct descriptors replayed in {time.time() - t0:.1f} s; worst err/bound {worst[0]:.3g}"
          + (f" ({worst[2]}; {worst[1]})" if worst[1] else ""))
    assert not failures, f"{len(failures)} of {len(todo)} {kind} descriptors fail:\n" + "\n".join(failures)


# ================================================================================================================ GPU: edges
def _ssim_f(n, c, vh, vw):
    return dict(x=1, y=1, n=n, c=c, h=vh + 10, w=vw + 10, ws=1, out=1)


def _pool_f(n, h, w, c, k, s, p, mode, xp=None, op=None, c_off=0):
    return dict(x=1, n=n, h=h, w=w, c=c, xp=xp or c, k=k, s=s, p=p, mode=mode, out=1, op=op or c_off + c, c_off=c_off)


def _lpips_f(n, h, w, c, pitch=None):
    return dict(fa=1, fb=1, n=n, h=h, w=w, c=c, pitch=pitch or c, lin=1, acc=1)


def _im2col_f(n, c, h, w, k, s, p, kpad, pitch=None, f32=0):
    (kh, kw), (sh, sw), (ph, pw) = k, s, p
    return dict(x=1, f32=f32, n=n, c=c, h=h, w=w, pitch=0 if f32 else (pitch or c), kh=kh, kw=kw, sh=sh, sw=sw, ph=ph, pw=pw, shift=f32,
                scale=f32, out=1, kpad=kpad)


def _resize_f(n, c, h, w, oh, ow):
    return dict(x=1, n=n, c=c, h=h, w=w, oh=oh, ow=ow, out=1)


EDGES = [
    # SSIM: valid extents 1, 15, 16, 17, 32, 33 on each axis (tile grids 1-3, last tiles of 1 and 16), c = 1, 3, 4
    *[(f"ssim valid {vh}x{vw} c{c}", "ssim", _ssim_f(3, c, vh, vw), {}) for vh, vw, c in
      [(1, 1, 1), (15, 33, 3), (16, 17, 4), (17, 16, 1), (32, 1, 3), (33, 15, 4), (1, 32, 3), (33, 33, 1)]],
    # partial counts around the reduce's 256-wide stride loop, and 1024x768
    ("ssim 255 partials", "ssim", _ssim_f(2, 3, 15 * 16, 17 * 16), {}),
    ("ssim 256 partials", "ssim", _ssim_f(2, 3, 256, 256), {}),
    ("ssim 257 partials", "ssim", _ssim_f(2, 1, 1, 257 * 16), {}),
    ("ssim 1024x768 (3072 partials)", "ssim", _ssim_f(2, 3, 1014, 758), {}),
    ("ssim constant images", "ssim", _ssim_f(4, 3, 40, 30), dict(inputs="const")),
    ("ssim near-white 512x384", "ssim", _ssim_f(4, 3, 502, 374), dict(inputs="white")),
    # pool2d: windows touching both borders in every mode, k = s, s > k, c_off + c == out_pitch, past the grid-stride cap
    *[(f"pool2d {hw}x{hw} k3 p1 mode {m}", "pool2d", _pool_f(2, hw, hw, 16, 3, 1, 1, m), {}) for hw in (1, 2, 3) for m in range(4)],
    *[(f"pool2d 3x3 k3 s2 p1 mode {m}", "pool2d", _pool_f(2, 3, 3, 8, 3, 2, 1, m), {}) for m in range(3)],
    *[(f"pool2d k = s = 2 mode {m}", "pool2d", _pool_f(2, 9, 7, 16, 2, 2, 0, m), {}) for m in range(3)],
    *[(f"pool2d s3 > k2 mode {m}", "pool2d", _pool_f(2, 11, 10, 16, 2, 3, 0, m), {}) for m in range(3)],
    *[(f"pool2d s4 > k3 p1 mode {m}", "pool2d", _pool_f(2, 13, 9, 8, 3, 4, 1, m), {}) for m in range(3)],
    *[(f"pool2d c_off + c == out_pitch mode {m}", "pool2d", _pool_f(2, 7, 5, 16, 3, 1, 1, m, xp=24, op=40, c_off=24), {}) for m in range(3)],
    ("pool2d past the grid-stride cap", "pool2d", _pool_f(4, 70, 70, 256, 3, 1, 1, POOL_EXCL), {}),
    # global average: hw = 1, c = 8, pitch > c, a channel window of a wider fp32 row
    ("global average hw 1 c 8", "pool2d", _pool_f(3, 1, 1, 8, 0, 0, 0, POOL_GLOBAL), {}),
    ("global average pitch > c", "pool2d", _pool_f(3, 5, 3, 8, 0, 0, 0, POOL_GLOBAL, xp=24, op=24, c_off=8), {}),
    # lpips_layer: hw 1, 15, 16, 17 and c 8, 40 (idle warps and lanes), pitch > c, a pair with itself, five accumulated calls
    *[(f"lpips hw {h * w} c {c}", "lpips_layer", _lpips_f(3, h, w, c), {}) for h, w in ((1, 1), (3, 5), (4, 4), (1, 17)) for c in (8, 40)],
    ("lpips pitch > c", "lpips_layer", _lpips_f(3, 5, 7, 40, pitch=56), {}),
    ("lpips pair with itself", "lpips_layer", _lpips_f(3, 31, 23, 256), dict(self_pair=True)),
    ("lpips five accumulated calls", "lpips_layer", _lpips_f(3, 9, 7, 64), dict(calls=5)),
    # im2col: k_pad >= kh*kw*c + 8, strides (2, 1) and (1, 2), windows hanging off both edges, rows past the grid-stride cap
    ("im2col k_pad past kh*kw*c + 8", "im2col", _im2col_f(2, 8, 6, 5, (3, 3), (1, 1), (1, 1), 88, pitch=16), {}),
    ("im2col stride (2, 1)", "im2col", _im2col_f(2, 16, 9, 8, (3, 3), (2, 1), (1, 1), 144), {}),
    ("im2col stride (1, 2)", "im2col", _im2col_f(2, 16, 8, 9, (1, 3), (1, 2), (0, 1), 48, pitch=24), {}),
    ("im2col windows off both edges", "im2col", _im2col_f(2, 8, 3, 3, (5, 5), (1, 1), (2, 2), 200), {}),
    ("im2col past the grid-stride cap", "im2col", _im2col_f(4, 16, 96, 96, (3, 3), (1, 1), (1, 1), 144), {}),
    ("im2col pixels stride (2, 1), AlexNet affine", "im2col", _im2col_f(2, 3, 30, 20, (11, 11), (2, 1), (2, 2), 384, f32=1), {}),
    ("im2col pixels windows off both edges", "im2col", _im2col_f(2, 3, 2, 3, (3, 3), (1, 2), (1, 1), 64, f32=1), {}),
    ("im2col pixels past the grid-stride cap", "im2col", _im2col_f(2, 3, 100, 100, (3, 3), (1, 1), (1, 1), 64, f32=1), {}),
    # resize_tf1_u8: identity (the truncated texels exactly), an up-scale, 512x384 and 1024x768 -> 299, inputs at k/255 and one ulp away
    ("resize identity", "resize_tf1", _resize_f(2, 3, 37, 29, 37, 29), {}),
    ("resize identity at k/255 +- 1 ulp", "resize_tf1", _resize_f(2, 3, 64, 48, 64, 48), dict(inputs="ties")),
    ("resize up-scale", "resize_tf1", _resize_f(2, 3, 20, 15, 47, 41), {}),
    ("resize 512x384 -> 299 at k/255 +- 1 ulp", "resize_tf1", _resize_f(2, 3, 512, 384, 299, 299), dict(inputs="ties")),
    ("resize 1024x768 -> 299", "resize_tf1", _resize_f(2, 3, 1024, 768, 299, 299), {}),
]


def test_edge_cases_are_what_they_say():
    """The edge shapes hit the limits they are named after (CPU)."""
    from ladi_vton_b200 import lib
    L = lib.load()
    e = {what: f for what, _, f, _ in EDGES}
    assert [L.ladi_ssim_partials(e[k]["h"], e[k]["w"]) for k in ("ssim 255 partials", "ssim 256 partials", "ssim 257 partials",
                                                                  "ssim 1024x768 (3072 partials)")] == [255, 256, 257, 3072]
    cap = SMS * 16 * 256
    assert _threads("pool2d", e["pool2d past the grid-stride cap"]) > cap
    assert all(_threads("im2col", e[k]) > cap for k in ("im2col past the grid-stride cap", "im2col pixels past the grid-stride cap"))
    f = e["im2col k_pad past kh*kw*c + 8"]
    assert f["kpad"] >= f["kh"] * f["kw"] * f["c"] + 8
    f = e["pool2d c_off + c == out_pitch mode 0"]
    assert f["c_off"] + f["c"] == f["op"]


@pytest.mark.gpu
@pytest.mark.parametrize("case", EDGES, ids=[c[0] for c in EDGES])
def test_metrics_edge_against_float64(cuda, case):
    what, kind, f, kw = case
    R = Replay(cuda, 2468)
    errs, res = REPLAY[kind](R, f, **kw)
    print(f"\n{what}: err/bound {res[0]:.3g} ({res[1]})")
    assert not errs, f"{what}:\n  " + "\n  ".join(errs)
