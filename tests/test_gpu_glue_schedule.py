"""The glue, cloth-warping and front-end kernels (csrc/warp.cu, the non-norm half of csrc/pointwise.cu, csrc/frontend.cu's small kernels)
at the edges of their launch policy and of their value ranges, against float64, and the placement rules of their entry points.

Shapes and values no workload reaches are driven through the glue census's replays (tests/kernel_check.py):
synthetic descriptors in the field names of its SCHEMA, so every case gets the census's float64 reference and per-element bound, its
NaN-poisoned outputs with a tail, its column-window checks and its second, bit-identical run.  The descriptors are not census rows: the
census records what the workloads run.

Launch policy.  The grid-stride kernels run min(ceil(work / 256), 16 SMs) blocks of 256 threads (grid_for in each .cu file).  With the
SM count of the device, selected cases sit at exactly one full pass (work = 16 SMs 256: every thread one element) and at the first work
count past it that the kind's shape can express (one element into a second pass where the work is any integer; 4 for space_to_depth2
with c = 1 and for ddim_cfg_step, whose work is a multiple of 4; 8 for patchify, whose k_pad is a multiple of 8; the next multiple of 3
for image_out_u8).  check_binarise's work is ceil(max(n_image, n_mask) / 4).  The image on the second pass is the last one, which the
census replays always check.

Value edges: NaN passes through the clamps of nhwc_to_nchw_clamp, image_out and posterior_sample's logvar, and through maxpool2's
window maximum, as the torch ops they restate pass it (torch.clamp, nn.MaxPool2d); image_out_u8 writes 0 for NaN (numpy's NaN -> uint8
cast is undefined, so the device's value is pinned).  A NaN's payload is not compared.

References added here (the census has none for these entry points):
  nhwc_to_nchw_f32   exact: the channel window [c_off, c_off + c) of an NHWC fp32 or bf16 tensor as NCHW fp32;
  upsample2x_nhwc    exact: nearest 2x, source pixel (y // 2, x // 2);
  pose_heatmaps      posemap.py's kpoint_to_heatmap in float64 (the maximum taken over the whole grid, not the kernel's closed form).
                     The kernel's exponent argument a = d / sigma^2 carries at most 7 * 2^-24 * a (the two fp32 differences and squares,
                     their sum, the fp32 1 / sigma^2 and the product), expf 2 ulp = 2^-22, so numerator and denominator each carry
                     7 * 2^-24 a + 2^-22 (amin for the denominator), plus 2^-24 for the eps addition and 2^-24 for the division:
                     bound (8 * 2^-24 (a + amin) + 2 * 2^-22 + 2 * 2^-24) |r| + 2^-125, the last term for an exponential that
                     underflows into fp32's subnormals (its absolute error 2^-149 over a denominator of at least eps = 2^-23).

CPU tests at the end show the new references have teeth (an fp32 emulation passes; x / y swapped, a nearest index off by one, floorf in
place of rintf and a NaN-dropping clamp or max are rejected), and check every placement rule in a process that sees no device."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from kernel_check import (A, EPS24, NAN, REPLAY, SCHEMA, SMS, Replay, check_placement, determinism, exact, flat_buf, ratio, sms, tail_nan, twice,
                          worst_at)

PASS = 16 * 256  # elements per SM in one full grid-stride pass
INF = float("inf")

# entry points the census does not record (kind -> argument names, in SCHEMA's format)
NEW_SCHEMA = {
    "nhwc_to_nchw_f32": "x:in f32 n c h w xp c_off out:out stream",
    "upsample2x_nhwc": "x:in n h w c out:out stream",
    "pose_heatmaps": "kpts:in n_maps h w sigma out:out stream",
}


def _fields(kind):
    spec = NEW_SCHEMA.get(kind) or next(a for k, a in SCHEMA.values() if k == kind)
    return [(t.split(":")[0], ":" in t) for t in spec.split() if t != "stream"]


def _f(kind, **kw):
    """A descriptor of `kind` in the schema's field names: every pointer present unless given as 0, every scalar given."""
    f = {}
    for name, is_ptr in _fields(kind):
        if is_ptr:
            f[name] = kw.pop(name, 1)
        else:
            assert name in kw, f"{kind}: scalar {name} missing"
            f[name] = kw.pop(name)
    assert not kw, f"{kind}: unknown fields {sorted(kw)}"
    return f


# ================================================================================================================ new references
def nhwc_to_nchw_expect(x, n, h, w, c, c_off):
    """x [n*h*w, pitch] (fp32 or bf16) -> NCHW fp32 [n, c, h, w] of channels [c_off, c_off + c)."""
    return x[:, c_off:c_off + c].float().reshape(n, h, w, c).permute(0, 3, 1, 2).contiguous()


def upsample_nearest_expect(x):
    """x NHWC [n, h, w, c] -> NHWC [n, 2h, 2w, c], pixel (y, x) <- (y // 2, x // 2)."""
    return x.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2)


def pose_expect(kpts, h, w, sigma):
    """kpts float64 [m, 2] (x, y) -> (r, bound) [m, h, w]: posemap.py's kpoint_to_heatmap in float64, per the module docstring."""
    ys, xs = torch.meshgrid(torch.arange(h, dtype=torch.float64, device=kpts.device), torch.arange(w, dtype=torch.float64, device=kpts.device),
                            indexing="ij")
    kx, ky = kpts[:, 0].view(-1, 1, 1), kpts[:, 1].view(-1, 1, 1)
    a = ((xs - kx) ** 2 + (ys - ky) ** 2) / float(sigma) ** 2
    e = torch.exp(-a)
    r = e / (e.amax(dim=(1, 2), keepdim=True) + float(np.finfo(np.float32).eps))
    drawn = (kpts > 0).any(dim=1).view(-1, 1, 1)
    r = torch.where(drawn, r, 0.0)
    amin = a.amin(dim=(1, 2), keepdim=True)
    return r, (8 * EPS24 * (a + amin) + 2 * 2.0 ** -22 + 2 * EPS24) * r.abs() + 2.0 ** -125


# ================================================================================================================ new replays (GPU)
def replay_nhwc_to_nchw_f32(R, f):
    from ladi_vton_b200 import lib
    f32, n, c, h, w, xp, c_off = (f[k] for k in ("f32", "n", "c", "h", "w", "xp", "c_off"))
    dt = torch.float32 if f32 else torch.bfloat16
    x = R.poisoned(n * h * w, xp, None, dtype=dt)
    x[:, c_off:c_off + c] = R.randn(n * h * w, c).to(dt)  # the rest of the row stays NaN: a read outside the window shows
    cnt = n * c * h * w

    def fresh():
        flat, o = flat_buf(R, cnt, torch.float32)
        return dict(flat=flat, out=o)
    runs = twice(lambda b: lib.call("ladi_nhwc_to_nchw_f32", C.c_void_p(x.data_ptr()), f32, n, c, h, w, xp, c_off, C.c_void_p(b["out"].data_ptr()),
                                     R.stream), fresh)
    errs = tail_nan(runs[0]["flat"], cnt, "output") + determinism(runs, ["flat"])
    e, res = exact(runs[0]["out"].view(n, c, h, w), nhwc_to_nchw_expect(x, n, h, w, c, c_off), "values")
    return errs + e, res


def replay_upsample2x_nhwc(R, f):
    from ladi_vton_b200 import lib
    n, h, w, c = f["n"], f["h"], f["w"], f["c"]
    x = R.randn(n, h, w, c).bfloat16()
    cnt = n * 4 * h * w * c

    def fresh():
        flat, o = flat_buf(R, cnt, torch.bfloat16)
        return dict(flat=flat, out=o)
    runs = twice(lambda b: lib.call("ladi_upsample2x_nhwc", C.c_void_p(x.data_ptr()), n, h, w, c, C.c_void_p(b["out"].data_ptr()), R.stream), fresh)
    errs = tail_nan(runs[0]["flat"], cnt, "output") + determinism(runs, ["flat"])
    e, res = exact(runs[0]["out"].view(n, 2 * h, 2 * w, c), upsample_nearest_expect(x), "values")
    return errs + e, res


POSE_KEYPOINTS = [(0.0, 0.0), (-3.0, -1.0), (0.0, 17.5), (12.25, 0.0), (-4.0, 30.0), (30.0, -6.0),  # missing / half-missing / negative
                  (100.0, 10.0), (5.0, 200.0), (-40.0, 200.0),                                    # off the map: nearest grid point clamped
                  (23.5, 31.5), (0.5, 7.5), (2.5, 0.5),                                           # half-integers: the rintf tie
                  (7.7, 3.2), (46.6, 63.4), (0.3, 0.2), (47.0, 63.0), (19.999, 40.501)]


def replay_pose_heatmaps(R, f, kpts=None):
    from ladi_vton_b200 import lib
    m, h, w, sigma = f["n_maps"], f["h"], f["w"], f["sigma"]
    k = torch.tensor(POSE_KEYPOINTS if kpts is None else kpts, dtype=torch.float32, device=R.dev)
    k = torch.cat([k, torch.cat([R.rand(m, 1) * (w + 4) - 2, R.rand(m, 1) * (h + 4) - 2], dim=1)])[:m].contiguous()
    cnt = m * h * w

    def fresh():
        flat, o = flat_buf(R, cnt, torch.float32)
        return dict(flat=flat, out=o)
    runs = twice(lambda b: lib.call("ladi_pose_heatmaps", C.c_void_p(k.data_ptr()), m, h, w, float(sigma), C.c_void_p(b["out"].data_ptr()),
                                     R.stream), fresh)
    errs = tail_nan(runs[0]["flat"], cnt, "output") + determinism(runs, ["flat"])
    r, bound = pose_expect(k.double(), h, w, float(np.float32(sigma)))
    e, res = worst_at(ratio(runs[0]["out"].view(m, h, w), r, bound), ("map", "y", "x"))
    return errs + e, res


def replay_check_binarise_values(R, f, image_values, mask_values, flags0):
    """check_binarise on the given values (padded to n_image / n_mask with in-range ones) with flags starting at flags0: the flags are
    flags0 OR the reference's range tests (NaN compares false), the mask binarised at 0.5 with NaN kept."""
    from ladi_vton_b200 import lib
    ni, nm = f["n_image"], f["n_mask"]
    image_flat, image = flat_buf(R, ni, torch.float32, fill=5.0)
    image.copy_(R.rand(ni) * 2 - 1)
    image[:len(image_values)] = torch.tensor(image_values, dtype=torch.float32)
    mflat, m = flat_buf(R, nm, torch.float32, fill=0.3)
    m.copy_(R.rand(nm))
    m[nm - len(mask_values):] = torch.tensor(mask_values, dtype=torch.float32)  # at the end: the last elements of the grid-stride walk
    src = m.clone()
    flags = torch.tensor(flags0, dtype=torch.int32, device=R.dev)
    lib.call("ladi_check_binarise", C.c_void_p(image.data_ptr()), ni, C.c_void_p(m.data_ptr()), nm, C.c_void_p(flags.data_ptr()), R.stream)
    torch.cuda.synchronize()
    im64, m64 = image.double(), src.double()
    want = [flags0[0] | int(bool(((im64 < -1) | (im64 > 1)).any())), flags0[1] | int(bool(((m64 < 0) | (m64 > 1)).any()))]
    errs = [] if flags.tolist() == want else [f"flags {flags.tolist()}, expected {want}"]
    if not bool((mflat[nm:] == 0.3).all()):
        errs.append("mask written past n_mask")
    errs += exact(m, torch.where(src < 0.5, 0.0, torch.where(src >= 0.5, 1.0, src)), "mask")[0]
    return errs, (0.0 if not errs else INF, "bit-exact mask and flags" if not errs else errs[0])


REPLAY_HERE = dict(REPLAY, nhwc_to_nchw_f32=replay_nhwc_to_nchw_f32, upsample2x_nhwc=replay_upsample2x_nhwc, pose_heatmaps=replay_pose_heatmaps,
                   check_binarise_values=replay_check_binarise_values)


# ================================================================================================================ value inputs
def _f32_ulp(v, d):
    return float(np.nextafter(np.float32(v), np.float32(d)))


def _exact_ties(count=255):
    """fp32 images v whose (v * 0.5 + 0.5) * 255 evaluates in fp32 to exactly k + 0.5 (round half to even decides), for the k < count
    where an fp32 v within 64 ulps reaches the tie (191 of the 255)."""
    out = []
    for k in range(count):
        v = np.float32((k + 0.5) / 127.5 - 1.0)
        for _ in range(64):
            t = (v * np.float32(0.5) + np.float32(0.5)) * np.float32(255.0)
            if t == np.float32(k + 0.5):
                out.append(float(v))
                break
            v = np.nextafter(v, np.float32(np.inf) if t < k + 0.5 else np.float32(-np.inf))
    return out


def _image_values(kind):
    def make(R, f):
        rows = f["n"] * f["h"] * f["w"]
        v = R.rand(rows, 3) * 2.4 - 1.2
        flat = v.view(-1)
        if kind == "ties":
            t = torch.tensor(_exact_ties(), dtype=torch.float32, device=R.dev)
            flat[:t.numel()] = t
        else:  # the clamp's ends and one ulp past them, +-inf, NaN
            special = [-1.0, 1.0, _f32_ulp(-1.0, -2), _f32_ulp(1.0, 2), _f32_ulp(-1.0, 0), _f32_ulp(1.0, 0), INF, -INF, NAN, 0.0, -0.0, NAN]
            flat[:len(special)] = torch.tensor(special, dtype=torch.float32, device=R.dev)
        return v
    return make


def _clamp_values(R, f):
    v = R.randn(f["n"] * f["h"] * f["w"], f["c"]) * 0.8
    special = [INF, -INF, NAN, 1e30, -1e30, f["lo"], f["hi"], NAN]
    v.view(-1)[:len(special)] = torch.tensor(special, device=R.dev)
    v.view(-1)[-3:] = torch.tensor([NAN, INF, -INF], device=R.dev)
    return v


def _logvar_values(R, f):
    rows = f["n"] * f["h"] * f["w"]
    lv = R.rand(rows, f["cz"]) * 60 - 36
    special = [-30.0, 20.0, _f32_ulp(-30.0, -31), _f32_ulp(20.0, 21), -30.5, 20.5, -1e30, 1e30, -INF, INF, NAN, _f32_ulp(-30.0, 0)]
    lv.view(-1)[:len(special)] = torch.tensor(special, device=R.dev)
    lv.view(-1)[-1] = NAN
    return lv


def _maxpool_values(kind):
    def make(R, f):
        n, h, w, c = f["n"], f["h"], f["w"], f["c"]
        x = -(R.rand(n * h * w, c) + 0.01)  # all-negative windows: a max seeded with 0 would show
        if kind == "nan":
            x = torch.where(R.rand(n * h * w, c) < 0.03, NAN, x)
            x[0, 0] = NAN  # the first window's first tap
            x[-1, -1] = NAN  # the last window's last tap
        return x
    return make


def _edge_grid(R, f):
    """Sampling grid with values exactly +-1 (the centres of the border texels' outer halves) and far outside on every side."""
    n, gh, gw = f["n"], f["gh"], f["gw"]
    choices = torch.tensor([-1.0, 1.0, -3.0, 3.0, -1e3, 1e3, 0.0, -0.999, 0.999], device=R.dev)
    idx = torch.randint(0, choices.numel(), (n, gh, gw, 2), device=R.dev, generator=R.g)
    return choices[idx]


def _zero_pixel(R, f):
    x = (R.randn(f["rows"], f["c"]).clamp_min(0)).bfloat16()
    x[0] = 0.0
    x[-1] = 0.0
    return x


# ================================================================================================================ the cases
def _ddim_capped_hw(sms):
    """(h, w) with B = 2 and CFG whose work 2 * 4 * h * w exceeds one full pass."""
    s = int(np.ceil(np.sqrt(PASS * sms / 8))) + 1
    return s, s


def edges(sms):
    """(name, kind, descriptor, replay keywords; a callable keyword is called with (R, descriptor) first) at `sms` SMs."""
    P = PASS * sms
    rz = lambda **k: _f("resize_aa", **k)  # noqa: E731
    cp = lambda **k: _f("clip_preprocess", **k)  # noqa: E731
    wg = lambda **k: _f("warp_grid_sample", **k)  # noqa: E731
    dd = lambda B=2, h=8, w=6, ep=4, inp=8, cfg=1, g=7.5, adv=1, noise=0: _f("ddim_cfg_step", ep=ep, inp=inp, B=B, h=h, w=w, cfg=cfg,  # noqa: E731
                                                                             guidance=g, advance=adv, noise=noise)
    io = lambda n=2, h=5, w=7, xp=3, f32=1: _f("image_out", f32=f32, n=n, h=h, w=w, xp=xp)  # noqa: E731
    npx_full, npx_next = P // 3, P // 3 + 1
    E = [
        # resize_aa: down-scale 5 and 4.99 with another factor on the other axis, identity, up-scale (from h = 1), 1x1 from 5x5,
        # c_off + c == out_pitch, one full pass and one image into the second
        ("resize_aa down 5 x 3.2", "resize_aa", rz(n=2, c=3, h=60, w=32, oh=12, ow=10, op=8, c_off=0), {}),
        ("resize_aa down 4.99 x 2", "resize_aa", rz(n=2, c=3, h=499, w=40, oh=100, ow=20, op=8, c_off=0), {}),
        ("resize_aa up 1.5 x down 5", "resize_aa", rz(n=2, c=3, h=10, w=50, oh=15, ow=10, op=8, c_off=0), {}),
        ("resize_aa identity", "resize_aa", rz(n=2, c=3, h=37, w=29, oh=37, ow=29, op=8, c_off=0), {}),
        ("resize_aa up from h 1", "resize_aa", rz(n=2, c=3, h=1, w=7, oh=9, ow=20, op=8, c_off=0), {}),
        ("resize_aa 1x1 from 5x5", "resize_aa", rz(n=3, c=3, h=5, w=5, oh=1, ow=1, op=8, c_off=0), {}),
        ("resize_aa c_off + c == out_pitch", "resize_aa", rz(n=2, c=3, h=20, w=15, oh=8, ow=6, op=8, c_off=5), {}),
        ("resize_aa one full pass", "resize_aa", rz(n=P, c=3, h=5, w=5, oh=1, ow=1, op=8, c_off=0), {}),
        ("resize_aa one element into a second pass", "resize_aa", rz(n=P + 1, c=3, h=5, w=5, oh=1, ow=1, op=8, c_off=0), {}),
        # clip_preprocess: the same scale edges, quantiser on and off
        *[(f"clip_preprocess {what} quantise {q}", "clip_preprocess", cp(n=2, c=3, h=h, w=w, oh=oh, ow=ow, quantise=q), {})
          for what, h, w, oh, ow in (("down 5 x 3.2", 60, 32, 12, 10), ("down 4.99 x 2", 499, 40, 100, 20), ("identity", 37, 29, 37, 29),
                                     ("up from h 1", 1, 7, 9, 20), ("1x1 from 5x5", 5, 5, 1, 1)) for q in (0, 1)],
        # warp_grid_sample: grid at +-1 and far outside, H = 1, W = 1, a 1x1 grid, c = 3 at c_off > 0 of a pitch-8 output, grid passes
        ("warp grid at +-1 and far outside", "warp_grid_sample", wg(gh=9, gw=7, n=2, c=3, H=12, W=10, op=8, c_off=0), dict(grid=_edge_grid)),
        ("warp H 1", "warp_grid_sample", wg(gh=3, gw=9, n=2, c=3, H=1, W=9, op=8, c_off=0), {}),
        ("warp W 1", "warp_grid_sample", wg(gh=7, gw=2, n=2, c=3, H=7, W=1, op=8, c_off=0), {}),
        ("warp 1x1 grid", "warp_grid_sample", wg(gh=1, gw=1, n=2, c=3, H=5, W=4, op=8, c_off=0), {}),
        ("warp c 3 at c_off 5 of pitch 8", "warp_grid_sample", wg(gh=16, gw=12, n=2, c=3, H=32, W=24, op=8, c_off=5), {}),
        ("warp one full pass", "warp_grid_sample", wg(gh=1, gw=1, n=P, c=16, H=1, W=1, op=16, c_off=0), {}),
        ("warp one element into a second pass", "warp_grid_sample", wg(gh=5, gw=5, n=P + 1, c=16, H=1, W=1, op=16, c_off=0), {}),
        # upsample2x_bilinear_ac: h = 1 (the sy = 0 branch), w = 1, both, c = 8 and c > 8
        *[(f"upsample2x_ac {h}x{w} c {c}", "upsample2x_ac", _f("upsample2x_ac", n=2, h=h, w=w, c=c), {})
          for h, w in ((1, 5), (5, 1), (1, 1)) for c in (8, 24)],
        # space_to_depth2: c = 3, x_pitch > c, out_pitch > 4c (padding untouched), grid passes with c = 1
        ("s2d c 3", "space_to_depth2", _f("space_to_depth2", n=2, h=6, w=4, c=3, xp=3, op=12), {}),
        ("s2d x_pitch > c", "space_to_depth2", _f("space_to_depth2", n=2, h=6, w=4, c=3, xp=8, op=12), {}),
        ("s2d out_pitch > 4c", "space_to_depth2", _f("space_to_depth2", n=2, h=6, w=4, c=3, xp=8, op=16), {}),
        ("s2d one full pass", "space_to_depth2", _f("space_to_depth2", n=P // 4, h=2, w=2, c=1, xp=1, op=4), {}),
        ("s2d four elements into a second pass", "space_to_depth2", _f("space_to_depth2", n=P // 4 + 1, h=2, w=2, c=1, xp=1, op=4), {}),
        # maxpool2: all-negative windows, windows holding a NaN
        ("maxpool2 all-negative windows", "maxpool2", _f("maxpool2", n=2, h=6, w=4, c=16), dict(values=_maxpool_values("neg"))),
        ("maxpool2 NaN in windows", "maxpool2", _f("maxpool2", n=2, h=6, w=4, c=16), dict(values=_maxpool_values("nan"))),
        # channel_affine / l2norm_channels: pitch > c, c = 8, 256, 264 (two lane passes), 512, rows 1..7 mod 8, an all-zero pixel
        *[(f"channel_affine c {c}", "channel_affine", _f("channel_affine", rows=8 * 5 + 3, c=c, pitch=c + 8), {}) for c in (8, 256, 264, 512)],
        *[(f"l2norm c {c}", "l2norm_channels", _f("l2norm_channels", rows=8 * 5 + 5, c=c, pitch=c + 16), {}) for c in (8, 256, 264, 512)],
        *[(f"l2norm rows {8 * 3 + r}", "l2norm_channels", _f("l2norm_channels", rows=8 * 3 + r, c=264, pitch=272), {}) for r in range(1, 8)],
        ("l2norm all-zero pixels", "l2norm_channels", _f("l2norm_channels", rows=13, c=64, pitch=72), dict(values=_zero_pixel)),
        # feature_correlation: h != w both ways, c = 8, out_pitch > h*w, n > 1, grid passes
        ("correlation 3x5 c 8", "feature_correlation", _f("feature_correlation", n=3, h=3, w=5, c=8, op=16), {}),
        ("correlation 5x3 out_pitch > hw", "feature_correlation", _f("feature_correlation", n=3, h=5, w=3, c=24, op=40), {}),
        ("correlation one full pass", "feature_correlation", _f("feature_correlation", n=P, h=1, w=1, c=8, op=8), {}),
        ("correlation one element into a second pass", "feature_correlation", _f("feature_correlation", n=P + 1, h=1, w=1, c=8, op=8), {}),
        # tps_grid: 1 and 64 control points, 1, 255, 256, 257 points, theta_pitch > 2 n_ctrl
        *[(f"tps n_ctrl {nc} points {npts}", "tps_grid", _f("tps_grid", tp=2 * nc + tp, n=2, n_ctrl=nc, npts=npts), {})
          for nc, npts, tp in ((1, 1, 6), (64, 255, 0), (64, 256, 8), (64, 257, 2), (25, 1, 4), (1, 257, 0))],
        # nhwc_to_nchw_clamp: x_pitch > c, lo == hi, +-inf and NaN
        ("clamp x_pitch > c with inf and NaN", "nhwc_to_nchw_clamp", _f("nhwc_to_nchw_clamp", n=2, c=3, h=5, w=4, xp=8, lo=-1.0, hi=1.0),
         dict(values=_clamp_values)),
        ("clamp lo == hi", "nhwc_to_nchw_clamp", _f("nhwc_to_nchw_clamp", n=2, c=3, h=5, w=4, xp=4, lo=0.25, hi=0.25), dict(values=_clamp_values)),
        # nchw_to_nhwc: f = 1, 2, 8; gates of exactly 0.5 and NaN; scale != 1; c_off + c == out_pitch
        *[(f"nchw_to_nhwc f {fct} gate 0.5 and NaN", "nchw_to_nhwc", _f("nchw_to_nhwc", n=2, c=3, h=5, w=4, f=fct, scale=1.0, op=8, c_off=0),
           dict(gate_nan=True)) for fct in (1, 2, 8)],
        ("nchw_to_nhwc scale != 1, c_off + c == out_pitch", "nchw_to_nhwc",
         _f("nchw_to_nhwc", n=2, c=4, h=6, w=5, f=1, scale=1 / 0.18215, gate=0, op=8, c_off=4), {}),
        # nhwc_to_nchw_f32: fp32 and bf16 sources, c_off > 0, x_pitch > c, n > 1
        *[(f"nhwc_to_nchw_f32 f32 {f32} c_off {co} pitch {xp}", "nhwc_to_nchw_f32",
           _f("nhwc_to_nchw_f32", f32=f32, n=3, c=4, h=5, w=7, xp=xp, c_off=co), {}) for f32 in (1, 0) for co, xp in ((0, 4), (4, 8), (3, 16))],
        # upsample2x_nhwc: h = 1, w = 1, c = 8 and 264, n > 1, past the grid-stride cap
        *[(f"upsample2x_nhwc {h}x{w} c {c}", "upsample2x_nhwc", _f("upsample2x_nhwc", n=3, h=h, w=w, c=c), {})
          for h, w, c in ((1, 5, 8), (5, 1, 264), (1, 1, 8), (7, 6, 16))],
        ("upsample2x_nhwc eight elements into a second pass", "upsample2x_nhwc", _f("upsample2x_nhwc", n=2, h=1, w=P // 8 + 1, c=8), {}),
        # posterior_sample: logvar at -30 and 20, one ulp past, beyond both, +-inf, NaN; m_pitch > 2 cz
        ("posterior logvar edges, m_pitch > 2 cz", "posterior_sample", _f("posterior_sample", mp=16, n=2, cz=4, h=5, w=3, scale=0.18215),
         dict(logvar=_logvar_values)),
        # inv_mask_rows / bilinear_down8: f = 1, H = W = 8
        ("inv_mask_rows f 1", "inv_mask_rows", _f("inv_mask_rows", n=2, H=5, W=3, f=1), {}),
        ("inv_mask_rows one output", "inv_mask_rows", _f("inv_mask_rows", n=2, H=8, W=8, f=8), {}),
        ("bilinear_down8 one output", "bilinear_down8", _f("bilinear_down8", n=2, c=3, H=8, W=8), {}),
        # ddim_cfg_step: one-block and capped grids (the ticket's reset of step_ptr[1]), device step > 0, advance 0, cfg off / on,
        # guidance 0 and 1, noise, pitches > 4 (columns >= 4 untouched), grid passes
        ("ddim one block", "ddim_cfg_step", dd(B=1, h=8, w=8, cfg=0), {}),
        ("ddim one partial block, cfg", "ddim_cfg_step", dd(B=1, h=4, w=3), {}),
        ("ddim capped grid, cfg", "ddim_cfg_step", dd(B=2, h=_ddim_capped_hw(sms)[0], w=_ddim_capped_hw(sms)[1]), {}),
        ("ddim from device step 2", "ddim_cfg_step", dd(), dict(start=2)),
        ("ddim advance 0", "ddim_cfg_step", dd(adv=0), dict(start=1)),
        ("ddim guidance 0", "ddim_cfg_step", dd(g=0.0), {}),
        ("ddim guidance 1", "ddim_cfg_step", dd(g=1.0), {}),
        ("ddim noise, pitches 8 and 16", "ddim_cfg_step", dd(ep=8, inp=16, noise=1), {}),
        ("ddim noise, no cfg", "ddim_cfg_step", dd(cfg=0, noise=1, ep=5, inp=9), {}),
        ("ddim one full pass", "ddim_cfg_step", dd(B=P // 4, h=1, w=1, cfg=0), {}),
        ("ddim four elements into a second pass", "ddim_cfg_step", dd(B=P // 4 + 1, h=1, w=1, cfg=0), {}),
        # check_binarise: n_image >> n_mask and the reverse, grid passes; value edges below
        ("check_binarise n_image >> n_mask", "check_binarise", _f("check_binarise", n_image=1 << 20, n_mask=100), {}),
        ("check_binarise n_mask >> n_image", "check_binarise", _f("check_binarise", n_image=100, n_mask=1 << 20), {}),
        ("check_binarise one full pass", "check_binarise", _f("check_binarise", n_image=4 * P, n_mask=4 * P), {}),
        ("check_binarise one element into a second pass", "check_binarise", _f("check_binarise", n_image=4 * P + 1, n_mask=3), {}),
        # image_out / image_out_u8: fp32 and bf16 sources, x_pitch > 3, exact rounding ties, values past [-1, 1], +-inf, NaN, grid passes
        *[(f"{k} f32 {f32} x_pitch {xp} {vals}", k, io(f32=f32, xp=xp), dict(values=_image_values(vals)))
          for k in ("image_out", "image_out_u8") for f32, xp in ((1, 3), (0, 8), (1, 8)) for vals in ("ties", "edges")],
        ("image_out_u8 one full pass", "image_out_u8", io(n=npx_full, h=1, w=1), {}),
        ("image_out_u8 three elements into a second pass", "image_out_u8", io(n=npx_next, h=1, w=1), {}),
        # pose_heatmaps: missing, half-missing, negative, off-map, half-integer key-points, sigma 1 and 9, a 1x1 map
        *[(f"pose_heatmaps {h}x{w} sigma {s}", "pose_heatmaps", _f("pose_heatmaps", n_maps=m, h=h, w=w, sigma=s), {})
          for h, w, s, m in ((64, 48, 9.0, 40), (64, 48, 1.0, 40), (1, 1, 9.0, 20), (7, 3, 1.0, 20))],
        # clip_embed, patchify, vit_assemble
        ("clip_embed 3 prompts with pseudo-words", "clip_embed", _f("clip_embed", rows=3 * 77, seq=77, c=64, op=72), {}),
        ("clip_embed no word_emb", "clip_embed", _f("clip_embed", wemb=0, rows=2 * 77, seq=77, c=64, op=64), {}),
        ("patchify k_pad > ch ps^2", "patchify", _f("patchify", n=2, ch=3, h=6, w=4, patch=2, kpad=24), {}),
        ("patchify ps 1", "patchify", _f("patchify", n=2, ch=3, h=5, w=3, patch=1, kpad=8), {}),
        ("patchify one full pass", "patchify", _f("patchify", n=P // 8, ch=3, h=1, w=1, patch=1, kpad=8), {}),
        ("patchify eight elements into a second pass", "patchify", _f("patchify", n=P // 8 + 1, ch=3, h=1, w=1, patch=1, kpad=8), {}),
        ("vit_assemble one patch", "vit_assemble", _f("vit_assemble", pp=64, n=3, np=1, c=64), {}),
        ("vit_assemble patch_pitch > c", "vit_assemble", _f("vit_assemble", pp=80, n=3, np=5, c=64), {}),
    ]
    return E


# value edges of check_binarise: (name, descriptor, image values, mask values, flags before)
_U = _f32_ulp
BINARISE_VALUES = [
    ("in range at the ends", [-1.0, 1.0, NAN], [0.0, 0.5, 1.0, _U(0.5, 0), _U(0.5, 1), NAN], [0, 0]),
    ("image one ulp below -1", [_U(-1.0, -2)], [0.5], [0, 0]),
    ("image one ulp above 1", [_U(1.0, 2)], [0.5], [0, 0]),
    ("mask one ulp below 0", [0.0], [_U(0.0, -1)], [0, 0]),
    ("mask one ulp above 1", [0.0], [_U(1.0, 2)], [0, 0]),
    ("image +inf, mask -inf", [INF], [-INF], [0, 0]),
    ("image -inf, mask +inf", [-INF], [INF], [0, 0]),
    ("flags already set stay set", [0.0], [0.5], [1, 1]),
    ("NaN only", [NAN, NAN], [NAN, NAN], [0, 0]),
]


def _work(kind, f):
    """Elements the grid-stride loop of `kind` walks (grid = min(ceil(work / 256), 16 SMs))."""
    return {"resize_aa": lambda: f["n"] * f["oh"] * f["ow"], "warp_grid_sample": lambda: f["n"] * f["H"] * f["W"],
            "space_to_depth2": lambda: f["n"] * (f["h"] // 2) * (f["w"] // 2) * 4 * f["c"],
            "feature_correlation": lambda: f["n"] * (f["h"] * f["w"]) ** 2, "ddim_cfg_step": lambda: f["B"] * 4 * f["h"] * f["w"],
            "check_binarise": lambda: -(-max(f["n_image"], f["n_mask"]) // 4), "patchify": lambda: f["n"] * f["h"] * f["w"] * f["kpad"],
            "image_out_u8": lambda: f["n"] * f["h"] * f["w"] * 3, "upsample2x_nhwc": lambda: f["n"] * 4 * f["h"] * f["w"] * f["c"] // 8}[kind]()


# ================================================================================================================ CPU: the cases
def test_edge_cases_are_what_they_say():
    """The cases hit the limits they are named after, at the H100 SXM's 132 SMs (CPU)."""
    E = {name: (kind, f) for name, kind, f, _ in edges(SMS)}
    P = PASS * SMS
    for name, (kind, f) in E.items():
        if "full pass" in name:
            assert _work(kind, f) == P, name
        elif "second pass" in name:
            assert P < _work(kind, f) <= P + 8, name
    assert _work("ddim_cfg_step", E["ddim capped grid, cfg"][1]) > P
    assert _work("ddim_cfg_step", E["ddim one block"][1]) == 256
    f = E["resize_aa down 5 x 3.2"][1]
    assert f["h"] / f["oh"] == 5.0
    f = E["resize_aa c_off + c == out_pitch"][1]
    assert f["c_off"] + f["c"] == f["op"]
    assert {nc for k, (kind, f) in E.items() if kind == "tps_grid" for nc in [f["n_ctrl"]]} >= {1, 64}
    assert {f["npts"] for k, (kind, f) in E.items() if kind == "tps_grid"} >= {1, 255, 256, 257}
    assert {f["rows"] % 8 for k, (kind, f) in E.items() if kind == "l2norm_channels"} >= set(range(1, 8))
    ties = np.array(_exact_ties(), dtype=np.float32)
    t = (ties * np.float32(0.5) + np.float32(0.5)) * np.float32(255.0)
    assert len(ties) > 150 and np.all(t - np.floor(t) == 0.5)
    for name, kind, f, _ in edges(114):  # another SM count gives the same limits
        if "full pass" in name:
            assert _work(kind, f) == PASS * 114 or kind == "image_out_u8", name


# ================================================================================================================ CPU: teeth
def test_teeth_nhwc_to_nchw_xy_swap():
    g = torch.Generator().manual_seed(1)
    n, h, w, c, xp, co = 2, 5, 7, 4, 8, 3
    x = torch.randn(n * h * w, xp, generator=g)
    r = nhwc_to_nchw_expect(x, n, h, w, c, co)
    good = x.view(n, h, w, xp)[..., co:co + c].permute(0, 3, 1, 2)
    assert not exact(good, r, "")[0]
    swapped = x.view(n, w, h, xp)[..., co:co + c].permute(0, 3, 2, 1)  # x / y swapped in the source index
    assert exact(swapped.contiguous(), r, "")[0]
    shifted = x.view(n, h, w, xp)[..., co - 1:co - 1 + c].permute(0, 3, 1, 2)  # c_off ignored by one
    assert exact(shifted.contiguous(), r, "")[0]


def test_teeth_upsample_nearest_off_by_one():
    g = torch.Generator().manual_seed(2)
    x = torch.randn(2, 4, 3, 8, generator=g).bfloat16()
    r = upsample_nearest_expect(x)
    oy, ox = torch.arange(8), torch.arange(6)
    good = x[:, oy // 2][:, :, ox // 2]
    assert not exact(good.contiguous(), r, "")[0]
    bad = x[:, ((oy + 1) // 2).clamp_max(3)][:, :, ox // 2]
    assert exact(bad.contiguous(), r, "")[0]


def _pose_emulate(k, h, w, sigma, rnd=torch.round):
    """The kernel's arithmetic in fp32 (closed-form maximum at the nearest grid point, clamped into the map)."""
    k = k.float()
    kx, ky = k[:, 0].view(-1, 1, 1), k[:, 1].view(-1, 1, 1)
    ys, xs = torch.meshgrid(torch.arange(h, dtype=torch.float32), torch.arange(w, dtype=torch.float32), indexing="ij")
    inv = torch.tensor(1.0, dtype=torch.float32) / torch.tensor(sigma * sigma, dtype=torch.float32)
    nx, ny = rnd(kx).clamp(0, w - 1), rnd(ky).clamp(0, h - 1)
    dmin = (nx - kx) ** 2 + (ny - ky) ** 2
    d = (xs - kx) ** 2 + (ys - ky) ** 2
    v = torch.exp(-d * inv) / (torch.exp(-dmin * inv) + torch.tensor(1.1920929e-07, dtype=torch.float32))
    return torch.where(((kx > 0) | (ky > 0)), v, 0.0)


@pytest.mark.parametrize("sigma", [1.0, 9.0])
def test_teeth_pose_heatmap_rint(sigma):
    k = torch.tensor(POSE_KEYPOINTS, dtype=torch.float32)
    h, w = 64, 48
    r, bound = pose_expect(k.double(), h, w, sigma)
    assert float(ratio(_pose_emulate(k, h, w, sigma), r, bound).max()) <= 1
    assert float(ratio(_pose_emulate(k, h, w, sigma, torch.floor), r, bound).max()) > 1  # floorf in place of rintf


def test_teeth_nan_dropping_clamp_and_max():
    x = torch.tensor([NAN, -2.0, 0.5, INF, -INF, 2.0, NAN, 0.0])
    ref = x.clamp(-1.0, 1.0)
    keep = torch.where(torch.isnan(x), x, torch.fmin(torch.fmax(x, torch.tensor(-1.0)), torch.tensor(1.0)))
    assert not exact(keep, ref, "")[0]
    drop = torch.fmin(torch.fmax(x, torch.tensor(-1.0)), torch.tensor(1.0))  # fmaxf / fminf: NaN -> the other operand
    assert exact(drop, ref, "")[0]
    X = torch.randn(1, 8, 4, 6).bfloat16()
    X[0, 3, 1, 2] = NAN
    ref = F.max_pool2d(X.float(), 2).bfloat16()
    win = X.float().unfold(2, 2, 2).unfold(3, 2, 2).reshape(1, 8, 2, 3, 4)
    keep = win.amax(-1).bfloat16()  # NaN-propagating
    assert not exact(keep, ref, "")[0]
    drop = torch.nan_to_num(win, nan=-INF).amax(-1).bfloat16()
    assert exact(drop, ref, "")[0]


# ================================================================================================================ CPU: placement rules
# (id, entry point, arguments with pointers as ints, expected message or None = the checks pass and the launch fails for lack of a device)
_ADD = lambda a=A, b=A, out=A: ("ladi_add_bf16", [a, b, out, 64])  # noqa: E731
_UP = lambda x=A, out=A: ("ladi_upsample2x_nhwc", [x, 1, 2, 2, 8, out])  # noqa: E731
_MAX = lambda x=A, out=A: ("ladi_maxpool2_nhwc", [x, 1, 4, 4, 8, out])  # noqa: E731
_UPAC = lambda x=A, out=A: ("ladi_upsample2x_bilinear_ac", [x, 1, 2, 2, 8, out])  # noqa: E731
_L2 = lambda x=A: ("ladi_l2norm_channels", [x, 4, 8, 8])  # noqa: E731
_AFF = lambda x=A, sc=A, sh=A: ("ladi_channel_affine", [x, 4, 8, 8, sc, sh])  # noqa: E731
_CORR = lambda fa=A, fb=A: ("ladi_feature_correlation", [fa, fb, 1, 2, 2, 8, A, 8])  # noqa: E731
_EMB = lambda tok=A, we=A, pos=A, out=A: ("ladi_clip_embed", [A, tok, we, pos, out, 2, 2, 8, 8])  # noqa: E731
_VIT = lambda patch=A, pp=8, cls=A, pos=A, out=A, n=2: ("ladi_vit_assemble", [patch, pp, cls, pos, out, n, 4, 8])  # noqa: E731
_TPS = lambda n=2: ("ladi_tps_grid", [A, 50, A, A, n, 25, 16, A, A])  # noqa: E731
_N2C = lambda x=A, xp=8, co=0, c=4: ("ladi_nhwc_to_nchw_f32", [x, 1, 1, c, 2, 2, xp, co, A])  # noqa: E731
_C2N = lambda op=8, co=0: ("ladi_nchw_f32_to_nhwc_bf16", [A, 1, 3, 2, 2, 1, 1.0, 0, A, op, co])  # noqa: E731
_POST = lambda mp=8: ("ladi_posterior_sample", [A, mp, A, 1, 4, 2, 2, 0.18215, A])  # noqa: E731
_IMG = lambda x=A, xp=3: ("ladi_image_out", [x, 1, 1, 2, 2, xp, A])  # noqa: E731
_DDIM = lambda ep=4, inp=8, step=A, adv=1: ("ladi_ddim_cfg_step", [A, ep, A, A, inp, 1, 2, 2, 1, 7.5, A, step, adv, 0])  # noqa: E731
PLACEMENT = [
    ("add a", *_ADD(a=A + 8), "a 0x100008 must be 16-byte aligned"),
    ("add b", *_ADD(b=A + 4), "b 0x100004 must be 16-byte aligned"),
    ("add out", *_ADD(out=A + 2), "out 0x100002 must be 16-byte aligned"),
    ("add ok", *_ADD(), None),
    ("upsample2x x", *_UP(x=A + 8), "x 0x100008 must be 16-byte aligned"),
    ("upsample2x out", *_UP(out=A + 8), "out 0x100008 must be 16-byte aligned"),
    ("upsample2x ok", *_UP(), None),
    ("maxpool2 x", *_MAX(x=A + 8), "x 0x100008 must be 16-byte aligned"),
    ("maxpool2 out", *_MAX(out=A + 2), "out 0x100002 must be 16-byte aligned"),
    ("maxpool2 ok", *_MAX(), None),
    ("upsample2x_ac x", *_UPAC(x=A + 8), "x 0x100008 must be 16-byte aligned"),
    ("upsample2x_ac out", *_UPAC(out=A + 8), "out 0x100008 must be 16-byte aligned"),
    ("upsample2x_ac ok", *_UPAC(), None),
    ("l2norm x", *_L2(x=A + 8), "x 0x100008 must be 16-byte aligned"),
    ("l2norm ok", *_L2(), None),
    ("channel_affine x", *_AFF(x=A + 8), "x 0x100008 must be 16-byte aligned"),
    ("channel_affine scale", *_AFF(sc=A + 4), "scale 0x100004 must be 16-byte aligned"),
    ("channel_affine shift", *_AFF(sh=A + 8), "shift 0x100008 must be 16-byte aligned"),
    ("channel_affine ok", *_AFF(sc=A + 16, sh=A + 48), None),
    ("correlation fa", *_CORR(fa=A + 8), "fa 0x100008 must be 16-byte aligned"),
    ("correlation fb", *_CORR(fb=A + 2), "fb 0x100002 must be 16-byte aligned"),
    ("correlation ok", *_CORR(), None),
    ("clip_embed tok", *_EMB(tok=A + 8), "tok 0x100008 must be 16-byte aligned"),
    ("clip_embed word_emb", *_EMB(we=A + 8), "word_emb 0x100008 must be 16-byte aligned"),
    ("clip_embed pos", *_EMB(pos=A + 4), "pos 0x100004 must be 16-byte aligned"),
    ("clip_embed out", *_EMB(out=A + 2), "out 0x100002 must be 16-byte aligned"),
    ("clip_embed ok without word_emb", *_EMB(we=0), None),
    ("vit_assemble patch", *_VIT(patch=A + 8), "patch 0x100008 must be 16-byte aligned"),
    ("vit_assemble cls", *_VIT(cls=A + 8), "cls 0x100008 must be 16-byte aligned"),
    ("vit_assemble pos", *_VIT(pos=A + 2), "pos 0x100002 must be 16-byte aligned"),
    ("vit_assemble out", *_VIT(out=A + 8), "out 0x100008 must be 16-byte aligned"),
    ("vit_assemble patch_pitch < c", *_VIT(pp=0), "patch_pitch 0 is below c"),
    ("vit_assemble n", *_VIT(n=65536), "n 65536 exceeds 65535"),
    ("vit_assemble ok at n = 65535", *_VIT(n=65535), None),
    ("tps_grid n", *_TPS(n=65536), "n 65536 exceeds 65535"),
    ("tps_grid ok at n = 65535", *_TPS(n=65535), None),
    ("nhwc_to_nchw x_pitch < c_off + c", *_N2C(xp=8, co=5), "channel window [5, 9) outside the input pitch 8"),
    ("nhwc_to_nchw c_off < 0", *_N2C(co=-1), "channel window [-1, 3) outside the input pitch 8"),
    ("nhwc_to_nchw null x", *_N2C(x=0), "nhwc_to_nchw: bad extent"),
    ("nhwc_to_nchw ok at c_off + c == x_pitch", *_N2C(xp=8, co=4), None),
    ("nchw_to_nhwc out_pitch < c_off + c", *_C2N(op=8, co=6), "channel window [6, 9) outside the output pitch 8"),
    ("nchw_to_nhwc c_off < 0", *_C2N(co=-2), "channel window [-2, 1) outside the output pitch 8"),
    ("nchw_to_nhwc ok at c_off + c == out_pitch", *_C2N(op=8, co=5), None),
    ("posterior m_pitch < 2 cz", *_POST(mp=7), "m_pitch 7 is below 2*cz (8)"),
    ("posterior ok", *_POST(mp=8), None),
    ("image_out x_pitch < 3", *_IMG(xp=2), "image_out: bad extent"),
    ("image_out null x", *_IMG(x=0), "image_out: bad extent"),
    ("image_out ok", *_IMG(), None),
    ("ddim eps_pitch < 4", *_DDIM(ep=3), "eps_pitch 3 is below the 4 latent channels"),
    ("ddim in_pitch < 4", *_DDIM(inp=3), "in_pitch 3 is below the 4 latent channels"),
    ("ddim advance without step_ptr", *_DDIM(step=0), "advance needs step_ptr"),
    ("ddim ok without step_ptr or advance", *_DDIM(step=0, adv=0), None),
    ("ddim ok", *_DDIM(), None),
    ("inv_mask_rows null mask", "ladi_inv_mask_rows", [0, 1, 8, 8, 8, A], "inv_mask: null operand"),
    ("inv_mask_rows ok", "ladi_inv_mask_rows", [A, 1, 8, 8, 8, A], None),
    ("bilinear_down8 null x", "ladi_bilinear_down8", [0, 1, 1, 8, 8, A], "bilinear_down8: null operand"),
    ("bilinear_down8 null out", "ladi_bilinear_down8", [A, 1, 1, 8, 8, 0], "bilinear_down8: null operand"),
    ("bilinear_down8 ok", "ladi_bilinear_down8", [A, 1, 1, 8, 8, A], None),
]


def test_placement_rules_without_a_device():
    """The placement rules of the glue, warping and front-end entry points (PLACEMENT), checked in a process that sees no device."""
    check_placement(PLACEMENT)


# ================================================================================================================ GPU


_EDGE_IDS = [e[0] for e in edges(SMS)]


@pytest.mark.gpu
@pytest.mark.parametrize("name", _EDGE_IDS)
def test_glue_edge_against_float64(cuda, name):
    case = {e[0]: e for e in edges(sms(cuda))}[name]
    _, kind, f, kw = case
    R = Replay(cuda, 1357)
    kw = {k: (v(R, f) if callable(v) else v) for k, v in kw.items()}
    errs, res = REPLAY_HERE[kind](R, f, **kw)
    print(f"\n{name} at {sms(cuda)} SMs: err/bound {res[0]:.3g} ({res[1]})")
    torch.cuda.empty_cache()
    assert not errs, f"{name}:\n  " + "\n  ".join(errs)


@pytest.mark.gpu
@pytest.mark.parametrize("case", BINARISE_VALUES, ids=[c[0] for c in BINARISE_VALUES])
@pytest.mark.parametrize("sizes", [(1 << 16, 97), (97, 1 << 16)], ids=["n_image >> n_mask", "n_mask >> n_image"])
def test_check_binarise_values(cuda, case, sizes):
    name, im, m, flags0 = case
    R = Replay(cuda, 97531)
    errs, res = replay_check_binarise_values(R, _f("check_binarise", n_image=sizes[0], n_mask=sizes[1]), im, m, flags0)
    print(f"\ncheck_binarise {name}: {res[1]}")
    assert not errs, f"{name}:\n  " + "\n  ".join(errs)
