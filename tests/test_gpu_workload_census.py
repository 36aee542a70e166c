"""Every distinct kernel call the engine modules issue in the benchmarked workloads (UNet, VAE encode and decode, EMASC, the inversion
adapter, and the `plan_context` GEMM), replayed one by one against a float64 reference with per-element error bounds.  The kernels the
Python sequencing issues around them (the pipeline's glue) and the inference CLI's front end (cloth warping, the CLIP towers) are
tests/test_gpu_glue_frontend_census.py's.

The census (CPU).  Plan-only engines for the full-size UNet, VAE, EMASC and inversion adapter (random weights packed on the CPU, library
defaults: no CTA pairs, no LayerNorm fold) are walked at the shapes of bench.py / BASELINE.json; the text-context GEMM of
`UNet2DConditionModel.plan_context` is recorded from the Python sequencing (`lib.RECORD`).  Addresses are stripped (an operand is only
"present" or "absent") and the descriptors deduplicated; each keeps the module and shape that issued it first.  The tile geometry, N tile
and split-K factor of `ladi_conv2d_bf16` and the launch shapes of the other kernels are functions of exactly these fields, so the census
is the set of code paths the workloads run.

The replay (GPU).  Each descriptor goes through the same ABI entry point with the same fields; only the pointers are new.  Inputs are
random bf16 at realistic magnitudes, every pitch padding of an input is NaN (a kernel that reads it produces NaN), the output is
NaN-poisoned over its full pitch before the call and must afterwards be finite in exactly the columns the call owns and still NaN in the
rest, and a second run must be bit-identical (the library has no floating-point atomics).  The reference is float64 on the GPU (chunked
where a full intermediate would not fit; for the largest descriptors on the first and last image of the batch).

The error bound is per element and is built from the error sources the kernels have.  Its constants:
  U_BF16   = 2^-7   bf16 output rounding (8-bit significand, round-to-nearest: unit roundoff 2^-8) doubled for the fp32 epilogue
                    arithmetic before it;
  U_F32    = 2^-21  fp32 output rounding (2^-24) with the same kind of margin;
  C_ACC    = 4      fp32 accumulation of K exact bf16 products (wgmma, split-K partials, fp32 norm sums): the error of a sum of K terms
                    behaves like 2^-24 * sqrt(K) * sum|terms| for rounding (and for the truncating alignment of the tensor core, whose
                    sign follows the random-walking partial sum); 4 covers the tail over millions of elements;
  SILU_REL = 2^-11  tanh.approx in SiLU (x/2 * (1 + tanh(x/2))): relative error 2^-11 of tanh, i.e. at most 2^-12 |x|, doubled;
  GELU_REL = 3e-5   the degree-8 erf polynomial of the GELU epilogue: |erf error| <= 4.8e-5 -> |gelu error| <= 2.4e-5 |x| (also past
                    the +-3 clamp, where erf(3) misses 1 by 2.2e-5);
  ACT_GAIN = 1.13   sup |act'| of SiLU (1.10) and GELU (1.13): how much an accumulation error grows through the activation;
  U_P      = 2^-7   attention: P is rounded to bf16 (2^-8) before P.V, doubled; the error it causes is at most U_P * sum p|v| / l;
  E_EXP    = 2^-16  attention: ex2.approx (2^-22 relative) plus the fp32 rounding of the exponent argument (|x| 2^-24, |x| < 2^6).
So  conv/GEMM:  |y - r| <= U * |r| + gain * C_ACC * sqrt(K) * 2^-24 * m + eps_act,  m = |A| (*) |W| + |bias| + |residual| in float64;
    attention:  |y - r| <= U * |r| + (U_P + C_ACC * sqrt(nkv) * 2^-24 + E_EXP) * sum p|v| / l   (from the float64 softmax);
    GroupNorm / LayerNorm: U * |r| + gain * |gamma| (|xhat| d_rstd + d_mean rstd) + eps_act, where the one-pass fp32 statistics give
                d_mean = delta (|mean| + std) and d_rstd = 1.5 delta (mean^2 + var) / var, delta = C_ACC sqrt(count) 2^-24: the term
                that grows with mean^2 / var, which is why the GroupNorm inputs carry per-channel offsets of a few sigma.
The CPU tests at the end show the bound has teeth: the same checker rejects five simulated kernel faults and accepts an honest fp32
emulation."""
import ctypes as C
import math
import re
import time
from collections import OrderedDict, defaultdict

import pytest
import torch
import torch.nn.functional as F

U_BF16, U_F32 = 2.0 ** -7, 2.0 ** -21
C_ACC = 4.0
SILU_REL, GELU_REL, ACT_GAIN = 2.0 ** -11, 3e-5, 1.13
U_P, E_EXP = 2.0 ** -7, 2.0 ** -16
EPS24 = 2.0 ** -24
SPLITK_WS_BYTES = 64 << 20  # what the engine allocates (csrc/engine.cu) and ops.SPLITK_WS_BYTES: the same split decisions

# ================================================================================================================ the census (CPU)
# per op: the fields the trace prints; the replay implements exactly these (an unknown op or field fails test_census_integrity)
FIELDS = {
    "conv": "k s p up n h w hin win cout nsrc src0 c0 p0 src1 c1 p1 nsc sc0 sc0c sc0p sc1 sc1c sc1p wt K wp bias bpr bss step res rp rs act out op f32",
    "gn_stats": "x0 c0 p0 x1 c1 p1 n hw groups",
    "gn_apply": "x0 c0 p0 x1 c1 p1 n hw groups gamma beta eps silu add ap out op",
    "ln": "x xp rows c gamma beta eps out op",
    "attn": "d batch heads nq nkv q qp qbs k kp kbs v vp vbs out op obs scale",
    "add": "a b out count",
    "cls_attn": "q qp kv kvp batch tokens heads hd out op",
    "timestep_embedding": "t n c kp out",
}
FIELDS = {k: v.split() for k, v in FIELDS.items()}
KINDS = ["conv", "attn_d64", "attn_d512", "gn", "ln", "cls_attn", "add", "timestep_embedding"]
M_UNET, M_ENC, M_DEC, M_EMASC, M_ADAPTER, M_PLAN = 0, 1, 2, 3, 4, 5
# (workload label, [(module, batch, height, width)]): the shapes of bench.py / BASELINE.json; "ctx" = plan_context GEMM at (UNet batch) x 77 rows
WORKLOADS = [
    ("512x384, 8 images, CFG (bench default; configs 1, 2, 4)",
     [(M_UNET, 16, 64, 48), (M_ENC, 8, 512, 384), (M_DEC, 8, 64, 48), (M_EMASC, 8, 512, 384), (M_PLAN, 50, 0, 0), ("ctx", 16, 77, 1024)]),
    ("512x384, 100 DDIM steps (config 4)", [(M_PLAN, 100, 0, 0)]),
    ("1024x768, 4 images, CFG (config 3)",
     [(M_UNET, 8, 128, 96), (M_ENC, 4, 1024, 768), (M_DEC, 4, 128, 96), (M_EMASC, 4, 1024, 768), (M_PLAN, 50, 0, 0), ("ctx", 8, 77, 1024)]),
    ("one 512x384 image, CFG, 20 DDIM steps (config 0 shape)",
     [(M_UNET, 2, 64, 48), (M_ENC, 1, 512, 384), (M_DEC, 1, 64, 48), (M_EMASC, 1, 512, 384), (M_PLAN, 20, 0, 0), ("ctx", 2, 77, 1024)]),
    ("inversion adapter, 8 images x 257 tokens (inference CLI path, not in the bench)", [(M_ADAPTER, 8, 257, 0)]),
]
MODULE_NAMES = {M_UNET: "UNet", M_ENC: "VAE encode", M_DEC: "VAE decode", M_EMASC: "EMASC", M_ADAPTER: "adapter", M_PLAN: "UNet plan_steps",
                "ctx": "UNet plan_context GEMM"}


def parse(line):
    """-> (op, {field: value}) with every @address replaced by 1 (operand present) or 0 (absent)."""
    op = line.split(" ", 1)[0]
    f = OrderedDict()
    for k, v in re.findall(r"(\w+)=(\S+)", line):
        f[k] = ("1" if int(v[1:], 16) else "0") if v.startswith("@") else v
    return op, f


def kind_of(op, f):
    if op == "attn":
        return "attn_d64" if f["d"] == "64" else "attn_d512"
    return {"gn_apply": "gn"}.get(op, op)


def _build_engines():
    from ladi_vton_b200 import EMASC, AutoencoderKL, InversionAdapter, UNet2DConditionModel, engine as eng, synthetic as S, unet_param_shapes
    from ladi_vton_b200.vae import vae_param_shapes

    def pack(model, shapes, seed):
        model._sd = S.random_state_dict(shapes, seed, fast=True)  # the walk depends on shapes only: tiled random values are enough
        model.device = torch.device("cpu")
        model._pack()
        model._sd = None
        return model

    unet = pack(UNet2DConditionModel(), unet_param_shapes({}), 1)
    vae = pack(AutoencoderKL(), vae_param_shapes({}), 2)
    ad = pack(InversionAdapter(), InversionAdapter().param_shapes(), 4)
    ein, eout = S.emasc_channels(vae.config.block_out_channels)
    em = pack(EMASC(ein, eout), S.emasc_param_shapes(ein, eout), 3)
    W = {}
    for i, (w1, b1, w2, b2) in enumerate(em.P):
        W.update({f"emasc.{i}.w1": w1, f"emasc.{i}.b1": b1, f"emasc.{i}.w2": w2, f"emasc.{i}.b2": b2})
    engines = {M_UNET: eng.Engine(eng.flatten(unet.P), plan_only=True, **unet.engine_config()),
               M_ENC: eng.Engine(eng.flatten(vae.P), plan_only=True, **vae.engine_config()),
               M_EMASC: eng.Engine(W, plan_only=True, emasc_scales=5, emasc_in=ein, emasc_out=eout, emasc_stride=[1, 1, 2, 4, 8]),
               M_ADAPTER: eng.Engine(eng.flatten(ad.P, "adapter."), plan_only=True, adapter_dim=ad.dim, adapter_heads=ad.heads,
                                     adapter_mlp=ad.mlp_dim, adapter_hidden=ad.hidden, adapter_out=ad.out_dim)}
    engines[M_DEC], engines[M_PLAN] = engines[M_ENC], engines[M_UNET]
    return unet, engines


def _context_trace(unet, batch, tokens, dim):
    """The plan_context GEMM as the Python sequencing issues it (recorded, not launched)."""
    import test_engine_trace as tt
    from ladi_vton_b200 import lib
    lib.RECORD = []
    try:
        unet._ctx = None
        unet.plan_context(torch.zeros((batch, tokens, dim), dtype=torch.bfloat16))
        return tt.python_trace(lib.RECORD)
    finally:
        lib.RECORD = None


_CENSUS = None


def census():
    """-> (descriptors, calls, unparsed): descriptors = OrderedDict stripped line -> {kind, op, f, first, n}; calls = {(workload, module
    label): Counter of calls and distinct descriptors per kind}; unparsed = lines with an unknown op or field set."""
    global _CENSUS
    if _CENSUS is not None:
        return _CENSUS
    import os
    for k in ("LADI_UP2X", "LADI_LN_FOLD", "LADI_CONV_2CTA"):  # library defaults only (the workload runs with them)
        assert k not in os.environ, f"census runs with library defaults; unset {k}"
    unet, engines = _build_engines()
    desc, calls, unparsed = OrderedDict(), OrderedDict(), []
    for wl, mods in WORKLOADS:
        for mod, b, h, w in mods:
            label = f"{MODULE_NAMES[mod]} {b}x{h}x{w}" if mod not in (M_PLAN, M_ADAPTER, "ctx") else \
                {M_PLAN: f"UNet plan_steps, {b} timesteps", M_ADAPTER: f"adapter {b}x{h}", "ctx": f"plan_context GEMM, {b}x{h} rows x {w}"}[mod]
            lines = _context_trace(unet, b, h, w) if mod == "ctx" else [l for l in engines[mod].trace(mod, b, h, w).splitlines() if l.strip()]
            cnt = calls.setdefault((wl, label), defaultdict(lambda: [0, set()]))
            prev = None
            for ln in lines:
                op, f = parse(ln)
                if op not in FIELDS or list(f) != FIELDS[op]:
                    unparsed.append(ln)
                    continue
                if op == "gn_stats":  # replayed together with the gn_apply that must follow it on the same operands
                    prev = f
                    continue
                if op == "gn_apply":
                    if prev is None or any(prev[k] != f[k] for k in FIELDS["gn_stats"]):
                        unparsed.append("gn_apply without its gn_stats: " + ln)
                    prev = None
                key = op + " " + " ".join(f"{k}={v}" for k, v in f.items())
                kd = kind_of(op, f)
                cnt[kd][0] += 1
                cnt[kd][1].add(key)
                if key not in desc:
                    desc[key] = dict(kind=kd, op=op, f={k: (float(v) if k in ("eps", "scale") else int(v)) for k, v in f.items()},
                                     first=f"{label} [{wl}]", n=0)
                desc[key]["n"] += 1
    _CENSUS = (desc, calls, unparsed)
    return _CENSUS


def print_census(desc, calls):
    print("\nworkload census: calls (distinct descriptors) per module and shape")
    for (wl, label), cnt in calls.items():
        print(f"  {label:44s} " + ", ".join(f"{k} {v[0]} ({len(v[1])})" for k, v in sorted(cnt.items())) + f"   [{wl}]")
    per = defaultdict(int)
    for d in desc.values():
        per[d["kind"]] += 1
    print("  distinct over all workloads: " + ", ".join(f"{k} {per[k]}" for k in KINDS if per[k]))


# ================================================================================================================ error bounds (CPU and GPU)
def silu64(x):
    return x * torch.sigmoid(x)


def gelu64(x):
    return 0.5 * x * (1.0 + torch.erf(x * (0.5 ** 0.5)))


def conv_expect(pre, m, K, act, res=None, rs=None, out_fp32=False):
    """pre = A W^T + bias and m = |A| |W|^T + |bias| (+|res|), float64 [..., c_out] -> (r, bound) [..., c_eff] per the module docstring."""
    e = C_ACC * math.sqrt(K) * EPS24 * m
    if act == 2:  # GEGLU: interleaved (value, gate) columns -> value * gelu(gate)
        v, g, ev, eg = pre[..., 0::2], pre[..., 1::2], e[..., 0::2], e[..., 1::2]
        gl = gelu64(g)
        r = v * gl
        err = ev * gl.abs() + ACT_GAIN * eg * (v.abs() + ev) + GELU_REL * g.abs() * v.abs()
    else:
        if act == 1:
            r, err = silu64(pre), ACT_GAIN * e + SILU_REL * pre.abs()
        elif act == 3:
            r, err = gelu64(pre), ACT_GAIN * e + GELU_REL * pre.abs()
        elif act == 4:
            r, err = pre.clamp_min(0), e
        else:
            r, err = pre, e
        if res is not None:
            r = r + res
    if rs is not None:
        r, err = r * rs, err * rs
    return r, (U_F32 if out_fp32 else U_BF16) * r.abs() + err


def attn_expect(o, sv, nkv, u_p=None):
    """o = softmax(s) v and sv = sum p|v| / l from the float64 softmax -> bound."""
    u_p = U_P if u_p is None else u_p
    return U_BF16 * o.abs() + (u_p + C_ACC * math.sqrt(nkv) * EPS24 + E_EXP) * sv


def norm_expect(x, mean, var, gamma, beta, eps, count, silu, add=None):
    """x [..., C] float64 with mean / var broadcast to it -> (r, bound) of (x - mean) rstd gamma + beta (+SiLU) (+add)."""
    rstd = 1.0 / torch.sqrt(var + eps)
    xhat = (x - mean) * rstd
    pre = xhat * gamma + beta
    delta = C_ACC * math.sqrt(count) * EPS24
    sd = var.sqrt()
    d_mean = delta * (mean.abs() + sd)
    d_rstd = 1.5 * delta * (mean * mean + var) / (var + eps) + 2.0 ** -22
    e = gamma.abs() * (xhat.abs() * d_rstd + d_mean * rstd + 2.0 ** -23 * (x.abs() + mean.abs()) * rstd)
    if silu:
        r, e = silu64(pre), ACT_GAIN * e + SILU_REL * pre.abs()
    else:
        r = pre
    if add is not None:
        r = r + add
    return r, U_BF16 * r.abs() + e


def ratio(y, r, bound):
    """|y - r| / bound, NaN (a poisoned value that leaked into the result) -> inf."""
    q = (y.double() - r).abs() / bound.clamp_min(1e-300)
    return torch.nan_to_num(q, nan=float("inf"))


# ================================================================================================================ replay (GPU)
def _lpd(v, cap):
    d = 1
    while d * 2 <= cap and v % (d * 2) == 0:
        d *= 2
    return d


class Replay:
    def __init__(self, dev, seed):
        self.dev = dev
        self.g = torch.Generator(device=dev).manual_seed(seed)
        self.stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def randn(self, *shape, std=1.0):
        return torch.randn(shape, device=self.dev, generator=self.g) * std

    def rand(self, *shape):
        return torch.rand(shape, device=self.dev, generator=self.g)

    def poisoned(self, rows, pitch, values=None, dtype=torch.bfloat16):
        """[rows, pitch] NaN, with `values` [rows, c] in the first c columns."""
        t = torch.full((rows, pitch), float("nan"), dtype=dtype, device=self.dev)
        if values is not None:
            t[:, :values.shape[1]] = values.to(dtype)
        return t


def _layout(out, c_eff, what):
    """The call wrote every element of its columns (finite) and nothing beyond them (still NaN)."""
    errs = []
    o = out.view(out.shape[0], -1) if out.dim() > 2 else out
    if not bool(torch.isfinite(o[:, :c_eff]).all()):
        bad = (~torch.isfinite(o[:, :c_eff])).nonzero()[0].tolist()
        errs.append(f"{what}: non-finite output at (row, column) {bad} (unwritten, or a poisoned input was read)")
    if o.shape[1] > c_eff and not bool(torch.isnan(o[:, c_eff:].float()).all()):
        bad = (~torch.isnan(o[:, c_eff:].float())).nonzero()[0].tolist()
        errs.append(f"{what}: wrote beyond its {c_eff} columns at (row, column - {c_eff}) {bad}")
    return errs


def _bitwise_equal(a, b):
    it = {torch.bfloat16: torch.int16, torch.float32: torch.int32}[a.dtype]
    return torch.equal(a.view(it), b.view(it))


def _pick(n, work, limit):
    """Images the reference evaluates: all, or the first and last when the work is large."""
    return list(range(n)) if n <= 2 or work <= limit else [0, n - 1]


def _conv_ref(xpad, w64, s, k, h, w):
    """float64 convolution (no padding) of xpad [nI, C, Hp, Wp] by w64 [cout, C, k, k] -> (acc, |x| (*) |w|) [nI, h, w, cout],
    im2col + GEMM in bands of output rows so no intermediate exceeds ~1 GB."""
    nI, Cin = xpad.shape[:2]
    wf = w64.reshape(w64.shape[0], -1)
    wa = wf.abs()
    xpad = xpad[:, :, :, :(w - 1) * s + k]
    acc = torch.empty((nI, h, w, wf.shape[0]), dtype=torch.float64, device=xpad.device)
    m = torch.empty_like(acc)
    band = max(1, (1 << 26) // (nI * w * wf.shape[1]))
    for y0 in range(0, h, band):
        y1 = min(h, y0 + band)
        cols = F.unfold(xpad[:, :, y0 * s:(y1 - 1) * s + k], k, stride=s)  # [nI, C k k, (y1-y0) w]
        acc[:, y0:y1] = (wf @ cols).view(nI, -1, y1 - y0, w).permute(0, 2, 3, 1)
        m[:, y0:y1] = (wa @ cols.abs_()).view(nI, -1, y1 - y0, w).permute(0, 2, 3, 1)
        del cols
    return acc, m


def _m_tile(f, img, y, x):
    up, k, s = f["up"], f["k"], f["s"]
    HO, WO = (f["h"] // 2, f["w"] // 2) if up else (f["h"], f["w"])
    yy, xx = (y // 2, x // 2) if up else (y, x)
    bw = 128 if (k == 1 and f["h"] == 1 and s == 1) else _lpd(WO, 128)
    bh = _lpd(HO, 128 // bw)
    bn = 128 // (bw * bh)
    tx, ty = -(-WO // bw), -(-HO // bh)
    t = ((img // bn) * ty + yy // bh) * tx + xx // bw
    par = f" parity ({y % 2}, {x % 2})" if up else ""
    return f"M tile {t} of {tx * ty * -(-f['n'] // bn)}{par} (tile = {bn} x {bh} x {bw} pixels)"


def replay_conv(R, f):
    from ladi_vton_b200 import lib, weights
    n, h, w, cout, k, s, pad, up, act = (f[x] for x in ("n", "h", "w", "cout", "k", "s", "p", "up", "act"))
    hin, win, K = f["hin"], f["win"], f["K"]
    srcs = [(f["c0"], f["p0"]), (f["c1"], f["p1"])][:f["nsrc"]]
    scs = [(f["sc0c"], f["sc0p"]), (f["sc1c"], f["sc1p"])][:f["nsc"]]
    rows = n * h * w
    c_eff = cout // 2 if act == 2 else cout
    xs = [R.poisoned(n * hin * win, p, R.randn(n * hin * win, c)) for c, p in srcs]
    sc = [R.poisoned(rows, p, R.randn(rows, c)) for c, p in scs]
    csum, scsum = sum(c for c, _ in srcs), sum(c for c, _ in scs)
    fan = k * k * csum + scsum
    wmain = R.randn(cout, csum, k, k, std=fan ** -0.5).bfloat16().float()
    wsc = R.randn(cout, scsum, std=fan ** -0.5).bfloat16().float() if scs else None
    if up:
        packed = weights.pack_conv_up2x(wmain, [c for c, _ in srcs])
        wref = weights.merge_up2x(wmain).bfloat16().double()  # what the kernel multiplies: the merged 2x2 weights, rounded once
    else:
        packed = weights.pack_conv(wmain, [c for c, _ in srcs], wsc[:, :, None, None] if scs else None, [c for c, _ in scs])
    assert packed.shape[1] == K, f"packed K {packed.shape[1]} != descriptor K {K}"
    wbuf = R.poisoned(packed.shape[0], f["wp"], packed)
    step = bias_eff = bias_buf = None
    if f["bias"]:
        if f["bpr"]:
            bias_buf = R.randn(rows)
            bias_eff = bias_buf[:, None]
        elif f["bss"]:  # per-step bias table: the kernel adds *step_ptr * stride; the engine points into the middle of the table
            tab = R.randn(4, f["bss"], std=0.5)
            off = (f["bss"] - cout) // 2 // 4 * 4
            step = torch.tensor([2, 0], dtype=torch.int32, device=R.dev)
            bias_buf, bias_eff = tab.view(-1)[off:], tab[2, off:off + cout]
        else:
            bias_buf = bias_eff = R.randn(cout, std=0.5)
    res = R.poisoned(rows, f["rp"], R.randn(rows, cout)) if f["res"] else None
    rs = R.rand(rows) if f["rs"] else None
    odt = torch.float32 if f["f32"] else torch.bfloat16
    ws = torch.empty(SPLITK_WS_BYTES // 4, dtype=torch.float32, device=R.dev)

    d = lib.ConvDesc()
    for fld, key in (("n", "n"), ("h_out", "h"), ("w_out", "w"), ("c_out", "cout"), ("h_in", "hin"), ("w_in", "win"), ("ksize", "k"), ("stride", "s"),
                     ("pad_lo", "p"), ("n_src", "nsrc"), ("n_sc", "nsc"), ("k_total", "K"), ("weight_pitch", "wp"), ("bias_per_row", "bpr"),
                     ("bias_step_stride", "bss"), ("residual_pitch", "rp"), ("act", "act"), ("out_pitch", "op"), ("out_fp32", "f32"), ("up2x", "up")):
        setattr(d, fld, f[key])
    for i, (c, p) in enumerate(srcs):
        d.src[i], d.src_c[i], d.src_pitch[i] = xs[i].data_ptr(), c, p
    for i, (c, p) in enumerate(scs):
        d.sc[i], d.sc_c[i], d.sc_pitch[i] = sc[i].data_ptr(), c, p
    d.weight = wbuf.data_ptr()
    d.bias = bias_buf.data_ptr() if bias_buf is not None else None
    d.step_ptr = step.data_ptr() if step is not None else None
    d.residual = res.data_ptr() if res is not None else None
    d.row_scale = rs.data_ptr() if rs is not None else None
    d.splitk_ws, d.splitk_ws_bytes = ws.data_ptr(), SPLITK_WS_BYTES
    outs = []
    for _ in range(2):
        o = R.poisoned(rows, f["op"], dtype=odt)
        d.out = o.data_ptr()
        lib.call("ladi_conv2d_bf16", C.byref(d), R.stream)
        outs.append(o)
    torch.cuda.synchronize()
    errs = _layout(outs[0], c_eff, "output")
    if not _bitwise_equal(outs[0], outs[1]):
        errs.append("two runs differ bitwise")
    if errs:
        return errs, None

    imgs = _pick(n, n * h * w * cout * K, 1 << 35)
    sel = torch.tensor(imgs, device=R.dev)
    nI = len(imgs)
    X = torch.cat([x.view(n, hin, win, -1)[sel, ..., :c].double() for x, (c, _) in zip(xs, srcs)], dim=3).permute(0, 3, 1, 2)
    if up:
        xpad = F.pad(X, (1, 1, 1, 1))
        acc = torch.empty((nI, h, w, cout), dtype=torch.float64, device=R.dev)
        m = torch.empty_like(acc)
        for p in range(4):
            py, px = p // 2, p % 2
            a_, m_ = _conv_ref(xpad[:, :, py:py + hin + 1, px:px + win + 1], wref[p], 1, 2, hin, win)
            acc[:, py::2, px::2], m[:, py::2, px::2] = a_, m_
    else:
        pe = pad if k == 3 else 0
        xpad = F.pad(X, (pe, max(0, (w - 1) * s + k - pe - win), pe, max(0, (h - 1) * s + k - pe - hin)))
        acc, m = _conv_ref(xpad, wmain.double(), s, k, h, w)
    del X, xpad
    if scs:
        Sx = torch.cat([t.view(n, h, w, -1)[sel, ..., :c].double() for t, (c, _) in zip(sc, scs)], dim=3)
        acc += Sx @ wsc.double().t()
        m += Sx.abs() @ wsc.double().abs().t()
        del Sx
    if bias_eff is not None:
        be = bias_eff.double()
        if f["bpr"]:
            be = be.view(n, h, w, 1)[sel]
        acc += be
        m += be.abs()
    rsel = res.view(n, h, w, -1)[sel, ..., :cout].double() if res is not None else None
    if rsel is not None:
        m += rsel.abs()
    rss = rs.view(n, h, w, 1)[sel].double() if rs is not None else None
    r, bound = conv_expect(acc, m, K, act, rsel, rss, bool(f["f32"]))
    del acc, m
    y = outs[0].view(n, h, w, -1)[sel, ..., :c_eff]
    q = ratio(y, r, bound)
    worst = float(q.max())
    i0, yy, xx, cc = (int(v) for v in torch.unravel_index(q.argmax(), q.shape))
    ac = 2 * cc if act == 2 else cc
    where = (f"image {imgs[i0]}, y {yy}, x {xx}, channel {cc}: {_m_tile(f, imgs[i0], yy, xx)}, accumulator columns [{ac // 64 * 64}, "
             f"{ac // 64 * 64 + 64}) (N tile {ac // 128} at BN 128, {ac // 64} at BN 64); got {float(y[i0, yy, xx, cc]):.6g}, "
             f"ref {float(r[i0, yy, xx, cc]):.6g}, bound {float(bound[i0, yy, xx, cc]):.3g}")
    return ([f"err/bound {worst:.3g} at {where}"] if worst > 1 else []), (worst, where)


def _strided(buf, batch, n, pitch, bstride):
    return buf.as_strided((batch, n, pitch), (bstride, pitch, 1))


def _attn_ref(q, k, v, heads, D, scale):
    """q [nq, heads*D], k/v [nkv, heads*D] float64 -> (o, sum p|v| / l) [nq, heads*D], chunked over queries."""
    nq, nkv = q.shape[0], k.shape[0]
    qh, kh, vh = (t.view(-1, heads, D).transpose(0, 1) for t in (q, k, v))
    o = torch.empty((heads, nq, D), dtype=torch.float64, device=q.device)
    sv = torch.empty_like(o)
    ch = max(1, (1 << 26) // (heads * nkv))
    for i in range(0, nq, ch):
        s = (qh[:, i:i + ch] @ kh.transpose(1, 2)) * scale
        p = torch.exp(s - s.amax(-1, keepdim=True))
        del s
        l = p.sum(-1, keepdim=True)
        o[:, i:i + ch] = (p @ vh) / l
        sv[:, i:i + ch] = (p @ vh.abs()) / l
        del p
    return o.transpose(0, 1).reshape(nq, heads * D), sv.transpose(0, 1).reshape(nq, heads * D)


def replay_attn(R, f):
    from ladi_vton_b200 import lib
    D, B, heads, nq, nkv = f["d"], f["batch"], f["heads"], f["nq"], f["nkv"]
    width = heads * D
    sd = 2 ** 0.5  # scores scale * q.k of std 2 (q, k ~ N(0, 2), scale = D^-1/2): a softmax that is not flat
    bufs = {}
    for name, n_, std in (("q", nq, sd), ("k", nkv, sd), ("v", nkv, 1.0)):
        p, bs = f[name + "p"], f[name + "bs"]
        t = torch.full(((B - 1) * bs + n_ * p,), float("nan"), dtype=torch.bfloat16, device=R.dev)
        _strided(t, B, n_, p, bs)[..., :width] = R.randn(B, n_, width, std=std).bfloat16()
        bufs[name] = t
    d = lib.AttnDesc()
    for fld in ("batch", "heads", "nq", "nkv"):
        setattr(d, fld, f[fld])
    d.q, d.q_pitch, d.q_batch_stride = bufs["q"].data_ptr(), f["qp"], f["qbs"]
    d.k, d.k_pitch, d.k_batch_stride = bufs["k"].data_ptr(), f["kp"], f["kbs"]
    d.v, d.v_pitch, d.v_batch_stride = bufs["v"].data_ptr(), f["vp"], f["vbs"]
    d.out_pitch, d.out_batch_stride, d.scale, d.variant = f["op"], f["obs"], f["scale"], 0
    d.head_dim = 0 if D == 64 else D
    outs = []
    for _ in range(2):
        o = torch.full(((B - 1) * f["obs"] + nq * f["op"],), float("nan"), dtype=torch.bfloat16, device=R.dev)
        d.out = o.data_ptr()
        lib.call("ladi_attention_bf16" if D == 64 else "ladi_attention_d512_bf16", C.byref(d), R.stream)
        outs.append(o)
    torch.cuda.synchronize()
    ov = _strided(outs[0], B, nq, f["op"], f["obs"])
    errs = _layout(ov.reshape(B * nq, f["op"]) if f["obs"] == nq * f["op"] else ov[..., :width].reshape(B * nq, width), width, "output")
    if not _bitwise_equal(outs[0], outs[1]):
        errs.append("two runs differ bitwise")
    if errs:
        return errs, None
    worst, where = 0.0, ""
    for b in _pick(B, B * heads * nq * nkv, 1 << 31):
        q, k, v = (_strided(bufs[nm], B, n_, f[nm + "p"], f[nm + "bs"])[b, :, :width].double() for nm, n_ in (("q", nq), ("k", nkv), ("v", nkv)))
        o, sv = _attn_ref(q, k, v, heads, D, f["scale"])
        qq = ratio(ov[b, :, :width], o, attn_expect(o, sv, nkv))
        if float(qq.max()) > worst:
            i, c = (int(t) for t in torch.unravel_index(qq.argmax(), qq.shape))
            worst = float(qq.max())
            where = (f"image {b}, query {i} (query tile {i // 128} of 128 rows, {i // 64} of 64), head {c // D}, column {c % D}: got "
                     f"{float(ov[b, i, c]):.6g}, ref {float(o[i, c]):.6g}")
    return ([f"err/bound {worst:.3g} at {where}"] if worst > 1 else []), (worst, where)


def replay_cls(R, f):
    B, T, heads, hd = f["batch"], f["tokens"], f["heads"], f["hd"]
    Cw = heads * hd
    q0 = R.poisoned(B, f["qp"], R.randn(B, Cw, std=2 ** 0.5))
    kv = R.poisoned(B * T, f["kvp"], torch.cat([R.randn(B * T, Cw, std=2 ** 0.5), R.randn(B * T, Cw)], dim=1))
    return check_cls(R, f, q0, kv, hd ** -0.5)  # the scale of csrc/engine.cu adapter_forward


CLS_TAIL = 3  # NaN rows after the output that no call may write


def check_cls(R, f, q0, kv, scale):
    """Run the descriptor f twice on q0 [B, qp] and kv [B * T, kvp] (NaN in their pitch gaps) into a NaN-poisoned output with CLS_TAIL
    extra rows, then check the layout, determinism and the float64 bound."""
    from ladi_vton_b200 import lib
    B, T, heads, hd = f["batch"], f["tokens"], f["heads"], f["hd"]
    Cw = heads * hd
    outs = []
    for _ in range(2):
        o = R.poisoned(B + CLS_TAIL, f["op"])
        lib.call("ladi_cls_attention", C.c_void_p(q0.data_ptr()), f["qp"], C.c_void_p(kv.data_ptr()), f["kvp"], B, T, heads, hd, scale,
                 C.c_void_p(o.data_ptr()), f["op"], R.stream)
        outs.append(o)
    torch.cuda.synchronize()
    errs = _layout(outs[0][:B], Cw, "output")
    if not bool(torch.isnan(outs[0][B:].float()).all()):
        errs.append("output: wrote past the last image")
    if not _bitwise_equal(outs[0], outs[1]):
        errs.append("two runs differ bitwise")
    if errs:
        return errs, None
    worst, where = 0.0, ""
    for b in range(B):
        kvb = kv[b * T:(b + 1) * T].double()
        o, sv = _attn_ref(q0[b:b + 1, :Cw].double(), kvb[:, :Cw], kvb[:, Cw:2 * Cw], heads, hd, scale)
        qq = ratio(outs[0][b:b + 1, :Cw], o, attn_expect(o, sv, T, u_p=2.0 ** -22))  # P stays fp32 in this kernel
        if float(qq.max()) > worst:
            c = int(qq.argmax())
            worst, where = float(qq.max()), f"image {b}, head {c // hd}, column {c % hd}"
    return ([f"err/bound {worst:.3g} at {where}"] if worst > 1 else []), (worst, where)


def _norm_input(R, rows, c):
    """bf16 values with per-channel scales and offsets of a few sigma (the regime where one-pass fp32 variance loses digits)."""
    return (R.randn(rows, c) * torch.exp(R.randn(c, std=0.5)) + R.randn(c, std=3.0)).bfloat16()


def replay_gn(R, f):
    from ladi_vton_b200 import lib
    n, hw, G, c0, c1, p0, p1 = f["n"], f["hw"], f["groups"], f["c0"], f["c1"], f["p0"], f["p1"]
    Ct = c0 + c1
    xs = [R.poisoned(n * hw, p0, _norm_input(R, n * hw, c0))]
    if c1:
        xs.append(R.poisoned(n * hw, p1, _norm_input(R, n * hw, c1)))
    gamma, beta = 1.0 + R.randn(Ct, std=0.25), R.randn(Ct, std=0.25)
    add = R.poisoned(n * hw, f["ap"], R.randn(n * hw, Ct)) if f["add"] else None
    chunks = lib.load().ladi_groupnorm_chunks(hw)
    P = lambda t: C.c_void_p(t.data_ptr() if t is not None else 0)
    outs = []
    for _ in range(2):
        ws = torch.full((n * chunks * G * 2,), float("nan"), dtype=torch.float32, device=R.dev)
        o = R.poisoned(n * hw, f["op"])
        x1 = xs[1] if c1 else None
        lib.call("ladi_groupnorm_stats", P(xs[0]), c0, p0, P(x1), c1, p1 if c1 else 0, n, hw, G, P(ws), R.stream)
        lib.call("ladi_groupnorm_apply", P(xs[0]), c0, p0, P(x1), c1, p1 if c1 else 0, n, hw, G, P(ws), P(gamma), P(beta), f["eps"], f["silu"],
                 P(add), f["ap"], P(o), f["op"], R.stream)
        outs.append(o)
    torch.cuda.synchronize()
    errs = _layout(outs[0], Ct, "output")
    if not _bitwise_equal(outs[0], outs[1]):
        errs.append("two runs differ bitwise")
    if errs:
        return errs, None
    worst, where = 0.0, ""
    for b in _pick(n, n * hw * Ct, 1 << 28):
        x = torch.cat([t[b * hw:(b + 1) * hw, :c].double() for t, c in zip(xs, (c0, c1))], dim=1)
        xg = x.view(hw, G, Ct // G)
        mean = xg.mean(dim=(0, 2), keepdim=True).expand_as(xg).reshape(hw, Ct)
        var = xg.var(dim=(0, 2), unbiased=False, keepdim=True).expand_as(xg).reshape(hw, Ct)
        a = add[b * hw:(b + 1) * hw, :Ct].double() if add is not None else None
        r, bound = norm_expect(x, mean, var, gamma.double(), beta.double(), f["eps"], hw * Ct // G, f["silu"], a)
        qq = ratio(outs[0][b * hw:(b + 1) * hw, :Ct], r, bound)
        if float(qq.max()) > worst:
            p, c = (int(t) for t in torch.unravel_index(qq.argmax(), qq.shape))
            worst, where = float(qq.max()), f"image {b}, pixel {p}, channel {c} (group {c // (Ct // G)})"
    return ([f"err/bound {worst:.3g} at {where}"] if worst > 1 else []), (worst, where)


def replay_ln(R, f):
    from ladi_vton_b200 import lib
    rows, c = f["rows"], f["c"]
    x = R.poisoned(rows, f["xp"], _norm_input(R, rows, c))
    gamma, beta = 1.0 + R.randn(c, std=0.25), R.randn(c, std=0.25)
    outs = []
    for _ in range(2):
        o = R.poisoned(rows, f["op"])
        lib.call("ladi_layernorm", C.c_void_p(x.data_ptr()), f["xp"], rows, c, C.c_void_p(gamma.data_ptr()), C.c_void_p(beta.data_ptr()), f["eps"],
                 C.c_void_p(o.data_ptr()), f["op"], R.stream)
        outs.append(o)
    torch.cuda.synchronize()
    errs = _layout(outs[0], c, "output")
    if not _bitwise_equal(outs[0], outs[1]):
        errs.append("two runs differ bitwise")
    if errs:
        return errs, None
    xd = x[:, :c].double()
    mean = xd.mean(dim=1, keepdim=True).expand_as(xd)
    var = xd.var(dim=1, unbiased=False, keepdim=True).expand_as(xd)
    r, bound = norm_expect(xd, mean, var, gamma.double(), beta.double(), f["eps"], c, False)
    qq = ratio(outs[0][:, :c], r, bound)
    i, j = (int(t) for t in torch.unravel_index(qq.argmax(), qq.shape))
    worst = float(qq.max())
    return ([f"err/bound {worst:.3g} at row {i}, column {j}"] if worst > 1 else []), (worst, f"row {i}, column {j}")


def _flat_io(R, count, pad=64):
    return torch.full((count + pad,), float("nan"), dtype=torch.bfloat16, device=R.dev)


def replay_add(R, f):
    from ladi_vton_b200 import lib
    cnt = f["count"]
    a, b = R.randn(cnt).bfloat16(), R.randn(cnt).bfloat16()
    outs = []
    for _ in range(2):
        o = _flat_io(R, cnt)
        lib.call("ladi_add_bf16", C.c_void_p(a.data_ptr()), C.c_void_p(b.data_ptr()), C.c_void_p(o.data_ptr()), cnt, R.stream)
        outs.append(o)
    torch.cuda.synchronize()
    errs = _layout(outs[0].view(1, -1), cnt, "output") + ([] if _bitwise_equal(outs[0], outs[1]) else ["two runs differ bitwise"])
    if errs:
        return errs, None
    r = a.double() + b.double()
    qq = ratio(outs[0][:cnt], r, U_BF16 * r.abs())
    worst = float(qq.max())
    return ([f"err/bound {worst:.3g} at element {int(qq.argmax())}"] if worst > 1 else []), (worst, "")


def replay_temb(R, f):
    from ladi_vton_b200 import lib
    n, c0, kp = f["n"], f["c"], f["kp"]
    t = torch.linspace(999, 1, n, device=R.dev).round()
    outs = []
    for _ in range(2):
        o = R.poisoned(n, 2 * kp)
        lib.call("ladi_timestep_embedding", C.c_void_p(t.data_ptr()), n, c0, kp, C.c_void_p(o.data_ptr()), R.stream)
        outs.append(o)
    torch.cuda.synchronize()
    errs = _layout(outs[0], 2 * kp, "output") + ([] if _bitwise_equal(outs[0], outs[1]) else ["two runs differ bitwise"])
    if errs:
        return errs, None
    half = c0 // 2
    arg = t.double()[:, None] * torch.exp(-math.log(10000.0) * torch.arange(half, dtype=torch.float64, device=R.dev) / half)[None, :]
    ref = torch.cat([torch.cos(arg), torch.sin(arg)], dim=1)
    got = outs[0][:, :c0].double() + outs[0][:, kp:kp + c0].double()
    # hi + lo carries ~17 bits (2^-16); the fp32 frequency (device expf) and product t * freq are good to a few ulp of the argument
    qq = ratio(got, ref, 2.0 ** -16 + 2.0 ** -21 * torch.cat([arg, arg], dim=1).abs())
    zero = float(outs[0][:, c0:kp].float().abs().sum() + outs[0][:, kp + c0:].float().abs().sum()) if kp > c0 else 0.0
    worst = float(qq.max())
    errs = ([f"err/bound {worst:.3g} at (timestep, column) {[int(v) for v in torch.unravel_index(qq.argmax(), qq.shape)]}"] if worst > 1 else [])
    return errs + ([] if zero == 0 else ["padding columns are not zero"]), (worst, "")


REPLAY = {"conv": replay_conv, "attn_d64": replay_attn, "attn_d512": replay_attn, "gn": replay_gn, "ln": replay_ln, "cls_attn": replay_cls,
          "add": replay_add, "timestep_embedding": replay_temb}


# ================================================================================================================ CPU: census integrity
def test_census_integrity():
    desc, calls, unparsed = census()
    print_census(desc, calls)
    assert not unparsed, "trace lines the replay does not implement (new op kind or field):\n  " + "\n  ".join(unparsed[:10])
    assert set(REPLAY) == set(KINDS) and {d["kind"] for d in desc.values()} <= set(REPLAY)
    convs = [d["f"] for d in desc.values() if d["kind"] == "conv"]
    # the paths the op tests do not reach, which this census exists to cover
    assert any(f["act"] == 3 for f in convs), "GELU epilogue (adapter MLP)"
    assert any(f["act"] == 3 and f["w"] == 8 and f["K"] >= 2048 for f in convs), "GELU GEMM at M = 8 eligible for split-K"
    assert any(f["nsc"] == 2 and f["K"] >= 2048 for f in convs), "split-K-eligible conv with a two-source fused 1x1 shortcut"
    assert any(f["k"] == 1 and f["h"] == 1 and f["p0"] > f["c0"] * 8 for f in convs), "row-strided A (adapter CLS projection)"
    assert any(f["res"] and f["rp"] > f["cout"] * 8 for f in convs), "row-strided residual (adapter CLS out-projection)"
    assert any(f["up"] for f in convs), "nearest-2x upsample fused into the 3x3 convolution"
    assert any(f["cout"] == 4 and f["op"] == 8 for f in convs), "post-quant GEMM writing 4 channels into pitch 8"
    assert any(f["bss"] and f["step"] for f in convs), "per-step bias table"
    gns = [d["f"] for d in desc.values() if d["kind"] == "gn"]
    assert any(f["add"] for f in gns), "GroupNorm with the add operand (VAE decoder image-level skip)"
    assert any(f["c1"] for f in gns), "two-source GroupNorm"
    assert any(d["kind"] == "cls_attn" for d in desc.values()), "CLS attention of the inversion adapter"
    attn = [d["f"] for d in desc.values() if d["kind"] == "attn_d64"]
    assert any(f["nq"] == 12288 for f in attn), "d = 64 attention at 12288 queries (1024x768)"
    assert any(f["nkv"] == 77 and f["kp"] > 2 * f["heads"] * 64 for f in attn), "cross-attention K/V read from the packed all-layer buffer"
    assert any(d["kind"] == "attn_d512" for d in desc.values())


# ================================================================================================================ CPU: the bound has teeth
def _gemm_case(seed, M=300, K=640, N=192):
    g = torch.Generator().manual_seed(seed)
    a = torch.randn((M, K), generator=g).bfloat16()
    w = (torch.randn((N, K), generator=g) * K ** -0.5).bfloat16()
    b = torch.randn((N,), generator=g) * 0.5
    pre = a.double() @ w.double().t() + b.double()
    m = a.double().abs() @ w.double().abs().t() + b.double().abs()
    return a, w, b, pre, m


def _emulate_gemm(a, w, b, act=0, drop_block=None, splits=1, drop_split=None):
    """fp32 accumulation over 64-wide K blocks, in REVERSE block order (an order no float64 reference uses), optionally split-K into
    `splits` fp32 partials summed in order; then bias, activation and bf16 rounding."""
    K = a.shape[1]
    nb = K // 64
    per = -(-nb // splits)
    parts = []
    for sp in range(splits):
        acc = torch.zeros((a.shape[0], w.shape[0]), dtype=torch.float32)
        for kb in reversed(range(sp * per, min(nb, (sp + 1) * per))):
            if kb != drop_block:
                acc += a[:, kb * 64:(kb + 1) * 64].float() @ w[:, kb * 64:(kb + 1) * 64].float().t()
        parts.append(acc)
    acc = sum(p for i, p in enumerate(parts) if i != drop_split)
    return acc, b


def _finish(acc, b, act):
    pre = acc + b
    if act == 1:
        y = F.silu(pre)
    elif act == 2:
        y = pre[:, 0::2] * F.gelu(pre[:, 1::2])
    elif act == 3:
        y = F.gelu(pre)
    else:
        y = pre
    return y.bfloat16()


@pytest.mark.parametrize("act", [0, 1, 2, 3])
def test_bound_accepts_honest_gemm(act):
    a, w, b, pre, m = _gemm_case(1)
    r, bound = conv_expect(pre, m, a.shape[1], act)
    acc, _ = _emulate_gemm(a, w, b)
    assert float(ratio(_finish(acc, b, act), r, bound).max()) <= 1.0
    acc, _ = _emulate_gemm(a, w, b, splits=4)  # split-K partials, summed in split order
    assert float(ratio(_finish(acc, b, act), r, bound).max()) <= 1.0


def test_bound_rejects_gemm_faults():
    a, w, b, pre, m = _gemm_case(2)
    K = a.shape[1]
    r, bound = conv_expect(pre, m, K, 0)
    check = lambda y: float(ratio(y, r, bound).max())
    acc, _ = _emulate_gemm(a, w, b, drop_block=5)  # 1. one 64-wide K block missing from the reduction
    assert check(_finish(acc, b, 0)) > 1
    acc, _ = _emulate_gemm(a, w, b, splits=4, drop_split=3)  # 2. one split-K partial missing
    assert check(_finish(acc, b, 0)) > 1
    acc, _ = _emulate_gemm(a, w, b)
    bad = b.clone()  # 3. one 8-column group of N tile 1 (BN = 64) reads the neighbouring group's bias
    bad[64 + 24:64 + 32] = b[64 + 32:64 + 40]
    assert check(_finish(acc, bad, 0)) > 1
    y = _finish(acc, b, 0)  # 4. the ragged last M tile (rows 256..299 of 300) holds a copy of the previous tile's rows
    y[256:] = y[128:128 + 44]
    assert check(y) > 1
    assert check(_finish(acc, b, 0)) <= 1  # and the honest result on the same data passes


def _attn_case(seed, nq, nkv, D=64):
    g = torch.Generator().manual_seed(seed)
    q = (torch.randn((nq, D), generator=g) * 2 ** 0.5).bfloat16()
    k = (torch.randn((nkv, D), generator=g) * 2 ** 0.5).bfloat16()
    v = torch.randn((nkv, D), generator=g).bfloat16()
    o, sv = _attn_ref(q.double(), k.double(), v.double(), 1, D, D ** -0.5)
    return q, k, v, o, sv


def _emulate_attn(q, k, v, scale, padded_keys_count=False, tile=128, skip_rescale=None):
    """Flash-style fp32 emulation over K/V tiles of 128: running max, exp2, P rounded to bf16 for P.V, l from the fp32 P.  The faults:
    the padded keys of the last tile (zero-filled K and V) enter the softmax as keys of score 0; skip_rescale = "l" / "o": a new running
    maximum does not rescale l / the O accumulator."""
    nkv = k.shape[0]
    nt = -(-nkv // tile)
    kp = torch.zeros((nt * tile, k.shape[1]), dtype=torch.float32)
    vp = torch.zeros_like(kp)
    kp[:nkv], vp[:nkv] = k.float(), v.float()
    mx = torch.full((q.shape[0], 1), -float("inf"))
    l = torch.zeros((q.shape[0], 1))
    acc = torch.zeros((q.shape[0], k.shape[1]))
    l2e = 1.4426950408889634
    for t in range(nt):
        s = (q.float() @ kp[t * tile:(t + 1) * tile].t()) * (scale * l2e)
        if not padded_keys_count:
            valid = torch.arange(t * tile, (t + 1) * tile) < nkv
            s[:, ~valid] = -float("inf")
        mn = torch.maximum(mx, s.amax(1, keepdim=True))
        p = torch.exp2(s - mn)
        corr = torch.exp2(mx - mn)
        l = (l if skip_rescale == "l" else l * corr) + p.sum(1, keepdim=True)
        acc = (acc if skip_rescale == "o" else acc * corr) + p.bfloat16().float() @ vp[t * tile:(t + 1) * tile]
        mx = mn
    return (acc / l).bfloat16()


@pytest.mark.parametrize("nkv", [77, 200])
def test_bound_attention_teeth(nkv):
    q, k, v, o, sv = _attn_case(3, 96, nkv)
    bound = attn_expect(o, sv, nkv)
    assert float(ratio(_emulate_attn(q, k, v, 0.125), o, bound).max()) <= 1.0  # honest: accepted
    assert float(ratio(_emulate_attn(q, k, v, 0.125, padded_keys_count=True), o, bound).max()) > 1  # 5. padded keys counted: rejected


@pytest.mark.parametrize("skip", ["l", "o"])
def test_bound_attention_rescale_teeth(skip):
    """Keys whose scores grow tile by tile (the maximum moves on every tile): skipping the rescale of l or of O is rejected."""
    g = torch.Generator().manual_seed(4)
    D, nq, nkv = 64, 96, 64 * 6
    u = torch.sign(torch.randn(D, generator=g))
    q = (torch.randn((nq, D), generator=g) * 0.5 + u).bfloat16()
    k = (torch.randn((nkv, D), generator=g) * 0.5 + (2.0 * (torch.arange(nkv) // 64) / (0.125 * D))[:, None] * u).bfloat16()
    v = torch.randn((nkv, D), generator=g).bfloat16()
    o, sv = _attn_ref(q.double(), k.double(), v.double(), 1, D, 0.125)
    bound = attn_expect(o, sv, nkv)
    assert float(ratio(_emulate_attn(q, k, v, 0.125, tile=64), o, bound).max()) <= 1.0
    assert float(ratio(_emulate_attn(q, k, v, 0.125, tile=64, skip_rescale=skip), o, bound).max()) > 1


# ================================================================================================================ GPU: replay
@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_replay_against_float64(cuda, kind):
    desc, calls, unparsed = census()
    todo = [(key, d) for key, d in desc.items() if d["kind"] == kind]
    assert todo, f"no {kind} descriptor in the census"
    R = Replay(cuda, 1234)
    failures, worst, t0 = [], (0.0, "", ""), time.time()
    for key, d in todo:
        errs, res = REPLAY[kind](R, d["f"])
        if errs:
            failures.append(f"{key}\n    first issued by {d['first']}\n    " + "\n    ".join(errs))
        if res is not None and res[0] > worst[0]:
            worst = (res[0], key, res[1])
        torch.cuda.empty_cache()
    print(f"\n{kind}: {len(todo)} distinct descriptors replayed in {time.time() - t0:.1f} s; worst err/bound {worst[0]:.3g}"
          + (f" ({worst[2]}; {worst[1]})" if worst[1] else ""))
    assert not failures, f"{len(failures)} of {len(todo)} {kind} descriptors fail:\n" + "\n".join(failures)
