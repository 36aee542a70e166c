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

The error bound is per element; its constants and their derivation are in tests/kernel_check.py's docstring.
The CPU tests at the end show the bound has teeth: the same checker rejects five simulated kernel faults and accepts an honest fp32
emulation."""
import ctypes as C
import math
import time
from collections import defaultdict

import pytest
import torch
import torch.nn.functional as F

from kernel_check import (U_BF16, Replay, argworst, attn_expect, attn_ref, census, check_cls, conv_expect, determinism, emulate_attn, flat_buf,
                          layout, norm_expect, norm_input, pick, ptr, ratio, replay_conv, replay_ln, twice)

# ================================================================================================================ the census (CPU)
# per op: the fields the trace prints; the replay implements exactly these (an unknown op or field fails test_census_integrity)
KINDS = ["conv", "attn_d64", "attn_d512", "gn", "ln", "cls_attn", "add", "timestep_embedding"]
# (workload label, [(module, batch, height, width)]): the shapes of bench.py / BASELINE.json; "ctx" = plan_context GEMM at (UNet batch) x 77 rows


def print_census(desc, calls):
    print("\nworkload census: calls (distinct descriptors) per module and shape")
    for (wl, label), cnt in calls.items():
        print(f"  {label:44s} " + ", ".join(f"{k} {v[0]} ({len(v[1])})" for k, v in sorted(cnt.items())) + f"   [{wl}]")
    per = defaultdict(int)
    for d in desc.values():
        per[d["kind"]] += 1
    print("  distinct over all workloads: " + ", ".join(f"{k} {per[k]}" for k in KINDS if per[k]))


# ================================================================================================================ replay (GPU)
def _strided(buf, batch, n, pitch, bstride):
    return buf.as_strided((batch, n, pitch), (bstride, pitch, 1))


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

    def call(b):
        d.out = b["out"].data_ptr()
        lib.call("ladi_attention_bf16" if D == 64 else "ladi_attention_d512_bf16", C.byref(d), R.stream)
    runs = twice(call, lambda: dict(out=torch.full(((B - 1) * f["obs"] + nq * f["op"],), float("nan"), dtype=torch.bfloat16, device=R.dev)))
    ov = _strided(runs[0]["out"], B, nq, f["op"], f["obs"])
    errs = layout(ov.reshape(B * nq, f["op"]) if f["obs"] == nq * f["op"] else ov[..., :width].reshape(B * nq, width), 0, width, "output")
    errs += determinism(runs, ["out"])
    if errs:
        return errs, None
    worst, where = 0.0, ""
    for b in pick(B, B * heads * nq * nkv, 1 << 31):
        q, k, v = (_strided(bufs[nm], B, n_, f[nm + "p"], f[nm + "bs"])[b, :, :width].double() for nm, n_ in (("q", nq), ("k", nkv), ("v", nkv)))
        o, sv = attn_ref(q, k, v, heads, D, f["scale"])
        w, (i, c) = argworst(ratio(ov[b, :, :width], o, attn_expect(o, sv, nkv)))
        if w > worst:
            worst = w
            where = (f"image {b}, query {i} (query tile {i // 128} of 128 rows, {i // 64} of 64), head {c // D}, column {c % D}: got "
                     f"{float(ov[b, i, c]):.6g}, ref {float(o[i, c]):.6g}")
    return ([f"err/bound {worst:.3g} at {where}"] if worst > 1 else []), (worst, where)


def replay_cls(R, f):
    B, T, heads, hd = f["batch"], f["tokens"], f["heads"], f["hd"]
    Cw = heads * hd
    q0 = R.poisoned(B, f["qp"], R.randn(B, Cw, std=2 ** 0.5))
    kv = R.poisoned(B * T, f["kvp"], torch.cat([R.randn(B * T, Cw, std=2 ** 0.5), R.randn(B * T, Cw)], dim=1))
    return check_cls(R, f, q0, kv, hd ** -0.5)  # the scale of csrc/engine.cu adapter_forward


def replay_gn(R, f):
    from ladi_vton_b200 import lib
    n, hw, G, c0, c1, p0, p1 = f["n"], f["hw"], f["groups"], f["c0"], f["c1"], f["p0"], f["p1"]
    Ct = c0 + c1
    xs = [R.poisoned(n * hw, p0, norm_input(R, n * hw, c0))]
    if c1:
        xs.append(R.poisoned(n * hw, p1, norm_input(R, n * hw, c1)))
    gamma, beta = 1.0 + R.randn(Ct, std=0.25), R.randn(Ct, std=0.25)
    add = R.poisoned(n * hw, f["ap"], R.randn(n * hw, Ct)) if f["add"] else None
    chunks = lib.load().ladi_groupnorm_chunks(hw)
    x1 = xs[1] if c1 else None

    def call(b):
        lib.call("ladi_groupnorm_stats", ptr(xs[0]), c0, p0, ptr(x1), c1, p1 if c1 else 0, n, hw, G, ptr(b["ws"]), R.stream)
        lib.call("ladi_groupnorm_apply", ptr(xs[0]), c0, p0, ptr(x1), c1, p1 if c1 else 0, n, hw, G, ptr(b["ws"]), ptr(gamma), ptr(beta), f["eps"],
                 f["silu"], ptr(add), f["ap"], ptr(b["out"]), f["op"], R.stream)
    runs = twice(call, lambda: dict(ws=torch.full((n * chunks * G * 2,), float("nan"), dtype=torch.float32, device=R.dev),
                                    out=R.poisoned(n * hw, f["op"])))
    out = runs[0]["out"]
    errs = layout(out, 0, Ct, "output") + determinism(runs, ["out"])
    if errs:
        return errs, None
    worst, where = 0.0, ""
    for b in pick(n, n * hw * Ct, 1 << 28):
        x = torch.cat([t[b * hw:(b + 1) * hw, :c].double() for t, c in zip(xs, (c0, c1))], dim=1)
        xg = x.view(hw, G, Ct // G)
        mean = xg.mean(dim=(0, 2), keepdim=True).expand_as(xg).reshape(hw, Ct)
        var = xg.var(dim=(0, 2), unbiased=False, keepdim=True).expand_as(xg).reshape(hw, Ct)
        a = add[b * hw:(b + 1) * hw, :Ct].double() if add is not None else None
        r, bound = norm_expect(x, mean, var, gamma.double(), beta.double(), f["eps"], hw * Ct // G, f["silu"], a)
        w, (p, c) = argworst(ratio(out[b * hw:(b + 1) * hw, :Ct], r, bound))
        if w > worst:
            worst, where = w, f"image {b}, pixel {p}, channel {c} (group {c // (Ct // G)})"
    return ([f"err/bound {worst:.3g} at {where}"] if worst > 1 else []), (worst, where)


def replay_add(R, f):
    from ladi_vton_b200 import lib
    cnt = f["count"]
    a, b = R.randn(cnt).bfloat16(), R.randn(cnt).bfloat16()
    runs = twice(lambda o: lib.call("ladi_add_bf16", ptr(a), ptr(b), ptr(o["out"]), cnt, R.stream),
                 lambda: dict(out=flat_buf(R, cnt, torch.bfloat16)[0]))
    errs = layout(runs[0]["out"].view(1, -1), 0, cnt, "output") + determinism(runs, ["out"])
    if errs:
        return errs, None
    r = a.double() + b.double()
    qq = ratio(runs[0]["out"][:cnt], r, U_BF16 * r.abs())
    worst = float(qq.max())
    return ([f"err/bound {worst:.3g} at element {int(qq.argmax())}"] if worst > 1 else []), (worst, "")


def replay_temb(R, f):
    from ladi_vton_b200 import lib
    n, c0, kp = f["n"], f["c"], f["kp"]
    t = torch.linspace(999, 1, n, device=R.dev).round()
    runs = twice(lambda b: lib.call("ladi_timestep_embedding", ptr(t), n, c0, kp, ptr(b["out"]), R.stream), lambda: dict(out=R.poisoned(n, 2 * kp)))
    outs = [r["out"] for r in runs]
    errs = layout(outs[0], 0, 2 * kp, "output") + determinism(runs, ["out"])
    if errs:
        return errs, None
    half = c0 // 2
    arg = t.double()[:, None] * torch.exp(-math.log(10000.0) * torch.arange(half, dtype=torch.float64, device=R.dev) / half)[None, :]
    ref = torch.cat([torch.cos(arg), torch.sin(arg)], dim=1)
    got = outs[0][:, :c0].double() + outs[0][:, kp:kp + c0].double()
    # hi + lo carries ~17 bits (2^-16); the fp32 frequency (device expf) and product t * freq are good to a few ulp of the argument
    qq = ratio(got, ref, 2.0 ** -16 + 2.0 ** -21 * torch.cat([arg, arg], dim=1).abs())
    zero = float(outs[0][:, c0:kp].float().abs().sum() + outs[0][:, kp + c0:].float().abs().sum()) if kp > c0 else 0.0
    worst, at = argworst(qq)
    errs = ([f"err/bound {worst:.3g} at (timestep, column) {at}"] if worst > 1 else [])
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
    o, sv = attn_ref(q.double(), k.double(), v.double(), 1, D, D ** -0.5)
    return q, k, v, o, sv


@pytest.mark.parametrize("nkv", [77, 200])
def test_bound_attention_teeth(nkv):
    q, k, v, o, sv = _attn_case(3, 96, nkv)
    bound = attn_expect(o, sv, nkv)
    assert float(ratio(emulate_attn(q, k, v, 0.125, 128), o, bound).max()) <= 1.0  # honest: accepted
    assert float(ratio(emulate_attn(q, k, v, 0.125, 128, "padded"), o, bound).max()) > 1  # 5. padded keys counted: rejected


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
