"""The 160-wide N tile's staged epilogue: bit for bit the fragment path's result, and right against float64.

A launch with N tile 160 and a long reduction (more than 8 K blocks) whose bf16 output rows are whole, 16-byte aligned chunks leaves the
kernel through a 40 KB shared-memory staging tile (20 chunks per row, its own swizzle) beside a 5-stage pipeline; with an output pitch of
c + 4 the same call stores from the accumulator fragment.  Each GPU case runs both on the same data (force_bn=160, the plan asserted
first) and checks
- the staged output against float64 with the census's per-element bound (conv_expect), its pitch gap still NaN;
- the two outputs bitwise equal (same arithmetic, same K-block order, one rounding to bf16).
The cases cover every epilogue form with both bias kinds, a ragged last M tile and c_out not a multiple of 160, 3x3 convolutions whose
M tiles span rows and images, the fused nearest-2x upsample, K-block counts around the 5-stage ring, work items around the SM count and an
in-place residual.

The CPU test pins where the library's plan takes the 160-wide tile for the benchmarked UNet step and the VAE at 132 SMs: only long
reductions that can be staged, every short reduction keeps its plan, and the VAE's 128 / 256 / 512-wide convolutions are left alone."""
import re

import pytest
import torch
import torch.nn.functional as F

from kernel_check import SMS, conv_expect, cpu_gen, ladi_lib, max_ratio, nan_buf, same, sms

FORMS = ["bias", "nobias", "stepbias", "rowbias", "silu", "gelu", "relu", "geglu", "residual", "inplace", "rowscale", "silu_res_rowscale"]


def _inputs(form, rows, c_out, c_eff, dev, seed):
    """Epilogue operands of one form: (ops kwargs, float64 column / row bias, residual bf16 [rows, c_eff] or None, row scale, act)."""
    from ladi_vton_b200 import ops
    g = cpu_gen(seed)
    act = {"silu": ops.ACT_SILU, "gelu": ops.ACT_GELU, "relu": ops.ACT_RELU, "geglu": ops.ACT_GEGLU,
           "silu_res_rowscale": ops.ACT_SILU}.get(form, ops.ACT_NONE)
    kw, bcol, brow, res, rs = {"act": act}, None, None, None, None
    if form == "stepbias":
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
    if form in ("residual", "inplace", "silu_res_rowscale"):
        res = torch.randn((rows, c_eff), generator=g).to(dev).bfloat16()
    if form in ("rowscale", "silu_res_rowscale"):
        rs = torch.rand((rows,), generator=g).to(dev)
        kw.update(row_scale=rs)
        rs = rs.double()
    return kw, bcol, brow, res, rs, act


def _run_both(call, form, rows, c_eff, res, dev, want):
    """call(out [rows, pitch] view, residual view or None, plan=False) at a staged pitch (c_eff + 8) and a fragment pitch (c_eff + 4);
    want(plan, staged) asserts each plan.  -> the staged output [rows, c_eff]."""
    outs = []
    for pitch, staged in ((c_eff + 8, 1), (c_eff + 4, 0)):
        if form == "inplace":
            buf = nan_buf((rows, pitch), torch.bfloat16, dev, res)
            rbuf = buf[:, :c_eff]
        else:
            buf = nan_buf((rows, pitch), torch.bfloat16, dev)
            rbuf = None if res is None else nan_buf((rows, pitch), torch.bfloat16, dev, res)[:, :c_eff]
        plan = call(buf, rbuf, plan=True)
        assert (plan.bn, plan.staged, plan.splits, plan.pair) == (160, staged, 1, 0), \
            f"pitch {pitch}: bn {plan.bn} staged {plan.staged} splits {plan.splits} pair {plan.pair}"
        want(plan, staged)
        call(buf, rbuf)
        outs.append(buf)
    torch.cuda.synchronize()
    staged, frag = outs
    assert bool(torch.isnan(staged[:, c_eff:].float()).all()), "the staged drain wrote into the pitch gap"
    assert bool(torch.isfinite(staged[:, :c_eff].float()).all()), "the staged drain left output elements unwritten"
    assert same(staged[:, :c_eff], frag[:, :c_eff]), "staged and fragment stores differ"
    return staged[:, :c_eff]


def _check(y, acc, m, K, bcol, brow, res, rs, act):
    pre, mm = acc.clone(), m.clone()
    if bcol is not None:
        pre += bcol
        mm += bcol.abs()
    if brow is not None:
        pre += brow[:, None]
        mm += brow.abs()[:, None]
    r64 = None
    if res is not None:
        r64 = res.double()
        mm += r64.abs()
    r, bound = conv_expect(pre, mm, K, act, r64, None if rs is None else rs[:, None])
    worst = max_ratio(y, r, bound)
    assert worst <= 1.0, f"err/bound {worst:.3g}"


def _gemm_case(dev, form, M, kb, c_out, want=lambda plan, staged: None, seed=31):
    from ladi_vton_b200 import ops, weights
    K = 64 * kb
    c_eff = c_out // 2 if form == "geglu" else c_out
    g = cpu_gen(seed)
    a = torch.randn((M, K), generator=g).to(dev).bfloat16()
    w = (torch.randn((c_out, K), generator=g) * K ** -0.5).to(dev).bfloat16()
    kw, bcol, brow, res, rs, act = _inputs(form, M, c_out, c_eff, dev, seed + 1)
    wp = weights.pack_linear(w.float())

    def call(out, resid, plan=False):
        return (ops.gemm_plan if plan else ops.gemm)(a, wp, c_out, out=out[:, :c_eff], residual=resid, force_bn=160, split_k=False, **kw)

    y = _run_both(call, form, M, c_eff, res, dev, want)
    _check(y, a.double() @ w.double().t(), a.double().abs() @ w.double().abs().t(), K, bcol, brow, res, rs, act)


@pytest.mark.gpu
@pytest.mark.parametrize("form", FORMS)
def test_staged160_gemm(cuda, form):
    """M 1000 (a ragged last M tile), K 640 (10 K blocks: the ring wraps twice), c_out 448 (2 full tiles and a 128-wide one; 896
    interleaved columns for GEGLU)."""
    _gemm_case(cuda, form, 1000, 10, 896 if form == "geglu" else 448)


def _stages(plan, staged):
    assert plan.stages == (5 if staged else 6), f"stages {plan.stages}"


@pytest.mark.gpu
@pytest.mark.parametrize("kb", [9, 10, 11, 14, 15, 16])
def test_staged160_k_depth(cuda, kb):
    """K-block counts around the 5-stage ring (9 is the shortest staged reduction): 2 st - 1 .. 2 st + 1 and 3 st - 1 .. 3 st + 1."""
    _gemm_case(cuda, "residual", 128 * 3 - 24, kb, 320, want=_stages, seed=kb)


@pytest.mark.gpu
@pytest.mark.parametrize("items", ["1", "sms-1", "sms", "sms+1", "2sms+1"])
def test_staged160_items(cuda, items):
    """Work items around the persistent grid (one 160-wide N tile, so items = M tiles); the last M tile is ragged."""
    s = sms(cuda)
    T = {"1": 1, "sms-1": s - 1, "sms": s, "sms+1": s + 1, "2sms+1": 2 * s + 1}[items]

    def want(plan, staged):
        assert plan.items() == T, f"items {plan.items()}, want {T}"
    _gemm_case(cuda, "silu", 128 * T - 40, 9, 160, want=want, seed=T)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["64x48", "8x6", "16x12", "up2x 8x6"])
@pytest.mark.parametrize("form", ["bias", "rowbias", "silu", "residual", "inplace", "rowscale"])
def test_staged160_conv(cuda, form, shape):
    """3x3 convolutions with c_out 320 over C 128 (18 K blocks): at batch 2 on a 64x48 latent (M tiles of 8 rows x 16 pixels) and at
    batch 16 on 8x6 / 16x12 (M tiles of several rows and images); and the fused nearest-2x upsample over C 192 (4 merged taps, 12 K
    blocks).  Weights are multiples of 1/64 below 1/8 in magnitude, so the upsample's merged taps are exact in bf16 and the float64
    reference is the plain convolution of the upsampled input."""
    from ladi_vton_b200 import ops, weights
    up = shape.startswith("up2x")
    if up and form not in ("bias", "silu"):
        pytest.skip("up2x takes a per-channel bias and an activation only")
    h, w = (int(v) for v in shape.split()[-1].split("x"))
    n = 2 if (h, w) == (64, 48) else 16
    C, c_out = (192 if up else 128), 320
    ho, wo = (2 * h, 2 * w) if up else (h, w)
    rows = n * ho * wo
    g = cpu_gen(41)
    x = torch.randn((n, h, w, C), generator=g).to(cuda).bfloat16()
    wt = (torch.randint(-7, 8, (c_out, C, 3, 3), generator=g).float() / 64).to(cuda)
    kw, bcol, brow, res, rs, act = _inputs(form, rows, c_out, c_out, cuda, 42)
    wp = weights.pack_conv_up2x(wt, [C]) if up else weights.pack_conv(wt, [C])

    def call(out, resid, plan=False):
        o4 = out.view(n, ho, wo, out.shape[1])[..., :c_out]
        r4 = None if resid is None else resid.view(n, ho, wo, c_out)
        return (ops.conv_plan if plan else ops.conv2d)([x], wp, c_out, ksize=3, out=o4, residual=r4, force_bn=160, split_k=False, up2x=up,
                                                       **kw)

    y = _run_both(call, form, rows, c_out, res, cuda, lambda plan, staged: None)
    xd = x.double().permute(0, 3, 1, 2)
    if up:
        xd = F.interpolate(xd, scale_factor=2, mode="nearest")
    acc = F.conv2d(xd, wt.double(), padding=1).permute(0, 2, 3, 1).reshape(rows, c_out)
    m = F.conv2d(xd.abs(), wt.double().abs(), padding=1).permute(0, 2, 3, 1).reshape(rows, c_out)
    _check(y, acc, m, 9 * C, bcol, brow, res, rs, act)


# ================================================================================================================ CPU: where 160 is planned
FIELDS = "k s p up n h w hin win cout nsrc c0 p0 c1 p1 nsc sc0c sc0p sc1c sc1p K wp bpr bss act op f32".split()


def _traced_plans(module, batch, h, w):
    """(trace fields, plan at SMS SMs) of every conv record of one module run, on fake 256-byte aligned addresses that keep the trace's
    null pointers null and its in-place residuals in place."""
    from ladi_vton_b200 import AutoencoderKL, UNet2DConditionModel, engine as eng, synthetic as S, unet_param_shapes
    from ladi_vton_b200.vae import vae_param_shapes
    model, shapes = (UNet2DConditionModel(), unet_param_shapes({})) if module == eng.MODULE_UNET else (AutoencoderKL(), vae_param_shapes({}))
    model._sd = S.random_state_dict(shapes, 1, fast=True)
    model.device = torch.device("cpu")
    model._pack()
    model._sd = None
    e = eng.Engine(eng.flatten(model.P), plan_only=True, **model.engine_config())
    lib = ladi_lib()
    out = []
    for line in e.trace(module, batch, h, w).splitlines():
        if not line.startswith("conv "):
            continue
        kv = dict(re.findall(r"(\w+)=@?([0-9a-fx]+)", line))
        f = {k: int(kv[k]) for k in FIELDS}
        a = {k: int(kv[k], 16) for k in ("bias", "step", "res", "rs", "out")}
        fake = lambda i: (1 << 40) + (i << 32)
        d = lib.ConvDesc()
        d.n, d.h_out, d.w_out, d.c_out, d.h_in, d.w_in = f["n"], f["h"], f["w"], f["cout"], f["hin"], f["win"]
        d.ksize, d.stride, d.pad_lo, d.up2x = f["k"], f["s"], f["p"], f["up"]
        d.n_src, d.src[0], d.src_c[0], d.src_pitch[0] = f["nsrc"], fake(1), f["c0"], f["p0"]
        if f["nsrc"] > 1:
            d.src[1], d.src_c[1], d.src_pitch[1] = fake(2), f["c1"], f["p1"]
        d.n_sc = f["nsc"]
        for i in range(f["nsc"]):
            d.sc[i], d.sc_c[i], d.sc_pitch[i] = fake(3 + i), f[f"sc{i}c"], f[f"sc{i}p"]
        d.weight, d.k_total, d.weight_pitch = fake(5), f["K"], f["wp"]
        if a["bias"]:
            d.bias, d.bias_per_row, d.bias_step_stride = fake(6), f["bpr"], f["bss"]
        if a["step"]:
            d.step_ptr = fake(7)
        d.out, d.out_pitch, d.out_fp32, d.act = fake(8), f["op"], f["f32"], f["act"]
        if a["res"]:
            d.residual, d.residual_pitch = (fake(8) if a["res"] == a["out"] else fake(9)), f["op"]
        if a["rs"]:
            d.row_scale = fake(10)
        d.splitk_ws, d.splitk_ws_bytes = fake(11), 64 << 20
        out.append((f, lib.conv_plan(d, SMS)))
    return out


def _old_rule_bn(tiles_m, total_kb, c_out):
    """The N tile before 160 was a candidate: min(ceil(tiles / SMs) * (BN + 64)) over 128 / 64 / 32, 128 for short reductions."""
    best, bn = None, 0
    for c in (128, 64, 32):
        if total_kb <= 8 and c_out >= 128 and c < 128:
            continue
        cost = -(-tiles_m * -(-c_out // c) // SMS) * (c + 64)
        if best is None or cost < best:
            best, bn = cost, c
    return bn


def test_plan_160_where_the_rule_says():
    """UNet step at 512x384, batch 8 with CFG (UNet batch 16, 64x48 latents), and the VAE encode / decode at the same size."""
    from ladi_vton_b200 import engine as eng
    moved = 0
    for module, b, h, w in ((eng.MODULE_UNET, 16, 64, 48), (eng.MODULE_VAE_ENCODE, 8, 512, 384), (eng.MODULE_VAE_DECODE, 8, 64, 48)):
        for f, p in _traced_plans(module, b, h, w):
            desc = f"module {module} conv {f}"
            if p.splits > 1:
                assert p.bn != 160, desc
                continue
            old = _old_rule_bn(p.tiles_m, p.total_kb, f["cout"])
            if p.total_kb <= 8:  # short reductions keep their plan: 128 for c_out >= 128
                assert (p.bn, p.staged) == (old, 1 if f["op"] % 8 == 0 and f["cout"] % 8 == 0 and not f["f32"] else p.staged), desc
                assert p.bn != 160, desc
                continue
            if module != eng.MODULE_UNET:
                assert p.bn == old, desc  # the VAE keeps its tiles
                continue
            if p.bn == 160:
                moved += 1
                assert p.staged == 1 and p.stages == 5 and f["cout"] >= 160 and not f["f32"], desc
            else:
                assert p.bn == old, desc
    assert moved > 0
