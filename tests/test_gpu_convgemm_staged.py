"""The two store paths of the conv/GEMM epilogue agree bit for bit, and the staged one is right against float64.

A bf16 output whose rows are whole, 16-byte aligned chunks (c_out, out_pitch and residual_pitch multiples of 8) leaves the kernel
through a shared-memory staging tile and 16-byte stores; any other output is stored from the accumulator fragment.  Each case here runs
once with a NaN-padded output pitch that is a multiple of 8 (staged) and once with a pitch of c + 4 (fragment), on the same data:
- the staged output is checked against float64 with the census's per-element bound (conv_expect), and its pitch gap must still be NaN;
- the two outputs must be bitwise equal (same arithmetic, same order, one rounding to bf16).
The cases cover every epilogue form, N tiles 32 / 64 / 128, M not a multiple of 128, c_out not a multiple of the N tile, convolution
tiles spanning several rows and images (8x6 and 16x12 latents at batch 16) and the fused nearest-2x upsample."""
import pytest
import torch
import torch.nn.functional as F

from kernel_check import conv_expect, cpu_gen, max_ratio, nan_buf, same

pytestmark = pytest.mark.gpu

FORMS = ["bias", "nobias", "stepbias", "rowbias", "silu", "gelu", "relu", "geglu", "residual", "inplace", "rowscale", "silu_res_rowscale"]


def _inputs(form, rows, c_out, c_eff, dev, seed):
    """Epilogue operands of one form: (ops kwargs, float64 column / row bias, residual bf16 [rows, c_eff] or None, row scale, act)."""
    from ladi_vton_b200 import ops
    g = cpu_gen(seed)
    act = {"silu": ops.ACT_SILU, "gelu": ops.ACT_GELU, "relu": ops.ACT_RELU, "geglu": ops.ACT_GEGLU,
           "silu_res_rowscale": ops.ACT_SILU}.get(form, ops.ACT_NONE)
    kw, bcol, brow, res, rs = {"act": act}, None, None, None, None
    if form == "stepbias":
        steps = 3
        table = torch.randn((steps, c_out), generator=g).to(dev)
        kw.update(bias=table, bias_step_stride=c_out, step_ptr=torch.tensor([2], dtype=torch.int32, device=dev))
        bcol = table[2].double()
    elif form == "rowbias":
        brow = torch.randn((rows,), generator=g).to(dev)
        kw.update(bias=brow, bias_per_row=True)
        brow = brow.double()
    elif form != "nobias":
        bcol = torch.randn((c_out,), generator=g).to(dev)
        kw.update(bias=bcol)
        bcol = bcol.double()
    if form in ("residual", "inplace", "silu_res_rowscale"):
        res = torch.randn((rows, c_eff), generator=g).to(dev).bfloat16()
    if form in ("rowscale", "silu_res_rowscale"):
        rs = torch.rand((rows,), generator=g).to(dev)
        kw.update(row_scale=rs)
        rs = rs.double()
    return kw, bcol, brow, res, rs, act


def _run_both(call, form, rows, c_eff, res, dev):
    """call(out [rows, pitch] view, residual view or None, plan=False) for a staged pitch (c_eff + 8) and a fragment pitch (c_eff + 4);
    call(..., plan=True) returns the plan (ladi_conv2d_plan) of the same call, which must be the staged one and the fragment one."""
    outs = []
    for pitch, staged in ((c_eff + 8, 1), (c_eff + 4, 0)):
        if form == "inplace":
            buf = nan_buf((rows, pitch), torch.bfloat16, dev, res)
            rbuf = buf[:, :c_eff]
        else:
            buf = nan_buf((rows, pitch), torch.bfloat16, dev)
            rbuf = None if res is None else nan_buf((rows, pitch), torch.bfloat16, dev, res)[:, :c_eff]
        plan = call(buf, rbuf, plan=True)
        assert (plan.staged, plan.splits, plan.pair) == (staged, 1, 0), f"pitch {pitch}: staged {plan.staged}, want {staged}"
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


@pytest.mark.parametrize("bn", [0, 32, 64, 128])
@pytest.mark.parametrize("form", FORMS)
def test_staged_gemm(cuda, form, bn):
    """M = 1000 (a partial last M tile); c_out 320 (not a multiple of 128; 640 interleaved columns for GEGLU)."""
    from ladi_vton_b200 import ops, weights
    M, K = 1000, 320
    c_out = 640 if form == "geglu" else 320
    c_eff = c_out // 2 if form == "geglu" else c_out
    g = cpu_gen(11)
    a = torch.randn((M, K), generator=g).to(cuda).bfloat16()
    w = (torch.randn((c_out, K), generator=g) * K ** -0.5).to(cuda).bfloat16()
    kw, bcol, brow, res, rs, act = _inputs(form, M, c_out, c_eff, cuda, 12)
    wp = weights.pack_linear(w.float())

    def call(out, resid, plan=False):
        return (ops.gemm_plan if plan else ops.gemm)(a, wp, c_out, out=out[:, :c_eff], residual=resid, force_bn=bn, split_k=False, **kw)

    y = _run_both(call, form, M, c_eff, res, cuda)
    acc = a.double() @ w.double().t()
    m = a.double().abs() @ w.double().abs().t()
    _check(y, acc, m, K, bcol, brow, res, rs, act)


@pytest.mark.parametrize("shape", ["8x6", "16x12", "up2x 8x6"])
@pytest.mark.parametrize("form", ["bias", "rowbias", "silu", "residual", "inplace", "rowscale"])
def test_staged_conv(cuda, form, shape):
    """3x3 convolutions at batch 16 on the small UNet latents (M tiles of several rows and images), c_out 320 at the 128-wide tile,
    and the fused nearest-2x upsample (parity-strided output rows).  Weights are multiples of 1/64 below 1/8 in magnitude, so the
    upsample's merged taps are exact in bf16 and the float64 reference is the plain convolution of the upsampled input."""
    from ladi_vton_b200 import ops, weights
    up = shape.startswith("up2x")
    if up and form not in ("bias", "silu"):
        pytest.skip("up2x takes a per-channel bias and an activation only")
    n, C, c_out = 16, 64, 320
    h, w = (8, 6) if shape.endswith("8x6") else (16, 12)
    ho, wo = (2 * h, 2 * w) if up else (h, w)
    rows = n * ho * wo
    g = cpu_gen(21)
    x = torch.randn((n, h, w, C), generator=g).to(cuda).bfloat16()
    wt = (torch.randint(-7, 8, (c_out, C, 3, 3), generator=g).float() / 64).to(cuda)
    kw, bcol, brow, res, rs, act = _inputs(form, rows, c_out, c_out, cuda, 22)
    wp = weights.pack_conv_up2x(wt, [C]) if up else weights.pack_conv(wt, [C])

    def call(out, resid, plan=False):
        o4 = out.view(n, ho, wo, out.shape[1])[..., :c_out]
        r4 = None if resid is None else resid.view(n, ho, wo, c_out)
        return (ops.conv_plan if plan else ops.conv2d)([x], wp, c_out, ksize=3, out=o4, residual=r4, force_bn=128, split_k=False, up2x=up,
                                                       **kw)

    y = _run_both(call, form, rows, c_out, res, cuda)
    xd = x.double().permute(0, 3, 1, 2)
    if up:
        xd = F.interpolate(xd, scale_factor=2, mode="nearest")
    acc = F.conv2d(xd, wt.double(), padding=1).permute(0, 2, 3, 1).reshape(rows, c_out)
    m = F.conv2d(xd.abs(), wt.double().abs(), padding=1).permute(0, 2, 3, 1).reshape(rows, c_out)
    _check(y, acc, m, 9 * C, bcol, brow, res, rs, act)
