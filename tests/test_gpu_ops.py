"""GPU parity of each hand-written kernel (through the C ABI) against a plain PyTorch fp32 computation of the same op on
the same bf16-rounded inputs.  Tolerances: outputs are bf16 (relative rounding 2^-9 = 0.2%) of fp32 accumulations, so the
normalised max error |y - ref|_inf / |ref|_inf must be < 1e-2 (bf16 out) / 2e-3 (fp32 out)."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

TOL_BF16, TOL_F32 = 1e-2, 2e-3


def nerr(y, ref):
    return ((y.float() - ref.float()).abs().max() / ref.float().abs().max().clamp_min(1e-6)).item()


def rnd(shape, dev, seed, scale=1.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(dev)


# ------------------------------------------------------------------------------------------------ GEMM
@pytest.mark.parametrize("M,K,N,bn", [(512, 320, 320, 0), (200, 64, 96, 0), (384, 1024, 640, 0), (128, 128, 4, 0),
                                      (256, 256, 256, 32), (256, 256, 256, 64), (256, 256, 256, 128), (256, 256, 320, 160),
                                      (256, 256, 384, 192), (256, 256, 512, 256), (3072, 320, 960, 0), (77 * 2, 1024, 640, 0)])
@pytest.mark.parametrize("direct", [False, True])
def test_gemm_plain(cuda, M, K, N, bn, direct):
    """direct=True: force_direct_epilogue is accepted and ignored (the library picks the store path, staged or fragment, from the rest of
    the descriptor), so it must leave the output bit-identical."""
    from ladi_vton_b200 import ops, weights
    a = rnd((M, K), cuda, 1).bfloat16()
    w = rnd((N, K), cuda, 2, K ** -0.5)
    b = rnd((N,), cuda, 3)
    y = ops.gemm(a, weights.pack_linear(w), N, bias=b, force_bn=bn, direct_epilogue=direct)
    torch.cuda.synchronize()
    assert y.shape == (M, N)
    if direct:
        assert torch.equal(y, ops.gemm(a, weights.pack_linear(w), N, bias=b, force_bn=bn))
        return
    ref = a.float() @ w.bfloat16().float().t() + b
    assert nerr(y, ref) < TOL_BF16


@pytest.mark.parametrize("bn", [0, 160, 256])
@pytest.mark.parametrize("mode", ["residual", "silu", "geglu", "fp32", "rowscale", "rowbias", "stepbias", "strided"])
def test_gemm_epilogues(cuda, mode, bn):
    from ladi_vton_b200 import ops, weights
    M, K, N = 300, 320, 640
    if mode == "geglu" and bn == 160:
        bn = 128
    a = rnd((M, K), cuda, 1).bfloat16()
    w = rnd((N, K), cuda, 2, K ** -0.5)
    b = rnd((N,), cuda, 3)
    wb = w.bfloat16().float()
    base = a.float() @ wb.t() + b
    if mode == "residual":
        r = rnd((M, N), cuda, 4).bfloat16()
        y = ops.gemm(a, weights.pack_linear(w), N, bias=b, residual=r, force_bn=bn)
        ref = base + r.float()
    elif mode == "silu":
        y = ops.gemm(a, weights.pack_linear(w), N, bias=b, act=ops.ACT_SILU, force_bn=bn)
        ref = F.silu(base)
    elif mode == "geglu":
        wi, bi = weights.interleave_geglu(w, b)
        y = ops.gemm(a, weights.pack_linear(wi), N, bias=bi.contiguous(), act=ops.ACT_GEGLU, force_bn=bn)
        v, g = base.chunk(2, dim=-1)
        ref = v * F.gelu(g)
        assert y.shape == (M, N // 2)
    elif mode == "fp32":
        y = ops.gemm(a, weights.pack_linear(w), N, bias=b, out_fp32=True, force_bn=bn)
        ref = base
        assert y.dtype == torch.float32
        torch.cuda.synchronize()
        assert nerr(y, ref) < TOL_F32
    elif mode == "rowscale":
        rs = torch.rand(M, device=cuda)
        y = ops.gemm(a, weights.pack_linear(w), N, bias=b, row_scale=rs, force_bn=bn)
        ref = base * rs[:, None]
    elif mode == "rowbias":
        rb = rnd((M,), cuda, 5)
        y = ops.gemm(a, weights.pack_linear(w), N, bias=rb, bias_per_row=True, force_bn=bn)
        ref = a.float() @ wb.t() + rb[:, None]
    elif mode == "stepbias":
        tab = rnd((5, N), cuda, 6)
        step = torch.tensor([3, 0], dtype=torch.int32, device=cuda)
        y = ops.gemm(a, weights.pack_linear(w), N, bias=tab, bias_step_stride=N, step_ptr=step, force_bn=bn)
        ref = a.float() @ wb.t() + tab[3]
    else:  # strided A (a column slice of a wider buffer) and strided weight rows
        big = rnd((M, 3 * K), cuda, 7).bfloat16()
        a2 = big[:, K:2 * K]
        wbig = weights.pack_linear(rnd((N, 2 * K), cuda, 8, K ** -0.5))
        y = ops.gemm(a2, wbig[:, :K], N, bias=b, force_bn=bn)
        ref = a2.float() @ wbig[:, :K].float().t() + b
    torch.cuda.synchronize()
    assert nerr(y, ref) < TOL_BF16


# ------------------------------------------------------------------------------------------------ conv
def conv_ref(xs, w, b, stride=1, pad=1, asym=False):
    x = torch.cat([t.float().permute(0, 3, 1, 2) for t in xs], dim=1)
    if asym:
        x = F.pad(x, (0, 1, 0, 1))
        pad = 0
    y = F.conv2d(x, w.bfloat16().float(), b, stride=stride, padding=pad)
    return y.permute(0, 2, 3, 1)


@pytest.mark.parametrize("n,h,w,cin,cout", [(2, 16, 12, 64, 128), (2, 64, 48, 320, 320), (3, 8, 6, 128, 192), (2, 32, 24, 192, 640),
                                            (1, 128, 96, 64, 64), (5, 8, 6, 64, 64), (2, 16, 12, 1280, 1280)])
def test_conv3x3(cuda, n, h, w, cin, cout):
    from ladi_vton_b200 import ops, weights
    x = rnd((n, h, w, cin), cuda, 1).bfloat16()
    wt = rnd((cout, cin, 3, 3), cuda, 2, (9 * cin) ** -0.5)
    b = rnd((cout,), cuda, 3)
    y = ops.conv2d([x], weights.pack_conv(wt, [cin]), cout, bias=b)
    ref = conv_ref([x], wt, b)
    torch.cuda.synchronize()
    assert nerr(y, ref) < TOL_BF16


def test_conv3x3_residual_rowscale_silu(cuda):
    """ResnetBlock2D conv2 (+x) and EMASC conv (SiLU, (1-mask) row scale) on ragged tile geometry (24x20, batch 3)."""
    from ladi_vton_b200 import ops, weights
    n, h, w, c = 3, 24, 20, 192
    x = rnd((n, h, w, c), cuda, 1).bfloat16()
    res = rnd((n, h, w, c), cuda, 2).bfloat16()
    wt = rnd((c, c, 3, 3), cuda, 3, (9 * c) ** -0.5)
    b = rnd((c,), cuda, 4)
    rs = torch.rand(n * h * w, device=cuda)
    ref = conv_ref([x], wt, b)
    for direct in (False, True):
        y = ops.conv2d([x], weights.pack_conv(wt, [c]), c, bias=b, residual=res, direct_epilogue=direct)
        torch.cuda.synchronize()
        assert nerr(y, ref + res.float()) < TOL_BF16
        y = ops.conv2d([x], weights.pack_conv(wt, [c]), c, bias=b, act=ops.ACT_SILU, row_scale=rs, direct_epilogue=direct)
        torch.cuda.synchronize()
        assert nerr(y, F.silu(ref) * rs.view(n, h, w, 1)) < TOL_BF16


@pytest.mark.parametrize("mode", ["plain", "residual", "silu", "stepbias"])
def test_conv3x3_split_k(cuda, mode):
    """8x6 UNet level (768 output rows, K = 11520): few tiles, long reduction -> split-K partial planes + deterministic reduce."""
    from ladi_vton_b200 import ops, weights
    n, h, w, c = 16, 8, 6, 1280
    x = rnd((n, h, w, c), cuda, 1).bfloat16()
    wt = rnd((c, c, 3, 3), cuda, 2, (9 * c) ** -0.5)
    b = rnd((c,), cuda, 3)
    ref = conv_ref([x], wt, b)
    kw = {}
    if mode == "residual":
        res = rnd((n, h, w, c), cuda, 4).bfloat16()
        kw["residual"] = res
        ref = ref + res.float()
    elif mode == "silu":
        kw["act"] = ops.ACT_SILU
        ref = F.silu(ref)
    packed = weights.pack_conv(wt, [c])
    if mode == "stepbias":
        tab = rnd((3, c), cuda, 5)
        step = torch.tensor([2, 0], dtype=torch.int32, device=cuda)
        y = ops.conv2d([x], packed, c, bias=tab, bias_step_stride=c, step_ptr=step)
        y0 = ops.conv2d([x], packed, c, bias=tab, bias_step_stride=c, step_ptr=step, split_k=False)
        ref = conv_ref([x], wt, tab[2])
    else:
        y = ops.conv2d([x], packed, c, bias=b, **kw)
        y0 = ops.conv2d([x], packed, c, bias=b, split_k=False, **kw)
    torch.cuda.synchronize()
    assert nerr(y, ref) < TOL_BF16 and nerr(y0, ref) < TOL_BF16
    assert torch.equal(y, ops.conv2d([x], packed, c, bias=(tab if mode == "stepbias" else b),
                                     **({"bias_step_stride": c, "step_ptr": step} if mode == "stepbias" else kw)))  # deterministic


def test_conv3x3_concat_shortcut(cuda):
    """UNet up-block resnet conv2: 3x3 over h + fused 1x1 conv_shortcut over the (virtual) concat [x, skip]."""
    from ladi_vton_b200 import ops, weights
    n, h, w, c0, c1, cm, cout = 2, 32, 24, 128, 64, 128, 128
    hmid = rnd((n, h, w, cm), cuda, 1).bfloat16()
    x0 = rnd((n, h, w, c0), cuda, 2).bfloat16()
    x1 = rnd((n, h, w, c1), cuda, 3).bfloat16()
    wt = rnd((cout, cm, 3, 3), cuda, 4, (9 * cm) ** -0.5)
    ws = rnd((cout, c0 + c1, 1, 1), cuda, 5, (c0 + c1) ** -0.5)
    b = rnd((cout,), cuda, 6)
    y = ops.conv2d([hmid], weights.pack_conv(wt, [cm], ws, [c0, c1]), cout, bias=b, shortcut=[x0, x1])
    ref = conv_ref([hmid], wt, b) + conv_ref([x0, x1], ws, None, pad=0)
    torch.cuda.synchronize()
    assert nerr(y, ref) < TOL_BF16
    # two-source 3x3 (concat never materialised)
    wt2 = rnd((cout, c0 + c1, 3, 3), cuda, 7, (9 * (c0 + c1)) ** -0.5)
    y2 = ops.conv2d([x0, x1], weights.pack_conv(wt2, [c0, c1]), cout, bias=b)
    torch.cuda.synchronize()
    assert nerr(y2, conv_ref([x0, x1], wt2, b)) < TOL_BF16


@pytest.mark.parametrize("asym", [False, True])
def test_conv3x3_stride2(cuda, asym):
    from ladi_vton_b200 import ops, weights
    n, h, w, c = 2, 32, 24, 128
    x = rnd((n, h, w, c), cuda, 1).bfloat16()
    wt = rnd((c, c, 3, 3), cuda, 2, (9 * c) ** -0.5)
    b = rnd((c,), cuda, 3)
    y = ops.conv2d([x], weights.pack_conv(wt, [c]), c, bias=b, stride=2, pad_lo=0 if asym else 1)
    ref = conv_ref([x], wt, b, stride=2, asym=asym)
    torch.cuda.synchronize()
    assert y.shape == ref.shape
    assert nerr(y, ref) < TOL_BF16


@pytest.mark.parametrize("cin,pitch,cout", [(31, 32, 320), (3, 8, 128), (4, 8, 512), (128, 128, 3), (320, 320, 4), (512, 512, 8)])
def test_conv3x3_odd_channels(cuda, cin, pitch, cout):
    """conv_in / conv_out shapes: channel counts that are not multiples of 64 ride on TMA zero fill + zero-padded weights."""
    from ladi_vton_b200 import ops, weights
    n, h, w = 2, 16, 24
    buf = torch.zeros((n, h, w, pitch), dtype=torch.bfloat16, device=cuda)
    buf[..., :cin] = rnd((n, h, w, cin), cuda, 1).bfloat16()
    buf[..., cin:] = 7.0  # garbage beyond C must never be read as data
    x = buf[..., :cin]
    wt = rnd((cout, cin, 3, 3), cuda, 2, (9 * cin) ** -0.5)
    b = rnd((cout,), cuda, 3)
    opitch = (cout + 7) // 8 * 8
    out = torch.zeros((n, h, w, opitch), dtype=torch.float32, device=cuda)
    y = ops.conv2d([x], weights.pack_conv(wt, [cin]), cout, bias=b, out=out, out_fp32=True)[..., :cout]
    ref = conv_ref([x], wt, b)
    torch.cuda.synchronize()
    assert nerr(y, ref) < TOL_F32 * 2


def test_conv_invalid_args_error(cuda):
    from ladi_vton_b200 import ops, weights
    x = torch.zeros((1, 8, 8, 64), dtype=torch.bfloat16, device=cuda)
    w = weights.pack_conv(torch.zeros(64, 64, 3, 3), [64]).to(cuda)
    with pytest.raises(RuntimeError, match="weight K"):
        ops.conv2d([x], w[:, :64].contiguous(), 64)


# ------------------------------------------------------------------------------------------------ attention
@pytest.mark.parametrize("B,heads,nq,nkv", [(2, 5, 768, 768), (1, 2, 128, 128), (2, 3, 192, 192), (3, 2, 48, 48), (2, 5, 768, 77),
                                            (1, 1, 3072, 3072), (2, 2, 200, 333), (2, 3, 384, 640), (16, 5, 3072, 77), (3, 20, 48, 77), (2, 1, 1000, 128)])
@pytest.mark.parametrize("variant", [0, 1, 2, 4, 5, 6, 8])
def test_attention(cuda, B, heads, nq, nkv, variant):
    """sm_90a runs one kernel for every accepted `variant` (include/ladi_b200.h): variant 0 is checked against the reference, every other
    variant must give bit-identical output, and variant 8 (a single K/V tile) must still reject nkv > 128."""
    from ladi_vton_b200 import ops
    C = heads * 64
    if nq == nkv:  # fused QKV buffer, per-head slices read in place
        qkv = rnd((B, nq, 3 * C), cuda, 1).bfloat16()
        q, k, v = qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:]
    else:
        q = rnd((B, nq, C), cuda, 1).bfloat16()
        kv = rnd((B, nkv, 2 * C), cuda, 2).bfloat16()
        k, v = kv[..., :C], kv[..., C:]
    if variant == 8 and nkv > 128:
        with pytest.raises(RuntimeError, match="bad attention variant 8"):
            ops.attention(q, k, v, heads, 0.125, variant=variant)
        return
    y = ops.attention(q, k, v, heads, 0.125, variant=variant)
    if variant != 0:
        assert torch.equal(y, ops.attention(q, k, v, heads, 0.125))
        return
    sp = lambda t: t.float().reshape(B, -1, heads, 64).transpose(1, 2)
    ref = F.scaled_dot_product_attention(sp(q), sp(k), sp(v)).transpose(1, 2).reshape(B, nq, C)
    torch.cuda.synchronize()
    assert nerr(y, ref) < 2e-2


# ------------------------------------------------------------------------------------------------ norms & glue
@pytest.mark.parametrize("n,hw,c0,c1,groups,silu", [(2, 3072, 320, 0, 32, True), (2, 768, 1280, 640, 32, True), (3, 48, 2560, 0, 32, False),
                                                    (2, 196608, 128, 0, 32, True), (2, 192, 64, 64, 32, True)])
def test_groupnorm(cuda, n, hw, c0, c1, groups, silu):
    from ladi_vton_b200 import ops
    h, w = (hw // 48, 48) if hw % 48 == 0 else (hw, 1)
    x0 = (rnd((n, h, w, c0), cuda, 1) * 2 + 0.5).bfloat16()
    srcs = [x0]
    if c1:
        srcs.append((rnd((n, h, w, c1), cuda, 2) - 1.0).bfloat16())
    C = c0 + c1
    gamma, beta = rnd((C,), cuda, 3) + 1, rnd((C,), cuda, 4)
    ws = ops.GroupNormWS(cuda)
    y = ops.groupnorm(srcs, gamma, beta, groups, 1e-5, ws, silu=silu)
    xc = torch.cat([s.float() for s in srcs], dim=-1).permute(0, 3, 1, 2)
    ref = F.group_norm(xc, groups, gamma, beta, 1e-5)
    if silu:
        ref = F.silu(ref)
    ref = ref.permute(0, 2, 3, 1)
    torch.cuda.synchronize()
    assert nerr(y, ref) < TOL_BF16


@pytest.mark.parametrize("rows,C", [(3072, 320), (100, 640), (77, 1280), (9, 1024)])
def test_layernorm(cuda, rows, C):
    from ladi_vton_b200 import ops
    x = (rnd((rows, C), cuda, 1) * 3 + 1).bfloat16()
    g, b = rnd((C,), cuda, 2) + 1, rnd((C,), cuda, 3)
    y = ops.layernorm(x, g, b, 1e-5)
    ref = F.layer_norm(x.float(), (C,), g, b, 1e-5)
    torch.cuda.synchronize()
    assert nerr(y, ref) < TOL_BF16


def test_softmax_rows(cuda):
    from ladi_vton_b200 import ops
    s = rnd((300, 3072), cuda, 1, 20.0)
    y = ops.softmax_rows(s, 512 ** -0.5)
    ref = torch.softmax(s * 512 ** -0.5, dim=-1)
    torch.cuda.synchronize()
    assert nerr(y, ref) < TOL_BF16


def test_pointwise_glue(cuda):
    from ladi_vton_b200 import ops
    a, b = rnd((2, 8, 6, 64), cuda, 1).bfloat16(), rnd((2, 8, 6, 64), cuda, 2).bfloat16()
    assert nerr(ops.add(a, b), a.float() + b.float()) < TOL_BF16
    up = ops.upsample2x(a)
    assert torch.equal(up, a.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2))
    x = rnd((2, 18, 64, 48), cuda, 3).abs()
    assert torch.allclose(ops.bilinear_down8(x), F.interpolate(x, size=(8, 6), mode="bilinear"), atol=1e-6)
    m = (rnd((2, 1, 64, 48), cuda, 4) > 0).float()
    for f in (1, 2, 4, 8):
        assert torch.equal(ops.inv_mask_rows(m, f), 1 - F.interpolate(m, size=(64 // f, 48 // f))[:, 0])
    nchw = rnd((2, 5, 8, 6), cuda, 5)
    buf = torch.zeros((2, 8, 6, 16), dtype=torch.bfloat16, device=cuda)
    ops.nchw_to_nhwc(nchw, buf, c_off=3, scale=2.0)
    assert torch.equal(buf[..., 3:8], (nchw * 2).bfloat16().permute(0, 2, 3, 1))
    assert torch.equal(ops.nhwc_to_nchw(buf, 5, 3), buf[..., 3:8].float().permute(0, 3, 1, 2))
    mom = rnd((2, 8, 6, 8), cuda, 6)
    noise = rnd((2, 4, 8, 6), cuda, 7)
    z = ops.posterior_sample(mom, noise, 0.18215)
    mean, logvar = mom[..., :4].permute(0, 3, 1, 2), mom[..., 4:].permute(0, 3, 1, 2).clamp(-30, 20)
    assert torch.allclose(z, (mean + torch.exp(0.5 * logvar) * noise) * 0.18215, rtol=1e-5, atol=1e-6)
    img = rnd((2, 8, 6, 4), cuda, 8)
    assert torch.allclose(ops.image_out(img), (img[..., :3] / 2 + 0.5).clamp(0, 1), atol=1e-6)
    torch.cuda.synchronize()


@pytest.mark.parametrize("cfg", [False, True])
@pytest.mark.parametrize("eta", [False, True])
def test_ddim_cfg_step(cuda, cfg, eta):
    from ladi_vton_b200 import ops
    B, h, w, g = 2, 8, 6, 7.5
    Bp = 2 * B if cfg else B
    eps = torch.zeros((Bp, h, w, 4), dtype=torch.float32, device=cuda)
    eps[:] = rnd((Bp, h, w, 4), cuda, 1)
    lat = rnd((B, 4, h, w), cuda, 2)
    lat0 = lat.clone()
    uin = torch.zeros((Bp, h, w, 32), dtype=torch.bfloat16, device=cuda)
    coef = torch.tensor([[1.1, 0.3, 0.9, 0.2, 0.7, 0, 0, 0], [1.2, 0.4, 0.8, 0.1, 0.5, 0, 0, 0]], device=cuda)
    step = torch.tensor([1, 0], dtype=torch.int32, device=cuda)
    noise = rnd((B, 4, h, w), cuda, 3) if eta else None
    ops.ddim_cfg_step(eps, lat, uin, cfg, g, coef, step, noise=noise)
    e = eps.permute(0, 3, 1, 2)
    if cfg:
        e = e[:B] + g * (e[B:] - e[:B])
    ref = 0.8 * ((lat0 - 0.4 * e) * 1.2) + 0.1 * e
    if eta:
        ref = ref + 0.5 * noise  # DDIMScheduler.step: prev_sample += sigma_t * variance_noise
    torch.cuda.synchronize()
    assert torch.allclose(lat, ref, rtol=1e-5, atol=1e-5)
    assert step.tolist() == [2, 0]
    assert torch.equal(uin[:B, ..., :4], lat.bfloat16().permute(0, 2, 3, 1))
    if cfg:
        assert torch.equal(uin[B:, ..., :4], uin[:B, ..., :4])


def test_check_binarise(cuda):
    """prepare_mask_and_masked_image's range checks + in-place binarisation on the device (tryon_pipe.py:630), flags instead of syncs."""
    from ladi_vton_b200 import ops
    img = (torch.rand((2, 3, 40, 24), device=cuda) * 2 - 1).contiguous()
    mask = torch.rand((2, 1, 40, 24), device=cuda).contiguous()
    ref = (mask >= 0.5).float()
    flags = torch.zeros(2, dtype=torch.int32, device=cuda)
    ops.check_binarise_(img, mask, flags)
    assert flags.tolist() == [0, 0] and torch.equal(mask, ref)
    img[1, 2, 7, 3] = 1.5
    ops.check_binarise_(img, mask, flags)
    assert flags.tolist() == [1, 0]
    mask[0, 0, 0, 0] = -0.25
    flags.zero_()
    ops.check_binarise_(img * 0, mask, flags)
    assert flags.tolist() == [0, 1] and float(mask[0, 0, 0, 0]) == 0.0


# ------------------------------------------------------------------------------------------------ wide single-head attention (VAE mid block)
@pytest.mark.parametrize("D,B,nq,nkv", [(512, 2, 128, 128), (512, 1, 3072, 3072), (512, 2, 200, 200), (512, 1, 384, 1000), (256, 2, 128, 128),
                                        (256, 3, 640, 640), (512, 1, 12288, 12288)])
def test_attention_d512(cuda, D, B, nq, nkv):
    """One head of width 512 (src/models/vae.py:81-90: diffusers AttentionBlock, softmax(q k^T / sqrt(C)) v), flash-style, vs fp32 torch on
    the same bf16 inputs; q/k/v are column slices of one fused [B, N, 3D] projection buffer like the VAE passes them."""
    from ladi_vton_b200 import ops
    if nq == nkv:
        qkv = rnd((B, nq, 3 * D), cuda, 1).bfloat16()
        q, k, v = qkv[..., :D], qkv[..., D:2 * D], qkv[..., 2 * D:]
    else:
        q = rnd((B, nq, D), cuda, 1).bfloat16()
        kv = rnd((B, nkv, 2 * D), cuda, 2).bfloat16()
        k, v = kv[..., :D], kv[..., D:]
    k = (k.float() * 2.0).bfloat16()  # scores of std ~2 after the 1/sqrt(D) scale: a softmax that is not flat
    scale = D ** -0.5
    y = ops.attention_d512(q, k, v, scale)
    torch.cuda.synchronize()
    ref = torch.empty((B, nq, D), dtype=torch.float32, device=cuda)
    for b in range(B):
        for i in range(0, nq, 2048):  # chunked fp32 reference (12288^2 scores would be 600 MB at once)
            sl = slice(i, min(nq, i + 2048))
            ref[b, sl] = torch.softmax((q[b, sl].float() @ k[b].float().t()) * scale, dim=-1) @ v[b].float()
    assert y.shape == (B, nq, D)
    assert nerr(y, ref) < TOL_BF16


# ------------------------------------------------------------------------------------------------ fused nearest-2x upsample + conv3x3
@pytest.mark.parametrize("n,h,w,ci,co,pair", [(2, 8, 6, 64, 64, None), (2, 8, 6, 96, 160, None), (16, 8, 6, 128, 256, None), (8, 16, 12, 320, 320, True),
                                               (3, 4, 4, 64, 72, None), (2, 32, 24, 128, 128, None), (1, 64, 48, 256, 256, None)])
def test_conv_up2x(cuda, n, h, w, ci, co, pair):
    """Upsample2D (F.interpolate(scale_factor=2, nearest) + conv3x3) as one sub-pixel convolution over the half-resolution tensor."""
    from ladi_vton_b200 import ops, weights
    x = rnd((n, h, w, ci), cuda, 1).bfloat16()
    wt = rnd((co, ci, 3, 3), cuda, 2, (9 * ci) ** -0.5)
    b = rnd((co,), cuda, 3)
    y = ops.conv2d([x], weights.pack_conv_up2x(wt, [ci]), co, bias=b, up2x=True, pair=pair)
    torch.cuda.synchronize()
    assert y.shape == (n, 2 * h, 2 * w, co)
    up = F.interpolate(x.float().permute(0, 3, 1, 2), scale_factor=2, mode="nearest")
    ref = F.conv2d(up, wt.bfloat16().float(), b, padding=1).permute(0, 2, 3, 1)
    assert nerr(y, ref) < TOL_BF16
    # and equal (up to the rounding of the merged weights) to the materialised form on the same kernels
    y2 = ops.conv2d([ops.upsample2x(x)], weights.pack_conv(wt, [ci]), co, bias=b)
    assert nerr(y, y2) < TOL_BF16


# ------------------------------------------------------------------------------------------------ LayerNorm folded into the GEMMs around it
@pytest.mark.parametrize("M,C,N,bn", [(300, 320, 320, 0), (3072, 320, 960, 0), (768, 1280, 1280, 0), (200, 64, 192, 0), (512, 640, 640, 160), (512, 640, 640, 256)])
def test_gemm_rowstat_and_ln_fold(cuda, M, C, N, bn):
    """Producer: out = a W1^T + b1 + residual, plus per-(row, 32-column chunk) {sum, sum of squares} of what it stores.
    Consumer: LayerNorm(out) W2^T + b2 computed from the RAW `out` with W2 diag(gamma) and the rank-1 epilogue correction."""
    from ladi_vton_b200 import ops, weights
    a = rnd((M, C), cuda, 1).bfloat16()
    w1 = rnd((C, C), cuda, 2, C ** -0.5)
    b1 = rnd((C,), cuda, 3)
    res = (rnd((M, C), cuda, 4) * 2 + 0.7).bfloat16()  # non-zero row means: the correction term matters
    stats = torch.empty((M, C // 32, 2), dtype=torch.float32, device=cuda)
    t = ops.gemm(a, weights.pack_linear(w1), C, bias=b1, residual=res, rowstat=stats, force_bn=bn)
    torch.cuda.synchronize()
    tref = a.float() @ w1.bfloat16().float().t() + b1 + res.float()
    assert nerr(t, tref) < TOL_BF16
    ch = tref.view(M, C // 32, 32)
    assert torch.allclose(stats[..., 0], ch.sum(-1), rtol=2e-3, atol=2e-2)
    assert torch.allclose(stats[..., 1], (ch * ch).sum(-1), rtol=2e-3, atol=2e-2)
    gamma, beta = torch.rand(C, device=cuda) + 0.5, rnd((C,), cuda, 5)
    w2 = rnd((N, C), cuda, 6, C ** -0.5)
    b2 = rnd((N,), cuda, 7)
    wp, cs, bp = weights.fold_layernorm(w2, gamma, beta, b2)
    y = ops.gemm(t, wp, N, bias=bp, ln=(stats, cs, 1e-5), force_bn=bn)
    torch.cuda.synchronize()
    ref = F.layer_norm(t.float(), (C,), gamma, beta, 1e-5) @ w2.float().t() + b2
    assert nerr(y, ref) < 1.5 * TOL_BF16
    # ... and it agrees with the stand-alone LayerNorm kernel followed by the plain GEMM
    y2 = ops.gemm(ops.layernorm(t, gamma, beta), weights.pack_linear(w2), N, bias=b2, force_bn=bn)
    assert nerr(y, y2) < 1.5 * TOL_BF16


def test_gemm_ln_fold_geglu(cuda):
    from ladi_vton_b200 import ops, weights
    M, C = 384, 320
    a = rnd((M, C), cuda, 1).bfloat16()
    w1 = rnd((C, C), cuda, 2, C ** -0.5)
    stats = torch.empty((M, C // 32, 2), dtype=torch.float32, device=cuda)
    t = ops.gemm(a, weights.pack_linear(w1), C, rowstat=stats)
    gamma, beta = torch.rand(C, device=cuda) + 0.5, rnd((C,), cuda, 5)
    w2 = rnd((8 * C, C), cuda, 6, C ** -0.5)
    b2 = rnd((8 * C,), cuda, 7)
    wi, bi = weights.interleave_geglu(w2, b2)
    wp, cs, bp = weights.fold_layernorm(wi, gamma, beta, bi)
    y = ops.gemm(t, wp, 8 * C, bias=bp, act=ops.ACT_GEGLU, ln=(stats, cs, 1e-5))
    torch.cuda.synchronize()
    h = F.layer_norm(t.float(), (C,), gamma, beta, 1e-5) @ w2.float().t() + b2
    v, g = h.chunk(2, dim=-1)
    assert y.shape == (M, 4 * C)
    assert nerr(y, v * F.gelu(g)) < 1.5 * TOL_BF16


# ------------------------------------------------------------------------------------------------ CTA pairs (2-CTA clusters, B tile shared by TMA multicast)
@pytest.mark.parametrize("M,K,N,bn", [(512, 320, 320, 160), (640, 256, 512, 256), (384, 1024, 640, 128), (300, 320, 640, 192),
                                      (3072 * 4, 320, 960, 0), (128 * 5, 128, 256, 256), (128 * 149, 64, 320, 160)])
@pytest.mark.parametrize("direct", [False, True])
def test_gemm_pair(cuda, M, K, N, bn, direct):
    """Same GEMMs through the CTA-pair kernel (M = 256 MMAs across two SMs, each staging half of B): odd numbers of M tiles (phantom
    tile of the last pair), ragged M (300 rows), N tiles that overhang c_out, more pairs than clusters (persistent loop)."""
    from ladi_vton_b200 import ops, weights
    a = rnd((M, K), cuda, 1).bfloat16()
    w = rnd((N, K), cuda, 2, K ** -0.5)
    b = rnd((N,), cuda, 3)
    y = ops.gemm(a, weights.pack_linear(w), N, bias=b, force_bn=bn, direct_epilogue=direct, pair=True, split_k=False)
    torch.cuda.synchronize()
    if direct:  # the ignored flag changes nothing on the pair kernel either
        assert torch.equal(y, ops.gemm(a, weights.pack_linear(w), N, bias=b, force_bn=bn, pair=True, split_k=False))
        return
    y1 = ops.gemm(a, weights.pack_linear(w), N, bias=b, force_bn=bn, pair=False, split_k=False)
    ref = a.float() @ w.bfloat16().float().t() + b
    torch.cuda.synchronize()
    assert nerr(y, ref) < TOL_BF16
    assert torch.equal(y, y1)  # same products in the same order: the pair kernel is bit-identical to the single-CTA kernel


@pytest.mark.parametrize("mode", ["residual", "silu", "geglu", "fp32", "rowscale", "stepbias"])
def test_gemm_pair_epilogues(cuda, mode):
    from ladi_vton_b200 import ops, weights
    M, K, N = 128 * 7 + 40, 320, 640
    a = rnd((M, K), cuda, 1).bfloat16()
    w = rnd((N, K), cuda, 2, K ** -0.5)
    b = rnd((N,), cuda, 3)
    base = a.float() @ w.bfloat16().float().t() + b
    kw = dict(pair=True, split_k=False, force_bn=128 if mode == "geglu" else 160)
    if mode == "residual":
        r = rnd((M, N), cuda, 4).bfloat16()
        y, ref = ops.gemm(a, weights.pack_linear(w), N, bias=b, residual=r, **kw), base + r.float()
    elif mode == "silu":
        y, ref = ops.gemm(a, weights.pack_linear(w), N, bias=b, act=ops.ACT_SILU, **kw), F.silu(base)
    elif mode == "geglu":
        wi, bi = weights.interleave_geglu(w, b)
        y = ops.gemm(a, weights.pack_linear(wi), N, bias=bi.contiguous(), act=ops.ACT_GEGLU, **kw)
        v, g = base.chunk(2, dim=-1)
        ref = v * F.gelu(g)
    elif mode == "fp32":
        y, ref = ops.gemm(a, weights.pack_linear(w), N, bias=b, out_fp32=True, **kw), base
    elif mode == "rowscale":
        rs = torch.rand(M, device=cuda)
        y, ref = ops.gemm(a, weights.pack_linear(w), N, bias=b, row_scale=rs, **kw), base * rs[:, None]
    else:
        tab = rnd((5, N), cuda, 6)
        step = torch.tensor([3, 0], dtype=torch.int32, device=cuda)
        y = ops.gemm(a, weights.pack_linear(w), N, bias=tab, bias_step_stride=N, step_ptr=step, **kw)
        ref = a.float() @ w.bfloat16().float().t() + tab[3]
    torch.cuda.synchronize()
    assert nerr(y, ref) < (TOL_F32 if mode == "fp32" else TOL_BF16)


@pytest.mark.parametrize("n,h,w,cin,cout,bn", [(2, 64, 48, 320, 320, 0), (2, 32, 24, 192, 640, 128), (1, 128, 96, 64, 128, 128),
                                               (3, 24, 20, 192, 192, 192), (16, 32, 24, 640, 640, 0)])
def test_conv3x3_pair(cuda, n, h, w, cin, cout, bn):
    from ladi_vton_b200 import ops, weights
    x = rnd((n, h, w, cin), cuda, 1).bfloat16()
    res = rnd((n, h, w, cout), cuda, 5).bfloat16()
    wt = rnd((cout, cin, 3, 3), cuda, 2, (9 * cin) ** -0.5)
    b = rnd((cout,), cuda, 3)
    wp = weights.pack_conv(wt, [cin])
    y = ops.conv2d([x], wp, cout, bias=b, residual=res, pair=True, split_k=False, force_bn=bn)
    y1 = ops.conv2d([x], wp, cout, bias=b, residual=res, pair=False, split_k=False, force_bn=bn)
    ref = conv_ref([x], wt, b) + res.float()
    torch.cuda.synchronize()
    assert nerr(y, ref) < TOL_BF16
    assert torch.equal(y, y1)


def test_conv_pair_concat_shortcut_stride2(cuda):
    """UNet up-block conv1 (two concatenated sources + fused 1x1 shortcut) and a stride-2 downsample through the pair kernel."""
    from ladi_vton_b200 import ops, weights
    n, h, w, c1, c2, cout = 2, 32, 24, 128, 64, 256
    x1, x2 = rnd((n, h, w, c1), cuda, 1).bfloat16(), rnd((n, h, w, c2), cuda, 2).bfloat16()
    wt = rnd((cout, c1 + c2, 3, 3), cuda, 3, (9 * (c1 + c2)) ** -0.5)
    b = rnd((cout,), cuda, 4)
    y = ops.conv2d([x1, x2], weights.pack_conv(wt, [c1, c2]), cout, bias=b, pair=True, split_k=False, force_bn=128)
    torch.cuda.synchronize()
    assert nerr(y, conv_ref([x1, x2], wt, b)) < TOL_BF16
    ws = rnd((cout, c1, 3, 3), cuda, 5, (9 * c1) ** -0.5)
    y = ops.conv2d([x1], weights.pack_conv(ws, [c1]), cout, bias=b, stride=2, pair=True, split_k=False, force_bn=128)
    torch.cuda.synchronize()
    assert nerr(y, conv_ref([x1], ws, b, stride=2)) < TOL_BF16


def test_pair_mode_errors(cuda):
    from ladi_vton_b200 import ops, weights
    a = rnd((100, 64), cuda, 1).bfloat16()  # one M tile: nothing to pair
    w = weights.pack_linear(rnd((128, 64), cuda, 2))
    with pytest.raises(RuntimeError, match="pair_mode=1"):
        ops.gemm(a, w, 128, force_bn=128, pair=True)


def test_timestep_embedding(cuda):
    """diffusers get_timestep_embedding (flip_sin_to_cos=True, downscale_freq_shift=0) as a (hi, lo) pair of bf16 column blocks."""
    import ctypes as C
    import math
    from ladi_vton_b200 import lib
    c0, kp = 320, 320
    t = torch.tensor([981.0, 501.0, 21.0, 1.0], device=cuda)
    out = torch.full((4, 2 * kp), 7.0, dtype=torch.bfloat16, device=cuda)
    lib.call("ladi_timestep_embedding", C.c_void_p(t.data_ptr()), 4, c0, kp, C.c_void_p(out.data_ptr()), C.c_void_p(torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    half = c0 // 2
    freq = torch.exp(-math.log(10000.0) * torch.arange(half, dtype=torch.float32) / half)
    arg = t.cpu()[:, None] * freq[None, :]
    ref = torch.cat([torch.cos(arg), torch.sin(arg)], dim=-1)
    got = out[:, :c0].float().cpu() + out[:, kp:kp + c0].float().cpu()
    # hi + lo carries ~17 bits; the dominant term is one fp32 ulp of the frequency (device expf vs torch.exp) times t <= 1000: ~6e-5 at the first columns
    assert (got - ref).abs().max() < 2e-4
    arg_dev = t.cpu()[:, None] * torch.exp((-math.log(10000.0) * torch.arange(half, dtype=torch.float64) / half)).float()[None, :]
    assert (got[:, half:] - torch.sin(arg_dev.double()).float()).abs().max() < 2e-4
    assert float(out[:, c0:kp].abs().max() if kp > c0 else 0.0) == 0.0
