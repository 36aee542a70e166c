"""GPU tests of the image-quality metrics (csrc/metrics.cu, ladi_vton_b200/metrics.py, ladi_vton_b200/val_metrics.py) on an H100:
each new kernel against fp32 / fp64 torch, the full-size FID Inception-v3 and LPIPS AlexNet against the fp32 oracle with random weights
(BatchNorm statistics calibrated on the test batch so activations stay O(1)), FID / KID / IS from engine features against the same
statistics from oracle features, determinism, and the CLI end to end on synthetic PNG folders."""
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

# Gates set from values measured on an H100 80GB HBM3 (700 W power limit), recorded in DESIGN.md section 7, with headroom.  With random
# weights and batch-calibrated BatchNorm every Inception block amplifies the error it receives about 1.5x, so the end-to-end numbers are
# far looser than what one stage adds: STAGE_REL_L2 is the strict check of every layer; the end-to-end gates guard against gross faults.
STAGE_REL_L2 = 2e-2       # each Inception stage fed the oracle's input (measured <= 7.9e-3)
FEATURE_REL_L2 = 0.3      # pool3 features / unbiased logits, end to end (measured 0.20)
LPIPS_REL = 2e-3          # per pair, AlexNet has 5 layers (measured 4.1e-4)
STAT_REL = {"fid": 5e-2, "kid": 0.3, "is": 1e-3}  # from engine vs oracle features of 16 + 16 images (measured 1.6e-2, 0.15, 1.8e-5)


@pytest.fixture(autouse=True)
def _fp32_reference():
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def rel_l2(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float((a - b).norm() / b.norm())


def _im2col_ref(x_nchw, kernel, stride, padding, k_pad):
    (kh, kw), (sh, sw), (ph, pw) = kernel, stride, padding
    xp = F.pad(x_nchw, (pw, pw, ph, ph))
    n, c = x_nchw.shape[:2]
    oh, ow = (xp.shape[2] - kh) // sh + 1, (xp.shape[3] - kw) // sw + 1
    cols = [xp[:, :, ky:ky + sh * (oh - 1) + 1:sh, kx:kx + sw * (ow - 1) + 1:sw] for ky in range(kh) for kx in range(kw)]
    rows = torch.stack(cols, 1).permute(0, 3, 4, 1, 2).reshape(n * oh * ow, kh * kw * c)
    return F.pad(rows, (0, k_pad - rows.shape[1]))


# ---- kernels ----------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kernel,stride,padding,c", [((1, 7), (1, 1), (0, 3), 16), ((7, 1), (1, 1), (3, 0), 24), ((5, 5), (1, 1), (2, 2), 48),
                                                    ((3, 3), (2, 2), (0, 0), 32), ((3, 3), (1, 1), (0, 0), 8), ((1, 3), (1, 1), (0, 1), 8)])
def test_im2col_nhwc_bit_exact(cuda, kernel, stride, padding, c):
    from ladi_vton_b200 import ops
    g = torch.Generator(device=cuda).manual_seed(1)
    full = torch.randn(2, 17, 13, c + 8, generator=g, device=cuda).to(torch.bfloat16)
    x = full[..., :c]  # channel-sliced view: pitch c + 8
    k_pad = -(-kernel[0] * kernel[1] * c // 64) * 64
    rows, (n, oh, ow) = ops.im2col(x, kernel, stride, padding, k_pad)
    assert torch.equal(rows, _im2col_ref(x.permute(0, 3, 1, 2).float(), kernel, stride, padding, k_pad).to(torch.bfloat16))


@pytest.mark.parametrize("kernel,stride,padding", [((11, 11), (4, 4), (2, 2)), ((3, 3), (2, 2), (0, 0))])
def test_im2col_pixels_affine_before_padding(cuda, kernel, stride, padding):
    from ladi_vton_b200 import ops
    x = torch.rand(2, 3, 45, 37, generator=torch.Generator(device=cuda).manual_seed(2), device=cuda)
    shift = torch.tensor([0.485, 0.456, 0.406], device=cuda)
    scale = torch.tensor([0.229, 0.224, 0.225], device=cuda)
    rows, _ = ops.im2col(x, kernel, stride, padding, 384 if kernel[0] == 11 else 64, shift=shift, scale=scale)
    want = _im2col_ref((x - shift.view(1, 3, 1, 1)) / scale.view(1, 3, 1, 1), kernel, stride, padding, rows.shape[1])
    assert torch.equal(rows, want.to(torch.bfloat16))  # zeros in the padding: the affine is not applied there


@pytest.mark.parametrize("k,s,p", [(3, 2, 0), (3, 1, 1), (2, 2, 0)])
def test_pool2d(cuda, k, s, p):
    from ladi_vton_b200 import ops
    x = torch.randn(3, 35, 17, 40, generator=torch.Generator(device=cuda).manual_seed(3), device=cuda).to(torch.bfloat16)
    xc = x.permute(0, 3, 1, 2).float()
    got = ops.pool2d(x, k, s, p, ops.POOL_MAX).permute(0, 3, 1, 2)
    assert torch.equal(got, F.max_pool2d(xc, k, s, p).to(torch.bfloat16))
    for mode, incl in ((ops.POOL_AVG, True), (ops.POOL_AVG_EXCLUDE_PAD, False)):
        got = ops.pool2d(x, k, s, p, mode).permute(0, 3, 1, 2).float()
        want = F.avg_pool2d(xc.double(), k, s, p, count_include_pad=incl)
        assert float(((got - want).abs() / (want.abs() + 1e-3)).max()) <= 2 ** -8  # one bf16 rounding of an fp32 mean
    # into a channel slice of a wider buffer, other channels untouched
    out = torch.full((3, ops.conv_out_size(35, k, s, p), ops.conv_out_size(17, k, s, p), 64), 7.0, dtype=torch.bfloat16, device=cuda)
    ops.pool2d(x, k, s, p, ops.POOL_MAX, out=out, c_off=16)
    assert torch.equal(out[..., 16:56].permute(0, 3, 1, 2), F.max_pool2d(xc, k, s, p).to(torch.bfloat16))
    assert bool((out[..., :16] == 7).all()) and bool((out[..., 56:] == 7).all())


def test_global_avg_pool(cuda):
    from ladi_vton_b200 import ops
    x = torch.randn(5, 8, 8, 2048, generator=torch.Generator(device=cuda).manual_seed(4), device=cuda).to(torch.bfloat16)
    got = ops.global_avg_pool(x)
    want = x.double().mean(dim=(1, 2))
    assert got.dtype == torch.float32 and got.shape == (5, 2048)
    assert float((got.double() - want).abs().max()) < 1e-6


@pytest.mark.parametrize("h,w,c", [(127, 95, 64), (31, 23, 192), (15, 11, 384), (15, 11, 256)])
def test_lpips_layer(cuda, h, w, c):
    from ladi_vton_b200 import ops
    g = torch.Generator(device=cuda).manual_seed(5)
    fa = torch.relu(torch.randn(3, h, w, c, generator=g, device=cuda)).to(torch.bfloat16)
    fb = torch.relu(fa.float() + 0.3 * torch.randn(3, h, w, c, generator=g, device=cuda)).to(torch.bfloat16)
    lin = torch.rand(c, generator=g, device=cuda) * 0.1
    acc = torch.full((3,), 0.25, device=cuda)
    ops.lpips_layer_(fa, fb, lin, acc)
    a, b = fa.double(), fb.double()
    na = a / (a.pow(2).sum(-1, keepdim=True).sqrt() + 1e-10)
    nb = b / (b.pow(2).sum(-1, keepdim=True).sqrt() + 1e-10)
    want = 0.25 + ((na - nb) ** 2 * lin.double()).sum(-1).mean(dim=(1, 2))
    assert float(((acc.double() - want).abs() / want).max()) < 1e-5


@pytest.mark.parametrize("h,w", [(512, 384), (37, 23), (11, 11), (100, 27)])
def test_ssim_kernel(cuda, h, w):
    from ladi_oracle import metrics as OM
    from ladi_vton_b200 import ops
    g = torch.Generator(device=cuda).manual_seed(6)
    x = torch.rand(4, 3, h, w, generator=g, device=cuda)
    y = (x + 0.2 * torch.randn(4, 3, h, w, generator=g, device=cuda)).clamp(0, 1)
    got = ops.ssim(x, y)
    want = OM.ssim(x, y, torch.float64)
    assert float((got.double() - want).abs().max()) < 2e-5, (got, want)
    assert float((ops.ssim(x, x).double() - 1).abs().max()) < 1e-5
    with pytest.raises(ValueError, match="at least 11"):
        ops.ssim(x[..., :10, :].contiguous(), y[..., :10, :].contiguous())


def test_resize_tf1(cuda):
    from ladi_oracle import metrics as OM
    from ladi_vton_b200 import ops
    x = torch.rand(2, 3, 512, 384, generator=torch.Generator(device=cuda).manual_seed(7), device=cuda)
    x[0, 0, :4, :4] = torch.tensor([0.0, 1.0, 3 / 255, 200 / 255], device=cuda)[None, :]  # values at and near integer multiples of 1/255
    got = ops.resize_tf1_u8(x, 299, 299)
    want = OM.resize_tf1_u8(x, 299, 299)
    assert float((got - want).abs().max()) < 1e-3


# ---- networks ----------------------------------------------------------------------------------------------------------------------------
def _inception_pair(cuda, n=8, seed=11):
    """engine FIDInceptionV3 and an oracle state dict sharing random weights whose BatchNorm statistics come from the test batch."""
    from ladi_oracle import metrics as OM
    from ladi_vton_b200.metrics import FIDInceptionV3, random_state_dict
    net = FIDInceptionV3()
    sd = {k: v.to(cuda) for k, v in random_state_dict(net.param_shapes(), seed).items()}
    g = torch.Generator(device=cuda).manual_seed(seed)
    x = F.interpolate(torch.rand(n, 3, 75, 75, generator=g, device=cuda), size=(299, 299), mode="bilinear") * 255
    with torch.no_grad():
        OM.calibrate_batchnorm(sd, x)
    net.load_state_dict({k: v.cpu() for k, v in sd.items()}).to(cuda)
    return net, sd, x


def test_inception_stages_vs_oracle(cuda):
    """Every stage (stem convolutions, pools, each Mixed block) fed the oracle's own input, rounded to bf16: the error one stage adds."""
    from ladi_oracle import metrics as OM
    from ladi_vton_b200 import ops
    net, sd, x = _inception_pair(cuda)
    L = net.layers
    o = OM._bconv(sd, "Conv2d_1a_3x3", (x - 128) / 128, stride=2)
    errs = {"Conv2d_1a_3x3": rel_l2(L["Conv2d_1a_3x3"](x, shift=net.shift, scale=net.scale).permute(0, 3, 1, 2), o)}
    stages = [("Conv2d_2a_3x3", L["Conv2d_2a_3x3"], lambda t: OM._bconv(sd, "Conv2d_2a_3x3", t)),
              ("Conv2d_2b_3x3", L["Conv2d_2b_3x3"], lambda t: OM._bconv(sd, "Conv2d_2b_3x3", t, padding=1)),
              ("maxpool1", lambda t: ops.pool2d(t, 3, 2, 0, ops.POOL_MAX), lambda t: F.max_pool2d(t, 3, 2)),
              ("Conv2d_3b_1x1", L["Conv2d_3b_1x1"], lambda t: OM._bconv(sd, "Conv2d_3b_1x1", t)),
              ("Conv2d_4a_3x3", L["Conv2d_4a_3x3"], lambda t: OM._bconv(sd, "Conv2d_4a_3x3", t)),
              ("maxpool2", lambda t: ops.pool2d(t, 3, 2, 0, ops.POOL_MAX), lambda t: F.max_pool2d(t, 3, 2))]
    stages += [(m, lambda t, m=m: net._block_a(t, m), lambda t, m=m: OM._a(sd, m, t)) for m in ("Mixed_5b", "Mixed_5c", "Mixed_5d")]
    stages += [("Mixed_6a", lambda t: net._block_b(t, "Mixed_6a"), lambda t: OM._b(sd, "Mixed_6a", t))]
    stages += [(m, lambda t, m=m: net._block_c(t, m), lambda t, m=m: OM._c(sd, m, t)) for m in ("Mixed_6b", "Mixed_6c", "Mixed_6d", "Mixed_6e")]
    stages += [("Mixed_7a", lambda t: net._block_d(t, "Mixed_7a"), lambda t: OM._d(sd, "Mixed_7a", t)),
               ("Mixed_7b", lambda t: net._block_e(t, "Mixed_7b", ops.POOL_AVG_EXCLUDE_PAD), lambda t: OM._e(sd, "Mixed_7b", t, False)),
               ("Mixed_7c", lambda t: net._block_e(t, "Mixed_7c", ops.POOL_MAX), lambda t: OM._e(sd, "Mixed_7c", t, True))]
    with torch.no_grad():
        for name, eng, orc in stages:
            e = eng(o.permute(0, 2, 3, 1).to(torch.bfloat16).contiguous())
            o = orc(o)
            errs[name] = rel_l2(e.permute(0, 3, 1, 2), o)
    print("\n[metrics] inception stage rel-L2: " + ", ".join(f"{k} {v:.2e}" for k, v in errs.items()))
    assert max(errs.values()) < STAGE_REL_L2, errs


def test_inception_vs_oracle(cuda):
    from ladi_oracle import metrics as OM
    net, sd, x = _inception_pair(cuda)
    feats = net(x)
    with torch.no_grad():
        of, ol = OM.inception_features(sd, x)
    e_f, e_l = rel_l2(feats, of), rel_l2(net.unbiased_logits(feats), ol.cpu())
    print(f"\n[metrics] inception pool3 rel-L2 {e_f:.3e}  logits rel-L2 {e_l:.3e}")
    assert feats.shape == (8, 2048) and e_f < FEATURE_REL_L2 and e_l < FEATURE_REL_L2
    # determinism: a second run gives the same bits
    assert torch.equal(net(x), feats)


def test_lpips_vs_oracle(cuda):
    from ladi_oracle import metrics as OM
    from ladi_vton_b200.metrics import LPIPSAlex, random_state_dict
    net = LPIPSAlex()
    sd = random_state_dict(net.param_shapes(), 12)
    net.load_state_dict(sd).to(cuda)
    g = torch.Generator(device=cuda).manual_seed(12)
    a = F.interpolate(torch.rand(4, 3, 64, 48, generator=g, device=cuda), size=(512, 384), mode="bilinear")
    b = (a + 0.1 * torch.randn(a.shape, generator=g, device=cuda)).clamp(0, 1)
    got = net(a, b)
    with torch.no_grad():
        want = OM.lpips({k: v.to(cuda) for k, v in sd.items()}, a, b)
    err = float(((got.double() - want.double()).abs() / want.double().abs()).max())
    print(f"\n[metrics] lpips per-pair max rel diff {err:.3e} (values {want.tolist()})")
    assert err < LPIPS_REL
    assert torch.equal(net(a, b), got)


def test_statistics_from_engine_vs_oracle_features(cuda):
    """FID / KID / IS computed on engine features vs on oracle features of the same synthetic images."""
    from ladi_oracle import metrics as OM
    from ladi_vton_b200.metrics import feature_stats, frechet_distance, inception_score, kernel_distance
    net, sd, x = _inception_pair(cuda, n=32, seed=13)
    gen, ref = x[:16], x[16:]
    with torch.no_grad():
        of_gen, ol_gen = OM.inception_features(sd, gen)
        of_ref, _ = OM.inception_features(sd, ref)
    ef_gen, ef_ref = net(gen), net(ref)
    el_gen = net.unbiased_logits(ef_gen)
    f = lambda a, b: frechet_distance(*feature_stats(a), *feature_stats(b))  # noqa: E731
    np_ = lambda t: t.double().cpu().numpy()  # noqa: E731
    pairs = {"fid": (f(np_(ef_gen), np_(ef_ref)), f(np_(of_gen), np_(of_ref))),
             "kid": (kernel_distance(np_(ef_ref), np_(ef_gen), seed=3), kernel_distance(np_(of_ref), np_(of_gen), seed=3)),
             "is": (inception_score(el_gen.numpy(), seed=3)[0], inception_score(ol_gen.cpu().numpy(), seed=3)[0])}
    for k, (e, o) in pairs.items():
        print(f"\n[metrics] {k}: engine {e:.6g} oracle {o:.6g} rel {abs(e - o) / abs(o):.3e}")
    for k, (e, o) in pairs.items():
        assert abs(e - o) <= STAT_REL[k] * abs(o), (k, e, o)


def test_ssim_wrapper_deterministic(cuda):
    from ladi_vton_b200.metrics import ssim
    g = torch.Generator(device=cuda).manual_seed(14)
    x, y = torch.rand(6, 3, 512, 384, generator=g, device=cuda), torch.rand(6, 3, 512, 384, generator=g, device=cuda)
    assert torch.equal(ssim(x, y), ssim(x, y))


# ---- CLI ------------------------------------------------------------------------------------------------------------------------------
def _write_tree(root, gen, n=6, seed=15):
    from PIL import Image
    rs = np.random.RandomState(seed)
    names = [f"{i:05d}_00.jpg" for i in range(n)]
    os.makedirs(os.path.join(root, "test", "image"))
    os.makedirs(os.path.join(gen, "upper_body"))
    with open(os.path.join(root, "test_pairs.txt"), "w") as f:
        f.write("".join(f"{a} {b}\n" for a, b in zip(names, reversed(names))))
    for nm in names:
        base = rs.randint(0, 256, size=(8, 6, 3)).astype(np.uint8)
        gt = Image.fromarray(base).resize((384, 512), Image.BILINEAR)
        gt.save(os.path.join(root, "test", "image", nm), quality=95)
        noisy = np.clip(np.asarray(gt, dtype=np.int16) + rs.randint(-20, 21, size=(512, 384, 3)), 0, 255).astype(np.uint8)
        Image.fromarray(noisy).save(os.path.join(gen, "upper_body", nm.replace(".jpg", ".png")))


def test_main_end_to_end(cuda, tmp_path):
    from ladi_vton_b200.val_metrics import main
    root, gen, cache = str(tmp_path / "vitonhd"), str(tmp_path / "gen"), str(tmp_path / "cache")
    _write_tree(root, gen)
    argv = ["--gen_folder", gen, "--test_order", "paired", "--dataset", "vitonhd", "--vitonhd_dataroot", root, "--batch_size", "4",
            "--workers", "0", "--random_init", "--cache_dir", cache]
    m = main(argv)
    out = json.load(open(os.path.join(gen, "metrics_paired_all.json")))
    assert list(out) == ['ssim_score', 'lpips_score', 'fid_score', 'kid_score', 'is_score'] and out == m
    assert all(np.isfinite(v) for v in out.values()), out
    assert 0 < out["ssim_score"] < 1 and out["lpips_score"] > 0 and out["is_score"] >= 1
    assert sorted(os.listdir(cache)) == ["vitonhd_all_random0.npz"]
    assert main(argv) == m  # cached statistics and fixed seeds: the same numbers
    print(f"\n[metrics] main(): {m}")
