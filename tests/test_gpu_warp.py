"""GPU parity of the cloth-warping front-end (SURVEY.md section 8(f) row 2) against torch CPU fp32 semantics and the fp32 oracle
(oracle/ladi_oracle/warp.py, pinned bit-exactly against the reference's ConvNet_TPS / UNetVanilla classes).

Tolerances: data-movement kernels exact; fp32 geometry kernels <= 1e-4 absolute; kernels with bf16 outputs within bf16 rounding of the
fp32 result (<= 1e-2 relative); assembled networks (bf16 activations, the reference runs them in fp32): control points and TPS grid
<= 1e-2 absolute in normalised [-1, 1] coordinates (measured 2e-3), refinement U-Net <= 2e-2 relative L2 (measured 6-8e-3), refined
warped cloth (end to end, smooth synthetic cloth) <= 3e-2 relative L2 (measured 5e-3).
"""
import pytest
import torch
import torch.nn.functional as F

from kernel_check import rel_l2
from model_pairs import tps_pair, unet_pair

pytestmark = pytest.mark.gpu


def nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous()


@pytest.mark.parametrize("h,w,oh,ow", [(512, 384, 256, 192), (64, 48, 32, 24), (30, 22, 13, 9), (16, 12, 32, 24)])
def test_resize_aa(cuda, h, w, oh, ow):
    from ladi_vton_b200 import ops
    x = torch.randn((2, 5, h, w), generator=torch.Generator().manual_seed(h))
    out = torch.zeros((2, oh, ow, 16), dtype=torch.bfloat16, device=cuda)
    ops.resize_aa(x.to(cuda), oh, ow, out=out, c_off=3)
    ref = F.interpolate(x, size=(oh, ow), mode="bilinear", antialias=True, align_corners=False)
    assert (out[..., 3:8].float().cpu() - nhwc(ref)).abs().max() < 2e-2  # bf16 rounding of O(3) values
    assert float(out[..., :3].abs().max()) == 0.0 and float(out[..., 8:].abs().max()) == 0.0


def test_layout_kernels_exact(cuda):
    from ladi_vton_b200 import ops
    g = torch.Generator().manual_seed(0)
    x = torch.randn((2, 6, 4, 24), generator=g).to(cuda, torch.bfloat16)  # NHWC, 21 valid channels of pitch 24
    y, c4 = ops.space_to_depth2(x, 21)
    assert c4 == 84 and y.shape == (2, 3, 2, 88)
    ref = x[..., :21].reshape(2, 3, 2, 2, 2, 21).permute(0, 1, 3, 2, 4, 5).reshape(2, 3, 2, 84)
    assert torch.equal(y[..., :84], ref)
    m = torch.randn((2, 8, 6, 16), generator=g).to(cuda, torch.bfloat16)
    ref = F.max_pool2d(m.float().permute(0, 3, 1, 2), 2).permute(0, 2, 3, 1).to(torch.bfloat16)
    assert torch.equal(ops.maxpool2(m), ref)
    f = torch.randn((2, 4, 3, 5), generator=g).to(cuda)
    out = ops.nhwc_f32_to_nchw_clamp(f, 3, -0.5, 0.5)
    assert torch.equal(out, f[..., :3].permute(0, 3, 1, 2).clamp(-0.5, 0.5))


def test_pointwise_kernels(cuda):
    from ladi_vton_b200 import ops
    g = torch.Generator().manual_seed(1)
    x = torch.randn((2, 5, 3, 64), generator=g).to(cuda, torch.bfloat16)
    s, t = torch.rand(64, generator=g).to(cuda) + 0.5, torch.randn(64, generator=g).to(cuda)
    ref = (x.float() * s + t)
    assert (ops.channel_affine_(x.clone(), s, t).float() - ref).abs().max() < 3e-2
    ref = x.float() / torch.sqrt((x.float() ** 2).sum(-1, keepdim=True) + 1e-6)
    assert (ops.l2norm_channels_(x.clone()).float() - ref).abs().max() < 2e-3
    u = torch.randn((2, 5, 7, 16), generator=g).to(cuda, torch.bfloat16)
    ref = F.interpolate(u.float().permute(0, 3, 1, 2), scale_factor=2, mode="bilinear", align_corners=True).permute(0, 2, 3, 1)
    assert (ops.upsample2x_bilinear_ac(u).float() - ref).abs().max() < 2e-2
    fa = torch.randn((2, 4, 3, 64), generator=g).to(cuda, torch.bfloat16)
    fb = torch.randn((2, 4, 3, 64), generator=g).to(cuda, torch.bfloat16)
    corr = ops.feature_correlation(fa, fb)  # NHWC [2, 4, 3, 12]
    A, Bm = fa.float().permute(0, 3, 1, 2), fb.float().permute(0, 3, 1, 2)  # NCHW
    n, c, h, w = A.shape
    mul = Bm.reshape(n, c, h * w).transpose(1, 2) @ A.transpose(2, 3).reshape(n, c, h * w)  # ConvNet_TPS.py:73-80
    ref = mul.view(n, h, w, h * w)
    assert rel_l2(corr, ref) < 1e-2


def test_tps_grid_and_sampling(cuda):
    from ladi_oracle import warp as ow
    from ladi_vton_b200 import ops, synthetic as S
    ctrl = ow.control_points()
    gen = ow.TPSGridGen(64, 48, ctrl)
    g = torch.Generator().manual_seed(2)
    theta = torch.atanh(ctrl).view(1, -1).repeat(3, 1) + torch.randn((3, 50), generator=g) * 0.2
    pts_ref = torch.tanh(theta).view(3, 25, 2)
    grid_ref = gen(pts_ref).view(3, 64, 48, 2)
    pts, grid = ops.tps_grid(theta.to(cuda), gen.inverse_kernel.to(cuda), gen.target_coordinate_repr.to(cuda), 25)
    assert (pts.cpu() - pts_ref).abs().max() < 1e-5 and (grid.cpu().view(3, 64, 48, 2) - grid_ref).abs().max() < 1e-4
    # inference.py:252-257 with the exact low-resolution grid: resize to (128, 96) + grid_sample(border)
    cloth = S.warp_inputs(3, 128, 96, seed=3)["cloth"]
    hi = F.interpolate(grid_ref.permute(0, 3, 1, 2), size=(128, 96), mode="bilinear", antialias=True).permute(0, 2, 3, 1)
    ref = F.grid_sample(cloth, hi, padding_mode="border", align_corners=False)
    out = torch.zeros((3, 128, 96, 8), dtype=torch.bfloat16, device=cuda)
    ops.warp_grid_sample(grid_ref.to(cuda).contiguous(), cloth.to(cuda), out, c_off=2)
    assert (out[..., 2:5].float().cpu() - nhwc(ref)).abs().max() < 8e-3


def test_conv4x4_stride2_through_space_to_depth(cuda):
    from ladi_vton_b200 import ops
    from ladi_vton_b200.warp import s2d_weight
    from ladi_vton_b200.weights import pack_conv
    g = torch.Generator().manual_seed(4)
    x = torch.randn((2, 21, 32, 24), generator=g)
    w = torch.randn((64, 21, 4, 4), generator=g) * 0.05
    b = torch.randn(64, generator=g)
    ref = F.relu(F.conv2d(x, w, b, stride=2, padding=1))
    xn = torch.zeros((2, 32, 24, 24), dtype=torch.bfloat16, device=cuda)
    ops.nchw_to_nhwc(x.to(cuda), xn)
    xs, c4 = ops.space_to_depth2(xn, 21)
    y = ops.conv2d([xs[..., :c4]], pack_conv(s2d_weight(w), [c4]).to(cuda), 64, bias=b.to(cuda), act=ops.ACT_RELU)
    assert rel_l2(y, nhwc(ref)) < 1e-2


def test_convnet_tps(cuda):
    """hubconf.py:57 configuration: ConvNet_TPS(256, 192, 21, 3) -> 25 control points and the [256, 192] sampling grid."""
    eng, o = tps_pair(cuda)
    g = torch.Generator().manual_seed(5)
    a, b = torch.rand((2, 3, 256, 192), generator=g) * 2 - 1, torch.rand((2, 21, 256, 192), generator=g)
    with torch.no_grad():
        grid_ref, pts_ref = o(a, b)
    out = eng(a, b)
    assert len(out) == 8 and out[0].shape == (2, 256, 192, 2) and out[1].shape == (2, 25, 2)
    e_pts, e_grid = (out[1].cpu() - pts_ref).abs().max().item(), (out[0].cpu() - grid_ref).abs().max().item()
    from ladi_oracle.warp import control_points
    moved = (pts_ref - control_points()).abs().max().item()
    print("TPS control points / grid max abs err:", e_pts, e_grid, "(warp moves the lattice by up to", moved, ")")
    assert moved > 0.05, "test weights must produce a non-identity warp"
    assert e_pts < 1e-2 and e_grid < 1e-2


@pytest.mark.parametrize("widths,hw", [((16, 32, 64, 128, 256), (64, 48)), ((64, 128, 256, 512, 1024), (64, 48))])
def test_unet_vanilla(cuda, widths, hw):
    eng, o = unet_pair(cuda, widths)
    x = torch.rand((2, 24, *hw), generator=torch.Generator().manual_seed(6)) * 2 - 1
    with torch.no_grad():
        ref = o(x)
    y = eng(x)
    err = rel_l2(y, ref)
    print("UNetVanilla rel-L2:", err)
    assert y.shape == ref.shape and err < 2e-2
    with pytest.raises(NotImplementedError):
        eng(torch.zeros((1, 24, 40, 48)))


def test_generate_warped_cloth_full_size(cuda):
    """src/inference.py:236-263 at 512x384: resizes, TPS, grid_sample, refinement, clamp."""
    from ladi_oracle import warp as ow
    from ladi_vton_b200 import generate_warped_cloth, ops, synthetic as S
    tps, otps = tps_pair(cuda)
    ref_net, oref = unet_pair(cuda)
    inp = S.warp_inputs(1, 512, 384, seed=7)
    with torch.no_grad():
        want, coarse, low_grid, pts = ow.warp_cloth(otps, oref, inp["cloth"], inp["im_mask"], inp["pose_map"], return_all=True)
    got = generate_warped_cloth(tps, ref_net, inp["cloth"], inp["im_mask"], inp["pose_map"])
    assert got.shape == want.shape == (1, 3, 512, 384) and float(got.abs().max()) <= 1.0
    err = rel_l2(got, want)
    sat = float((want.abs() >= 1.0).float().mean())
    print("refined warped cloth rel-L2:", err, "mean |diff|:", float((got.cpu() - want).abs().mean()), "clamped fraction:", sat)
    assert err < 3e-2
    # stage check with the oracle's own low-resolution grid: the fused grid-resize + grid_sample kernel alone
    x = torch.zeros((1, 512, 384, 8), dtype=torch.bfloat16, device=cuda)
    ops.warp_grid_sample(low_grid.to(cuda).contiguous(), inp["cloth"].to(cuda), x)
    assert (x[..., :3].float().cpu() - nhwc(coarse)).abs().max() < 8e-3


def test_hub_warping_module_roundtrip(cuda, tmp_path):
    from ladi_vton_b200 import hub, synthetic as S
    from ladi_vton_b200.warp import ConvNet_TPS, UNetVanilla, control_points
    tps_sd = S.warp_state_dict(ConvNet_TPS(256, 192, 21, 3).param_shapes(), 11, ctrl_bias=torch.atanh(control_points()).view(-1))
    unet_sd = S.warp_state_dict(UNetVanilla(24, 3, True).param_shapes(), 12)
    torch.save({"tps": tps_sd, "refinement": unet_sd}, tmp_path / "warping_vitonhd.pth")
    tps, refinement = hub.warping_module("vitonhd", checkpoint_dir=str(tmp_path))
    tps.to(cuda), refinement.to(cuda)
    a = tps(torch.zeros((1, 3, 256, 192)), torch.zeros((1, 21, 256, 192)))
    assert a[0].shape == (1, 256, 192, 2) and torch.isfinite(a[0]).all()
