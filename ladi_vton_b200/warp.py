"""H100-native cloth-warping front-end (SURVEY.md section 8(f) row 2): the module pair returned by the reference's
`warping_module` hub constructor (hubconf.py:56-66) and the batch body that uses it (src/inference.py:236-263).

  * `ConvNet_TPS(height, width, input_nc, n_layer)`  <- src/models/ConvNet_TPS.py:287-337.  `__call__(inputA, inputB)` returns the same
    8-tuple; the six regularisation scalars (:207-225, training losses, discarded at inference.py:248) are returned as None.
  * `UNetVanilla(n_channels, n_classes, bilinear)`   <- src/models/UNet.py:4-34 + unet_parts.py (bilinear variant).
  * `generate_warped_cloth(tps, refinement, cloth, im_mask, pose_map)` <- inference.py:236-263 -> `warped_cloth` NCHW fp32 in [-1, 1].

State-dict keys are the reference's (nn.Sequential indices, BatchNorm running statistics, the TPSGridGen buffers).  How it maps to
the hot-path kernels: every convolution and the regression linear run on the wgmma implicit-GEMM kernel (ReLU epilogue); eval-mode
BatchNorm that directly follows a convolution is folded into its weights; BatchNorm that follows a ReLU (FeatureExtraction) is one
in-place per-channel affine pass; the 4x4 stride-2 pad-1 convolutions are computed as 3x3 stride-1 pad-1 convolutions over a
space-to-depth tensor (their 16 taps land in 16 of the 36 (tap, sub-pixel) slots; the rest of the weights are zero); geometry (control
points, TPS grid, sampling coordinates) stays fp32.  The reference runs this module in fp32 (inference.py:205-206); here activations are
bf16 with fp32 accumulation, like the rest of the engine -- tests/test_gpu_warp.py states the resulting tolerances.  No CPU path.
"""
import itertools

import torch

from . import ops
from .module import PackedModule
from .weights import f32, pack_conv, pack_linear

BN_EPS = 1e-5


class _Module(PackedModule):
    def optional(self, key):  # BatchNorm's step counter is unused in eval; TPSGridGen's buffers are recomputed when absent (tps_matrices)
        return key.endswith("num_batches_tracked") or key.startswith("gridGen.")

    def _g(self, k):
        return self._sd[k].to(self.device, torch.float32)

    def _bn(self, p):
        """eval-mode BatchNorm2d `p` as (scale, shift): y = x * scale + shift."""
        s = self._g(p + ".weight") / torch.sqrt(self._g(p + ".running_var") + BN_EPS)
        return s, self._g(p + ".bias") - self._g(p + ".running_mean") * s


def _bn_shapes(S, p, c):
    for n in ("weight", "bias", "running_mean", "running_var"):
        S[f"{p}.{n}"] = (c,)
    S[f"{p}.num_batches_tracked"] = ()


def s2d_weight(w4):
    """[co, c, 4, 4] stride-2 pad-1 weight -> [co, 4c, 3, 3] stride-1 pad-1 weight over the space-to-depth input (channel
    (sy*2+sx)*c + ch): tap (dy, dx) of sub-pixel (sy, sx) holds w4[..., 2*dy+sy-1, 2*dx+sx-1] where that index exists."""
    co, c = w4.shape[:2]
    w3 = w4.new_zeros((co, 4 * c, 3, 3))
    for dy, dx, sy, sx in itertools.product(range(3), range(3), range(2), range(2)):
        ky, kx = 2 * dy + sy - 1, 2 * dx + sx - 1
        if 0 <= ky < 4 and 0 <= kx < 4:
            s = sy * 2 + sx
            w3[:, s * c:(s + 1) * c, dy, dx] = w4[:, :, ky, kx]
    return w3


def control_points(r=0.9, grid=5):
    """5x5 lattice in [-0.9, 0.9]^2, row-major over (y, x), stored as (x, y)  (ConvNet_TPS.py:300-307)."""
    step = 2.0 * r / (grid - 1)
    axis = [-r + i * step for i in range(grid)]
    return torch.tensor([[x, y] for y, x in itertools.product(axis, axis)], dtype=torch.float32)


def _radial(a, b):
    d = a[:, None, :] - b[None, :, :]
    d2 = d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]
    u = 0.5 * d2 * torch.log(d2)
    return torch.where(torch.isnan(u), torch.zeros_like(u), u)


def tps_matrices(height, width, ctrl):
    """One-time host constants of TPSGridGen.__init__ (ConvNet_TPS.py:145-181): inverse of the padded kernel matrix and the
    [H*W, N+3] representation of the target pixel lattice.  Used only when a checkpoint does not carry the `gridGen.*` buffers."""
    n = ctrl.shape[0]
    k = torch.zeros(n + 3, n + 3)
    k[:n, :n] = _radial(ctrl, ctrl)
    k[:n, n] = 1
    k[n, :n] = 1
    k[:n, n + 1:] = ctrl
    k[n + 1:, :n] = ctrl.t()
    ys, xs = torch.meshgrid(torch.arange(height, dtype=torch.float32), torch.arange(width, dtype=torch.float32), indexing="ij")
    coord = torch.stack([xs.reshape(-1) * 2 / (width - 1) - 1, ys.reshape(-1) * 2 / (height - 1) - 1], dim=1)
    rep = torch.cat([_radial(coord, ctrl), torch.ones(height * width, 1), coord], dim=1)
    return torch.inverse(k), rep


class ConvNet_TPS(_Module):
    def __init__(self, height, width, input_nc=6, n_layer=4):
        f = 2 ** (n_layer + 1)
        if height % (4 * f) or width % (4 * f):
            raise ValueError(f"height and width must be multiples of {4 * f} (feature maps are down-scaled {f}x, then twice more by 2)")
        self.height, self.width, self.input_nc, self.n_layer = height, width, input_nc, n_layer
        self.fh, self.fw = height // f, width // f
        self.n_ctrl = 25

    def _extraction_plan(self, cin):
        """[(sequential index of the conv, c_in, c_out, kernel, index of the BatchNorm after the ReLU or None)]."""
        plan, idx, c = [], 0, cin
        widths = [64] + [(2 ** (i + 1) * 64 if 2 ** i * 64 < 512 else 512) for i in range(self.n_layer)]
        for co in widths:
            plan.append((idx, c, co, 4, idx + 2))
            idx, c = idx + 3, co
        plan.append((idx, 512, 512, 3, idx + 2))
        plan.append((idx + 3, 512, 512, 3, None))
        return plan

    REG = [(0, None, 512, 4, 1), (3, 512, 256, 4, 4), (6, 256, 128, 3, 7), (9, 128, 64, 3, 10)]  # conv idx, cin, cout, k, bn idx

    def param_shapes(self):
        S = {}
        for name, cin in (("extractionA", 3), ("extractionB", self.input_nc)):
            for idx, ci, co, k, bn in self._extraction_plan(cin):
                S[f"{name}.model.{idx}.weight"], S[f"{name}.model.{idx}.bias"] = (co, ci, k, k), (co,)
                if bn is not None:
                    _bn_shapes(S, f"{name}.model.{bn}", co)
        hw = self.fh * self.fw
        for idx, ci, co, k, bn in self.REG:
            ci = hw if ci is None else ci
            S[f"loc_net.regression.conv.{idx}.weight"], S[f"loc_net.regression.conv.{idx}.bias"] = (co, ci, k, k), (co,)
            _bn_shapes(S, f"loc_net.regression.conv.{bn}", co)
        flat = 64 * (self.fh // 4) * (self.fw // 4)
        S["loc_net.regression.linear.weight"], S["loc_net.regression.linear.bias"] = (2 * self.n_ctrl, flat), (2 * self.n_ctrl,)
        n = self.n_ctrl + 3
        S["gridGen.inverse_kernel"], S["gridGen.padding_matrix"] = (n, n), (3, 2)
        S["gridGen.target_coordinate_repr"] = (self.height * self.width, n)
        return S

    def _pack_weights(self):
        g, P = self._g, {}
        for name, cin in (("extractionA", 3), ("extractionB", self.input_nc)):
            layers = []
            for idx, ci, co, k, bn in self._extraction_plan(cin):
                w = g(f"{name}.model.{idx}.weight")
                w = pack_conv(s2d_weight(w), [4 * ci]) if k == 4 else pack_conv(w, [ci])
                aff = tuple(f32(t) for t in self._bn(f"{name}.model.{bn}")) if bn is not None else None
                layers.append((w, f32(g(f"{name}.model.{idx}.bias")), co, k, aff))
            P[name] = layers
        reg = []
        for idx, ci, co, k, bn in self.REG:
            ci = self.fh * self.fw if ci is None else ci
            s, t = self._bn(f"loc_net.regression.conv.{bn}")  # conv -> BN -> ReLU: fold BN into the conv
            w = g(f"loc_net.regression.conv.{idx}.weight") * s[:, None, None, None]
            b = g(f"loc_net.regression.conv.{idx}.bias") * s + t
            reg.append((pack_conv(s2d_weight(w), [4 * ci]) if k == 4 else pack_conv(w, [ci]), f32(b), co, k))
        P["reg"] = reg
        qh, qw = self.fh // 4, self.fw // 4
        lw = g("loc_net.regression.linear.weight")
        P["lin.w"] = pack_linear(lw.view(-1, 64, qh, qw).permute(0, 2, 3, 1).reshape(lw.shape[0], -1))  # NCHW flatten -> NHWC flatten
        P["lin.b"] = f32(g("loc_net.regression.linear.bias"))
        if "gridGen.inverse_kernel" in self._sd and "gridGen.target_coordinate_repr" in self._sd:
            inv, rep = g("gridGen.inverse_kernel"), g("gridGen.target_coordinate_repr")
        else:
            inv, rep = (t.to(self.device) for t in tps_matrices(self.height, self.width, control_points()))
        P["inv"], P["rep"] = inv.contiguous(), rep.contiguous()
        self.P = P

    def _extract(self, name, x, c):
        """x NHWC bf16 [B, H, W, pitch] (first c channels valid) -> features NHWC bf16 [B, fh, fw, 512]."""
        for w, b, co, k, aff in self.P[name]:
            if k == 4:
                x, c = ops.space_to_depth2(x, c)
            x = ops.conv2d([x[..., :c]], w, co, bias=b, act=ops.ACT_RELU)
            c = co
            if aff is not None:
                ops.channel_affine_(x, *aff)
        return x

    def forward_nhwc(self, a, ca, b, cb):
        """a / b: NHWC bf16 inputs at (height, width) with ca / cb valid channels -> (grid fp32 [B, H, W, 2], points fp32 [B, 25, 2])."""
        if self.P is None:
            raise RuntimeError("ConvNet_TPS: load_state_dict(...) and .to('cuda') first")
        B = a.shape[0]
        fa = ops.l2norm_channels_(self._extract("extractionA", a, ca))
        fb = ops.l2norm_channels_(self._extract("extractionB", b, cb))
        x = ops.feature_correlation(fa, fb)  # NHWC [B, fh, fw, fh*fw]
        c = self.fh * self.fw
        for w, bias, co, k in self.P["reg"]:
            if k == 4:
                x, c = ops.space_to_depth2(x, c)
            x = ops.conv2d([x[..., :c]], w, co, bias=bias, act=ops.ACT_RELU)
            c = co
        theta = ops.gemm(x.reshape(B, -1), self.P["lin.w"], 2 * self.n_ctrl, bias=self.P["lin.b"], out_fp32=True)
        points, grid = ops.tps_grid(theta, self.P["inv"], self.P["rep"], self.n_ctrl)
        return grid.view(B, self.height, self.width, 2), points

    def __call__(self, inputA, inputB):
        B, ca, H, W = inputA.shape
        cb = inputB.shape[1]
        if (H, W) != (self.height, self.width) or tuple(inputB.shape[-2:]) != (H, W) or ca != 3 or cb != self.input_nc:
            raise ValueError(f"expected inputA [B,3,{self.height},{self.width}] and inputB [B,{self.input_nc},{self.height},{self.width}]")
        a = torch.zeros((B, H, W, 8), dtype=torch.bfloat16, device=self.device)
        b = torch.zeros((B, H, W, (cb + 7) // 8 * 8), dtype=torch.bfloat16, device=self.device)
        ops.nchw_to_nhwc(inputA.to(self.device, torch.float32).contiguous(), a)
        ops.nchw_to_nhwc(inputB.to(self.device, torch.float32).contiguous(), b)
        grid, points = self.forward_nhwc(a, ca, b, cb)
        return grid, points, None, None, None, None, None, None


class UNetVanilla(_Module):
    def __init__(self, n_channels, n_classes, bilinear=False, widths=(64, 128, 256, 512, 1024)):
        if not bilinear:
            raise NotImplementedError("only the bilinear-upsampling variant built by the reference hub constructor (hubconf.py:58) exists")
        self.n_channels, self.n_classes, self.bilinear, self.widths = n_channels, n_classes, bilinear, tuple(widths)

    def _blocks(self):
        """[(state-dict prefix of the DoubleConv, [source channels], mid, out)] in forward order."""
        w = self.widths
        return [("inc.double_conv", [self.n_channels], w[0], w[0]),
                ("down1.maxpool_conv.1.double_conv", [w[0]], w[1], w[1]), ("down2.maxpool_conv.1.double_conv", [w[1]], w[2], w[2]),
                ("down3.maxpool_conv.1.double_conv", [w[2]], w[3], w[3]), ("down4.maxpool_conv.1.double_conv", [w[3]], w[4] // 2, w[4] // 2),
                ("up1.conv.double_conv", [w[3], w[4] // 2], w[4] // 2, w[3] // 2), ("up2.conv.double_conv", [w[2], w[3] // 2], w[3] // 2, w[2] // 2),
                ("up3.conv.double_conv", [w[1], w[2] // 2], w[2] // 2, w[1] // 2), ("up4.conv.double_conv", [w[0], w[1] // 2], w[1] // 2, w[0])]

    def param_shapes(self):
        S = {}
        for p, srcs, mid, out in self._blocks():
            S[p + ".0.weight"], S[p + ".3.weight"] = (mid, sum(srcs), 3, 3), (out, mid, 3, 3)
            _bn_shapes(S, p + ".1", mid)
            _bn_shapes(S, p + ".4", out)
        S["outc.conv.weight"], S["outc.conv.bias"] = (self.n_classes, self.widths[0], 1, 1), (self.n_classes,)
        return S

    def _pack_weights(self):
        g, P = self._g, {}
        for p, srcs, mid, out in self._blocks():
            s1, t1 = self._bn(p + ".1")
            s2, t2 = self._bn(p + ".4")
            P[p] = (pack_conv(g(p + ".0.weight") * s1[:, None, None, None], srcs), f32(t1), mid,
                    pack_conv(g(p + ".3.weight") * s2[:, None, None, None], [mid]), f32(t2), out)
        P["outc.w"], P["outc.b"] = pack_conv(g("outc.conv.weight"), [self.widths[0]]), f32(g("outc.conv.bias"))
        self.P = P

    def _double(self, p, srcs):
        w1, b1, mid, w2, b2, out = self.P[p]
        h = ops.conv2d(srcs, w1, mid, bias=b1, act=ops.ACT_RELU)
        return ops.conv2d([h], w2, out, bias=b2, act=ops.ACT_RELU)

    def forward_nhwc(self, x):
        """x NHWC bf16 [B, H, W, pitch] (first n_channels valid) -> NHWC fp32 [B, H, W, n_classes]."""
        if self.P is None:
            raise RuntimeError("UNetVanilla: load_state_dict(...) and .to('cuda') first")
        if x.shape[1] % 16 or x.shape[2] % 16:
            raise NotImplementedError("H and W must be multiples of 16 (the reference pads odd sizes in Up.forward; not built)")
        B = self._blocks()
        skips = [self._double(B[0][0], [x[..., :self.n_channels]])]
        for i in range(1, 5):
            skips.append(self._double(B[i][0], [ops.maxpool2(skips[-1])]))
        y = skips.pop()
        for i in range(5, 9):
            y = self._double(B[i][0], [skips.pop(), ops.upsample2x_bilinear_ac(y)])  # torch.cat([x2, x1]) stays virtual (unet_parts.py:63)
        return ops.conv2d([y], self.P["outc.w"], self.n_classes, ksize=1, bias=self.P["outc.b"], out_fp32=True)

    def __call__(self, x):
        B, c, H, W = x.shape
        if c != self.n_channels:
            raise ValueError(f"expected {self.n_channels} input channels, got {c}")
        xn = torch.zeros((B, H, W, (c + 7) // 8 * 8), dtype=torch.bfloat16, device=self.device)
        ops.nchw_to_nhwc(x.to(self.device, torch.float32).contiguous(), xn)
        y = self.forward_nhwc(xn)
        return ops.nhwc_f32_to_nchw_clamp(y, self.n_classes, -3.0e38, 3.0e38)


def _low_grid(tps, cloth_d, mask_d, pose_d):
    """inference.py:236-247 (= train_tps.py:53-68): the three antialiased resizes to the TPS resolution and the TPS forward ->
    low-resolution sampling grid fp32 [B, lh, lw, 2]."""
    B, cc = cloth_d.shape[:2]
    lh, lw = tps.height, tps.width  # (256, 192): the TPS parameters are predicted at low resolution
    cm, cp = mask_d.shape[1], pose_d.shape[1]
    low_cloth = ops.resize_aa(cloth_d, lh, lw)
    agnostic = torch.zeros((B, lh, lw, (cm + cp + 7) // 8 * 8), dtype=torch.bfloat16, device=cloth_d.device)
    ops.resize_aa(mask_d, lh, lw, out=agnostic, c_off=0)
    ops.resize_aa(pose_d, lh, lw, out=agnostic, c_off=cm)  # torch.cat([low_im_mask, low_pose_map], 1)  (:247)
    low_grid, _ = tps.forward_nhwc(low_cloth, cc, agnostic, cm + cp)
    return low_grid


def _on(dev, *ts):
    return [t.to(dev, torch.float32).contiguous() for t in ts]


def _refine(tps, refinement, cloth, im_mask, pose_map, lo, hi):
    dev = tps.device
    cloth_d, mask_d, pose_d = _on(dev, cloth, im_mask, pose_map)
    B, cc, H, W = cloth_d.shape
    cm, cp = mask_d.shape[1], pose_d.shape[1]
    low_grid = _low_grid(tps, cloth_d, mask_d, pose_d)
    x = torch.zeros((B, H, W, (cm + cp + cc + 7) // 8 * 8), dtype=torch.bfloat16, device=dev)
    ops.nchw_to_nhwc(mask_d, x, c_off=0)  # torch.cat([im_mask, pose_map, warped_cloth], 1)  (:260)
    ops.nchw_to_nhwc(pose_d, x, c_off=cm)
    ops.warp_grid_sample(low_grid, cloth_d, x, c_off=cm + cp)  # grid resize (:252-255) + grid_sample (:257)
    y = refinement.forward_nhwc(x)
    return ops.nhwc_f32_to_nchw_clamp(y, refinement.n_classes, lo, hi)


def generate_warped_cloth(tps, refinement, cloth, im_mask, pose_map):
    """The warping part of the reference's inference loop body (src/inference.py:236-263): cloth [B,3,H,W] in [-1,1], im_mask [B,3,H,W],
    pose_map [B,18,H,W] -> refined warped cloth NCHW fp32 in [-1,1] (the `warped_cloth` argument of the try-on pipeline)."""
    return _refine(tps, refinement, cloth, im_mask, pose_map, -1.0, 1.0)  # :262


def refine_warped_cloth(tps, refinement, cloth, im_mask, pose_map):
    """generate_warped_cloth without the final clamp: the refinement network's output as the TPS trainer scores it (train_tps.py:77-80;
    UNetVanilla.__call__ returns it unclamped too)."""
    return _refine(tps, refinement, cloth, im_mask, pose_map, -3.0e38, 3.0e38)


def tps_warped_cloth(tps, cloth, im_mask, pose_map):
    """The TPS-only warp of the trainer's validation (train_tps.py:53-75, `refinement=None`): the same resizes, TPS and grid sampling as
    generate_warped_cloth -> the sampled cloth itself, NCHW fp32 [B, 3, H, W], unrounded (`ladi_warp_grid_sample_f32`)."""
    cloth_d, mask_d, pose_d = _on(tps.device, cloth, im_mask, pose_map)
    return ops.warp_grid_sample_f32(_low_grid(tps, cloth_d, mask_d, pose_d), cloth_d)
