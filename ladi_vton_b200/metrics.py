"""Image-quality metrics on the H100 engine: the networks and statistics behind the reference's src/utils/val_metrics.py (clean-fid's FID
and KID, torchmetrics' SSIM, LPIPS and Inception Score), without cleanfid, torchmetrics or a network connection.

  * `FIDInceptionV3` -- the TF "2015-12-05" Inception-v3 of FID / KID / IS in its torchvision restatement (pytorch-fid, torch-fidelity):
    1008 classes, no aux logits, average pools of the A, C and E_1 blocks with count_include_pad=False, a 3x3 max pool in E_2's pool
    branch.  State dict: `pt_inception-2015-12-05-6726825d.pth`.  `__call__` -> pool3 features fp32 [n, 2048]; `unbiased_logits` ->
    features @ fc.weight^T (no bias), fp64 on the host, [n, 1008].
  * `LPIPSAlex` -- torchmetrics LearnedPerceptualImagePatchSimilarity(net='alex', normalize=True): [0, 1] -> [-1, 1], the LPIPS scaling
    layer, torchvision AlexNet `features` tapped after ReLU 1-5, one `ladi_lpips_layer` per tap.  Weights: `alexnet-owt-7be5be79.pth`
    (`features.*`) and the LPIPS v0.1 `alex.pth` (`lin<k>.model.1.weight`).
  * `ssim` -- per-image SSIM (`ladi_ssim_f32`).
  * `frechet_distance`, `kernel_distance`, `inception_score` -- host fp64 statistics, as clean-fid and torchmetrics compute them.

How the networks map onto the kernels: BatchNorm (eval mode, eps 1e-3) is folded into the convolution weights at load and ReLU is the GEMM
epilogue.  1x1 convolutions are GEMMs over the NHWC rows; 3x3 stride-1 pad-1 convolutions whose output width is a multiple of 8 use the
implicit-GEMM ksize-3 path of `ladi_conv2d_bf16`; every other convolution (the 3-channel stems, 11x11/4, 5x5, 1x7, 7x1, 1x3, 3x1, valid and
strided 3x3, and 3x3 at odd widths, where the implicit path's 128-row tile would hold one pixel of the batch) is `ladi_im2col_bf16` + one GEMM.
Branch outputs and pools are written straight into their block's channel concatenation.  Activations are bf16 with fp32 accumulation; the
input affine ((x - 128) / 128 for Inception, the LPIPS scaling layer for AlexNet) is applied in fp32 by the pixel im2col before the
padding.  No CPU path: `.to("cpu")` raises.

`precision="tf32"` (both networks' constructors; the default is "bf16") is the precision the reference computes in on a GPU: clean-fid's and
torchmetrics' fp32 modules under PyTorch's default `torch.backends.cudnn.allow_tf32 = True`.  Activations are fp32 NHWC, the weights fp32
(BatchNorm folded in float64, K padded with zeros to a multiple of 4), and every convolution is one `ladi_gemm_tf32` (TF32 tensor cores,
operands rounded to nearest TF32 inside the kernel, fp32 accumulation): a 1x1 convolution directly over the NHWC rows, every other one
over `ladi_im2col_f32` rows.  Pools and the LPIPS layers run their fp32 forms.
"""
import math

import numpy as np
import torch

from . import lib, ops
from .module import PackedModule
from .weights import pad64

PRECISIONS = ("bf16", "tf32")
INCEPTION_BN_EPS = 1e-3
INCEPTION_FILE = "pt_inception-2015-12-05-6726825d.pth"
ALEXNET_FILE = "alexnet-owt-7be5be79.pth"
LPIPS_FILE = "alex.pth"
# LPIPS ScalingLayer (lpips/pretrained_networks.py, v0.1): (x - shift) / scale on [-1, 1] images
LPIPS_SHIFT = (-0.030, -0.088, -0.188)
LPIPS_SCALE = (0.458, 0.448, 0.450)


def pad4(k):
    return (k + 3) // 4 * 4


def _pair(v):
    return (v, v) if isinstance(v, int) else tuple(v)


# ---- layer tables ---------------------------------------------------------------------------------------------------------------------
def _inception_layers():
    """name -> (c_in, c_out, kernel, stride, padding) of every BasicConv2d of the FID Inception-v3 (torchvision key names)."""
    L = {}

    def add(name, ci, co, k, s=1, p=0):
        L[name] = (ci, co, _pair(k), _pair(s), _pair(p))

    add("Conv2d_1a_3x3", 3, 32, 3, 2)
    add("Conv2d_2a_3x3", 32, 32, 3)
    add("Conv2d_2b_3x3", 32, 64, 3, 1, 1)
    add("Conv2d_3b_1x1", 64, 80, 1)
    add("Conv2d_4a_3x3", 80, 192, 3)
    for name, ci, pf in (("Mixed_5b", 192, 32), ("Mixed_5c", 256, 64), ("Mixed_5d", 288, 64)):
        add(f"{name}.branch1x1", ci, 64, 1)
        add(f"{name}.branch5x5_1", ci, 48, 1)
        add(f"{name}.branch5x5_2", 48, 64, 5, 1, 2)
        add(f"{name}.branch3x3dbl_1", ci, 64, 1)
        add(f"{name}.branch3x3dbl_2", 64, 96, 3, 1, 1)
        add(f"{name}.branch3x3dbl_3", 96, 96, 3, 1, 1)
        add(f"{name}.branch_pool", ci, pf, 1)
    add("Mixed_6a.branch3x3", 288, 384, 3, 2)
    add("Mixed_6a.branch3x3dbl_1", 288, 64, 1)
    add("Mixed_6a.branch3x3dbl_2", 64, 96, 3, 1, 1)
    add("Mixed_6a.branch3x3dbl_3", 96, 96, 3, 2)
    for name, c7 in (("Mixed_6b", 128), ("Mixed_6c", 160), ("Mixed_6d", 160), ("Mixed_6e", 192)):
        add(f"{name}.branch1x1", 768, 192, 1)
        add(f"{name}.branch7x7_1", 768, c7, 1)
        add(f"{name}.branch7x7_2", c7, c7, (1, 7), 1, (0, 3))
        add(f"{name}.branch7x7_3", c7, 192, (7, 1), 1, (3, 0))
        add(f"{name}.branch7x7dbl_1", 768, c7, 1)
        add(f"{name}.branch7x7dbl_2", c7, c7, (7, 1), 1, (3, 0))
        add(f"{name}.branch7x7dbl_3", c7, c7, (1, 7), 1, (0, 3))
        add(f"{name}.branch7x7dbl_4", c7, c7, (7, 1), 1, (3, 0))
        add(f"{name}.branch7x7dbl_5", c7, 192, (1, 7), 1, (0, 3))
        add(f"{name}.branch_pool", 768, 192, 1)
    add("Mixed_7a.branch3x3_1", 768, 192, 1)
    add("Mixed_7a.branch3x3_2", 192, 320, 3, 2)
    add("Mixed_7a.branch7x7x3_1", 768, 192, 1)
    add("Mixed_7a.branch7x7x3_2", 192, 192, (1, 7), 1, (0, 3))
    add("Mixed_7a.branch7x7x3_3", 192, 192, (7, 1), 1, (3, 0))
    add("Mixed_7a.branch7x7x3_4", 192, 192, 3, 2)
    for name, ci in (("Mixed_7b", 1280), ("Mixed_7c", 2048)):
        add(f"{name}.branch1x1", ci, 320, 1)
        add(f"{name}.branch3x3_1", ci, 384, 1)
        add(f"{name}.branch3x3_2a", 384, 384, (1, 3), 1, (0, 1))
        add(f"{name}.branch3x3_2b", 384, 384, (3, 1), 1, (1, 0))
        add(f"{name}.branch3x3dbl_1", ci, 448, 1)
        add(f"{name}.branch3x3dbl_2", 448, 384, 3, 1, 1)
        add(f"{name}.branch3x3dbl_3a", 384, 384, (1, 3), 1, (0, 1))
        add(f"{name}.branch3x3dbl_3b", 384, 384, (3, 1), 1, (1, 0))
        add(f"{name}.branch_pool", ci, 192, 1)
    return L


INCEPTION_LAYERS = _inception_layers()
# torchvision AlexNet `features` index -> (c_in, c_out, kernel, stride, padding); the LPIPS taps follow the ReLUs of all five
ALEX_LAYERS = {0: (3, 64, (11, 11), (4, 4), (2, 2)), 3: (64, 192, (5, 5), (1, 1), (2, 2)), 6: (192, 384, (3, 3), (1, 1), (1, 1)),
               8: (384, 256, (3, 3), (1, 1), (1, 1)), 10: (256, 256, (3, 3), (1, 1), (1, 1))}
LPIPS_CHANNELS = (64, 192, 384, 256, 256)


# ---- weight packing -------------------------------------------------------------------------------------------------------------------
def uses_implicit_3x3(kernel, stride, padding, w_out):
    """True where ladi_conv2d_bf16's ksize-3 path runs the layer (see the module docstring); otherwise im2col + GEMM."""
    return kernel == (3, 3) and stride == (1, 1) and padding == (1, 1) and w_out % 8 == 0


def pack_im2col_weight(w, dtype=torch.bfloat16):
    """[c_out, c_in, kh, kw] -> [c_out, K'] in the im2col (ky, kx, c) column order, zeros in the columns past kh*kw*c_in: bf16 with
    K' = pad64(kh*kw*c_in) for ladi_conv2d_bf16, or fp32 with K' = pad4(kh*kw*c_in) for ladi_gemm_tf32."""
    co, ci, kh, kw = w.shape
    flat = w.permute(0, 2, 3, 1).reshape(co, kh * kw * ci)
    out = flat.new_zeros((co, (pad4 if dtype == torch.float32 else pad64)(kh * kw * ci)))
    out[:, :flat.shape[1]] = flat
    return out.to(dtype).contiguous()


def fold_bn(w, gamma, beta, mean, var, eps):
    """Eval-mode BatchNorm after a bias-free convolution -> (w', b') in fp64: conv(x, w') + b' == bn(conv(x, w))."""
    s = gamma.double() / torch.sqrt(var.double() + eps)
    return w.double() * s[:, None, None, None], beta.double() - mean.double() * s


class _Conv:
    """One convolution + ReLU.  bf16: packed for both paths (the choice needs the output width, known at call time).  tf32: one fp32
    [c_out, pad4(K)] weight for ladi_gemm_tf32, from the float64 `w`."""

    def __init__(self, w, b, stride, padding, device, precision="bf16"):
        self.c_in, self.c_out = int(w.shape[1]), int(w.shape[0])
        self.kernel, self.stride, self.padding = tuple(w.shape[2:]), stride, padding
        self.tf32 = precision == "tf32"
        self.bias = b.float().contiguous().to(device)
        self.w_3x3 = None
        if self.tf32:
            self.w_cols = pack_im2col_weight(w.double(), torch.float32).to(device)
            return
        self.w_cols = pack_im2col_weight(w.float()).to(device)
        if self.kernel == (3, 3) and stride == (1, 1) and padding == (1, 1):
            from .weights import pack_conv
            self.w_3x3 = pack_conv(w.float(), [self.c_in]).to(device)

    def __call__(self, x, out=None, c_off=0, shift=None, scale=None):
        """x NHWC bf16 [n, h, w, c_in] (fp32 with tf32; or NCHW fp32 pixels with shift / scale) -> ReLU(conv) NHWC bf16 (fp32 with tf32),
        written to channels [c_off, c_off + c_out) of `out` when given."""
        if self.tf32:
            return self._call_tf32(x, out, c_off, shift, scale)
        if x.dtype == torch.float32:
            n, _, h, w = x.shape
        else:
            n, h, w, _ = x.shape
        oh = ops.conv_out_size(h, self.kernel[0], self.stride[0], self.padding[0])
        ow = ops.conv_out_size(w, self.kernel[1], self.stride[1], self.padding[1])
        if out is None:
            out = torch.empty((n, oh, ow, self.c_out), dtype=torch.bfloat16, device=x.device)
        dst = out[..., c_off:c_off + self.c_out]
        if x.dtype == torch.bfloat16 and self.w_3x3 is not None and uses_implicit_3x3(self.kernel, self.stride, self.padding, ow):
            ops.conv2d([x], self.w_3x3, self.c_out, ksize=3, stride=1, pad_lo=1, bias=self.bias, act=ops.ACT_RELU, out=dst)
            return out
        if self.kernel == (1, 1) and self.stride == (1, 1) and self.padding == (0, 0) and x.dtype == torch.bfloat16:
            assert x.is_contiguous()
            a = x.view(n * h * w, self.c_in)
        else:
            a, _ = ops.im2col(x, self.kernel, self.stride, self.padding, self.w_cols.shape[1], shift=shift, scale=scale)
        ops.gemm(a, self.w_cols, self.c_out, bias=self.bias, act=ops.ACT_RELU, out=out.view(n * oh * ow, out.shape[3])[:, c_off:c_off + self.c_out])
        return out

    def _call_tf32(self, x, out, c_off, shift, scale):
        pixels = shift is not None
        n, h, w = (x.shape[0], x.shape[2], x.shape[3]) if pixels else x.shape[:3]
        oh = ops.conv_out_size(h, self.kernel[0], self.stride[0], self.padding[0])
        ow = ops.conv_out_size(w, self.kernel[1], self.stride[1], self.padding[1])
        if out is None:
            out = torch.empty((n, oh, ow, self.c_out), dtype=torch.float32, device=x.device)
        if self.kernel == (1, 1) and self.stride == (1, 1) and self.padding == (0, 0) and not pixels:
            assert x.dtype == torch.float32 and x.is_contiguous()
            a = x.view(n * h * w, self.c_in)
        else:
            a, _ = ops.im2col(x, self.kernel, self.stride, self.padding, self.w_cols.shape[1], shift=shift, scale=scale, dtype=torch.float32)
        ops.gemm_tf32(a, self.w_cols, self.c_out, out.view(n * oh * ow, out.shape[3]), c_off, bias=self.bias, relu=True)
        return out


class _Net(PackedModule):
    layers = None

    def __init__(self, precision="bf16"):
        if precision not in PRECISIONS:
            raise ValueError(f"{type(self).__name__}: precision must be one of {PRECISIONS}, got {precision!r}")
        self.precision = precision
        self.dtype = torch.float32 if precision == "tf32" else torch.bfloat16  # the activations'

    def _check_ready(self):
        if self.layers is None:
            raise RuntimeError(f"{type(self).__name__}: load a state dict and move it to a CUDA device first")


class FIDInceptionV3(_Net):
    def param_shapes(self):
        S = {}
        for name, (ci, co, k, _, _) in INCEPTION_LAYERS.items():
            S[f"{name}.conv.weight"] = (co, ci) + k
            for p in ("weight", "bias", "running_mean", "running_var"):
                S[f"{name}.bn.{p}"] = (co,)
            S[f"{name}.bn.num_batches_tracked"] = ()
        S["fc.weight"], S["fc.bias"] = (1008, 2048), (1008,)
        return S

    def _pack_weights(self):
        sd, dev = self._sd, self.device
        self.layers = {}
        for name, (_, _, _, s, p) in INCEPTION_LAYERS.items():
            w, b = fold_bn(sd[f"{name}.conv.weight"], sd[f"{name}.bn.weight"], sd[f"{name}.bn.bias"], sd[f"{name}.bn.running_mean"],
                           sd[f"{name}.bn.running_var"], INCEPTION_BN_EPS)
            self.layers[name] = _Conv(w, b, s, p, dev, self.precision)
        self.fc_weight = sd["fc.weight"].double().cpu()
        self.shift = torch.full((3,), 128.0, device=dev)
        self.scale = torch.full((3,), 128.0, device=dev)

    def _block_a(self, x, m):
        L = self.layers
        n, h, w, _ = x.shape
        pf = L[f"{m}.branch_pool"].c_out
        out = torch.empty((n, h, w, 224 + pf), dtype=self.dtype, device=x.device)
        L[f"{m}.branch1x1"](x, out, 0)
        L[f"{m}.branch5x5_2"](L[f"{m}.branch5x5_1"](x), out, 64)
        L[f"{m}.branch3x3dbl_3"](L[f"{m}.branch3x3dbl_2"](L[f"{m}.branch3x3dbl_1"](x)), out, 128)
        L[f"{m}.branch_pool"](ops.pool2d(x, 3, 1, 1, ops.POOL_AVG_EXCLUDE_PAD), out, 224)
        return out

    def _block_b(self, x, m):
        L = self.layers
        n, h, w, c = x.shape
        oh, ow = ops.conv_out_size(h, 3, 2, 0), ops.conv_out_size(w, 3, 2, 0)
        out = torch.empty((n, oh, ow, 480 + c), dtype=self.dtype, device=x.device)
        L[f"{m}.branch3x3"](x, out, 0)
        L[f"{m}.branch3x3dbl_3"](L[f"{m}.branch3x3dbl_2"](L[f"{m}.branch3x3dbl_1"](x)), out, 384)
        ops.pool2d(x, 3, 2, 0, ops.POOL_MAX, out=out, c_off=480)
        return out

    def _block_c(self, x, m):
        L = self.layers
        n, h, w, _ = x.shape
        out = torch.empty((n, h, w, 768), dtype=self.dtype, device=x.device)
        L[f"{m}.branch1x1"](x, out, 0)
        L[f"{m}.branch7x7_3"](L[f"{m}.branch7x7_2"](L[f"{m}.branch7x7_1"](x)), out, 192)
        t = x
        for i in range(1, 5):
            t = L[f"{m}.branch7x7dbl_{i}"](t)
        L[f"{m}.branch7x7dbl_5"](t, out, 384)
        L[f"{m}.branch_pool"](ops.pool2d(x, 3, 1, 1, ops.POOL_AVG_EXCLUDE_PAD), out, 576)
        return out

    def _block_d(self, x, m):
        L = self.layers
        n, h, w, c = x.shape
        oh, ow = ops.conv_out_size(h, 3, 2, 0), ops.conv_out_size(w, 3, 2, 0)
        out = torch.empty((n, oh, ow, 512 + c), dtype=self.dtype, device=x.device)
        L[f"{m}.branch3x3_2"](L[f"{m}.branch3x3_1"](x), out, 0)
        t = x
        for i in range(1, 4):
            t = L[f"{m}.branch7x7x3_{i}"](t)
        L[f"{m}.branch7x7x3_4"](t, out, 320)
        ops.pool2d(x, 3, 2, 0, ops.POOL_MAX, out=out, c_off=512)
        return out

    def _block_e(self, x, m, pool_mode):
        L = self.layers
        n, h, w, _ = x.shape
        out = torch.empty((n, h, w, 2048), dtype=self.dtype, device=x.device)
        L[f"{m}.branch1x1"](x, out, 0)
        t = L[f"{m}.branch3x3_1"](x)
        L[f"{m}.branch3x3_2a"](t, out, 320)
        L[f"{m}.branch3x3_2b"](t, out, 704)
        t = L[f"{m}.branch3x3dbl_2"](L[f"{m}.branch3x3dbl_1"](x))
        L[f"{m}.branch3x3dbl_3a"](t, out, 1088)
        L[f"{m}.branch3x3dbl_3b"](t, out, 1472)
        L[f"{m}.branch_pool"](ops.pool2d(x, 3, 1, 1, pool_mode), out, 1856)
        return out

    @torch.no_grad()
    def __call__(self, pixels):
        """pixels: NCHW fp32 [n, 3, 299, 299] with values in [0, 255] -> pool3 features fp32 [n, 2048] (device)."""
        self._check_ready()
        # CPU tensors only while the ABI calls are recorded instead of launched (tests/test_gpu_metrics_census.py)
        assert pixels.dtype == torch.float32 and pixels.dim() == 4 and pixels.shape[1] == 3 and (pixels.device.type == "cuda" or lib.RECORD is not None)
        L = self.layers
        x = L["Conv2d_1a_3x3"](pixels.contiguous(), shift=self.shift, scale=self.scale)
        x = L["Conv2d_2b_3x3"](L["Conv2d_2a_3x3"](x))
        x = ops.pool2d(x, 3, 2, 0, ops.POOL_MAX)
        x = L["Conv2d_4a_3x3"](L["Conv2d_3b_1x1"](x))
        x = ops.pool2d(x, 3, 2, 0, ops.POOL_MAX)
        for m in ("Mixed_5b", "Mixed_5c", "Mixed_5d"):
            x = self._block_a(x, m)
        x = self._block_b(x, "Mixed_6a")
        for m in ("Mixed_6b", "Mixed_6c", "Mixed_6d", "Mixed_6e"):
            x = self._block_c(x, m)
        x = self._block_d(x, "Mixed_7a")
        x = self._block_e(x, "Mixed_7b", ops.POOL_AVG_EXCLUDE_PAD)
        x = self._block_e(x, "Mixed_7c", ops.POOL_MAX)
        return ops.global_avg_pool(x)

    def unbiased_logits(self, features):
        """torch-fidelity's `logits_unbiased`: features @ fc.weight^T without the bias, in fp64 on the host -> CPU fp64 [n, 1008]."""
        self._check_ready()
        return features.detach().to("cpu", torch.float64) @ self.fc_weight.T

    def is_features(self, images01):
        """torchmetrics InceptionScore(normalize=True) input path: (x * 255).byte(), TF1 bilinear resize to 299 x 299, then the network;
        images01 NCHW fp32 in [0, 1] (device) -> unbiased logits CPU fp64 [n, 1008]."""
        return self.unbiased_logits(self(ops.resize_tf1_u8(images01.contiguous(), 299, 299)))


class LPIPSAlex(_Net):
    def param_shapes(self):
        S = {}
        for i, (ci, co, k, _, _) in ALEX_LAYERS.items():
            S[f"features.{i}.weight"], S[f"features.{i}.bias"] = (co, ci) + k, (co,)
        for t, c in enumerate(LPIPS_CHANNELS):
            S[f"lin{t}.model.1.weight"] = (1, c, 1, 1)
        return S

    def ignorable(self, key):
        return key.startswith("classifier.")  # torchvision's AlexNet file also holds the classifier

    def _pack_weights(self):
        sd, dev = self._sd, self.device
        self.layers = {i: _Conv(sd[f"features.{i}.weight"].double(), sd[f"features.{i}.bias"].double(), s, p, dev, self.precision)
                       for i, (_, _, _, s, p) in ALEX_LAYERS.items()}
        self.lins = [sd[f"lin{t}.model.1.weight"].reshape(-1).float().contiguous().to(dev) for t in range(5)]
        # [0,1] -> 2x - 1 -> (v - shift) / scale  ==  (x - (1 + shift) / 2) / (scale / 2)
        self.shift = torch.tensor([(1.0 + s) / 2 for s in LPIPS_SHIFT], dtype=torch.float32, device=dev)
        self.scale = torch.tensor([s / 2 for s in LPIPS_SCALE], dtype=torch.float32, device=dev)

    @torch.no_grad()
    def taps(self, images01):
        """AlexNet relu1..relu5 of NCHW fp32 images in [0, 1] (after the scaling layer): list of NHWC bf16 (fp32 with tf32) tensors."""
        self._check_ready()
        L = self.layers
        t1 = L[0](images01.contiguous(), shift=self.shift, scale=self.scale)
        t2 = L[3](ops.pool2d(t1, 3, 2, 0, ops.POOL_MAX))
        t3 = L[6](ops.pool2d(t2, 3, 2, 0, ops.POOL_MAX))
        t4 = L[8](t3)
        t5 = L[10](t4)
        return [t1, t2, t3, t4, t5]

    @torch.no_grad()
    def __call__(self, img0, img1):
        """LPIPS distance of each pair: NCHW fp32 [n, 3, H, W] in [0, 1] (device) -> fp32 [n] (device)."""
        assert img0.shape == img1.shape and img0.dtype == torch.float32 and img1.dtype == torch.float32
        n = img0.shape[0]
        taps = self.taps(torch.cat([img0, img1], dim=0))
        acc = torch.zeros(n, dtype=torch.float32, device=img0.device)
        for t, lin in zip(taps, self.lins):
            ops.lpips_layer_(t[:n], t[n:], lin, acc)
        return acc


def ssim(x, y):
    """Per-image SSIM of NCHW fp32 images in [0, 1] (device) -> fp32 [n] (device); torchmetrics averages these over the images."""
    return ops.ssim(x.contiguous(), y.contiguous())


def random_state_dict(shapes, seed):
    """Seeded random weights of the right shapes (He-normal convolutions, identity BatchNorm statistics, non-negative LPIPS `lin`
    weights), for synthetic runs without the weight files."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for k, shp in sorted(shapes.items()):
        if k.endswith("num_batches_tracked"):
            sd[k] = torch.zeros((), dtype=torch.long)
        elif k.endswith("running_var") or k.endswith("bn.weight"):
            sd[k] = torch.ones(shp)
        elif k.endswith("running_mean") or k.endswith("bias"):
            sd[k] = torch.zeros(shp)
        elif k.startswith("lin"):
            sd[k] = torch.rand(shp, generator=g) * 0.1
        else:
            fan_in = math.prod(shp[1:])
            sd[k] = torch.randn(shp, generator=g) * math.sqrt(2.0 / fan_in)
    return sd


# ---- host statistics (fp64) -----------------------------------------------------------------------------------------------------------
def feature_stats(feats):
    """(mu, sigma) of features [n, d] as clean-fid stores them: mean over rows, np.cov(rowvar=False)."""
    f = np.asarray(feats, dtype=np.float64)
    return f.mean(axis=0), np.cov(f, rowvar=False)


def frechet_distance(mu1, sigma1, mu2, sigma2, eps=1e-6):
    """|mu1 - mu2|^2 + tr(sigma1 + sigma2 - 2 sqrtm(sigma1 sigma2)); when the product's square root is not finite, it is retried with
    eps added to both diagonals (clean-fid's frechet_distance)."""
    from scipy import linalg
    mu1, mu2 = np.atleast_1d(mu1).astype(np.float64), np.atleast_1d(mu2).astype(np.float64)
    sigma1, sigma2 = np.atleast_2d(sigma1).astype(np.float64), np.atleast_2d(sigma2).astype(np.float64)
    diff = mu1 - mu2
    covmean = linalg.sqrtm(sigma1.dot(sigma2))
    if not np.isfinite(covmean).all():
        offset = np.eye(sigma1.shape[0]) * eps
        covmean = linalg.sqrtm((sigma1 + offset).dot(sigma2 + offset))
    if np.iscomplexobj(covmean):
        if not np.allclose(np.diagonal(covmean).imag, 0, atol=1e-3):
            raise ValueError(f"frechet_distance: imaginary component {np.max(np.abs(covmean.imag))}")
        covmean = covmean.real
    return float(diff.dot(diff) + np.trace(sigma1) + np.trace(sigma2) - 2 * np.trace(covmean))


def kernel_distance(feats1, feats2, num_subsets=100, max_subset_size=1000, seed=0):
    """clean-fid's KID: unbiased MMD^2 with the polynomial kernel k(x, y) = (x.y / d + 1)^3, averaged over `num_subsets` random subsets
    of m = min(n1, n2, max_subset_size) rows of each set (drawn without replacement, feats2 first) from a generator seeded with `seed`."""
    f1, f2 = np.asarray(feats1, dtype=np.float64), np.asarray(feats2, dtype=np.float64)
    rng = np.random.RandomState(seed)
    d = f1.shape[1]
    m = min(f1.shape[0], f2.shape[0], max_subset_size)
    t = 0.0
    for _ in range(num_subsets):
        x = f2[rng.choice(f2.shape[0], m, replace=False)]
        y = f1[rng.choice(f1.shape[0], m, replace=False)]
        a = (x @ x.T / d + 1) ** 3 + (y @ y.T / d + 1) ** 3
        b = (x @ y.T / d + 1) ** 3
        t += (a.sum() - np.diag(a).sum()) / (m - 1) - b.sum() * 2 / m
    return float(t / num_subsets / m)


def inception_score(logits, splits=10, seed=0):
    """torchmetrics InceptionScore.compute on unbiased logits [n, classes]: rows shuffled by a seeded permutation, cut into chunks of
    ceil(n / splits) rows (torch.chunk), per chunk exp(mean_i KL(p_i || mean p)) -> (mean, unbiased std) over the chunks."""
    z = np.asarray(logits, dtype=np.float64)
    z = z[np.random.RandomState(seed).permutation(z.shape[0])]
    z = z - z.max(axis=1, keepdims=True)
    log_p = z - np.log(np.exp(z).sum(axis=1, keepdims=True))
    p = np.exp(log_p)
    size = -(-z.shape[0] // splits)
    scores = []
    for i in range(0, z.shape[0], size):
        pc, lc = p[i:i + size], log_p[i:i + size]
        kl = (pc * (lc - np.log(pc.mean(axis=0, keepdims=True)))).sum(axis=1).mean()
        scores.append(math.exp(kl))
    scores = np.array(scores)
    return float(scores.mean()), float(scores.std(ddof=1)) if len(scores) > 1 else float("nan")
