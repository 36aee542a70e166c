"""The perceptual loss of the reference's warping trainer (src/utils/vgg_loss.py) on the H100 engine.

  * `VGG19` -- torchvision's `vgg19().features[0:30]`, the five slices of vgg_loss.py:7-37 (relu1_1, relu2_1, relu3_1, relu4_1, relu5_1).
    State dict: torchvision's own keys (`features.<N>.weight / bias`, file `vgg19-dcbb9e9d.pth`); the classifier and the convolutions
    past relu5_1 (`features.30` on) are accepted and dropped.  `taps(images)` takes NCHW fp32 images in [-1, 1] and applies the loss's
    `(x + 1) / 2` and ImageNet normalisation itself, inside the first im2col, before the zero padding.
  * `VGGLoss` -- vgg_loss.py:40-68: `Resize(256, antialias=True)` (the short side to 256: 512x384 -> 341x256), the normalisation, and
    1/32, 1/16, 1/8, 1/4, 1 times the `L1Loss` of each tap.  x and y run as one batch of 2B, so each layer is one GEMM per image chunk.
  * `L1Loss` -- nn.L1Loss() (mean reduction).

One precision, TF32: the reference runs this module in fp32, and cuDNN runs fp32 convolutions on TF32 tensor cores by default on Ampere
and Hopper (the argument of metrics.py's precision="tf32").  Activations are fp32 NHWC; every 3x3 convolution is `ladi_im2col_f32` over
a chunk of images (the im2col rows of conv1_2 at 341x256 are 200 MB per image; a chunk holds at most IM2COL_BYTES) and one
`ladi_gemm_tf32` with the ReLU epilogue; the max pools are `ladi_pool2d_f32`; each L1 term is one `ladi_l1_mean_f32`, which adds
weight * mean|a - b| to a device accumulator in a fixed order, so a loss is read back once and two runs give the same bits.
"""
import torch

from . import ops
from .metrics import pack_im2col_weight
from .module import PackedModule

VGG_FILE = "vgg19-dcbb9e9d.pth"
# torchvision vgg19().features up to relu5_1: index of each 3x3 pad-1 convolution -> (c_in, c_out); a ReLU follows each
CONVS = {0: (3, 64), 2: (64, 64), 5: (64, 128), 7: (128, 128), 10: (128, 256), 12: (256, 256), 14: (256, 256), 16: (256, 256),
         19: (256, 512), 21: (512, 512), 23: (512, 512), 25: (512, 512), 28: (512, 512)}
POOLS = (4, 9, 18, 27)  # MaxPool2d(2, 2)
TAPS = (0, 5, 10, 19, 28)  # the convolutions whose ReLUs end slice1..slice5 (vgg_loss.py:17-26)
LAST = 30
LOSS_WEIGHTS = (1.0 / 32, 1.0 / 16, 1.0 / 8, 1.0 / 4, 1.0)  # vgg_loss.py:51
MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)  # vgg_loss.py:52-53
RESIZE = 256  # vgg_loss.py:54
IM2COL_BYTES = 512 << 20
GEMM_MAX_ROWS = 8388480  # ladi_gemm_tf32: at most 65535 tiles of 128 rows


def resized_size(h, w, size=RESIZE):
    """torchvision Resize(size) with an int size: the short side becomes `size`, the long one int(size * long / short)."""
    return (int(size * h / w), size) if w <= h else (size, int(size * w / h))


class VGG19(PackedModule):
    def param_shapes(self):
        S = {}
        for i, (ci, co) in CONVS.items():
            S[f"features.{i}.weight"], S[f"features.{i}.bias"] = (co, ci, 3, 3), (co,)
        return S

    def ignorable(self, key):
        parts = key.split(".")
        return parts[0] == "classifier" or (parts[0] == "features" and parts[1].isdigit() and int(parts[1]) >= LAST)

    def _pack_weights(self):
        sd, dev = self._sd, self.device
        self.P = {i: (pack_im2col_weight(sd[f"features.{i}.weight"].double(), torch.float32).to(dev),
                      sd[f"features.{i}.bias"].float().contiguous().to(dev)) for i in CONVS}
        # (x + 1) / 2, then (v - mean) / std  ==  (x - (2 mean - 1)) / (2 std), applied by the pixel im2col before the zero padding
        self.shift = torch.tensor([2 * m - 1 for m in MEAN], dtype=torch.float32, device=dev)
        self.scale = torch.tensor([2 * s for s in STD], dtype=torch.float32, device=dev)

    def _conv(self, i, x):
        """ReLU(conv3x3 pad 1) of NHWC fp32 activations, or of NCHW fp32 [-1, 1] images for the first layer -> NHWC fp32."""
        w, b = self.P[i]
        co, k = CONVS[i][1], w.shape[1]
        pixels = i == 0
        n, h, wd = (x.shape[0], x.shape[2], x.shape[3]) if pixels else x.shape[:3]
        out = torch.empty((n, h, wd, co), dtype=torch.float32, device=x.device)
        chunk = max(1, min(IM2COL_BYTES // (h * wd * k * 4), GEMM_MAX_ROWS // (h * wd)))
        for s in range(0, n, chunk):
            e = min(n, s + chunk)
            a, _ = ops.im2col(x[s:e], (3, 3), (1, 1), (1, 1), k, shift=self.shift if pixels else None, scale=self.scale if pixels else None,
                              dtype=torch.float32)
            ops.gemm_tf32(a, w, co, out[s:e].view(-1, co), 0, bias=b, relu=True)
        return out

    @torch.no_grad()
    def taps(self, images):
        """relu1_1, relu2_1, relu3_1, relu4_1, relu5_1 (NHWC fp32) of NCHW fp32 images in [-1, 1], normalised as VGGLoss does."""
        if self.P is None:
            raise RuntimeError("VGG19: load_state_dict(...) and .to('cuda') first")
        assert images.dtype == torch.float32 and images.dim() == 4 and images.shape[1] == 3
        x, out = images.contiguous(), []
        for i in range(LAST):
            if i in CONVS:
                x = self._conv(i, x)
                if i in TAPS:
                    out.append(x)
            elif i in POOLS:
                x = ops.pool2d(x, 2, 2, 0, ops.POOL_MAX)
        return out


class L1Loss:
    """nn.L1Loss(): mean |a - b| of two fp32 tensors of one shape, on the device."""

    def __call__(self, a, b, acc=None, weight=1.0):
        """Adds weight * mean|a - b| to `acc` (one-element fp32 device tensor) when given; returns the accumulator (a new one otherwise)."""
        if acc is None:
            acc = torch.zeros(1, dtype=torch.float32, device=a.device)
        return ops.l1_mean_(a.contiguous(), b.contiguous(), acc, weight)


class VGGLoss:
    """vgg_loss.py:40-68.  `load_state_dict` takes torchvision's vgg19 state dict; `.to("cuda")` packs it."""

    def __init__(self, vgg=None):
        self.vgg = vgg if vgg is not None else VGG19()
        self.weights = list(LOSS_WEIGHTS)
        self.criterion = L1Loss()

    def load_state_dict(self, sd, strict=True):
        self.vgg.load_state_dict(sd, strict)
        return self

    def to(self, device=None, dtype=None, **kw):
        self.vgg.to(device, dtype, **kw)
        return self

    def eval(self):
        return self

    @property
    def device(self):
        return self.vgg.device

    @torch.no_grad()
    def __call__(self, x, y, acc=None):
        """x, y NCHW fp32 [B, 3, H, W] in [-1, 1] -> `acc` + the loss (one-element fp32 device tensor), summed over the taps in the
        reference's order."""
        assert x.shape == y.shape and x.dim() == 4 and x.shape[1] == 3
        dev = self.vgg.device
        B, _, H, W = x.shape
        oh, ow = resized_size(H, W)
        xy = torch.empty((2 * B, 3, oh, ow), dtype=torch.float32, device=dev)
        ops.resize_aa_f32(x.to(dev, torch.float32).contiguous(), oh, ow, out=xy[:B])
        ops.resize_aa_f32(y.to(dev, torch.float32).contiguous(), oh, ow, out=xy[B:])
        if acc is None:
            acc = torch.zeros(1, dtype=torch.float32, device=dev)
        for t, w in zip(self.vgg.taps(xy), self.weights):
            c = t.shape[3]
            ops.l1_mean_(t[:B].view(-1, c), t[B:].view(-1, c), acc, w)
        return acc
