"""TEST INFRASTRUCTURE ONLY (see oracle/ladi_oracle/__init__.py) -- fp32 CPU restatement of the warping trainer's perceptual loss,
src/utils/vgg_loss.py:

  * `VGG19`   <- vgg_loss.py:7-37: torchvision's `vgg19().features[0:30]` (Conv2d 3x3 pad 1, ReLU(inplace=True), MaxPool2d(2, 2)) with
                 its module indices, so torchvision's state-dict keys `features.<N>.*` load unchanged (`load_torchvision` drops the
                 classifier and `features.30` on); `forward` -> [relu1_1, relu2_1, relu3_1, relu4_1, relu5_1].
  * `VGGLoss` <- vgg_loss.py:40-68: Resize(256, antialias=True) (the short side to 256), (x + 1) / 2, ImageNet mean / std, and
                 1/32 .. 1 times the L1Loss of each tap.

Pinned: the taps bit for bit against torchvision's own `vgg19().features` slices, and the loss through tests/golden/tps_val_small.npz.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

CFG = [64, 64, "M", 128, 128, "M", 256, 256, 256, 256, "M", 512, 512, 512, 512, "M", 512]  # torchvision cfg "E" up to conv5_1
TAP_INDEX = (1, 6, 11, 20, 29)  # the last module of slice1..slice5 (vgg_loss.py:17-26)


def resized_size(h, w, size=256):
    """torchvision Resize(size) with an int size: the short side becomes `size`, the long one int(size * long / short)."""
    return (int(size * h / w), size) if w <= h else (size, int(size * w / h))


class VGG19(nn.Module):
    def __init__(self):
        super().__init__()
        layers, c = [], 3
        for v in CFG:
            if v == "M":
                layers.append(nn.MaxPool2d(kernel_size=2, stride=2))
            else:
                layers += [nn.Conv2d(c, v, kernel_size=3, padding=1), nn.ReLU(inplace=True)]
                c = v
        self.features = nn.Sequential(*layers)
        assert len(self.features) == 30

    def load_torchvision(self, sd):
        keep = {k: v for k, v in sd.items() if k.startswith("features.") and int(k.split(".")[1]) < 30}
        self.load_state_dict(keep)
        return self

    def forward(self, x):
        out = []
        for i, m in enumerate(self.features):
            x = m(x)
            if i in TAP_INDEX:
                out.append(x)
        return out


class VGGLoss(nn.Module):
    def __init__(self, vgg):
        super().__init__()
        self.vgg = vgg.eval()
        self.weights = [1.0 / 32, 1.0 / 16, 1.0 / 8, 1.0 / 4, 1.0]
        self.register_buffer("mean", torch.tensor([0.485, 0.456, 0.406]).view(1, 3, 1, 1))
        self.register_buffer("std", torch.tensor([0.229, 0.224, 0.225]).view(1, 3, 1, 1))

    def prepare(self, x):
        x = F.interpolate(x, size=resized_size(*x.shape[-2:]), mode="bilinear", align_corners=False, antialias=True)
        return ((x + 1) / 2 - self.mean) / self.std

    def forward(self, x, y):
        xv, yv = self.vgg(self.prepare(x)), self.vgg(self.prepare(y))
        loss = 0
        for w, a, b in zip(self.weights, xv, yv):
            loss += w * F.l1_loss(a, b)
        return loss
