"""fp32 / fp64 PyTorch restatement of the five metrics of the reference's src/utils/val_metrics.py and of the two networks behind them, the
checker for ladi_vton_b200/metrics.py and ladi_vton_b200/val_metrics.py.

The libraries the reference calls (clean-fid, torchmetrics, lpips, torch-fidelity) are not installed here, so their constants are
restated from memory of their public sources.  Every such constant is in the RECALLED block below and marked [recalled]; agreement with
the real libraries' numbers cannot be checked offline.  The networks are functional forwards over torchvision-layout state dicts
(F.conv2d / F.batch_norm / pools in fp32), checked against torchvision's own Inception-v3 and AlexNet modules by tests/test_metrics.py.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

# ---- RECALLED ---------------------------------------------------------------------------------------------------------------------------
LPIPS_SHIFT = (-0.030, -0.088, -0.188)   # [recalled] lpips ScalingLayer shift (v0.1)
LPIPS_SCALE = (0.458, 0.448, 0.450)      # [recalled] lpips ScalingLayer scale
LPIPS_EPS = 1e-10                        # [recalled] lpips normalize_tensor: x / (sqrt(sum x^2) + eps)
SSIM_KERNEL, SSIM_SIGMA = 11, 1.5        # [recalled] torchmetrics SSIM defaults: gaussian window 11, sigma 1.5
SSIM_CROP = (SSIM_KERNEL - 1) // 2       # [recalled] torchmetrics reflect-pads by 5, convolves, crops 5 on every side
SSIM_K1, SSIM_K2 = 0.01, 0.03            # [recalled] C1 = (K1 * data_range)^2, C2 = (K2 * data_range)^2
CLEAN_RESIZE = (299, 299)                # [recalled] clean-fid "clean": per-channel PIL mode 'F' BICUBIC resize, then clip(0, 255)
INCEPTION_NORM = (128.0, 128.0)          # [recalled] (x - 128) / 128 on 0..255 inputs (FID Inception input scaling)
KID_SUBSETS, KID_SUBSET_SIZE = 100, 1000 # [recalled] clean-fid kernel_distance: 100 subsets of <= 1000, kernel (x.y / d + 1)^3
TF1_RESIZE = "o * in / out, floor, +1 clamped"  # [recalled] torch-fidelity interpolate_bilinear_2d_like_tensorflow1x (align_corners=False)
UNBIASED_LOGITS = "features @ fc.weight.T"      # [recalled] torch-fidelity 'logits_unbiased': the fc layer without its bias
IS_SPLITS = 10                           # [recalled] torchmetrics InceptionScore(splits=10), torch.chunk splits, torch.randperm order
INCEPTION_BN_EPS = 1e-3                  # torchvision BasicConv2d BatchNorm2d(eps=0.001)


# ---- FID Inception-v3 -------------------------------------------------------------------------------------------------------------------
def _bconv(sd, name, x, stride=1, padding=0):
    x = F.conv2d(x, sd[f"{name}.conv.weight"], None, stride, padding)
    x = F.batch_norm(x, sd[f"{name}.bn.running_mean"], sd[f"{name}.bn.running_var"], sd[f"{name}.bn.weight"], sd[f"{name}.bn.bias"],
                     False, 0.0, INCEPTION_BN_EPS)
    return F.relu(x)


def _a(sd, m, x):
    b1 = _bconv(sd, f"{m}.branch1x1", x)
    b5 = _bconv(sd, f"{m}.branch5x5_2", _bconv(sd, f"{m}.branch5x5_1", x), padding=2)
    b3 = _bconv(sd, f"{m}.branch3x3dbl_1", x)
    b3 = _bconv(sd, f"{m}.branch3x3dbl_3", _bconv(sd, f"{m}.branch3x3dbl_2", b3, padding=1), padding=1)
    bp = _bconv(sd, f"{m}.branch_pool", F.avg_pool2d(x, 3, 1, 1, count_include_pad=False))
    return torch.cat([b1, b5, b3, bp], 1)


def _b(sd, m, x):
    b3 = _bconv(sd, f"{m}.branch3x3", x, stride=2)
    bd = _bconv(sd, f"{m}.branch3x3dbl_2", _bconv(sd, f"{m}.branch3x3dbl_1", x), padding=1)
    bd = _bconv(sd, f"{m}.branch3x3dbl_3", bd, stride=2)
    return torch.cat([b3, bd, F.max_pool2d(x, 3, 2)], 1)


def _c(sd, m, x):
    b1 = _bconv(sd, f"{m}.branch1x1", x)
    b7 = _bconv(sd, f"{m}.branch7x7_1", x)
    b7 = _bconv(sd, f"{m}.branch7x7_2", b7, padding=(0, 3))
    b7 = _bconv(sd, f"{m}.branch7x7_3", b7, padding=(3, 0))
    bd = _bconv(sd, f"{m}.branch7x7dbl_1", x)
    for i, p in ((2, (3, 0)), (3, (0, 3)), (4, (3, 0)), (5, (0, 3))):
        bd = _bconv(sd, f"{m}.branch7x7dbl_{i}", bd, padding=p)
    bp = _bconv(sd, f"{m}.branch_pool", F.avg_pool2d(x, 3, 1, 1, count_include_pad=False))
    return torch.cat([b1, b7, bd, bp], 1)


def _d(sd, m, x):
    b3 = _bconv(sd, f"{m}.branch3x3_2", _bconv(sd, f"{m}.branch3x3_1", x), stride=2)
    b7 = _bconv(sd, f"{m}.branch7x7x3_1", x)
    b7 = _bconv(sd, f"{m}.branch7x7x3_2", b7, padding=(0, 3))
    b7 = _bconv(sd, f"{m}.branch7x7x3_3", b7, padding=(3, 0))
    b7 = _bconv(sd, f"{m}.branch7x7x3_4", b7, stride=2)
    return torch.cat([b3, b7, F.max_pool2d(x, 3, 2)], 1)


def _e(sd, m, x, max_pool):
    b1 = _bconv(sd, f"{m}.branch1x1", x)
    t = _bconv(sd, f"{m}.branch3x3_1", x)
    b3 = torch.cat([_bconv(sd, f"{m}.branch3x3_2a", t, padding=(0, 1)), _bconv(sd, f"{m}.branch3x3_2b", t, padding=(1, 0))], 1)
    t = _bconv(sd, f"{m}.branch3x3dbl_2", _bconv(sd, f"{m}.branch3x3dbl_1", x), padding=1)
    bd = torch.cat([_bconv(sd, f"{m}.branch3x3dbl_3a", t, padding=(0, 1)), _bconv(sd, f"{m}.branch3x3dbl_3b", t, padding=(1, 0))], 1)
    pool = F.max_pool2d(x, 3, 1, 1) if max_pool else F.avg_pool2d(x, 3, 1, 1, count_include_pad=False)
    return torch.cat([b1, b3, bd, _bconv(sd, f"{m}.branch_pool", pool)], 1)


def inception_trunk(sd, x):
    """FID Inception-v3 (torchvision layout, FID pool variants) on already-normalised NCHW fp32 input -> pool3 features [n, 2048]."""
    x = _bconv(sd, "Conv2d_1a_3x3", x, stride=2)
    x = _bconv(sd, "Conv2d_2a_3x3", x)
    x = _bconv(sd, "Conv2d_2b_3x3", x, padding=1)
    x = F.max_pool2d(x, 3, 2)
    x = _bconv(sd, "Conv2d_4a_3x3", _bconv(sd, "Conv2d_3b_1x1", x))
    x = F.max_pool2d(x, 3, 2)
    for m in ("Mixed_5b", "Mixed_5c", "Mixed_5d"):
        x = _a(sd, m, x)
    x = _b(sd, "Mixed_6a", x)
    for m in ("Mixed_6b", "Mixed_6c", "Mixed_6d", "Mixed_6e"):
        x = _c(sd, m, x)
    x = _d(sd, "Mixed_7a", x)
    x = _e(sd, "Mixed_7b", x, max_pool=False)
    x = _e(sd, "Mixed_7c", x, max_pool=True)
    return F.adaptive_avg_pool2d(x, 1).flatten(1)


def inception_features(sd, pixels255):
    """pixels NCHW fp32 in [0, 255], 299 x 299 -> (pool3 features fp32 [n, 2048], unbiased logits fp64 [n, 1008])."""
    shift, scale = INCEPTION_NORM
    f = inception_trunk(sd, (pixels255 - shift) / scale)
    return f, f.double() @ sd["fc.weight"].double().T


def calibrate_batchnorm(sd, pixels255):
    """Set every BatchNorm's running statistics to the batch statistics of one pass over `pixels255` (in place), layer by layer, so
    that a randomly initialised network keeps O(1) activations: each BN sees the output of the already-calibrated layers before it."""
    shift, scale = INCEPTION_NORM
    orig = F.batch_norm

    def bn(x, running_mean, running_var, weight=None, bias=None, training=False, momentum=0.1, eps=1e-5):
        xd = x.double()
        mean, var = xd.mean(dim=(0, 2, 3)), xd.var(dim=(0, 2, 3), unbiased=False)
        running_mean.copy_(mean.float())
        running_var.copy_(var.float())
        return orig(x, running_mean, running_var, weight, bias, False, 0.0, eps)

    F.batch_norm = bn
    try:
        inception_trunk(sd, (pixels255 - shift) / scale)
    finally:
        F.batch_norm = orig


# ---- LPIPS (AlexNet) -------------------------------------------------------------------------------------------------------------------
def alexnet_taps(sd, x):
    """torchvision AlexNet `features` on NCHW fp32 input, outputs after ReLU 1..5 (lpips.pretrained_networks.alexnet slices)."""
    t = []
    x = F.relu(F.conv2d(x, sd["features.0.weight"], sd["features.0.bias"], 4, 2)); t.append(x)
    x = F.max_pool2d(x, 3, 2)
    x = F.relu(F.conv2d(x, sd["features.3.weight"], sd["features.3.bias"], 1, 2)); t.append(x)
    x = F.max_pool2d(x, 3, 2)
    x = F.relu(F.conv2d(x, sd["features.6.weight"], sd["features.6.bias"], 1, 1)); t.append(x)
    x = F.relu(F.conv2d(x, sd["features.8.weight"], sd["features.8.bias"], 1, 1)); t.append(x)
    x = F.relu(F.conv2d(x, sd["features.10.weight"], sd["features.10.bias"], 1, 1)); t.append(x)
    return t


def lpips_scaling(img01):
    """torchmetrics normalize=True ([0, 1] -> [-1, 1]) then the LPIPS ScalingLayer."""
    shift = torch.tensor(LPIPS_SHIFT, dtype=img01.dtype, device=img01.device).view(1, 3, 1, 1)
    scale = torch.tensor(LPIPS_SCALE, dtype=img01.dtype, device=img01.device).view(1, 3, 1, 1)
    return (2 * img01 - 1 - shift) / scale


def lpips(sd, img0, img1):
    """LPIPS distance per pair, fp32 [n]."""
    t0, t1 = alexnet_taps(sd, lpips_scaling(img0)), alexnet_taps(sd, lpips_scaling(img1))
    out = 0
    for k, (a, b) in enumerate(zip(t0, t1)):
        na = a / (torch.sqrt((a * a).sum(1, keepdim=True)) + LPIPS_EPS)
        nb = b / (torch.sqrt((b * b).sum(1, keepdim=True)) + LPIPS_EPS)
        d = F.conv2d((na - nb) ** 2, sd[f"lin{k}.model.1.weight"])
        out = out + d.mean(dim=(2, 3)).flatten()
    return out


# ---- SSIM -------------------------------------------------------------------------------------------------------------------------------
def ssim(x, y, dtype=torch.float64):
    """Per-image SSIM (torchmetrics, data_range = 1): mean over channels and the positions whose window lies inside the image."""
    x, y = x.to(dtype), y.to(dtype)
    c = x.shape[1]
    d = torch.arange(SSIM_KERNEL, dtype=dtype) - (SSIM_KERNEL - 1) / 2
    g = torch.exp(-0.5 * (d / SSIM_SIGMA) ** 2)
    g = g / g.sum()
    k2 = (g[:, None] * g[None, :]).expand(c, 1, SSIM_KERNEL, SSIM_KERNEL).to(x.device)
    x_p = F.pad(x, [SSIM_CROP] * 4, mode="reflect")
    y_p = F.pad(y, [SSIM_CROP] * 4, mode="reflect")
    outs = F.conv2d(torch.cat([x_p, y_p, x_p * x_p, y_p * y_p, x_p * y_p]), k2, groups=c)
    n = x.shape[0]
    mx, my, exx, eyy, exy = outs.split(n)
    c1, c2 = SSIM_K1 ** 2, SSIM_K2 ** 2
    vx, vy, cxy = exx - mx * mx, eyy - my * my, exy - mx * my
    s = ((2 * mx * my + c1) * (2 * cxy + c2)) / ((mx * mx + my * my + c1) * (vx + vy + c2))
    s = s[..., SSIM_CROP:-SSIM_CROP, SSIM_CROP:-SSIM_CROP]
    return s.reshape(n, -1).mean(-1)


# ---- resizes ----------------------------------------------------------------------------------------------------------------------------
def resize_tf1_u8(img01, oh, ow):
    """(x * 255).byte() then TF1-style bilinear resize (NCHW fp32)."""
    x = (img01 * 255).to(torch.uint8).float()
    h, w = x.shape[2:]
    fy = torch.arange(oh, dtype=torch.float32) * (h / oh)
    fx = torch.arange(ow, dtype=torch.float32) * (w / ow)
    y0 = fy.floor().long().clamp(max=h - 1); x0 = fx.floor().long().clamp(max=w - 1)
    y1 = (y0 + 1).clamp(max=h - 1); x1 = (x0 + 1).clamp(max=w - 1)
    ly = (fy - y0.float()).view(1, 1, oh, 1).to(x.device); lx = (fx - x0.float()).view(1, 1, 1, ow).to(x.device)
    y0, y1, x0, x1 = (t.to(x.device) for t in (y0, y1, x0, x1))
    tl, tr = x[:, :, y0][:, :, :, x0], x[:, :, y0][:, :, :, x1]
    bl, br = x[:, :, y1][:, :, :, x0], x[:, :, y1][:, :, :, x1]
    top, bot = tl + (tr - tl) * lx, bl + (br - bl) * lx
    return top + (bot - top) * ly


def clean_resize(img_u8_hwc):
    """clean-fid "clean" resize of one uint8 HWC RGB image -> float32 HWC 299 x 299 in [0, 255]."""
    from PIL import Image
    chans = [np.asarray(Image.fromarray(img_u8_hwc[:, :, c].astype(np.float32), mode="F").resize(CLEAN_RESIZE, resample=Image.BICUBIC))
             .clip(0, 255) for c in range(3)]
    return np.stack(chans, axis=2).astype(np.float32)


# ---- statistics -------------------------------------------------------------------------------------------------------------------------
def frechet_distance(mu1, sigma1, mu2, sigma2):
    from scipy import linalg
    covmean = linalg.sqrtm(sigma1 @ sigma2)
    if np.iscomplexobj(covmean):
        covmean = covmean.real
    diff = mu1 - mu2
    return float(diff @ diff + np.trace(sigma1) + np.trace(sigma2) - 2 * np.trace(covmean))


def kernel_distance_direct(feats1, feats2, num_subsets=KID_SUBSETS, max_subset_size=KID_SUBSET_SIZE, seed=0):
    """KID with explicit double loops over each subset's pairs (same subsets as ladi_vton_b200.metrics.kernel_distance)."""
    rng = np.random.RandomState(seed)
    d = feats1.shape[1]
    m = min(feats1.shape[0], feats2.shape[0], max_subset_size)
    k = lambda a, b: (float(a @ b) / d + 1) ** 3  # noqa: E731
    total = 0.0
    for _ in range(num_subsets):
        x = feats2[rng.choice(feats2.shape[0], m, replace=False)]
        y = feats1[rng.choice(feats1.shape[0], m, replace=False)]
        kxx = sum(k(x[i], x[j]) for i in range(m) for j in range(m) if i != j)
        kyy = sum(k(y[i], y[j]) for i in range(m) for j in range(m) if i != j)
        kxy = sum(k(x[i], y[j]) for i in range(m) for j in range(m))
        total += (kxx + kyy) / (m * (m - 1)) - 2 * kxy / (m * m)
    return total / num_subsets


def inception_score(logits, splits=IS_SPLITS, seed=0):
    z = torch.as_tensor(np.asarray(logits), dtype=torch.float64)
    z = z[torch.as_tensor(np.random.RandomState(seed).permutation(z.shape[0]))]
    p, lp = z.softmax(1), z.log_softmax(1)
    scores = []
    for pc, lc in zip(p.chunk(splits, 0), lp.chunk(splits, 0)):
        scores.append((pc * (lc - pc.mean(0, keepdim=True).log())).sum(1).mean().exp())
    s = torch.stack(scores)
    return float(s.mean()), float(s.std()) if len(scores) > 1 else math.nan
