"""Synthetic workload of BASELINE.json / SURVEY.md section 8(d): person/garment/pose/mask tensors shaped like the outputs of
src/dataset/vitonhd.py (image, cloth in [-1,1]; 18 Gaussian pose heat-maps; binary inpaint mask) and
random-init weights of the reference architectures (hubconf.py:16-53), all seeded (CLI default seed 1234,
src/inference.py:57).  No dataset, checkpoint or network access is needed."""
import math

import torch

from .unet import unet_param_shapes
from .vae import vae_param_shapes

EMASC_IN, EMASC_OUT = [128, 128, 128, 256, 512], [128, 256, 512, 512, 512]  # hubconf.py:41-42


def emasc_channels(vae_ch):
    c = list(vae_ch)
    return [c[0], c[0], c[0], c[1], c[2]], [c[0], c[1], c[2], c[3], c[3]]


def emasc_param_shapes(cin, cout, kernel_size=3, type="nonlinear"):
    """State-dict shapes of src/models/emasc.py's EMASC (the linear form is always 3x3, emasc.py:21-24)."""
    S = {}
    for i, (a, b) in enumerate(zip(cin, cout)):
        if type == "linear":
            S[f"conv.{i}.weight"], S[f"conv.{i}.bias"] = (b, a, 3, 3), (b,)
            continue
        k = kernel_size
        S[f"conv.{i}.0.weight"], S[f"conv.{i}.0.bias"] = (a, a, k, k), (a,)
        S[f"conv.{i}.2.weight"], S[f"conv.{i}.2.bias"] = (b, a, k, k), (b,)
    return S


def is_norm_key(k):
    """True for the weight / bias of a GroupNorm or LayerNorm (UNet, VAE, CLIP and inversion-adapter key names)."""
    leaf = k.rsplit(".", 1)[0].rsplit(".", 1)[-1]
    return leaf.startswith("norm") or leaf in ("group_norm", "conv_norm_out", "layer_norm1", "layer_norm2", "post_layernorm", "final_layer_norm", "pre_layrnorm")


def random_state_dict(shapes, seed, device="cpu", fast=False):
    """PyTorch-default-like init (U(-1/sqrt(fan_in), 1/sqrt(fan_in)) for conv/linear weights and biases, ones/zeros for
    norms), drawn in key order from one seeded generator on `device` (CPU draws are reproducible across machines and are
    what the parity tests share between oracle and engine; bench.py draws on the GPU to skip the host cost)."""
    g = torch.Generator(device=device).manual_seed(seed)
    sd = {}
    fan = {}
    block = torch.empty(1 << 22, device=device).uniform_(-1.0, 1.0, generator=g) if fast else None
    for k, shp in shapes.items():
        base = k.rsplit(".", 1)[0]
        if is_norm_key(k):
            sd[k] = torch.ones(shp, device=device) if k.endswith("weight") else torch.zeros(shp, device=device)
            continue
        if k.endswith("weight"):
            fan[base] = math.prod(shp[1:])
            bound = 1.0 / math.sqrt(fan[base])
        else:
            bound = 1.0 / math.sqrt(fan.get(base, shp[0]))
        if fast:  # timing-only weights (CPU baseline legs): tile one random block instead of drawing ~1e9 values
            n = math.prod(shp)
            t = torch.empty(n, device=device)
            for o in range(0, n, block.numel()):  # in-place tiling: one pass over fresh memory, no temporaries
                m = min(block.numel(), n - o)
                torch.mul(block[:m], bound, out=t[o:o + m])
            sd[k] = t.view(shp)
        else:
            sd[k] = torch.empty(shp, device=device).uniform_(-bound, bound, generator=g)
    return sd


def synthetic_inputs(B, H, W, seed=1234, ctx_dim=1024, n_pose=18):
    g = torch.Generator().manual_seed(seed)
    image = torch.rand((B, 3, H, W), generator=g) * 2 - 1
    cloth = torch.rand((B, 3, H, W), generator=g) * 2 - 1
    mask = torch.zeros((B, 1, H, W))
    mh, mw = int(H * 0.6), int(W * 0.58)  # centred rectangle, ~35 % of the pixels
    mask[:, :, (H - mh) // 2:(H - mh) // 2 + mh, (W - mw) // 2:(W - mw) // 2 + mw] = 1.0
    ys = torch.arange(H, dtype=torch.float32)[None, None, :, None]
    xs = torch.arange(W, dtype=torch.float32)[None, None, None, :]
    cy = torch.rand((B, n_pose, 1, 1), generator=g) * H
    cx = torch.rand((B, n_pose, 1, 1), generator=g) * W
    pose = torch.exp(-((ys - cy) ** 2 + (xs - cx) ** 2) / 81.0)  # sigma = 9 as src/utils/posemap.py:29-31
    prompt = torch.randn((B, 77, ctx_dim), generator=g)
    negative = torch.randn((B, 77, ctx_dim), generator=g)
    return dict(image=image, mask_image=mask, pose_map=pose, warped_cloth=cloth, prompt_embeds=prompt, negative_prompt_embeds=negative)


SMALL_UNET = dict(block_out_channels=(64, 128, 256, 256), attention_head_dim=(1, 2, 4, 4), cross_attention_dim=128, sample_size=16)
SMALL_VAE = dict(block_out_channels=(64, 128, 256, 256))


def build_state_dicts(unet_cfg=None, vae_cfg=None, seed=1234, device="cpu"):
    unet_cfg, vae_cfg = unet_cfg or {}, vae_cfg or {}
    from .vae import SD2_VAE
    vch = {**SD2_VAE, **vae_cfg}["block_out_channels"]
    ein, eout = emasc_channels(vch)
    return dict(unet=random_state_dict(unet_param_shapes(unet_cfg), seed, device),
                vae=random_state_dict(vae_param_shapes(vae_cfg), seed + 1, device),
                emasc=random_state_dict(emasc_param_shapes(ein, eout), seed + 2, device),
                emasc_channels=(ein, eout))


def build_pipeline(device, unet_cfg=None, vae_cfg=None, seed=1234, sds=None, weights_on_device=False):
    """Random-init engine pipeline (the hubconf.py constructors' architectures, no checkpoint)."""
    from . import EMASC, AutoencoderKL, DDIMScheduler, StableDiffusionTryOnePipeline, UNet2DConditionModel
    sds = sds or build_state_dicts(unet_cfg, vae_cfg, seed, device if weights_on_device else "cpu")
    unet = UNet2DConditionModel(**(unet_cfg or {})).load_state_dict(sds["unet"])
    vae = AutoencoderKL(**(vae_cfg or {})).load_state_dict(sds["vae"])
    emasc = EMASC(*sds["emasc_channels"]).load_state_dict(sds["emasc"])
    pipe = StableDiffusionTryOnePipeline(vae=vae, text_encoder=None, tokenizer=None, unet=unet, scheduler=DDIMScheduler(),
                                         emasc=emasc, emasc_int_layers=[1, 2, 3, 4, 5])
    return pipe.to(device), sds


def warp_state_dict(shapes, seed, ctrl_bias=None):
    """Seeded weights for the warping modules (ConvNet_TPS / UNetVanilla key sets): variance-preserving conv weights
    (U(+-sqrt(6/fan_in)), the nets are ReLU stacks up to 18 layers deep), BatchNorm affine ~ U(0.5,1.5) / N(0,0.1), running statistics
    N(0,0.1) / U(0.5,1.5); the TPS regression head starts at the identity lattice (`ctrl_bias` = atanh(control points), as
    ConvNet_TPS.py:199-203) plus a small random linear part so the predicted warp is not the identity."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for k, shp in shapes.items():
        leaf = k.rsplit(".", 1)[-1]
        if k.startswith("gridGen."):
            continue
        if leaf == "num_batches_tracked":
            sd[k] = torch.zeros((), dtype=torch.long)
        elif leaf == "running_var":
            sd[k] = torch.rand(shp, generator=g) + 0.5
        elif leaf == "running_mean":
            sd[k] = torch.randn(shp, generator=g) * 0.1
        elif len(shp) == 1 and leaf == "weight":
            sd[k] = torch.rand(shp, generator=g) + 0.5
        elif len(shp) == 1:
            sd[k] = torch.randn(shp, generator=g) * 0.1
        elif k.endswith("linear.weight"):
            sd[k] = torch.randn(shp, generator=g) * (0.5 / math.sqrt(shp[1]))
        else:
            bound = math.sqrt(6.0 / math.prod(shp[1:]))
            sd[k] = torch.empty(shp).uniform_(-bound, bound, generator=g)
            if k.startswith("outc."):
                sd[k] *= 0.15  # keep the refinement output mostly inside the [-1, 1] clamp of inference.py:262
    if ctrl_bias is not None:
        sd["loc_net.regression.linear.bias"] = ctrl_bias.clone()
    return sd


def warp_inputs(B, H, W, seed=1234, n_pose=18):
    """Smooth synthetic cloth (low-frequency colour field, so that a sub-pixel difference in the sampling grid is a small difference in
    the warped image), a 3-channel person mask and Gaussian pose heat-maps as in synthetic_inputs."""
    g = torch.Generator().manual_seed(seed)
    ys = torch.linspace(0, 1, H)[None, None, :, None]
    xs = torch.linspace(0, 1, W)[None, None, None, :]
    ph = torch.rand((B, 3, 1, 1), generator=g) * 6.28
    fy = torch.rand((B, 3, 1, 1), generator=g) * 3 + 1
    fx = torch.rand((B, 3, 1, 1), generator=g) * 3 + 1
    cloth = torch.sin(6.28 * (fy * ys + fx * xs) + ph) * 0.9
    im_mask = (torch.rand((B, 3, H, W), generator=g) * 2 - 1) * (ys > 0.3).float()
    cy = torch.rand((B, n_pose, 1, 1), generator=g) * H
    cx = torch.rand((B, n_pose, 1, 1), generator=g) * W
    yy = torch.arange(H, dtype=torch.float32)[None, None, :, None]
    xx = torch.arange(W, dtype=torch.float32)[None, None, None, :]
    pose = torch.exp(-((yy - cy) ** 2 + (xx - cx) ** 2) / 81.0)
    return dict(cloth=cloth, im_mask=im_mask, pose_map=pose)
