"""TEST INFRASTRUCTURE (oracle) -- never imported by the product.

fp32 restatement of the per-batch body of `extract_save_vae_images` (src/utils/image_from_pipe.py:221-258, the validation of
src/train_emasc.py), composed from the oracle VAE (vae.py), an EMASC form (parts.EMASC or emasc_forms.EMASC) and parts.mask_features:
  * the posterior of `image` and the skips `int_layers` of `im_mask` (:234-237);
  * EMASC, then mask_features with `inpaint_mask` (:240-242);
  * one posterior draw from the global RNG of the moments' device, as diffusers' randn_tensor does without a generator (:243);
  * the decode with the skips (:244), and `(x + 1) / 2` (:252), the tensor the reference hands to torchvision.utils.save_image.
emasc_type "none": encode, sample, decode without skips (the reference's branch, :245-249, crashes on the tuple `encode` returns).
Runs on whatever device its modules and the batch are on.  Pinned against the reference's own function by
tests/golden/emasc_val_small.npz (tests/golden/make_emasc_val_golden.py).
"""
import torch

from .parts import mask_features


def save_image_u8(t):
    """torchvision.utils.save_image's quantisation of one [3,H,W] (or a batch [B,3,H,W]) image: `mul(255).add_(0.5).clamp_(0, 255)`, then
    the uint8 cast, channels last."""
    return t.mul(255).add_(0.5).clamp_(0, 255).movedim(-3, -1).to(torch.uint8)


@torch.no_grad()
def run_batch(batch, vae, emasc, int_layers, emasc_type):
    """-> fp32 [B,3,H,W], `(decoded + 1) / 2` before save_image."""
    posterior_im, _ = vae.encode(batch["image"])
    inter = None
    if emasc_type != "none":
        _, feats = vae.encode(batch["im_mask"])
        inter = mask_features(emasc([feats[i] for i in int_layers]), batch["inpaint_mask"])
    dist = posterior_im.latent_dist
    latents = dist.mean + dist.std * torch.randn(dist.mean.shape, device=dist.mean.device, dtype=dist.mean.dtype)
    if inter is None:
        images = vae.decode(latents).sample
    else:
        images = vae.decode(latents, list(inter), list(int_layers)).sample
    return (images + 1) / 2
