"""ORACLE (test infrastructure only) -- CPU fp32 restatement of diffusers 0.14 `StableDiffusionInpaintPipeline.__call__` as
src/train_inversion_adapter.py:546-563 runs it: the try-on pipeline (pipeline.py, tryon_pipe.py:494-765) with a 9-channel UNet input
(latents4 | mask1 | masked4), no pose, no cloth, no EMASC, plus `num_images_per_prompt` and the broadcast of the images passed:
  * prompt embeddings and the initial latents grouped per prompt, `repeat(1, n, 1).view(...)` (tryon_pipe.py:255-257, 410-425): [a, a, b, b];
  * the masked-image posterior drawn once per image passed, then mask and masked-image latents tiled by `.repeat(B // b_img, 1, 1, 1)`
    (:427-477): [a, b, a, b].

PARITY STATUS: with num_images_per_prompt=1 and one image per prompt it is bit-identical to OracleTryOnPipeline with cloth_input_type
'none' on the same 9 UNet input channels (tests/test_inpaint_pipeline.py).

Only tests/ and tools/ may import this module.
"""
import numpy as np
import torch
import torch.nn.functional as F

from .parts import prepare_mask_and_masked_image, randn_tensor
from .pipeline import OracleTryOnPipeline


class OracleInpaintPipeline(OracleTryOnPipeline):
    def __init__(self, vae, unet, scheduler):
        super().__init__(vae, unet, scheduler)

    @torch.no_grad()
    def __call__(self, image, mask_image, prompt_embeds, negative_prompt_embeds=None, height=None, width=None, num_inference_steps=50,
                 guidance_scale=7.5, num_images_per_prompt=1, generator=None, latents=None, output_type="np", eta=0.0, callback=None):
        height = height or self.unet.config.sample_size * self.vae_scale_factor
        width = width or self.unet.config.sample_size * self.vae_scale_factor
        if height % 8 or width % 8:
            raise ValueError(f"`height` and `width` have to be divisible by 8 but are {height} and {width}.")
        n = num_images_per_prompt
        cfg = guidance_scale > 1.0
        wdtype = self.unet.dtype
        bs, seq, _ = prompt_embeds.shape
        B = bs * n
        ctx = prompt_embeds.to(wdtype).repeat(1, n, 1).view(B, seq, -1)  # :255-257
        if cfg:
            neg = negative_prompt_embeds.to(wdtype)
            ctx = torch.cat([neg.repeat(1, n, 1).view(B, neg.shape[1], -1), ctx])  # :305-315  [neg, pos]
        mask, masked_image = prepare_mask_and_masked_image(image, mask_image)
        self.scheduler.set_timesteps(num_inference_steps)
        timesteps = self.scheduler.timesteps
        h, w = height // self.vae_scale_factor, width // self.vae_scale_factor
        if latents is None:  # prepare_latents :410-425
            latents = randn_tensor((B, self.vae.config.latent_channels, h, w), generator=generator, dtype=ctx.dtype)
        latents = latents * self.scheduler.init_noise_sigma
        # prepare_mask_latents :427-492: one posterior draw per image passed (a generator list needs one image per sample, :442-446)
        mask_l = F.interpolate(mask, size=(h, w)).to(ctx.dtype)
        post, _ = self.vae.encode(masked_image.to(ctx.dtype))
        masked_l = self.vae.config.scaling_factor * self._sample(post.latent_dist, generator)
        b_img = mask_l.shape[0]
        if B % b_img:
            raise ValueError(f"{b_img} images cannot be repeated to an effective batch of {B}")
        mask_l, masked_l = mask_l.repeat(B // b_img, 1, 1, 1), masked_l.repeat(B // b_img, 1, 1, 1)  # :464-477
        self._rec("mask_latents", mask_l)
        self._rec("masked_latents", masked_l)
        if cfg:
            mask_l, masked_l = torch.cat([mask_l] * 2), torch.cat([masked_l] * 2)
        for i, t in enumerate(timesteps):
            x = torch.cat([latents] * 2) if cfg else latents
            x = torch.cat([x, mask_l, masked_l], dim=1)
            eps = self.unet(x, t, encoder_hidden_states=ctx).sample
            if i == 0:
                self._rec("unet_in0", x)
                self._rec("eps0", eps)
            if cfg:
                e_u, e_t = eps.chunk(2)
                eps = e_u + guidance_scale * (e_t - e_u)
            latents = self.scheduler.step(eps, t, latents, eta=eta, generator=generator).prev_sample.to(self.vae.dtype)
            if callback is not None:
                callback(i, t, latents)
        self._rec("final_latents", latents)
        img = self.vae.decode(1 / self.vae.config.scaling_factor * latents).sample
        img = (img / 2 + 0.5).clamp(0, 1).cpu().permute(0, 2, 3, 1).float().numpy()
        if output_type == "uint8":
            img = (img * 255).round().astype(np.uint8)
        return img
