"""DDIM scheduler with the SD-2-inpainting scheduler config -- the object the reference creates at
src/inference.py:123-124 and uses at src/vto_pipelines/tryon_pipe.py:650-651,722,740 (diffusers 0.14
`DDIMScheduler`, SURVEY.md Appendix A.6).  Host side only holds the tables; the update itself is the fused CFG+DDIM kernel
(`ladi_ddim_cfg_step`), fed by a per-step coefficient table so no host sync happens inside the denoising loop.
"""
import numpy as np
import torch

from . import ops
from .module import _Cfg


class _Step:
    def __init__(self, prev_sample):
        self.prev_sample = prev_sample


class DDIMScheduler:
    order = 1
    init_noise_sigma = 1.0

    def __init__(self, num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear",
                 steps_offset=1, clip_sample=False, set_alpha_to_one=False, prediction_type="epsilon", **unused):
        if beta_schedule != "scaled_linear" or prediction_type != "epsilon" or clip_sample:
            raise NotImplementedError("only the SD-2-inpainting DDIM config (scaled_linear, epsilon, clip_sample=False)")
        self.config = _Cfg(num_train_timesteps=num_train_timesteps, beta_start=beta_start, beta_end=beta_end,
                         beta_schedule=beta_schedule, steps_offset=steps_offset, clip_sample=clip_sample,
                         set_alpha_to_one=set_alpha_to_one, prediction_type=prediction_type, skip_prk_steps=True)
        betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, num_train_timesteps, dtype=torch.float32) ** 2
        self.alphas_cumprod = torch.cumprod(1.0 - betas, dim=0)
        self.final_alpha_cumprod = torch.tensor(1.0) if set_alpha_to_one else self.alphas_cumprod[0]
        self.num_inference_steps = None
        self.timesteps = torch.from_numpy(np.arange(0, num_train_timesteps)[::-1].copy().astype(np.int64))

    def set_timesteps(self, num_inference_steps, device=None):
        self.num_inference_steps = num_inference_steps
        ratio = self.config.num_train_timesteps // num_inference_steps
        ts = (np.arange(0, num_inference_steps) * ratio).round()[::-1].copy().astype(np.int64) + self.config.steps_offset
        self.timesteps_host = [int(t) for t in ts]
        self.timesteps = torch.from_numpy(ts).to(device) if device is not None else torch.from_numpy(ts)

    def scale_model_input(self, sample, timestep=None):
        return sample

    def coefficients(self, timesteps=None, eta=0.0):
        """fp32 [steps, 8] = {1/sqrt(a_t), sqrt(1-a_t), sqrt(a_prev), sqrt(1-a_prev-sigma_t^2), sigma_t, 0, 0, 0} with DDIM's
        sigma_t = eta * sqrt((1-a_prev)/(1-a_t) * (1 - a_t/a_prev))  (DDIMScheduler._get_variance / step; 0 for the CLI's eta = 0)."""
        timesteps = self.timesteps_host if timesteps is None else timesteps
        ratio = self.config.num_train_timesteps // self.num_inference_steps
        rows = []
        zero = torch.tensor(0.0)
        for t in timesteps:
            tp = t - ratio
            a_t = self.alphas_cumprod[t]
            a_p = self.alphas_cumprod[tp] if tp >= 0 else self.final_alpha_cumprod
            var = (1 - a_p) / (1 - a_t) * (1 - a_t / a_p)
            sigma = eta * var ** 0.5
            rows.append(torch.stack([1.0 / a_t ** 0.5, (1 - a_t) ** 0.5, a_p ** 0.5, (1 - a_p - sigma ** 2) ** 0.5, sigma + zero, zero, zero, zero]))
        return torch.stack(rows).to(torch.float32)

    def step(self, model_output, timestep, sample, eta=0.0, generator=None, return_dict=True):
        """Generic one-step API (NCHW tensors on the CUDA device), kept for signature parity (tryon_pipe.py:337-345
        introspects `eta`/`generator`); the pipeline itself calls the fused kernel directly."""
        dev = sample.device
        coef = self.coefficients([int(timestep)], eta=eta).to(dev)
        B, c, h, w = sample.shape
        eps = model_output.float().permute(0, 2, 3, 1).contiguous()
        lat = sample.float().contiguous().clone()
        scratch = torch.empty((B, h, w, 8), dtype=torch.bfloat16, device=dev)
        noise = None
        if eta > 0:  # variance noise drawn like diffusers' randn_tensor(model_output.shape, generator=generator, device=...)
            gdev = generator.device if generator is not None else dev
            noise = torch.randn(tuple(model_output.shape), generator=generator, device=gdev, dtype=torch.float32).to(dev).contiguous()
        ops.ddim_cfg_step(eps, lat, scratch, False, 1.0, coef, None, advance=False, noise=noise)
        return _Step(lat.to(sample.dtype))
