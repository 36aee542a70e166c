"""`StableDiffusionTryOnePipeline` -- same constructor, `.to()`, `__call__` signature/defaults/return types and error
behaviour as the reference's src/vto_pipelines/tryon_pipe.py:27-765 -- and `StableDiffusionInpaintPipeline`, the diffusers 0.14
inpainting pipeline the reference validates inversion adapters with (src/train_inversion_adapter.py:546-556).  Both run one body
(`_EnginePipeline._generate`) that differs only in the conditioning layout of the UNet input, re-built H100-first:

  * all model arithmetic runs in the hand-written sm_90a kernels (ops.py) -- NHWC bf16 activations, fp32 latents;
  * step-invariant work is hoisted out of the loop (27 of the 31 UNet input channels, text K/V, time-embedding tables);
  * one denoising step (UNet forward + CFG + DDIM update + re-assembly of the next UNet input) is captured ONCE as a CUDA
    graph per (batch, size, CFG) and replayed; the step index lives on the device, so there is no host sync in the loop;
  * RNG draws happen in the reference's order (cloth posterior -> initial latents -> masked-image posterior,
    tryon_pipe.py:640,419,458) with `randn_tensor` semantics, so a CPU generator reproduces the oracle's noise exactly.
"""
import inspect
import os
from dataclasses import dataclass
from typing import Any

import torch

from . import lib, ops


@dataclass
class StableDiffusionPipelineOutput:
    images: Any
    nsfw_content_detected: Any


def _randn(shape, generator, device):
    """diffusers.utils.randn_tensor (SURVEY.md Appendix A.8): sample on the generator's device, then move.  A LIST of generators
    (one per sample) draws every sample's (1, ...) slice from its own generator, as randn_tensor's list branch does."""
    if isinstance(generator, (list, tuple)):
        if len(generator) == 1:
            generator = generator[0]
        else:
            if len(generator) != shape[0]:
                raise ValueError(f"You have passed a list of generators of length {len(generator)}, but requested an effective batch"
                                 f" size of {shape[0]}. Make sure the batch size matches the length of the generators.")
            return torch.cat([torch.randn((1,) + tuple(shape[1:]), generator=g, device=g.device, dtype=torch.float32).to(device)
                              for g in generator], dim=0)
    gdev = generator.device if generator is not None else device
    return torch.randn(shape, generator=generator, device=gdev, dtype=torch.float32).to(device)


class _Session:
    """Everything one (batch, size, conditioning layout) shape needs to be replayable: static input buffers, the persistent UNet input /
    latents / step counter, and the captured CUDA graphs -- `pre` (mask + pose preprocessing, VAE encode x2, posterior samples, EMASC,
    UNet input assembly, text K/V), `loop` (all N denoising steps; or `step`, one step replayed N times, when something has to happen on the
    host between steps: eta > 0, cloth_cond_rate < 1, a callback) and `post` (VAE decode with the EMASC skips + image conversion)."""

    def __init__(self, B, Bp, h, w, H, W, in_pitch, n_pose, ctx_shape, kv_total, device, Bi=None):
        """`Bi`: the number of images / masks passed (default B); `pre` tiles them to the effective batch B."""
        f32 = dict(dtype=torch.float32, device=device)
        Bi = Bi or B
        self.image = torch.zeros((Bi, 3, H, W), **f32)
        self.mask = torch.zeros((Bi, 1, H, W), **f32)
        self.pose = torch.zeros((B, n_pose, H, W), **f32)
        self.cloth = torch.zeros((B, 3, H, W), **f32)
        # cloth posterior, initial latents, masked-image posterior (one draw per image passed)
        self.noise = [torch.zeros((B, 4, h, w), **f32), torch.zeros((B, 4, h, w), **f32), torch.zeros((Bi, 4, h, w), **f32)]
        self.step_noise = torch.zeros((B, 4, h, w), **f32)                 # eta > 0: DDIM variance noise of the current step
        self.ctx = torch.zeros(ctx_shape, dtype=torch.bfloat16, device=device)
        self.ctx_kv = torch.zeros((ctx_shape[0], ctx_shape[1], kv_total), dtype=torch.bfloat16, device=device)
        self.flags = torch.zeros(2, dtype=torch.int32, device=device)
        self.unet_in = torch.zeros((Bp, h, w, in_pitch), dtype=torch.bfloat16, device=device)
        self.latents = torch.zeros((B, 4, h, w), **f32)
        self.step = torch.zeros(2, dtype=torch.int32, device=device)
        self.coef = None
        self.inter = None          # EMASC outputs (mask_features applied), produced by `pre`, consumed by `post`
        self.out_f32 = self.out_u8 = None
        self.host_f32 = self.host_u8 = None  # pinned staging for the D2H of the result
        self.calls = 0
        self.g_pre = self.g_step = self.g_post = self.g_loop = None
        self.step_key = self.pre_key = self.post_key = self.loop_key = None
        self.step_nodes = self.pre_nodes = self.post_nodes = self.loop_nodes = 0


class _EnginePipeline:
    """What the try-on and the inpainting pipeline share: constructor state, `.to()`, prompt encoding, mask / image preparation, the
    captured `pre` / `step` / `post` pieces and the call body `_generate`, parameterised by the UNet input layout `lay`
    (latents4 | mask1 | masked4 [| pose | cloth4])."""
    _optional_components = ["safety_checker"]

    def __init__(self, vae, text_encoder, tokenizer, unet, scheduler, safety_checker=None, feature_extractor=None,
                 requires_safety_checker: bool = False, emasc=None, emasc_int_layers=None):
        if safety_checker is not None and feature_extractor is None:
            raise ValueError("Make sure to define a feature extractor when loading {self.__class__} if you want to use the safety"
                             " checker. If you do not want to use the safety checker, you can pass `'safety_checker=None'` instead.")
        self.vae, self.text_encoder, self.tokenizer, self.unet, self.scheduler = vae, text_encoder, tokenizer, unet, scheduler
        self.safety_checker, self.feature_extractor = safety_checker, feature_extractor
        self.emasc, self.emasc_int_layers = emasc, emasc_int_layers
        self.vae_scale_factor = 2 ** (len(self.vae.config.block_out_channels) - 1)
        self.device = torch.device("cpu")
        self.use_cuda_graph = True
        self._sessions = {}
        self._pack_gens = None

    def to(self, device):
        device = torch.device(device)
        if device.type != "cuda":
            raise RuntimeError("ladi_vton_b200 pipeline runs on CUDA (sm_90a) only; there is no CPU path")
        self.device = device
        for m in (self.vae, self.unet, self.emasc, self.text_encoder):
            if m is not None and hasattr(m, "to"):
                m.to(device)
        return self

    @property
    def _execution_device(self):
        return self.device

    # ---- copied semantics: tryon_pipe.py:362-407 ----------------------------------------------------------------------
    def check_inputs(self, prompt, height, width, callback_steps, negative_prompt=None, prompt_embeds=None,
                     negative_prompt_embeds=None):
        if height % 8 != 0 or width % 8 != 0:
            raise ValueError(f"`height` and `width` have to be divisible by 8 but are {height} and {width}.")
        if (callback_steps is None) or (callback_steps is not None and (not isinstance(callback_steps, int) or callback_steps <= 0)):
            raise ValueError(f"`callback_steps` has to be a positive integer but is {callback_steps} of type {type(callback_steps)}.")
        if prompt is not None and prompt_embeds is not None:
            raise ValueError(f"Cannot forward both `prompt`: {prompt} and `prompt_embeds`: {prompt_embeds}. Please make sure to"
                             " only forward one of the two.")
        elif prompt is None and prompt_embeds is None:
            raise ValueError("Provide either `prompt` or `prompt_embeds`. Cannot leave both `prompt` and `prompt_embeds` undefined.")
        elif prompt is not None and (not isinstance(prompt, str) and not isinstance(prompt, list)):
            raise ValueError(f"`prompt` has to be of type `str` or `list` but is {type(prompt)}")
        if negative_prompt is not None and negative_prompt_embeds is not None:
            raise ValueError(f"Cannot forward both `negative_prompt`: {negative_prompt} and `negative_prompt_embeds`:"
                             f" {negative_prompt_embeds}. Please make sure to only forward one of the two.")
        if prompt_embeds is not None and negative_prompt_embeds is not None:
            if prompt_embeds.shape != negative_prompt_embeds.shape:
                raise ValueError("`prompt_embeds` and `negative_prompt_embeds` must have the same shape when passed directly, but"
                                 f" got: `prompt_embeds` {prompt_embeds.shape} != `negative_prompt_embeds` {negative_prompt_embeds.shape}.")

    def prepare_extra_step_kwargs(self, generator, eta):
        params = set(inspect.signature(self.scheduler.step).parameters.keys())
        kw = {}
        if "eta" in params:
            kw["eta"] = eta
        if "generator" in params:
            kw["generator"] = generator
        return kw

    def _encode_text(self, texts, max_length):
        if self.tokenizer is None or self.text_encoder is None:
            raise ValueError("no tokenizer/text_encoder available: pass `prompt_embeds` (and `negative_prompt_embeds` when "
                             "guidance_scale > 1) instead of strings")
        ids = self.tokenizer(texts, padding="max_length", max_length=max_length, truncation=True, return_tensors="pt").input_ids
        return self.text_encoder(ids.to(self.device))[0]

    def _encode_prompt(self, prompt, device, num_images_per_prompt, do_cfg, negative_prompt=None, prompt_embeds=None,
                       negative_prompt_embeds=None):
        """tryon_pipe.py:184-317 -> [B', 77, D] with the CFG batch ordered [negative, positive] (:315)."""
        if prompt is not None:
            batch_size = 1 if isinstance(prompt, str) else len(prompt)
        else:
            batch_size = prompt_embeds.shape[0]
        if prompt_embeds is None:
            prompt_embeds = self._encode_text(prompt, self.tokenizer.model_max_length if self.tokenizer is not None else 77)
        prompt_embeds = prompt_embeds.to(device=device, dtype=torch.float32)
        bs, seq, _ = prompt_embeds.shape
        prompt_embeds = prompt_embeds.repeat(1, num_images_per_prompt, 1).view(bs * num_images_per_prompt, seq, -1)
        if do_cfg and negative_prompt_embeds is None:
            if negative_prompt is None:
                uncond = [""] * batch_size
            elif type(prompt) is not type(negative_prompt):
                raise TypeError(f"`negative_prompt` should be the same type to `prompt`, but got {type(negative_prompt)} !="
                                f" {type(prompt)}.")
            elif isinstance(negative_prompt, str):
                uncond = [negative_prompt]
            elif batch_size != len(negative_prompt):
                raise ValueError(f"`negative_prompt`: {negative_prompt} has batch size {len(negative_prompt)}, but `prompt`:"
                                 f" {prompt} has batch size {batch_size}. Please make sure that passed `negative_prompt` matches"
                                 " the batch size of `prompt`.")
            else:
                uncond = negative_prompt
            negative_prompt_embeds = self._encode_text(uncond, prompt_embeds.shape[1])
        if do_cfg:
            seq = negative_prompt_embeds.shape[1]
            negative_prompt_embeds = negative_prompt_embeds.to(device=device, dtype=torch.float32)
            negative_prompt_embeds = negative_prompt_embeds.repeat(1, num_images_per_prompt, 1).view(batch_size * num_images_per_prompt, seq, -1)
            prompt_embeds = torch.cat([negative_prompt_embeds, prompt_embeds])
        return prompt_embeds

    @staticmethod
    def _pil_to_tensors(image, mask):
        """diffusers prepare_mask_and_masked_image, PIL / ndarray branch (called at tryon_pipe.py:630): image -> float32 [-1, 1] NCHW,
        mask -> float32 [0, 1] N1HW.  Host-side conversion (the reference does the same with numpy)."""
        import numpy as np
        from PIL import Image
        if isinstance(image, (Image.Image, np.ndarray)):
            image = [image]
        if isinstance(image, list) and isinstance(image[0], Image.Image):
            image = np.concatenate([np.array(i.convert("RGB"))[None, :] for i in image], axis=0)
        elif isinstance(image, list) and isinstance(image[0], np.ndarray):
            image = np.concatenate([i[None, :] for i in image], axis=0)
        image = torch.from_numpy(np.ascontiguousarray(image.transpose(0, 3, 1, 2))).to(dtype=torch.float32) / 127.5 - 1.0
        if isinstance(mask, (Image.Image, np.ndarray)):
            mask = [mask]
        if isinstance(mask, list) and isinstance(mask[0], Image.Image):
            mask = np.concatenate([np.array(m.convert("L"))[None, None, :] for m in mask], axis=0).astype(np.float32) / 255.0
        elif isinstance(mask, list) and isinstance(mask[0], np.ndarray):
            mask = np.concatenate([m[None, None, :] for m in mask], axis=0).astype(np.float32)
        return image, torch.from_numpy(np.ascontiguousarray(mask))

    def _as_tensors(self, image, mask):
        """The shape half of diffusers prepare_mask_and_masked_image: PIL / ndarray inputs converted, both made 4-D (views of the
        caller's tensors, so the binarisation below still writes the caller's mask), batch and size checked."""
        if not isinstance(image, torch.Tensor) or not isinstance(mask, torch.Tensor):
            if isinstance(image, torch.Tensor) or isinstance(mask, torch.Tensor):
                raise TypeError("`image` and `mask_image` must both be torch tensors or both PIL images / arrays")
            if self.emasc:  # the reference hands mask_image to mask_features (tryon_pipe.py:685), which needs a tensor
                raise TypeError("with EMASC, `mask_image` must be a torch tensor (mask_features interpolates it, src/utils/data_utils.py:9)")
            image, mask = self._pil_to_tensors(image, mask)
        if image.ndim == 3:
            image = image.unsqueeze(0)
        if mask.ndim == 2:
            mask = mask.unsqueeze(0).unsqueeze(0)
        if mask.ndim == 3:
            mask = mask.unsqueeze(0) if mask.shape[0] == 1 else mask.unsqueeze(1)
        assert image.ndim == 4 and mask.ndim == 4, "Image and Mask must have 4 dimensions"
        assert image.shape[-2:] == mask.shape[-2:], "Image and Mask must have the same spatial dimensions"
        assert image.shape[0] == mask.shape[0], "Image and Mask must have the same batch size"
        return image, mask

    def _prepare_mask_and_image(self, image, mask, flags):
        """diffusers prepare_mask_and_masked_image (called at tryon_pipe.py:630): shape normalisation, the [-1,1] / [0,1] range checks and
        the IN-PLACE binarisation of the caller's mask at 0.5.  Device tensors: one kernel, the range flags are read back with the
        result (no host sync before the work is queued); host tensors: checked on the host, raising at once like the reference.
        `image * (mask < 0.5)` itself is fused into the layout kernel (ops.nchw_to_nhwc gate)."""
        image, mask = self._as_tensors(image, mask)
        fast = all(t.is_cuda and t.dtype == torch.float32 and t.is_contiguous() for t in (image, mask))
        if fast:
            ops.check_binarise_(image, mask, flags)
        else:
            if image.min() < -1 or image.max() > 1:
                raise ValueError("Image should be in [-1, 1] range")
            if mask.min() < 0 or mask.max() > 1:
                raise ValueError("Mask should be in [0, 1] range")
            mask[mask < 0.5] = 0
            mask[mask >= 0.5] = 1
        return mask, image

    def numpy_to_pil(self, images):
        from PIL import Image
        if images.ndim == 3:
            images = images[None]
        images = (images * 255).round().astype("uint8")
        return [Image.fromarray(im) for im in images]

    # ---- the three captured pieces of one call ----------------------------------------------------------------------------
    def _pre(self, s, lay):
        """Steps 4-7a of tryon_pipe.py:629-705 on the session's static buffers."""
        B, cfg, vsf, sf = lay["B"], lay["cfg"], self.vae_scale_factor, self.vae.config.scaling_factor
        s.unet_in.zero_()
        cond = s.unet_in[B:] if cfg else s.unet_in  # conditional half of the CFG batch ([uncond, cond], tryon_pipe.py:315,702-705)
        if not lay["no_pose"]:
            ops.nchw_to_nhwc(ops.bilinear_down8(s.pose), cond, c_off=lay["c_pose"])  # :632-634
        if lay["cloth"]:  # 4b. warped cloth latents (RNG draw #1)
            mom, _ = self.vae.encode_nhwc(s.cloth)
            ops.nchw_to_nhwc(ops.posterior_sample(mom, s.noise[0], sf), cond, c_off=lay["c_cloth"])
        s.latents.copy_(s.noise[1])  # 6. latents (RNG draw #2, already times init_noise_sigma)
        # 7. masked image -> latents + encoder skips (RNG draw #3, one per image passed); EMASC with mask_features fused
        Bi, H, W = s.image.shape[0], s.image.shape[2], s.image.shape[3]
        masked = torch.zeros((Bi, H, W, 8), dtype=torch.bfloat16, device=self.device)
        ops.nchw_to_nhwc(s.image, masked, gate=s.mask)  # image * (mask < 0.5)
        mom, feats = self.vae.encode_nhwc(masked, nhwc=True)
        masked_lat = ops.posterior_sample(mom, s.noise[2], sf)
        s.inter = None
        if self.emasc:
            sel = [feats[i] for i in self.emasc_int_layers]  # :460-461
            inv = [ops.inv_mask_rows(s.mask, H // f.shape[1]) for f in sel]  # data_utils.py:9-14 (chained nearest == direct)
            s.inter = self.emasc(sel, inv)  # :684-685
        for half in ((s.unet_in[:B], s.unet_in[B:]) if cfg else (s.unet_in,)):  # :482-485
            for r in range(0, B, Bi):  # :462-477: mask and masked latents repeated to the effective batch, rows [a, b, a, b]
                ops.nchw_to_nhwc(s.mask, half[r:r + Bi], c_off=lay["c_mask"], f=vsf)  # nearest /8 (:434-436)
                ops.nchw_to_nhwc(masked_lat, half[r:r + Bi], c_off=lay["c_masked"])
            ops.nchw_to_nhwc(s.latents, half, c_off=0)
        self.unet.plan_context(s.ctx, out=s.ctx_kv)  # step-invariant: text K/V of all 16 cross-attention layers
        s.step.zero_()

    def _step(self, s, cfg, guidance, eta_noise=False, advance=True):
        eps = self.unet.forward_nhwc(s.unet_in, s.step)
        ops.ddim_cfg_step(eps, s.latents, s.unet_in, cfg, guidance, s.coef, s.step, advance=advance, noise=s.step_noise if eta_noise else None)

    def _post(self, s, lay):
        """decode_latents (tryon_pipe.py:349-359) with the EMASC skips, then both image conversions (fp32 [0,1] and numpy_to_pil's uint8)."""
        sf = self.vae.config.scaling_factor
        img = self.vae.decode_nhwc(s.latents, s.inter, self.emasc_int_layers if s.inter is not None else None, scale=1.0 / sf)
        s.out_f32 = ops.image_out(img)     # [B, H, W, 3] fp32 in [0, 1]  (:356)
        s.out_u8 = ops.image_out_u8(img)   # (x * 255).round().astype(uint8)  (:760)

    def _run(self, s, which, fn, key, use_graph):
        """Run one of the three pieces eagerly (first call of a shape = warm-up, or graphs off) or as a captured graph."""
        g_attr, k_attr, n_attr = f"g_{which}", f"{which}_key", f"{which}_nodes"
        if not use_graph:
            # an eager run re-binds the tensors the pieces hand to each other (e.g. the EMASC outputs): a graph of this piece captured earlier
            # would keep writing its own, older buffers -- drop it so that the next graphed call re-captures
            if which != "step":
                setattr(s, g_attr, None)
                setattr(s, k_attr, None)
            return fn()
        if getattr(s, g_attr) is None or getattr(s, k_attr) != key:
            g = torch.cuda.CUDAGraph()
            n0 = lib.launches
            with torch.cuda.graph(g):
                fn()
            setattr(s, n_attr, lib.launches - n0)
            lib.launches = n0  # capture records, it does not launch
            setattr(s, g_attr, g)
            setattr(s, k_attr, key)
        getattr(s, g_attr).replay()
        lib.launches += getattr(s, n_attr)

    def _generate(self, lay, Bi, image, mask_image, pose_map, warped_cloth, prompt, height, width, num_inference_steps, guidance_scale,
                  negative_prompt, num_images_per_prompt, eta, prompt_embeds, negative_prompt_embeds, generator, latents, output_type,
                  return_dict, callback, callback_steps, cloth_cond_rate=1.0, noise=None):
        """The call body of both pipelines (tryon_pipe.py:578-765) for the UNet input layout `lay` (c_mask, c_masked, c_pose, c_cloth,
        no_pose, cloth).  `Bi`: the number of images / masks passed, tiled to the effective batch as prepare_mask_latents does
        (None: the images already have the effective batch)."""
        dev = self.device
        if prompt is not None:
            batch_size = 1 if isinstance(prompt, str) else len(prompt)
        else:
            batch_size = prompt_embeds.shape[0]
        B = batch_size * num_images_per_prompt
        if isinstance(generator, (list, tuple)) and len(generator) != 1 and len(generator) != B:  # prepare_latents :412-416
            raise ValueError(f"You have passed a list of generators of length {len(generator)}, but requested an effective batch"
                             f" size of {B}. Make sure the batch size matches the length of the generators.")
        Bi = Bi or B
        _check_tiling(Bi, Bi, B)
        if isinstance(generator, (list, tuple)) and len(generator) != 1 and Bi < B:
            # prepare_mask_latents :442-446 encodes masked_image[i] with generator[i] for every i < B: past the end of the images passed
            raise ValueError(f"a list of {len(generator)} generators draws one masked-image latent per sample, but only {Bi} images were"
                             f" passed for an effective batch of {B}: pass {B} images, or one generator")
        cfg = guidance_scale > 1.0
        ctx = self._encode_prompt(prompt, dev, num_images_per_prompt, cfg, negative_prompt, prompt_embeds, negative_prompt_embeds)
        Bp = 2 * B if cfg else B
        vsf = self.vae_scale_factor
        h, w = height // vsf, width // vsf

        # ---- session (static buffers + graphs) for this shape / conditioning layout
        n_pose = lay["c_cloth"] - lay["c_pose"]
        lay = dict(lay, B=B, cfg=cfg)
        gens = (self.unet.pack_gen, self.vae.pack_gen, self.emasc.pack_gen if self.emasc else 0)
        if gens != self._pack_gens:  # weights were re-packed: every captured graph points at freed memory
            self._sessions.clear()
            self._pack_gens = gens
        key = (B, Bp, Bi, h, w, n_pose, lay["no_pose"], lay["cloth"], bool(self.emasc), tuple(ctx.shape[1:]))
        s = self._sessions.get(key)
        if s is None:
            s = self._sessions[key] = _Session(B, Bp, h, w, height, width, self.unet.in_pitch, n_pose, tuple(ctx.shape), self.unet.kv_total, dev, Bi)
        use_graph = self.use_cuda_graph and s.calls > 0  # the first call of a shape runs eagerly: lazy kernel attributes, allocations

        # 4. mask / image validation + in-place binarisation (flags read back with the result), inputs -> static buffers
        s.flags.zero_()
        mask, image = self._prepare_mask_and_image(image, mask_image, s.flags)
        s.image.copy_(image, non_blocking=True)
        s.mask.copy_(mask, non_blocking=True)
        if not lay["no_pose"]:
            s.pose.copy_(pose_map, non_blocking=True)
        s.ctx.copy_(ctx, non_blocking=True)
        # RNG draws in the reference's order: cloth posterior (:640), initial latents (:419), masked-image posterior (:458)
        if lay["cloth"]:
            s.cloth.copy_(warped_cloth, non_blocking=True)
            s.noise[0].copy_(noise[0] if noise is not None else _randn((B, 4, h, w), generator, dev), non_blocking=True)
        # 5. timesteps
        self.scheduler.set_timesteps(num_inference_steps, device=dev)
        ts = self.scheduler.timesteps_host
        cloth_steps = (1 - cloth_cond_rate) * num_inference_steps
        if latents is None:
            latents = noise[1] if noise is not None else _randn((B, 4, h, w), generator, dev)
        s.noise[1].copy_(latents.to(dev, torch.float32) * self.scheduler.init_noise_sigma, non_blocking=True)
        s.noise[2].copy_(noise[2] if noise is not None else _randn((Bi, 4, h, w), generator, dev), non_blocking=True)
        self._run(s, "pre", lambda: self._pre(s, lay), (self.unet.ws.buf.data_ptr() if self.unet.ws.buf is not None else 0,
                                                       self.vae.ws.buf.data_ptr() if self.vae.ws.buf is not None else 0), use_graph)
        self.unet._ctx = s.ctx_kv  # (a replayed `pre` graph did not run plan_context's Python)
        # step-invariant UNet tables
        self.unet.plan_steps(ts)
        coef = self.scheduler.coefficients(eta=eta)
        if s.coef is None or s.coef.shape != coef.shape:
            s.coef = coef.to(dev)
        else:
            s.coef.copy_(coef, non_blocking=True)
        # 9. denoising loop
        n_zero_from = num_inference_steps - cloth_steps  # :718-719
        stochastic = eta > 0
        step_graph = self.use_cuda_graph and callback is None
        step_key = self._graph_key() + (s.coef.data_ptr(), float(guidance_scale), stochastic)
        per_step_host_work = stochastic or (lay["cloth"] and cloth_steps > 0)  # noise draw / cloth zeroing between steps
        if step_graph and use_graph and not per_step_host_work and os.environ.get("LADI_LOOP_GRAPH", "0") == "1":
            # opt-in: ALL N steps as one captured graph (one launch instead of N).  Measured neutral in a same-box A/B (659.4 vs 659.3 ms per call,
            # round 2): N replays of the step graph already queue back to back, so the default stays the cheaper-to-capture single step.
            self._run(s, "loop", lambda: [self._step(s, cfg, guidance_scale) for _ in range(num_inference_steps)], step_key + (num_inference_steps,), True)
            steps_left = range(0)
        else:
            steps_left = range(num_inference_steps)
        for i in steps_left:
            if lay["cloth"] and i >= n_zero_from and cloth_steps > 0:
                s.unet_in[..., lay["c_cloth"]:lay["c_cloth"] + 4].zero_()
            if stochastic:  # DDIMScheduler.step draws randn_tensor(model_output.shape, generator=...) once per step (after the 3 initial draws)
                s.step_noise.copy_(_randn((B, 4, h, w), generator, dev), non_blocking=True)
            stale = s.g_step is None or s.step_key != step_key
            if not step_graph or (i == 0 and stale):
                self._step(s, cfg, guidance_scale, stochastic)  # first step of a new shape runs eagerly: the warm-up before capture
            else:
                self._run(s, "step", lambda: self._step(s, cfg, guidance_scale, stochastic), step_key, True)
            if callback is not None and i % callback_steps == 0:
                callback(i, ts[i], s.latents)
        # 11. decode with the EMASC skips, clamp, D2H
        post_key = (self.vae.ws.buf.data_ptr() if self.vae.ws.buf is not None else 0,) + tuple(t.data_ptr() for t in (s.inter or ()))
        self._run(s, "post", lambda: self._post(s, lay), post_key, use_graph)
        s.calls += 1
        if output_type in ("pt", "pt_u8"):  # extensions: leave the result on the device (fp32 [0,1] / numpy_to_pil's uint8) for device-resident
            out = (s.out_f32 if output_type == "pt" else s.out_u8).clone()  # timing and the NCCL gather; the range flags stay unchecked
            return StableDiffusionPipelineOutput(images=out, nsfw_content_detected=None) if return_dict else (out, None)
        if output_type == "pil":  # numpy_to_pil's uint8 conversion already happened on the device: a quarter of the D2H bytes (:358-760)
            if s.host_u8 is None:
                s.host_u8 = torch.empty(s.out_u8.shape, dtype=torch.uint8, pin_memory=True)
            s.host_u8.copy_(s.out_u8, non_blocking=True)
        else:
            if s.host_f32 is None:
                s.host_f32 = torch.empty(s.out_f32.shape, dtype=torch.float32, pin_memory=True)
            s.host_f32.copy_(s.out_f32, non_blocking=True)
        flags = s.flags.cpu()  # synchronises the stream: the pinned result above is complete too
        if int(flags[0]):
            raise ValueError("Image should be in [-1, 1] range")
        if int(flags[1]):
            raise ValueError("Mask should be in [0, 1] range")
        if output_type == "pil":
            from PIL import Image
            out = [Image.fromarray(im) for im in s.host_u8.numpy().copy()]
        else:
            out = s.host_f32.numpy().copy()  # (:358) the staging buffer is reused by the next call
        if not return_dict:
            return (out, None)
        return StableDiffusionPipelineOutput(images=out, nsfw_content_detected=None)


    def _graph_key(self):
        # the captured step graph bakes in the addresses of the planned step table, the text K/V buffer and the GroupNorm workspace
        ws = self.unet.ws.buf
        return (self.unet._steps.data_ptr(), self.unet._ctx.data_ptr(), self.unet._steps.shape[0], ws.data_ptr() if ws is not None else 0)


def _check_tiling(n_masks, n_images, batch_size):
    """prepare_mask_latents (tryon_pipe.py:462-477): the masks and the masked-image latents passed are repeated to the effective batch,
    whole copies only.  More images than samples has no repeat that fits (the reference fails in torch.cat, :724)."""
    if n_masks < batch_size and batch_size % n_masks != 0:
        raise ValueError("The passed mask and the required batch size don't match. Masks are supposed to be duplicated to"
                         f" a total batch size of {batch_size}, but {n_masks} masks were passed. Make sure the number"
                         " of masks that you pass is divisible by the total requested batch size.")
    if n_images < batch_size and batch_size % n_images != 0:
        raise ValueError("The passed images and the required batch size don't match. Images are supposed to be duplicated"
                         f" to a total batch size of {batch_size}, but {n_images} images were passed."
                         " Make sure the number of images that you pass is divisible by the total requested batch size.")
    if max(n_masks, n_images) > batch_size:
        raise ValueError(f"{max(n_masks, n_images)} images / masks were passed for an effective batch of {batch_size}"
                         " (prompts x num_images_per_prompt): pass at most one image per sample")


class StableDiffusionTryOnePipeline(_EnginePipeline):

    @torch.no_grad()
    def __call__(self, image, mask_image, pose_map, warped_cloth, prompt=None, height=None, width=None,
                 num_inference_steps: int = 50, guidance_scale: float = 7.5, negative_prompt=None, num_images_per_prompt=1,
                 eta: float = 0.0, prompt_embeds=None, negative_prompt_embeds=None, generator=None, latents=None,
                 output_type="pil", return_dict: bool = True, callback=None, callback_steps=1, cloth_cond_rate: float = 1.0,
                 no_pose: bool = False, cloth_input_type: str = "warped", noise=None):
        """Same arguments as the reference `__call__` (tryon_pipe.py:495-520).  Extensions: output_type="pt" returns the
        device tensor; `noise=(cloth, latents, masked)` supplies the three RNG draws explicitly (batch-sharded runs slice
        one full-batch draw, distributed.draw_noise)."""
        if self.device.type != "cuda":
            raise RuntimeError("call .to('cuda') first: ladi_vton_b200 has no CPU path")
        height = height or self.unet.config.sample_size * self.vae_scale_factor
        width = width or self.unet.config.sample_size * self.vae_scale_factor
        self.check_inputs(prompt, height, width, callback_steps, negative_prompt, prompt_embeds, negative_prompt_embeds)
        if image is None:
            raise ValueError("`image` input cannot be undefined.")
        if mask_image is None:
            raise ValueError("`mask_image` input cannot be undefined.")
        if cloth_input_type not in ("warped", "none"):
            raise ValueError(f"Invalid cloth_input_type {cloth_input_type}")
        if num_images_per_prompt != 1:
            # the reference accepts the argument but its own body then concatenates [B*num, ...] latents with [B, ...] pose / cloth
            # tensors (tryon_pipe.py:702-726) and fails inside torch.cat; say so instead of failing somewhere in a kernel wrapper
            raise ValueError("num_images_per_prompt != 1 is not supported by the try-on pipeline: pose_map / warped_cloth are not repeated "
                             "to the effective batch (the reference fails in torch.cat at tryon_pipe.py:724); repeat the inputs instead")
        n_pose = pose_map.shape[1]
        lay = dict(no_pose=bool(no_pose), cloth=cloth_input_type == "warped", c_mask=4, c_masked=5, c_pose=9, c_cloth=9 + n_pose)
        assert self.unet.config.in_channels == lay["c_cloth"] + (4 if lay["cloth"] else 0), "UNet in_channels does not match the conditioning"
        return self._generate(lay, None, image, mask_image, pose_map, warped_cloth, prompt, height, width, num_inference_steps, guidance_scale,
                              negative_prompt, num_images_per_prompt, eta, prompt_embeds, negative_prompt_embeds, generator, latents,
                              output_type, return_dict, callback, callback_steps, cloth_cond_rate, noise)


class StableDiffusionInpaintPipeline(_EnginePipeline):
    """diffusers 0.14 `StableDiffusionInpaintPipeline` on the engine: the stock SD-2 inpainting model (9-channel UNet input
    latents4 | mask1 | masked4), as src/train_inversion_adapter.py:546-556 builds it to validate an inversion adapter.  The same
    body as the try-on pipeline without pose, cloth and EMASC, plus `num_images_per_prompt > 1`: prompt embeddings and initial
    latents grouped per prompt ([a, a, b, b]), the images passed encoded once each and tiled ([a, b, a, b]).  No safety checker
    is built: `nsfw_content_detected` is None."""

    def __init__(self, vae, text_encoder, tokenizer, unet, scheduler, safety_checker=None, feature_extractor=None,
                 requires_safety_checker: bool = True):
        super().__init__(vae, text_encoder, tokenizer, unet, scheduler, safety_checker, feature_extractor, requires_safety_checker)

    @torch.no_grad()
    def __call__(self, prompt=None, image=None, mask_image=None, height=None, width=None, num_inference_steps: int = 50,
                 guidance_scale: float = 7.5, negative_prompt=None, num_images_per_prompt=1, eta: float = 0.0, generator=None,
                 latents=None, prompt_embeds=None, negative_prompt_embeds=None, output_type="pil", return_dict: bool = True,
                 callback=None, callback_steps=1):
        """Same arguments, defaults and return types as diffusers 0.14; output_type="pt" (extension) returns the device tensor."""
        if self.device.type != "cuda":
            raise RuntimeError("call .to('cuda') first: ladi_vton_b200 has no CPU path")
        height = height or self.unet.config.sample_size * self.vae_scale_factor
        width = width or self.unet.config.sample_size * self.vae_scale_factor
        self.check_inputs(prompt, height, width, callback_steps, negative_prompt, prompt_embeds, negative_prompt_embeds)
        if image is None:
            raise ValueError("`image` input cannot be undefined.")
        if mask_image is None:
            raise ValueError("`mask_image` input cannot be undefined.")
        if 4 + 1 + 4 != self.unet.config.in_channels:
            raise ValueError(f"Incorrect configuration settings! The config of `pipeline.unet` expects {self.unet.config.in_channels} input"
                             " channels but received `num_channels_latents`: 4 + `num_channels_mask`: 1 + `num_channels_masked_image`: 4"
                             " = 9. Please verify the config of `pipeline.unet` or your `mask_image` or `image` input.")
        image, mask_image = self._as_tensors(image, mask_image)
        lay = dict(no_pose=True, cloth=False, c_mask=4, c_masked=5, c_pose=9, c_cloth=9)
        return self._generate(lay, image.shape[0], image, mask_image, None, None, prompt, height, width, num_inference_steps, guidance_scale,
                              negative_prompt, num_images_per_prompt, eta, prompt_embeds, negative_prompt_embeds, generator, latents,
                              output_type, return_dict, callback, callback_steps)
