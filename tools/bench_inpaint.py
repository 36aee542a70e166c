#!/usr/bin/env python
"""Images/s of `StableDiffusionInpaintPipeline` (the SD-2 inpainting pipeline inversion-adapter validation runs) on one GPU.

Full-size random-init weights (9-channel SD-2 inpainting UNet, SD-2 VAE), seeded synthetic images and masks, precomputed prompt
embeddings; by default 512x384, batch 8, 50 DDIM steps, guidance 7.5 (UNet batch 16).  Each timed call is the public `__call__`
with device-resident inputs and output_type="pt", timed with CUDA events after `--warmup` calls (the first call of a shape runs
eagerly and captures the CUDA graphs).  Prints one JSON line with the median and spread of the per-call time, images/s, and the
card's name and power limit read in the same run.

    python tools/bench_inpaint.py [--batch 8] [--steps 50] [--guidance 7.5] [--calls 5] [--warmup 2]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                       capture_output=True, text=True, check=True).stdout.strip().split(", ")
    return dict(name=q[0], power_limit=q[1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--height", type=int, default=512)
    ap.add_argument("--width", type=int, default=384)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--guidance", type=float, default=7.5)
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    from ladi_vton_b200 import AutoencoderKL, DDIMScheduler, StableDiffusionInpaintPipeline, UNet2DConditionModel, lib, synthetic as S
    from ladi_vton_b200.vae import vae_param_shapes
    lib.load()
    dev = torch.device("cuda", torch.cuda.current_device())
    unet = UNet2DConditionModel(in_channels=9)
    unet.load_state_dict(S.random_state_dict(unet.param_shapes(), 1234, device=dev, fast=True))
    vae = AutoencoderKL().load_state_dict(S.random_state_dict(vae_param_shapes({}), 1235, device=dev, fast=True))
    pipe = StableDiffusionInpaintPipeline(vae=vae, text_encoder=None, tokenizer=None, unet=unet, scheduler=DDIMScheduler(),
                                          safety_checker=None, feature_extractor=None, requires_safety_checker=False).to(dev)
    inp = {k: v.to(dev) for k, v in S.synthetic_inputs(args.batch, args.height, args.width).items()}
    neg = inp["negative_prompt_embeds"] if args.guidance > 1.0 else None

    def call():
        return pipe(image=inp["image"], mask_image=inp["mask_image"], prompt_embeds=inp["prompt_embeds"], negative_prompt_embeds=neg,
                    height=args.height, width=args.width, num_inference_steps=args.steps, guidance_scale=args.guidance,
                    generator=torch.Generator(dev).manual_seed(0), output_type="pt").images

    for _ in range(args.warmup):
        call()
    torch.cuda.synchronize()
    ms = []
    for _ in range(args.calls):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        call()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    ms.sort()
    med = ms[len(ms) // 2]
    print(json.dumps(dict(workload=f"inpaint {args.height}x{args.width} batch {args.batch}, {args.steps} DDIM steps, guidance {args.guidance}",
                          ms_per_call_median=round(med, 2), ms_per_call_min=round(ms[0], 2), ms_per_call_max=round(ms[-1], 2),
                          images_per_s=round(args.batch * 1000.0 / med, 3), calls=args.calls, gpu=card())))


if __name__ == "__main__":
    main()
