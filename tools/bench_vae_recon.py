#!/usr/bin/env python
"""Images/s of the EMASC trainer's validation body on one GPU: `eval.vae_recon_batch` + `ops.image_save_u8`.

Full-size random-init weights (SD-2 VAE, the hub's nonlinear 3x3 EMASC), seeded synthetic images and masks; by default 512x384, batch 16
(the trainer's --test_batch_size).  Each timed call runs from the host-to-device copy of the batch (pinned host tensors) to the
device-to-host copy of the uint8 images: two VAE encodes, EMASC with mask_features, the posterior sample, the decode with the skips and
the quantisation.  Data loading and the JPEG encode are not in it.  Timed with CUDA events after `--warmup` calls; prints one JSON line
with the median and spread of the per-call time, images/s, the achieved TFLOP/s from the analytic count of SURVEY.md Appendix C
(encode 0.831 TFLOP, EMASC 0.435, decode 1.879 per 512x384 image: 3.976 with the two encodes), and the card's name and power limit
read in the same run.

    python tools/bench_vae_recon.py [--batch 16] [--calls 5] [--warmup 2]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

TFLOP_PER_IMAGE_512x384 = 2 * 0.831 + 0.435 + 1.879


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                       capture_output=True, text=True, check=True).stdout.strip().split(", ")
    return dict(name=q[0], power_limit=q[1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--height", type=int, default=512)
    ap.add_argument("--width", type=int, default=384)
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    from ladi_vton_b200 import EMASC, AutoencoderKL, lib, ops, synthetic as S
    from ladi_vton_b200.eval import EMASC_IN, EMASC_OUT, INT_LAYERS, vae_recon_batch
    from ladi_vton_b200.vae import vae_param_shapes
    lib.load()
    dev = torch.device("cuda", torch.cuda.current_device())
    vae = AutoencoderKL().load_state_dict(S.random_state_dict(vae_param_shapes({}), 1235, device=dev, fast=True)).to(dev)
    emasc = EMASC(EMASC_IN, EMASC_OUT).load_state_dict(S.random_state_dict(S.emasc_param_shapes(EMASC_IN, EMASC_OUT), 1236, device=dev,
                                                                            fast=True)).to(dev)
    inp = S.synthetic_inputs(args.batch, args.height, args.width, ctx_dim=8)
    mask = (inp["mask_image"] >= 0.5).float()
    host = {k: v.contiguous().pin_memory() for k, v in dict(image=inp["image"], im_mask=inp["image"] * (1 - mask), inpaint_mask=mask).items()}
    out = torch.empty((args.batch, args.height, args.width, 3), dtype=torch.uint8).pin_memory()

    def call():
        batch = {k: v.to(dev, non_blocking=True) for k, v in host.items()}
        out.copy_(ops.image_save_u8(vae_recon_batch(vae, emasc, batch, INT_LAYERS, "nonlinear")), non_blocking=True)

    torch.cuda.manual_seed(0)
    with torch.no_grad():
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
    tflop = TFLOP_PER_IMAGE_512x384 * args.batch * (args.height * args.width) / (512 * 384)
    print(json.dumps(dict(workload=f"EMASC validation (2 VAE encodes, EMASC, decode, save_image quantisation) {args.height}x{args.width} "
                                   f"batch {args.batch}, H2D to D2H",
                          ms_per_batch_median=round(med, 2), ms_per_batch_min=round(ms[0], 2), ms_per_batch_max=round(ms[-1], 2),
                          images_per_s=round(args.batch * 1000.0 / med, 2), tflops=round(tflop / (med / 1000.0), 1), calls=args.calls,
                          gpu=card())))


if __name__ == "__main__":
    main()
