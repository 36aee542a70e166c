"""Throughput of the metric networks on the engine: FID Inception-v3 images/s (299 x 299, the FID / KID path), LPIPS AlexNet pairs/s and
SSIM pairs/s (512 x 384), at batch 32 and 64, with seeded random weights (the speed does not depend on the weight values), with the
networks in `--precision` bf16 (default) or tf32.  Prints one JSON line per measurement with the card's name and power limit.  Needs a
CUDA device; writes nothing.

    python tools/bench_metrics.py [--iters 10] [--warmup 3] [--precision bf16|tf32]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        name, limit = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
        return name, limit
    except Exception:  # noqa: BLE001 -- the numbers stay meaningful without the label, but say so
        return torch.cuda.get_device_name(), "unknown"


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / 1e3 / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--precision", choices=["bf16", "tf32"], default="bf16")
    a = ap.parse_args()
    from ladi_vton_b200.metrics import FIDInceptionV3, LPIPSAlex, random_state_dict, ssim
    dev = torch.device("cuda:0")
    name, limit = card()
    inc = FIDInceptionV3(a.precision)
    inc.load_state_dict(random_state_dict(inc.param_shapes(), 0)).to(dev)
    lp = LPIPSAlex(a.precision)
    lp.load_state_dict(random_state_dict(lp.param_shapes(), 1)).to(dev)
    g = torch.Generator(device=dev).manual_seed(0)
    for batch in (32, 64):
        px = torch.rand(batch, 3, 299, 299, generator=g, device=dev) * 255
        x = torch.rand(batch, 3, 512, 384, generator=g, device=dev)
        y = torch.rand(batch, 3, 512, 384, generator=g, device=dev)
        for what, fn, unit in (("inception_fid", lambda: inc(px), "images/s"), ("lpips_alex", lambda: lp(x, y), "pairs/s"),
                               ("ssim", lambda: ssim(x, y), "pairs/s")):
            s = timed(fn, a.iters, a.warmup)
            print(json.dumps(dict(metric=what, precision=a.precision, batch=batch, seconds_per_batch=round(s, 6), rate=round(batch / s, 1), unit=unit, gpu=name,
                                  power_limit=limit)))


if __name__ == "__main__":
    main()
