"""Throughput of the warping trainer's validation on the engine (eval_tps.compute_metric with refinement and the VGG loss): validation
pairs per second at 512 x 384, batch 16, full-width random weights, timed with CUDA events over the batches after a warm-up; reports the
card's name and power limit beside the number, and the peak memory of one VGG-loss call.

    python tools/bench_tps_val.py [--batches 8] [--warmup 2] [--batch_size 16] [--dense]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True).strip()
    except (OSError, subprocess.CalledProcessError):
        return "unknown"


def main():
    import torch
    from ladi_vton_b200 import synthetic as S
    from ladi_vton_b200.eval_tps import OUTPUTLIST, compute_metric
    from ladi_vton_b200.inference import SyntheticTryOnDataset
    from ladi_vton_b200.metrics import random_state_dict
    from ladi_vton_b200.vgg import VGG19, L1Loss, VGGLoss
    from ladi_vton_b200.warp import ConvNet_TPS, UNetVanilla, control_points
    p = argparse.ArgumentParser()
    p.add_argument("--batches", type=int, default=8)
    p.add_argument("--warmup", type=int, default=2)
    p.add_argument("--batch_size", type=int, default=16)
    p.add_argument("--dense", action="store_true")
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_tps_val: needs a CUDA device")
    dev = torch.device("cuda", 0)
    tps, ref = ConvNet_TPS(256, 192, 5 if a.dense else 21, 3), UNetVanilla(8 if a.dense else 24, 3, bilinear=True)
    tps.load_state_dict(S.warp_state_dict(tps.param_shapes(), 1, ctrl_bias=torch.atanh(control_points()).view(-1))).to(dev)
    ref.load_state_dict(S.warp_state_dict(ref.param_shapes(), 2)).to(dev)
    vgg = VGGLoss().load_state_dict(random_state_dict(VGG19().param_shapes(), 3)).to(dev)
    B = a.batch_size
    ds = SyntheticTryOnDataset(B, (512, 384), outputlist=OUTPUTLIST + (["dense_uv"] if a.dense else []))
    batch = torch.utils.data.default_collate([ds[i] for i in range(B)])
    batch = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in batch.items()}  # host loading is not what is timed
    compute_metric([batch] * a.warmup, tps, L1Loss(), vgg, refinement=ref)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    compute_metric([batch] * a.batches, tps, L1Loss(), vgg, refinement=ref)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    vgg(batch["im_cloth"], batch["cloth"])
    torch.cuda.synchronize()
    peak = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
    print(json.dumps(dict(card=card(), batch=B, batches=a.batches, dense=a.dense, ms_per_batch=round(ms / a.batches, 2),
                          pairs_per_s=round(B * a.batches / ms * 1e3, 1), vgg_loss_peak_mib=round(peak))))


if __name__ == "__main__":
    main()
