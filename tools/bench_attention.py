#!/usr/bin/env python
"""Times every distinct attention call of the benchmarked workload, one descriptor at a time, with CUDA events.

The descriptors come from the engine's plan-mode op trace (ladi_engine_trace) of the UNet step (512x384, batch 8, CFG: UNet batch 16)
and of the VAE encode and decode at the same size; identical calls are counted once with their multiplicity.  Each descriptor is run on
seeded random inputs laid out with its own pitches and batch strides (so fused-QKV slices are read in place, as in the step), warmed
up, then timed over --iters back-to-back launches.  Prints one row per descriptor (launches per step, us per launch, TFLOP/s from
4 * batch * heads * nq * nkv * d) and the per-step attention total, with the card's name and power limit.

  python tools/bench_attention.py [--iters 200] [--dump DIR] [--out FILE.json]

--dump DIR writes each descriptor's output (bf16 bits, one .npy per descriptor) from the same seeded inputs.  Two builds of the library
(LADI_B200_LIB selects the .so) dumped to two directories can then be compared bit for bit.
"""
import argparse
import ctypes as C
import json
import os
import re
import sys
from collections import OrderedDict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

FIELDS = "d batch heads nq nkv qp qbs kp kbs vp vbs op obs scale".split()


def descriptors(batch, height, width, guidance):
    """-> OrderedDict key -> {module, f: {field: value}, n: calls per module run} from plan-only engines (CPU; random packed weights)."""
    import torch
    from ladi_vton_b200 import AutoencoderKL, UNet2DConditionModel, engine as eng, synthetic as S, unet_param_shapes
    from ladi_vton_b200.vae import vae_param_shapes

    def plan(model, shapes):
        model._sd = S.random_state_dict(shapes, 1, fast=True)  # the trace depends on shapes only
        model.device = torch.device("cpu")
        model._pack()
        model._sd = None
        return eng.Engine(eng.flatten(model.P), plan_only=True, **model.engine_config())

    unet, vae = plan(UNet2DConditionModel(), unet_param_shapes({})), plan(AutoencoderKL(), vae_param_shapes({}))
    ub = 2 * batch if guidance > 1.0 else batch
    runs = [("unet step", unet, eng.MODULE_UNET, ub, height // 8, width // 8),
            ("vae encode", vae, eng.MODULE_VAE_ENCODE, batch, height, width),
            ("vae decode", vae, eng.MODULE_VAE_DECODE, batch, height // 8, width // 8)]
    out = OrderedDict()
    for label, e, mod, b, h, w in runs:
        for line in e.trace(mod, b, h, w).splitlines():
            if not line.startswith("attn "):
                continue
            f = {k: v for k, v in re.findall(r"(\w+)=(\S+)", line) if k in FIELDS}
            f = {k: (float(v) if k == "scale" else int(v)) for k, v in f.items()}
            key = (label,) + tuple(f[k] for k in FIELDS)
            out.setdefault(key, dict(module=label, f=f, n=0))["n"] += 1
    return out


def make_call(f, dev, seed):
    """Seeded bf16 inputs in the descriptor's layout -> (descriptor, output buffer, entry point)."""
    import torch
    from ladi_vton_b200 import lib
    D, B, heads, nq, nkv = f["d"], f["batch"], f["heads"], f["nq"], f["nkv"]
    width = heads * D
    g = torch.Generator(device=dev).manual_seed(seed)
    bufs = {}
    for name, n_, std in (("q", nq, 2 ** 0.5), ("k", nkv, 2 ** 0.5), ("v", nkv, 1.0)):
        p, bs = f[name + "p"], f[name + "bs"]
        t = torch.zeros(((B - 1) * bs + n_ * p,), dtype=torch.bfloat16, device=dev)
        t.as_strided((B, n_, p), (bs, p, 1))[..., :width] = (torch.randn((B, n_, width), device=dev, generator=g) * std).bfloat16()
        bufs[name] = t
    out = torch.zeros(((B - 1) * f["obs"] + nq * f["op"],), dtype=torch.bfloat16, device=dev)
    d = lib.AttnDesc()
    d.batch, d.heads, d.nq, d.nkv = B, heads, nq, nkv
    d.q, d.q_pitch, d.q_batch_stride = bufs["q"].data_ptr(), f["qp"], f["qbs"]
    d.k, d.k_pitch, d.k_batch_stride = bufs["k"].data_ptr(), f["kp"], f["kbs"]
    d.v, d.v_pitch, d.v_batch_stride = bufs["v"].data_ptr(), f["vp"], f["vbs"]
    d.out, d.out_pitch, d.out_batch_stride = out.data_ptr(), f["op"], f["obs"]
    d.scale, d.variant, d.head_dim = f["scale"], 0, 0 if D == 64 else D
    name = "ladi_attention_bf16" if D == 64 else "ladi_attention_d512_bf16"
    return d, bufs, out, name


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--height", type=int, default=512)
    ap.add_argument("--width", type=int, default=384)
    ap.add_argument("--guidance", type=float, default=7.5)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--dump", metavar="DIR", default=None)
    ap.add_argument("--out", metavar="FILE", default=None)
    args = ap.parse_args()

    import numpy as np
    import torch
    from bench import gpu_identity
    from ladi_vton_b200 import lib
    if not torch.cuda.is_available():
        raise SystemExit("bench_attention.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    gpu = gpu_identity(0)
    rows, step_us = [], {}
    for i, (key, e) in enumerate(descriptors(args.batch, args.height, args.width, args.guidance).items()):
        f = e["f"]
        d, bufs, out, name = make_call(f, dev, 1000 + i)
        for _ in range(3):
            lib.call(name, C.byref(d), stream)
        torch.cuda.synchronize()
        if args.dump:
            os.makedirs(args.dump, exist_ok=True)
            np.save(os.path.join(args.dump, f"attn{i:02d}.npy"), out.view(torch.int16).cpu().numpy())
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(args.iters):
            lib.call(name, C.byref(d), stream)
        t1.record()
        torch.cuda.synchronize()
        us = t0.elapsed_time(t1) * 1e3 / args.iters
        flop = 4.0 * f["batch"] * f["heads"] * f["nq"] * f["nkv"] * f["d"]
        r = dict(idx=i, module=e["module"], calls=e["n"], us=us, tflops=flop / (us * 1e-6) / 1e12, flop=flop,
                 **{k: f[k] for k in ("d", "batch", "heads", "nq", "nkv", "qp", "kp", "vp", "op")})
        rows.append(r)
        step_us[e["module"]] = step_us.get(e["module"], 0.0) + us * e["n"]
        del bufs, out
    print(f"# {gpu['name']}, power limit {gpu['power_limit']}; {args.height}x{args.width}, batch {args.batch}; "
          f"{args.iters} timed launches per descriptor, CUDA events")
    print(f"{'#':>3} {'module':<11}{'d':>4}{'batch':>6}{'heads':>6}{'nq':>6}{'nkv':>6}{'qp':>6}{'calls':>6}{'us':>9}{'TFLOP/s':>9}")
    for r in rows:
        print(f"{r['idx']:>3} {r['module']:<11}{r['d']:>4}{r['batch']:>6}{r['heads']:>6}{r['nq']:>6}{r['nkv']:>6}{r['qp']:>6}"
              f"{r['calls']:>6}{r['us']:>9.1f}{r['tflops']:>9.1f}")
    for m, us in step_us.items():
        print(f"# {m}: attention {us / 1e3:.3f} ms (sum of calls x time per call)")
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(dict(gpu=gpu, iters=args.iters, lib=lib.LIB_PATH, rows=rows, module_ms={k: v / 1e3 for k, v in step_us.items()}), fh, indent=1)


if __name__ == "__main__":
    main()
