#!/usr/bin/env python
"""Times every distinct conv/GEMM call of one benchmarked UNet step at every N tile its shape allows, with CUDA events.

The descriptors come from the engine's plan-mode op trace (ladi_engine_trace) of the UNet step (512x384, batch 8, CFG: UNet batch 16),
the same records tools/profile_unet_step.py joins with its kernels; identical calls are counted once with their multiplicity.  Each
descriptor is run on seeded random inputs laid out with its own pitches (an in-place residual stays in place, a per-step bias table is
read at step 0, split-K gets the engine's 64 MiB workspace), warmed up, then timed over --iters back-to-back launches: once as the
library plans it, and once per N tile through force_bn (which also rules out split-K).  Prints one row per descriptor and, with the
card's name and power limit, the launch-weighted per-step total of three policies:
  old rule  -- min(ceil(tiles / SMs) * (BN + 64)) over 128 / 64 / 32, 128 for short reductions (the rule before 160 was a candidate);
  library   -- the plan of the library being timed (ladi_conv2d_plan);
  best      -- the fastest of 128 / 64 / 32 / 160 per descriptor.
Split-K plans are the same under every policy and count with the time of the library's plan.

  python tools/sweep_conv_tiles.py [--iters 200] [--out FILE.json] [--text FILE.txt] [--dump DIR]
  python tools/sweep_conv_tiles.py --replan FILE.json     (CPU: the policies' totals of a saved sweep under this library's plan)

--dump DIR writes each descriptor's output under the library's plan (bf16 bits, one .npy per descriptor) from the same seeded inputs.
Two builds of the library (LADI_B200_LIB selects the .so) dumped to two directories can then be compared bit for bit.
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

FIELDS = "k s p up n h w hin win cout nsrc c0 p0 c1 p1 nsc sc0c sc0p sc1c sc1p K wp bpr bss act op f32".split()
PTRS = "bias step res rs out".split()
TILES = (32, 64, 128, 160, 192, 256)
PLAN_TILES = (128, 64, 32, 160)  # what choose_plan may pick (192 / 256 only through force_bn)
SPLITK_WS_BYTES = 64 << 20  # the engine's split-K workspace
FAKE = 1 << 40  # 256-byte aligned fake device addresses for plan queries (nothing is dereferenced)


def descriptors(batch, height, width, guidance):
    """-> OrderedDict key -> {f: numeric fields, ptr: which pointers are set (res_inplace: residual == out), n: calls per step}."""
    import torch
    from ladi_vton_b200 import UNet2DConditionModel, engine as eng, synthetic as S, unet_param_shapes
    model = UNet2DConditionModel()
    model._sd = S.random_state_dict(unet_param_shapes({}), 1, fast=True)  # the trace depends on shapes only
    model.device = torch.device("cpu")
    model._pack()
    model._sd = None
    e = eng.Engine(eng.flatten(model.P), plan_only=True, **model.engine_config())
    ub = 2 * batch if guidance > 1.0 else batch
    out = OrderedDict()
    for line in e.trace(eng.MODULE_UNET, ub, height // 8, width // 8).splitlines():
        if not line.startswith("conv "):
            continue
        kv = dict(re.findall(r"(\w+)=@?([0-9a-fx]+)", line))
        f = {k: int(kv[k]) for k in FIELDS}
        a = {k: int(kv[k], 16) for k in PTRS}
        ptr = {"bias": a["bias"] != 0, "step": a["step"] != 0, "res": a["res"] != 0, "res_inplace": a["res"] != 0 and a["res"] == a["out"],
               "rs": a["rs"] != 0}
        key = tuple(f[k] for k in FIELDS) + tuple(ptr.values())
        out.setdefault(key, dict(f=f, ptr=ptr, n=0))["n"] += 1
    return out


def tag(f):
    kind = "gemm" if (f["k"] == 1 and f["h"] == 1) else ("up2x" if f["up"] else f"conv{f['k']}x{f['k']}" + ("s2" if f["s"] == 2 else ""))
    return f"{kind} {f['h']}x{f['w']}" if kind != "gemm" else f"gemm {f['w']}"


def fill_desc(d, f, ptr, addrs):
    """The conv descriptor of trace fields f; addrs: name -> device address (real buffers, or fake ones for a plan query)."""
    d.n, d.h_out, d.w_out, d.c_out, d.h_in, d.w_in = f["n"], f["h"], f["w"], f["cout"], f["hin"], f["win"]
    d.ksize, d.stride, d.pad_lo, d.up2x = f["k"], f["s"], f["p"], f["up"]
    d.n_src = f["nsrc"]
    d.src[0], d.src_c[0], d.src_pitch[0] = addrs["src0"], f["c0"], f["p0"]
    if f["nsrc"] > 1:
        d.src[1], d.src_c[1], d.src_pitch[1] = addrs["src1"], f["c1"], f["p1"]
    d.n_sc = f["nsc"]
    for i in range(f["nsc"]):
        d.sc[i], d.sc_c[i], d.sc_pitch[i] = addrs[f"sc{i}"], f[f"sc{i}c"], f[f"sc{i}p"]
    d.weight, d.k_total, d.weight_pitch = addrs["wt"], f["K"], f["wp"]
    if ptr["bias"]:
        d.bias, d.bias_per_row, d.bias_step_stride = addrs["bias"], f["bpr"], f["bss"]
    if ptr["step"]:
        d.step_ptr = addrs["step"]
    if ptr["res"]:
        d.residual, d.residual_pitch = addrs["out"] if ptr["res_inplace"] else addrs["res"], f["op"]
    if ptr["rs"]:
        d.row_scale = addrs["rs"]
    d.act, d.out, d.out_pitch, d.out_fp32 = f["act"], addrs["out"], f["op"], f["f32"]
    d.splitk_ws, d.splitk_ws_bytes = addrs["ws"], SPLITK_WS_BYTES
    return d


def fake_addrs():
    return {k: FAKE + (i << 32) for i, k in enumerate("src0 src1 sc0 sc1 wt bias step res rs out ws".split())}


def allowed_tiles(c_out):
    """N tiles worth timing: every tile up to c_out, and the narrowest one that covers it."""
    return [bn for bn in TILES if bn <= c_out or bn == min(t for t in TILES if t >= min(c_out, 256))]


def old_rule_bn(tiles_m, total_kb, c_out, sms):
    """choose_plan's N tile before 160 became a candidate (no split-K, no forced tile, no pairs)."""
    best, bn = None, 0
    for c in (128, 64, 32):
        if total_kb <= 8 and c_out >= 128 and c < 128:
            continue
        cost = -(-tiles_m * -(-c_out // c) // sms) * (c + 64)
        if best is None or cost < best:
            best, bn = cost, c
    return bn


def policies(rows, sms):
    """Per-step totals (us, launch-weighted) of the old rule, the library's plan and the per-descriptor best."""
    tot = {"old rule": 0.0, "library": 0.0, "best": 0.0}
    for r in rows:
        t, n = r["us"], r["calls"]
        if r["plan"]["splits"] > 1:
            for k in tot:
                tot[k] += n * r["plan_us"]
            continue
        tot["old rule"] += n * t[str(old_rule_bn(r["plan"]["tiles_m"], r["plan"]["total_kb"], r["f"]["cout"], sms))]
        tot["library"] += n * r["plan_us"]
        tot["best"] += n * min(t[str(b)] for b in PLAN_TILES if str(b) in t)
    return tot


def plan_dict(p):
    return {k: getattr(p, k) for k in ("bn", "splits", "staged", "stages", "tiles_m", "tiles_n", "total_kb")}


def report(res):
    g = res["gpu"]
    lines = [f"# {g['name']}, power limit {g['power_limit']}; {res['workload']}; {res['iters']} timed launches per descriptor and tile, "
             f"CUDA events; library {res['lib']}",
             f"{'#':>3} {'call':<14}{'M':>7}{'N':>6}{'K':>6} {'form':<10}{'n':>3} {'plan':<10}{'plan us':>9}"
             + "".join(f"{'bn' + str(b):>9}" for b in TILES)]
    for r in res["rows"]:
        f, p = r["f"], r["plan"]
        form = "+".join(x for x in [{1: "silu", 2: "geglu", 3: "gelu", 4: "relu"}.get(f["act"], ""), "res" if r["ptr"]["res"] else "",
                                    "rs" if r["ptr"]["rs"] else "", "step" if r["ptr"]["step"] else ""] if x) or "bias"
        pl = f"{p['bn']}" + (f"/S{p['splits']}" if p["splits"] > 1 else ("s" if p["staged"] else "f"))
        lines.append(f"{r['idx']:>3} {tag(f):<14}{r['M']:>7}{f['cout']:>6}{r['k_true']:>6} {form:<10}{r['calls']:>3} {pl:<10}{r['plan_us']:>9.1f}"
                     + "".join(f"{r['us'][str(b)]:>9.1f}" if str(b) in r["us"] else f"{'':>9}" for b in TILES))
    for k, v in res["step_ms"].items():
        lines.append(f"# per step, {k}: {v:.3f} ms of conv/GEMM (sum of calls x time per call)")
    return "\n".join(lines)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--height", type=int, default=512)
    ap.add_argument("--width", type=int, default=384)
    ap.add_argument("--guidance", type=float, default=7.5)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--dump", metavar="DIR", default=None)
    ap.add_argument("--out", metavar="FILE", default=None)
    ap.add_argument("--text", metavar="FILE", default=None)
    ap.add_argument("--replan", metavar="FILE", default=None)
    args = ap.parse_args()

    from ladi_vton_b200 import lib
    if args.replan:
        with open(args.replan) as fh:
            res = json.load(fh)
        for r in res["rows"]:
            r["plan"] = plan_dict(lib.conv_plan(fill_desc(lib.ConvDesc(), r["f"], r["ptr"], fake_addrs()), res["sms"]))
            b = r["plan"]["bn"]
            if r["plan"]["splits"] == 1:
                r["plan_us"] = r["us"][str(b)]
        res["step_ms"] = {k: v / 1e3 for k, v in policies(res["rows"], res["sms"]).items()}
        res["lib"] = lib.LIB_PATH + " (replanned; times from the saved sweep)"
        print(report(res))
        return

    import numpy as np
    import torch
    from bench import gpu_identity
    if not torch.cuda.is_available():
        raise SystemExit("sweep_conv_tiles.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    gpu = gpu_identity(0)
    ws = torch.empty(SPLITK_WS_BYTES // 4, dtype=torch.float32, device=dev)
    rows = []
    for i, e in enumerate(descriptors(args.batch, args.height, args.width, args.guidance).values()):
        f, ptr = e["f"], e["ptr"]
        g = torch.Generator(device=dev).manual_seed(1000 + i)
        rnd = lambda n, dt=torch.bfloat16, s=1.0: (torch.randn((n,), device=dev, generator=g) * s).to(dt)
        rows_out = f["n"] * f["h"] * f["w"]
        k_true = f["k"] ** 2 * (f["c0"] + f["c1"]) + f["sc0c"] + f["sc1c"]
        bufs = {"src0": rnd(f["n"] * f["hin"] * f["win"] * f["p0"]), "ws": ws,
                "wt": rnd(f["cout"] * (4 if f["up"] else 1) * f["wp"], s=k_true ** -0.5),
                "out": torch.zeros((rows_out * f["op"],), dtype=torch.float32 if f["f32"] else torch.bfloat16, device=dev)}
        if f["nsrc"] > 1:
            bufs["src1"] = rnd(f["n"] * f["hin"] * f["win"] * f["p1"])
        for s in range(f["nsc"]):
            bufs[f"sc{s}"] = rnd(rows_out * f[f"sc{s}p"])
        if ptr["bias"]:
            bufs["bias"] = rnd(rows_out if f["bpr"] else max(f["bss"], f["cout"]), torch.float32)
        if ptr["step"]:
            bufs["step"] = torch.zeros((2,), dtype=torch.int32, device=dev)
        if ptr["res"] and not ptr["res_inplace"]:
            bufs["res"] = rnd(rows_out * f["op"])
        if ptr["rs"]:
            bufs["rs"] = torch.rand((rows_out,), device=dev, generator=g)
        addrs = {k: v.data_ptr() for k, v in bufs.items()}
        init = None
        if ptr["res_inplace"]:
            bufs["out"].copy_(rnd(bufs["out"].numel()))
            init = bufs["out"].clone()

        def timed(force_bn):
            d = fill_desc(lib.ConvDesc(), f, ptr, addrs)
            d.force_bn = force_bn
            for _ in range(3):
                lib.call("ladi_conv2d_bf16", C.byref(d), stream)
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            for _ in range(args.iters):
                lib.call("ladi_conv2d_bf16", C.byref(d), stream)
            t1.record()
            torch.cuda.synchronize()
            return t0.elapsed_time(t1) * 1e3 / args.iters

        plan = plan_dict(lib.conv_plan(fill_desc(lib.ConvDesc(), f, ptr, addrs), sms))
        if args.dump:  # one launch of the library's plan on fresh inputs (an in-place residual is read before it is overwritten)
            if init is not None:
                bufs["out"].copy_(init)
            lib.call("ladi_conv2d_bf16", C.byref(fill_desc(lib.ConvDesc(), f, ptr, addrs)), stream)
            torch.cuda.synchronize()
            os.makedirs(args.dump, exist_ok=True)
            np.save(os.path.join(args.dump, f"conv{i:02d}.npy"), bufs["out"].view(torch.int32 if f["f32"] else torch.int16).cpu().numpy())
        r = dict(idx=i, f=f, ptr=ptr, calls=e["n"], M=rows_out, k_true=k_true, plan=plan, plan_us=timed(0),
                 us={str(b): timed(b) for b in allowed_tiles(f["cout"])})
        r["tflops"] = 2.0 * rows_out * f["cout"] * k_true / (r["plan_us"] * 1e-6) / 1e12
        rows.append(r)
        del bufs
    res = dict(gpu=gpu, sms=sms, iters=args.iters, lib=lib.LIB_PATH, rows=rows,
               workload=f"UNet step {args.height}x{args.width}, batch {args.batch}, UNet batch {2 * args.batch if args.guidance > 1 else args.batch}")
    res["step_ms"] = {k: v / 1e3 for k, v in policies(rows, sms).items()}
    text = report(res)
    print(text)
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)
    if args.text:
        with open(args.text, "w") as fh:
            fh.write(text + "\n")


if __name__ == "__main__":
    main()
