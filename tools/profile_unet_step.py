#!/usr/bin/env python
"""Per-launch profile of the benchmarked denoising step: where the step's time goes, launch by launch.

Builds the pipeline the way bench.py does (512x384, batch 8, CFG: UNet batch 16), runs one call, then traces ONE replay of the captured
step graph with torch.profiler (CUDA activities).  The kernels are joined, in launch order, with the engine's plan-mode op trace
(ladi_engine_trace) of the same UNet forward: every convgemm_kernel launch is one `conv` record (a split-K reduce belongs to the
conv before it), and every attention kernel launch is one `attn` record.  Kernel times are exclusive, as in bench.py's in_graph figures: with programmatic dependent launch a kernel starts
while its predecessor drains, and only the part after the predecessor's end is charged to it.

Writes OUT/profile.json (one row per launch) and OUT/profile.txt (launches and descriptors sorted by time), with the card's name and
power limit.  Exits non-zero when the kernel and trace counts of the conv or attention family disagree, or when the rows do not add
up to the step's wall time within 1%.

  python tools/profile_unet_step.py --out DIR [--batch 8 --height 512 --width 384]
"""
import argparse
import json
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PEAK_TFLOPS, PEAK_GBS = 989.0, 3350.0  # H100 SXM data sheet (dense bf16, HBM3) at up to 700 W: ceilings, not rates seen here
ACT = {0: "", 1: "silu", 2: "geglu", 3: "gelu", 4: "relu"}


def parse_conv(line):
    f = dict(re.findall(r"(\w+)=@?([0-9a-fx]+)", line))
    i = lambda k: int(f[k], 16) if k in ("res", "rs") else int(f[k])
    k, up = i("k"), i("up")
    M, N = i("n") * i("h") * i("w"), i("cout")
    k_true = k * k * (i("c0") + i("c1")) + i("sc0c") + i("sc1c")
    n_eff = N // 2 if i("act") == 2 else N
    a_bytes = 2 * i("n") * i("hin") * i("win") * (i("c0") + i("c1")) + 2 * M * (i("sc0c") + i("sc1c"))
    hbm = a_bytes + 2 * N * i("K") * (4 if up else 1) + (4 if i("f32") else 2) * M * n_eff + (2 * M * N if i("res") else 0)
    kind = "gemm" if (k == 1 and i("h") == 1) else ("up2x" if up else f"conv{k}x{k}" + ("s2" if i("s") == 2 else ""))
    form = "+".join(x for x in [ACT[i("act")], "res" if i("res") else "", "rowscale" if i("rs") else "",
                                "rowbias" if i("bpr") else "", "stepbias" if i("bss") else "", "fp32" if i("f32") else ""] if x) or "bias"
    return dict(kind=kind, level=f"{i('h')}x{i('w')}", M=M, N=N, K=k_true, form=form, flop=2.0 * M * N * k_true, hbm_bytes=hbm)


def parse_attn(line):
    f = {k: int(v) for k, v in re.findall(r"(\w+)=(\d+)\b(?![.@])", line) if k in ("d", "batch", "heads", "nq", "nkv")}
    B, h, nq, nkv, d = f["batch"], f["heads"], f["nq"], f["nkv"], f["d"]
    # Q, K, V read once and O written once (bf16): the least traffic the call needs
    return dict(kind="attn", shape=f"d={d} B={B} h={h} nq={nq} nkv={nkv}", flop=4.0 * B * h * nq * nkv * d,
                hbm_bytes=2 * B * h * d * (2 * nq + 2 * nkv))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--height", type=int, default=512)
    ap.add_argument("--width", type=int, default=384)
    ap.add_argument("--ddim-steps", type=int, default=50)
    ap.add_argument("--guidance", type=float, default=7.5)
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile
    from bench import gpu_identity
    from ladi_vton_b200 import engine as eng, synthetic as S
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    B, H, W = args.batch, args.height, args.width
    pipe, _ = S.build_pipeline(dev, weights_on_device=True)
    inp = {k: v.to(dev) for k, v in S.synthetic_inputs(B, H, W, seed=1234).items()}
    gen = torch.Generator(device=dev).manual_seed(1234)
    for _ in range(2):  # the first call captures the graphs
        pipe(image=inp["image"], mask_image=inp["mask_image"], pose_map=inp["pose_map"], warped_cloth=inp["warped_cloth"],
             prompt_embeds=inp["prompt_embeds"], negative_prompt_embeds=inp["negative_prompt_embeds"], height=H, width=W,
             num_inference_steps=args.ddim_steps, guidance_scale=args.guidance, generator=gen, output_type="pt")
    torch.cuda.synchronize()
    s = next(iter(pipe._sessions.values()))
    if s.g_step is None:
        raise SystemExit("the pipeline captured no step graph")
    s.step.zero_()
    s.g_step.replay()
    torch.cuda.synchronize()
    s.step.zero_()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        s.g_step.replay()
        torch.cuda.synchronize()
    ev = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "Memcpy" not in e.name
                 and "Memset" not in e.name), key=lambda e: e.time_range.start)

    Bp = 2 * B if args.guidance > 1.0 else B
    trace = pipe.unet.engine.trace(eng.MODULE_UNET, Bp, H // 8, W // 8).splitlines()
    convs = [parse_conv(l) for l in trace if l.startswith("conv ")]
    attns = [parse_attn(l) for l in trace if l.startswith("attn ")]
    n_attn_trace = len(attns)

    rows, prev_end, ci, ai = [], None, 0, 0
    for e in ev:
        st = e.time_range.start if prev_end is None else max(e.time_range.start, prev_end)
        us = max(0.0, e.time_range.end - st)
        prev_end = e.time_range.end if prev_end is None else max(prev_end, e.time_range.end)
        m = re.search(r"convgemm_kernel<(\d+), (true|false)>", e.name)
        if m:
            if ci >= len(convs):
                ci += 1
                continue
            r = dict(convs[ci], module=f"{convs[ci]['kind']} {convs[ci]['level']}", kernel="convgemm_kernel", BN=int(m.group(1)),
                     pair=m.group(2) == "true", us=us, idx=ci)
            rows.append(r)
            ci += 1
        elif "attention_" in e.name and ai < len(attns):
            rows.append(dict(attns[ai], module="attention", kernel=re.sub(r"\(.*", "", e.name)[-80:], us=us, idx=ai))
            ai += 1
        elif "splitk_reduce" in e.name and rows and rows[-1].get("kernel") == "convgemm_kernel":
            rows[-1]["us"] += us
            rows[-1]["splitk_reduce"] = True
        else:
            fam = ("attention" if "attention_" in e.name else "norm" if ("gn_" in e.name or "layernorm" in e.name) else "other")
            rows.append(dict(module=fam, kernel=re.sub(r"\(.*", "", e.name)[-80:], us=us))
    wall = (prev_end - ev[0].time_range.start) if ev else 0.0
    total = sum(r["us"] for r in rows)
    n_conv_k = sum(1 for e in ev if "convgemm_kernel" in e.name)
    n_attn_k = sum(1 for e in ev if "attention_" in e.name)
    for r in rows:
        r["share"] = r["us"] / wall if wall else None
        if "flop" in r:
            t = r["us"] * 1e-6
            r["tflops"] = r["flop"] / t / 1e12 if t else None
            t_tc, t_mem = r["flop"] / (PEAK_TFLOPS * 1e12), r["hbm_bytes"] / (PEAK_GBS * 1e9)
            r["bound"] = "tensor" if t_tc >= t_mem else "hbm"
            r["roofline_frac"] = max(t_tc, t_mem) / t if t else None

    errors = []
    if n_conv_k != len(convs):
        errors.append(f"conv family: {n_conv_k} convgemm_kernel launches in the step graph, {len(convs)} conv records in the engine trace")
    if n_attn_k != n_attn_trace:
        errors.append(f"attention family: {n_attn_k} attention kernel launches, {n_attn_trace} attn records in the engine trace")
    if wall and abs(total - wall) > 0.01 * wall:
        errors.append(f"rows sum to {total:.1f} us, the step's wall time is {wall:.1f} us")

    # descriptors: identical (kind, level, M, N, K, form, BN) launches summed
    desc = {}
    for r in rows:
        if "BN" not in r:
            continue
        key = (r["module"], r["M"], r["N"], r["K"], r["form"], r["BN"])
        d = desc.setdefault(key, dict(module=r["module"], M=r["M"], N=r["N"], K=r["K"], form=r["form"], BN=r["BN"], launches=0, us=0.0, flop=0.0))
        d["launches"] += 1; d["us"] += r["us"]; d["flop"] += r["flop"]
    descs = sorted(desc.values(), key=lambda d: -d["us"])
    for d in descs:
        d["tflops"] = d["flop"] / (d["us"] * 1e-6) / 1e12 if d["us"] else None
        d["share"] = d["us"] / wall if wall else None
    adesc = {}
    for r in rows:
        if "shape" in r:
            d = adesc.setdefault(r["shape"], dict(shape=r["shape"], launches=0, us=0.0, flop=0.0))
            d["launches"] += 1; d["us"] += r["us"]; d["flop"] += r["flop"]
    adescs = sorted(adesc.values(), key=lambda d: -d["us"])
    for d in adescs:
        d["tflops"] = d["flop"] / (d["us"] * 1e-6) / 1e12 if d["us"] else None
        d["share"] = d["us"] / wall if wall else None
    fam = {}
    for r in rows:
        k = "conv" if "BN" in r else r["module"]
        fam[k] = fam.get(k, 0.0) + r["us"]

    os.makedirs(args.out, exist_ok=True)
    gpu = gpu_identity(0)
    res = {"gpu": gpu, "workload": f"{H}x{W}, batch {B}, UNet batch {Bp}, one replay of the step graph", "step_wall_us": wall,
           "rows_sum_us": total, "family_us": fam, "conv_launches": n_conv_k, "conv_records": len(convs), "errors": errors,
           "peak_source": "H100 SXM data sheet: 989 TFLOP/s dense bf16, 3.35 TB/s HBM3 (700 W)", "descriptors": descs,
           "attention_descriptors": adescs, "launches": rows}
    with open(os.path.join(args.out, "profile.json"), "w") as f:
        json.dump(res, f, indent=1)
    lines = [f"# {gpu['name']}, power limit {gpu['power_limit']}; {res['workload']}",
             f"# step wall {wall / 1e3:.3f} ms, rows sum {total / 1e3:.3f} ms; " + ", ".join(f"{k} {v / 1e3:.3f} ms" for k, v in fam.items()),
             "", "## conv/GEMM descriptors, by total time",
             f"{'module':<16}{'M':>7}{'N':>6}{'K':>6} {'form':<16}{'BN':>4}{'n':>4}{'ms':>8}{'TFLOP/s':>9}{'share':>7}"]
    for d in descs:
        lines.append(f"{d['module']:<16}{d['M']:>7}{d['N']:>6}{d['K']:>6} {d['form']:<16}{d['BN']:>4}{d['launches']:>4}{d['us'] / 1e3:>8.3f}"
                     f"{d['tflops']:>9.1f}{100 * d['share']:>6.1f}%")
    lines += ["", "## attention descriptors, by total time", f"{'shape':<42}{'n':>4}{'ms':>8}{'TFLOP/s':>9}{'share':>7}"]
    for d in adescs:
        lines.append(f"{d['shape']:<42}{d['launches']:>4}{d['us'] / 1e3:>8.3f}{d['tflops']:>9.1f}{100 * d['share']:>6.1f}%")
    lines += ["", "## launches, by time",
              f"{'#':>4} {'module':<16}{'M':>7}{'N':>6}{'K':>6} {'form':<16}{'BN':>4}{'us':>9}{'TFLOP/s':>9}{'MB':>8} {'bound':<7}{'share':>7}"]
    for r in sorted(rows, key=lambda r: -r["us"]):
        if "BN" in r:
            lines.append(f"{r['idx']:>4} {r['module']:<16}{r['M']:>7}{r['N']:>6}{r['K']:>6} {r['form']:<16}{r['BN']:>4}{r['us']:>9.1f}"
                         f"{r['tflops']:>9.1f}{r['hbm_bytes'] / 1e6:>8.1f} {r['bound']:<7}{100 * r['share']:>6.2f}%")
        elif "shape" in r:
            lines.append(f"{r['idx']:>4} {'attention':<16}{r['shape']:>42}{'':>4}{r['us']:>9.1f}{r['tflops']:>9.1f}"
                         f"{r['hbm_bytes'] / 1e6:>8.1f} {r['bound']:<7}{100 * r['share']:>6.2f}%")
        else:
            lines.append(f"{'':>4} {r['module']:<16}{r['kernel'][-40:]:>31}{'':>4}{r['us']:>9.1f}{'':>26}{100 * r['share']:>6.2f}%")
    with open(os.path.join(args.out, "profile.txt"), "w") as f:
        f.write("\n".join(lines + [""] + [f"ERROR: {e}" for e in errors]) + "\n")
    print("\n".join(lines[:2] + lines[3:25]))
    if errors:
        raise SystemExit("profile mismatch: " + "; ".join(errors))


if __name__ == "__main__":
    main()
