"""The kernel calls that tests/test_gpu_workload_census.py does not see, replayed one by one against a float64 reference with
per-element error bounds: the kernels the try-on pipeline launches from Python around the engine modules, and the front end of the
inference CLI.

The census (CPU).  The Python sequencing runs on CPU tensors with the ABI calls recorded instead of launched (`lib.RECORD`):
  * the pipeline pieces of bench.py's shapes -- the device path of `_prepare_mask_and_image` (`check_binarise`), `_pre`, one `_step` and
    `_post` -- at 8 x 512x384 with and without CFG, 4 x 1024x768 and 1 x 512x384.  The engine modules (VAE encode / decode, EMASC, UNet
    forward, `plan_context`) are stubbed down to what they launch from Python before their one module-level ABI call: the VAE's
    NCHW -> NHWC packing of its input, with the 1 / scaling_factor scale for the decoder's latents (the bodies behind the ABI calls are
    the other census's);
  * grids down-scaled by warp_grid_sample's grid resize up to the factor 5 its host check allows (SYNTHETIC: no workload does this);
  * the inference CLI's front end at batch 8, 512x384: `generate_warped_cloth` (ConvNet_TPS(256, 192, 21, 3) + UNetVanilla(24, 3)),
    `clip_preprocess`, the ViT-H/14 vision tower and the SD-2 text tower through `encode_text_word_embedding` with 16 pseudo-words.
    Modules are packed on the CPU from random weights; the towers pack one encoder layer and reuse it for every layer (all layers have
    the same shapes, so the call sequence is the full-depth one).
Each call is reduced to (entry point, scalar arguments, pointer operand present / absent) and deduplicated.  Convolutions / GEMMs and
LayerNorms use the workload census's field format; those it already replays are skipped.  Every other entry point must have a row in
SCHEMA (tests/kernel_check.py) (its argument names, with each pointer's role), or test_glue_census_integrity fails: a kernel added later cannot go unreplayed.

The replay (GPU).  Each descriptor goes through the same entry point with the same scalars on fresh buffers: inputs realistic for the
kind (images in [-1, 1], binary masks with values exactly 0.5, post-ReLU features, sampling grids inside and slightly outside [-1, 1]),
input pitch padding NaN, outputs NaN-poisoned over their full pitch plus a tail (finite afterwards in exactly the columns the call owns,
NaN elsewhere; in-place kernels leave their padding alone), and a second run must be bit-identical.

References and bounds (per element; the constants and the replays are tests/kernel_check.py's):
  exact     nhwc_to_nchw_clamp, inv_mask_rows, space_to_depth2, maxpool2, patchify,
            check_binarise (mask values with NaN kept, and both flags), image_out, image_out_u8 (numpy's round-half-even of the fp32 value);
  ROUND1    clip_embed, vit_assemble: two bf16 values summed in fp32 and rounded to bf16: 2^-8 |r|.  The fp32 sum is exact unless the
            exponents differ by more than ~16; then the fp32 and the bf16 rounding compound, and the error is at most
            (2^-8 + 2^-24) 2^e over a result of at least (1 + 2^-8 - 2^-24) 2^e, still below 2^-8 |r|.  The bound is the exact worst case
            of one rounding, so a measured ratio near 1 is expected;
  nchw_to_nhwc  (gate `mask < 0.5`, nearest /f) bit-equal to the fp32 product x * scale rounded to bf16, and within ROUND1 (1 + 2^-15) |r| of float64 (the decoder
            loads the latents with scale 1 / scaling_factor, whose fp32 product carries 2^-24 before the bf16 rounding);
  bilinear_down8   bit-equal to fp32 F.interpolate on the same device, and within 2^-23 sum|w x| of float64;
  ddim_cfg_step    three consecutive calls on distinct coefficient rows; after each step_ptr = [s + 1, 0], unet_in holds bf16(latents)
            bit-exactly in both CFG halves with channels >= 4 untouched, and the latents are within DDIM_ULPS * 2^-24 * M + 2^-24 |r| of
            float64, M = |sap / sqrt(a)| (|x| + sqrt(1-a) E) + |s1ap| E, E = |e_u| + g |e_t - e_u|: the CFG amplification enters through E;
  posterior_sample (2^-22 expf + 2^-23 rounding) on sigma*noise and the sum, logvar clamped to [-30, 20] as the reference clamps it;
  resampling (resize_aa, clip_preprocess, warp_grid_sample, upsample2x_bilinear_ac): torch's antialiased triangle filter restated in
            float64 (border renormalisation, truncation toward zero) and align_corners=True for the 2x upsample.  Bound: output rounding +
            2^-24 (taps_x + taps_y + 2) sum|w x| for the fp32 FMA chains + the fp32 weights' error, which comes from the sample position
            the kernel computes in fp32 (AA_POS below) and moves each normalised weight by at most (taps + 1) position errors / total.
            warp_grid_sample adds the grid's own resize error times W/2 times the local texel difference; clip_preprocess accepts every
            uint8 level its quantiser can reach within the bound of the value it quantises;
  feature_correlation   C_ACC sqrt(c) 2^-24 sum|a b| + bf16 rounding, reference from ConvNet_TPS's own bmm / view / transpose formula;
  l2norm_channels / channel_affine   (0.5 C_ACC sqrt(c) 2^-24 + 2^-22) |r| (fp32 sum of squares, sqrt, reciprocal) / one FMA, + bf16;
  tps_grid  tanhf 2^-22 relative, then the 25-term and 28-term fp32 dot products: C_ACC sqrt(K) 2^-24 sum|a b| with the points' and
            mapping's errors propagated through |inverse_kernel| and |target_coordinate_repr|;
  attention_small   float64 softmax with the causal mask applied in the reference, attn_expect with u_p = 2^-22 (P stays fp32), every
            query row checked;
  conv / ln  the workload census's replay_conv / replay_ln.
The CPU tests at the end show the bounds have teeth: the same checkers reject six simulated faults and accept honest fp32 emulations."""
import ctypes as C
import time
from collections import defaultdict

import pytest
import torch
import torch.nn.functional as F

from kernel_check import (GRID_DOWNSCALE, MODULE_ABI, REPLAY, SCHEMA, TRACED, U_BF16, Replay, aa_weights, assert_all_known, corr_expect,
                          ddim_expect, exact, glue_collect, glue_census, max_ratio, resample_expect, small_attn_expect, warp_expect)

# ================================================================================================================ the census (CPU)
WORKLOAD_CENSUS_ABI = ("ladi_attention_bf16", "ladi_attention_d512_bf16", "ladi_groupnorm_stats", "ladi_groupnorm_apply", "ladi_cls_attention",
                       "ladi_add_bf16", "ladi_timestep_embedding")  # what the engine modules' bodies issue (the other census)
KINDS = ["conv", "ln"] + sorted({k for k, _ in SCHEMA.values()})
# (label, images, height, width, guidance): bench.py's default, config 3 and config 0 shapes, and the call without guidance


# warp_grid_sample with the sampling grid DOWN-scaled, up to the factor 5 its host check allows (the CLI up-scales 256x192 -> 512x384):
# the antialiased branch of the grid resize, at an integer and at a non-integer factor


# ================================================================================================================ CPU: census integrity
def print_glue_census(desc, calls):
    print("\nglue and front-end census: calls (distinct descriptors not in the workload census) per kind")
    for wl, cnt in calls.items():
        tot = sum(v[0] for v in cnt.values())
        print(f"  {wl}: {tot} calls, {len(set().union(*(v[1] for v in cnt.values())))} new descriptors")
        print("    " + ", ".join(f"{k} {v[0]} ({len(v[1])})" for k, v in sorted(cnt.items())))
    per = defaultdict(int)
    for d in desc.values():
        per[d["kind"]] += 1
    print("  distinct over all workloads: " + ", ".join(f"{k} {per[k]}" for k in KINDS if per[k]))


def test_glue_census_integrity():
    from ladi_vton_b200 import lib
    desc, calls, unknown = glue_census()
    print_glue_census(desc, calls)
    issued = set()
    for wl, cnt in calls.items():
        assert sum(v[0] for v in cnt.values()) > 0, f"no calls recorded for {wl}"
    for d in desc.values():
        issued.add(d["kind"])
    unused = sorted(n for n in lib.SIGNATURES if n in SCHEMA and SCHEMA[n][0] not in issued)
    unused += sorted(n for n in lib.SIGNATURES if n not in SCHEMA and n not in TRACED and n not in MODULE_ABI and not n.startswith(
        ("ladi_abi", "ladi_last", "ladi_launch", "ladi_engine", "ladi_workspace", "ladi_unet_plan", "ladi_groupnorm_chunks", "ladi_ssim_partials"))
        and n not in WORKLOAD_CENSUS_ABI)
    print("  exported kernel entry points neither census issues (information): " + ", ".join(unused))
    assert_all_known(unknown)
    assert set(REPLAY) == set(KINDS) and {d["kind"] for d in desc.values()} <= set(REPLAY)
    for name, (kind, spec) in SCHEMA.items():
        assert name in lib.SIGNATURES and len(spec.split()) == len(lib.SIGNATURES[name][0]), f"SCHEMA row of {name} does not match its signature"
        assert any(a.endswith((":out", ":io")) for a in spec.split()), f"SCHEMA row of {name} names no output"
    by = defaultdict(list)
    for d in desc.values():
        by[d["kind"]].append(d["f"])
    # the paths this census exists to cover
    dd = by["ddim_cfg_step"]
    assert any(f["cfg"] and f["B"] * 4 * f["h"] * f["w"] > 256 for f in dd), "DDIM update with CFG over more than one CTA"
    assert any(not f["cfg"] and f["B"] * 4 * f["h"] * f["w"] > 256 for f in dd), "DDIM update without CFG over more than one CTA"
    assert any(f["n_image"] > 1 << 20 for f in by["check_binarise"]), "range check over more than 1 M image elements"
    assert {f["f"] for f in by["inv_mask_rows"]} >= {1, 2, 4, 8}, "inverse mask rows at factors 1, 2, 4 and 8"
    n2n = by["nchw_to_nhwc"]
    assert any(f["gate"] for f in n2n) and any(f["f"] == 8 for f in n2n), "layout kernel with the mask gate and with nearest /8"
    assert any(f["c_off"] > 0 and f["op"] > f["c_off"] + f["c"] for f in n2n), "layout kernel into a channel window of a wider pitch"
    assert any(f["scale"] != 1.0 and f["c"] == 4 for f in n2n), "latents loaded by the VAE decoder with the 1 / scaling_factor scale"
    assert any(not f["gate"] and f["c"] == 3 and f["op"] == 8 and f["h"] in (512, 1024) for f in n2n), "cloth packed for the VAE encoder"
    assert any(d["first"] == GRID_DOWNSCALE and d["f"]["gh"] == 5 * d["f"]["H"] for d in desc.values()), "grid down-scale at the limit"
    att = by["attention_small"]
    assert any(f["hd"] == 80 and not f["causal"] for f in att), "small attention with head width 80 (vision tower)"
    assert any(f["causal"] and f["nq"] == f["nkv"] == 77 for f in att), "causal small attention over 77 tokens (text tower)"
    rs = by["resize_aa"]
    assert any(f["h"] > f["oh"] for f in rs) and any(f["c_off"] > 0 for f in rs), "antialiased resize down-scaling, and into a channel window"
    assert any(f["h"] == 16 and f["w"] == 12 for f in by["feature_correlation"]), "feature correlation with h != w (16 x 12)"
    convs = by["conv"]
    s2d_out = {(f["n"], f["h"] // 2, f["w"] // 2, f["op"]) for f in by["space_to_depth2"]}
    assert any(f["act"] == 4 and (f["n"], f["hin"], f["win"], f["p0"]) in s2d_out for f in convs), "ReLU conv over a space-to-depth input"
    assert any(f["k"] == 1 and f["f32"] and f["cout"] == 3 and f["h"] == 512 for f in convs), "UNetVanilla 1x1 outc, fp32 out, 3 channels"
    for k in ("clip_preprocess", "warp_grid_sample", "tps_grid", "upsample2x_ac", "l2norm_channels", "channel_affine", "clip_embed", "patchify",
              "vit_assemble", "posterior_sample", "image_out", "image_out_u8", "bilinear_down8", "maxpool2", "nhwc_to_nchw_clamp", "ln"):
        assert by[k], f"no {k} descriptor in the census"


def test_glue_census_rejects_unknown_entry_point():
    """A workload that records an entry point without a SCHEMA row next to a known one: the census reports it, the integrity check fails."""
    known = ("ladi_inv_mask_rows", (C.c_void_p(16), 1, 8, 8, 2, C.c_void_p(32), C.c_void_p(0)))
    desc, calls, unknown = glue_collect([("fake workload", lambda: [known, ("ladi_not_in_the_schema", (C.c_void_p(16), 3, C.c_void_p(0)))])])
    assert unknown == ["ladi_not_in_the_schema"] and [d["kind"] for d in desc.values()] == ["inv_mask_rows"]
    with pytest.raises(AssertionError, match="ladi_not_in_the_schema"):
        assert_all_known(unknown)


# ================================================================================================================ CPU: the bounds have teeth


def test_teeth_correlation_index():
    g = torch.Generator().manual_seed(1)
    n, h, w, c = 2, 16, 12, 64
    fa, fb = (torch.randn((n, h, w, c), generator=g) / 8).bfloat16(), (torch.randn((n, h, w, c), generator=g) / 8).bfloat16()
    r, bound = corr_expect(fa.double(), fb.double())

    def emulate(transposed):
        a, b = fa.float().view(n, h * w, c), fb.float().view(n, h * w, c)
        ia = torch.arange(h * w)
        ya, xa = (ia // w, ia % w) if transposed else (ia % h, ia // h)  # honest: ia = xA * h + yA; fault: ia = yA * w + xA
        return (b @ a[:, ya * w + xa].transpose(1, 2)).view(n, h, w, h * w).bfloat16()
    assert max_ratio(emulate(False), r, bound) <= 1
    assert max_ratio(emulate(True), r, bound) > 1  # 1. correlation index transposed


def test_teeth_causal_mask():
    g = torch.Generator().manual_seed(2)
    T, heads, hd = 77, 2, 64
    q, k = ((torch.randn((T, heads * hd), generator=g) * 2 ** 0.5).bfloat16() for _ in range(2))
    v = torch.randn((T, heads * hd), generator=g).bfloat16()
    o, bound = small_attn_expect(q.double(), k.double(), v.double(), heads, hd ** -0.5, True)

    def emulate(extra):
        qh, kh, vh = (t.float().view(T, heads, hd).transpose(0, 1) for t in (q, k, v))
        s = (qh @ kh.transpose(1, 2)) * hd ** -0.5
        s = s.masked_fill(torch.ones((T, T), dtype=torch.bool).triu(1 + extra), -float("inf"))
        return (torch.softmax(s, -1) @ vh).transpose(0, 1).reshape(T, heads * hd).bfloat16()
    assert max_ratio(emulate(0), o, bound) <= 1
    assert max_ratio(emulate(1), o, bound) > 1  # 2. the mask admits key r + 1


def test_teeth_ddim_cfg_halves():
    g = torch.Generator().manual_seed(3)
    B, h, w, gs = 2, 8, 6, 7.5
    x, eu = torch.randn((B, 4, h, w), generator=g), torch.randn((B, 4, h, w), generator=g)
    et = eu + 0.3 * torch.randn((B, 4, h, w), generator=g)
    ab, abp = 0.3, 0.7
    row = torch.tensor([ab ** -0.5, (1 - ab) ** 0.5, abp ** 0.5, (1 - abp) ** 0.5, 0.0])
    r, bound = ddim_expect(x.double(), eu.double(), et.double(), row.double(), gs, True)

    def emulate(swap):
        a, b = (et, eu) if swap else (eu, et)
        e = a + gs * (b - a)
        return row[2] * ((x - row[1] * e) * row[0]) + row[3] * e
    assert max_ratio(emulate(False), r, bound) <= 1
    assert max_ratio(emulate(True), r, bound) > 1  # 3. CFG halves swapped


@pytest.mark.parametrize("gh,gw", [(16, 12), (160, 120)])  # the CLI's 2x up-scale of the grid, and a 5x down-scale (the host limit)
def test_teeth_grid_sample_align_corners(gh, gw):
    g = torch.Generator().manual_seed(4)
    n, c, H, W = 1, 3, 32, 24
    ys, xs = torch.meshgrid(torch.linspace(-1.06, 1.06, gh), torch.linspace(-1.06, 1.06, gw), indexing="ij")
    grid = torch.stack([xs + 0.02 * torch.randn((gh, gw), generator=g), ys + 0.02 * torch.randn((gh, gw), generator=g)], dim=2)[None]
    cloth = torch.rand((n, c, H, W), generator=g) * 2 - 1
    r, bound = warp_expect(grid.double(), cloth.double())

    def emulate(ac):
        hi = F.interpolate(grid.permute(0, 3, 1, 2), size=(H, W), mode="bilinear", antialias=True, align_corners=False).permute(0, 2, 3, 1)
        return F.grid_sample(cloth, hi, mode="bilinear", padding_mode="border", align_corners=ac).bfloat16()
    assert max_ratio(emulate(False), r, bound) <= 1
    assert max_ratio(emulate(True), r, bound) > 1  # 4. grid_sample with align_corners=True


def test_teeth_resize_border_tap():
    g = torch.Generator().manual_seed(5)
    x = torch.rand((2, 3, 64, 48), generator=g) * 2 - 1
    r, bound = resample_expect(x.double(), 28, 21, U_BF16)  # the clip_preprocess scale (512 -> 224)
    honest = F.interpolate(x, size=(28, 21), mode="bilinear", antialias=True, align_corners=False).bfloat16()
    Wy, _ = aa_weights(64, 28)
    Wx, _ = aa_weights(48, 21)
    Wx = Wx.clone()
    last = int(Wx[-1].nonzero().max())
    Wx[-1, last] = 0.0  # 5. the right-most output drops its last tap (weights renormalised over the rest)
    Wx[-1] /= Wx[-1].sum()
    faulty = (Wy.float() @ x @ Wx.float().t()).bfloat16()
    assert max_ratio(honest, r, bound) <= 1
    assert max_ratio(faulty, r, bound) > 1


def test_teeth_gate_threshold():
    g = torch.Generator().manual_seed(6)
    x = torch.rand((2, 3, 16, 12), generator=g) * 2 - 1
    m = (torch.rand((2, 1, 16, 12), generator=g) < 0.4).float()
    m[:, :, ::5, ::3] = 0.5
    ref = (x * (m < 0.5)).bfloat16()
    assert exact(ref, (x.double() * (m < 0.5)).float().bfloat16(), "")[0] == []
    assert exact((x * (m <= 0.5)).bfloat16(), ref, "")[0] != []  # 6. gate at mask <= 0.5 instead of < 0.5


# ================================================================================================================ GPU: replay
@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_glue_replay_against_float64(cuda, kind):
    desc, calls, unknown = glue_census()
    todo = [(key, d) for key, d in desc.items() if d["kind"] == kind]
    assert todo, f"no {kind} descriptor in the glue census"
    R = Replay(cuda, 4321)
    failures, worst, t0 = [], (0.0, "", ""), time.time()
    for key, d in todo:
        errs, res = REPLAY[kind](R, d["f"])
        if errs:
            failures.append(f"{key}\n    first issued by {d['first']}\n    " + "\n    ".join(errs))
        if res is not None and res[0] >= worst[0]:
            worst = (res[0], key, res[1])
        torch.cuda.empty_cache()
    print(f"\n{kind}: {len(todo)} distinct descriptors replayed in {time.time() - t0:.1f} s; worst err/bound {worst[0]:.3g}"
          + (f" ({worst[2]}; {worst[1]})" if worst[1] else ""))
    assert not failures, f"{len(failures)} of {len(todo)} {kind} descriptors fail:\n" + "\n".join(failures)
