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
LayerNorms use the other census's field format; those it already replays are skipped.  Every other entry point must have a row in
SCHEMA (its argument names, with each pointer's role), or test_glue_census_integrity fails: a kernel added later cannot go unreplayed.

The replay (GPU).  Each descriptor goes through the same entry point with the same scalars on fresh buffers: inputs realistic for the
kind (images in [-1, 1], binary masks with values exactly 0.5, post-ReLU features, sampling grids inside and slightly outside [-1, 1]),
input pitch padding NaN, outputs NaN-poisoned over their full pitch plus a tail (finite afterwards in exactly the columns the call owns,
NaN elsewhere; in-place kernels leave their padding alone), and a second run must be bit-identical.

References and bounds (per element; U_BF16, U_F32, C_ACC and EPS24 as in the other census):
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
  conv / ln  the other census's replay_conv / replay_ln, unchanged.
The CPU tests at the end show the bounds have teeth: the same checkers reject six simulated faults and accept honest fp32 emulations."""
import ctypes as C
import functools
import math
import time
from collections import OrderedDict, defaultdict

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from test_gpu_workload_census import (C_ACC, EPS24, U_BF16, U_F32, Replay, _bitwise_equal, _layout, _pick, attn_expect, census, parse,
                                      ratio, replay_conv, replay_ln)

ROUND1 = 2.0 ** -8     # one round-to-nearest to bf16 (8-bit significand)
DDIM_ULPS = 8.0        # the DDIM update's seven fp32 roundings (CFG difference, product, sum, two products, difference, scale), plus one
AA_POS = 2.0 ** -23    # relative error of the fp32 sample position (center = scale (o + 0.5), argument (j - center + 0.5) / scale)
NAN = float("nan")

# ================================================================================================================ the census (CPU)
# entry point -> (kind, its arguments in order: pointers are "name:role" with role in / out / io (in place); "stream" is dropped)
SCHEMA = {
    "ladi_check_binarise": ("check_binarise", "image:in n_image mask:io n_mask flags:io stream"),
    "ladi_bilinear_down8": ("bilinear_down8", "x:in n c H W out:out stream"),
    "ladi_nchw_f32_to_nhwc_bf16": ("nchw_to_nhwc", "x:in n c h w f scale gate:in out:out op c_off stream"),
    "ladi_posterior_sample": ("posterior_sample", "mom:in mp noise:in n cz h w scale out:out stream"),
    "ladi_inv_mask_rows": ("inv_mask_rows", "mask:in n H W f out:out stream"),
    "ladi_ddim_cfg_step": ("ddim_cfg_step", "eps:in ep lat:io uin:io inp B h w cfg guidance coef:in step:io advance noise:in stream"),
    "ladi_image_out": ("image_out", "x:in f32 n h w xp out:out stream"),
    "ladi_image_out_u8": ("image_out_u8", "x:in f32 n h w xp out:out stream"),
    "ladi_resize_aa": ("resize_aa", "x:in n c h w oh ow out:out op c_off stream"),
    "ladi_clip_preprocess": ("clip_preprocess", "x:in n c h w oh ow mean:in std:in quantise out:out stream"),
    "ladi_space_to_depth2": ("space_to_depth2", "x:in n h w c xp out:out op stream"),
    "ladi_channel_affine": ("channel_affine", "x:io rows c pitch scale:in shift:in stream"),
    "ladi_l2norm_channels": ("l2norm_channels", "x:io rows c pitch stream"),
    "ladi_feature_correlation": ("feature_correlation", "fa:in fb:in n h w c out:out op stream"),
    "ladi_tps_grid": ("tps_grid", "theta:in tp inv:in rep:in n n_ctrl npts points:out grid:out stream"),
    "ladi_warp_grid_sample": ("warp_grid_sample", "grid:in gh gw cloth:in n c H W out:out op c_off stream"),
    "ladi_maxpool2_nhwc": ("maxpool2", "x:in n h w c out:out stream"),
    "ladi_upsample2x_bilinear_ac": ("upsample2x_ac", "x:in n h w c out:out stream"),
    "ladi_nhwc_f32_to_nchw_clamp": ("nhwc_to_nchw_clamp", "x:in n c h w xp lo hi out:out stream"),
    "ladi_attention_small": ("attention_small", "q:in k:in v:in out:out B heads nq nkv hd qp kp vp op qbs kbs vbs obs scale causal stream"),
    "ladi_clip_embed": ("clip_embed", "src:in tok:in wemb:in pos:in out:out rows seq c op stream"),
    "ladi_patchify": ("patchify", "px:in out:out n ch h w patch kpad stream"),
    "ladi_vit_assemble": ("vit_assemble", "patch:in pp cls:in pos:in out:out n np c stream"),
}
TRACED = {"ladi_conv2d_bf16": "conv", "ladi_layernorm": "ln"}  # through test_engine_trace.python_trace, in the other census's fields
MODULE_ABI = ("ladi_unet_forward", "ladi_vae_encode", "ladi_vae_decode_emasc", "ladi_emasc_forward", "ladi_inversion_adapter_forward",
              "ladi_denoise_loop")
WORKLOAD_CENSUS_ABI = ("ladi_attention_bf16", "ladi_attention_d512_bf16", "ladi_groupnorm_stats", "ladi_groupnorm_apply", "ladi_cls_attention",
                       "ladi_add_bf16", "ladi_timestep_embedding")  # what the engine modules' bodies issue (the other census)
KINDS = ["conv", "ln"] + sorted({k for k, _ in SCHEMA.values()})
# (label, images, height, width, guidance): bench.py's default, config 3 and config 0 shapes, and the call without guidance
PIPE_WORKLOADS = [("512x384, 8 images, CFG (bench default)", 8, 512, 384, 7.5),
                  ("1024x768, 4 images, CFG (bench config 3)", 4, 1024, 768, 7.5),
                  ("one 512x384 image, CFG (bench config 0 shape)", 1, 512, 384, 7.5),
                  ("512x384, 8 images, no guidance", 8, 512, 384, 1.0)]
FRONTEND = "inference CLI front end, 8 x 512x384 (warping, CLIP preprocess, vision tower, text tower)"


class _Stub:
    """Stands in for the pipeline's engine modules: right shapes, and only the kernels the real methods launch from Python before their
    one module-level ABI call (the workload census covers the bodies behind that call).  `AutoencoderKL.encode_nhwc` packs an NCHW input
    into a zeroed NHWC buffer of pitch 8, and `decode_nhwc` packs the latents the same way with the 1 / scaling_factor scale (vae.py);
    `UNet2DConditionModel.forward_nhwc`, `plan_context` and `EMASC.__call__` launch nothing before theirs."""

    def __init__(self, H, W):
        self.H, self.W = H, W
        self.config = type("Cfg", (), {"scaling_factor": 0.18215})()

    def encode_nhwc(self, x, nhwc=False):
        from ladi_vton_b200 import ops
        B = x.shape[0]
        if not nhwc:
            ops.nchw_to_nhwc(x.contiguous(), torch.zeros((B, self.H, self.W, 8), dtype=torch.bfloat16))
        e = lambda f, c: torch.empty((B, self.H // f, self.W // f, c), dtype=torch.bfloat16)  # noqa: E731
        return torch.empty((B, self.H // 8, self.W // 8, 8)), [None, e(1, 128), e(1, 128), e(2, 256), e(4, 512), e(8, 512)]

    def decode_nhwc(self, z, feats=None, int_layers=None, scale=1.0):
        from ladi_vton_b200 import ops
        B, _, h, w = z.shape
        ops.nchw_to_nhwc(z.contiguous(), torch.zeros((B, h, w, 8), dtype=torch.bfloat16), scale=scale)
        return torch.empty((B, self.H, self.W, 4))

    def forward_nhwc(self, x_in, step):
        return torch.empty((x_in.shape[0], x_in.shape[1], x_in.shape[2], 4))

    def plan_context(self, ctx, out=None):
        return out

    def __call__(self, sel, inv):
        return list(sel)


def _record(fn):
    from ladi_vton_b200 import lib
    lib.RECORD = []
    try:
        with torch.no_grad():
            fn()
        return lib.RECORD
    finally:
        lib.RECORD = None


def _pipeline_calls(B, H, W, guidance):
    from ladi_vton_b200 import ops
    from ladi_vton_b200.pipeline import StableDiffusionTryOnePipeline as Pipe, _Session
    cfg = guidance > 1.0
    h, w = H // 8, W // 8
    stub = _Stub(H, W)
    pipe = type("PipeStub", (), {})()
    pipe.vae = pipe.unet = pipe.emasc = stub
    pipe.emasc_int_layers, pipe.vae_scale_factor, pipe.device = [1, 2, 3, 4, 5], 8, torch.device("cpu")
    s = _Session(B, 2 * B if cfg else B, h, w, H, W, 32, 18, (2 * B if cfg else B, 77, 1024), 8, torch.device("cpu"))
    s.coef = torch.zeros((50, 8))
    lay = dict(B=B, cfg=cfg, no_pose=False, cloth=True, c_mask=4, c_masked=5, c_pose=9, c_cloth=27)

    def run():
        ops.check_binarise_(s.image, s.mask, s.flags)  # _prepare_mask_and_image's device path (CUDA inputs)
        Pipe._pre(pipe, s, lay)
        Pipe._step(pipe, s, cfg, guidance)
        Pipe._post(pipe, s, lay)
    return _record(run)


def _cpu_pack(m, sd):
    m._sd, m.device = sd, torch.device("cpu")
    m._pack()
    m._sd = None
    return m


def _cpu_tower(cls, seed):
    from ladi_vton_b200 import synthetic as S
    depth = cls().config.num_hidden_layers
    t = cls(num_hidden_layers=1)
    _cpu_pack(t, S.random_state_dict(t.param_shapes(), seed, fast=True))
    p0 = f"{t.prefix}.encoder.layers.0."
    for i in range(1, depth):
        t.P.update({k.replace(p0, f"{t.prefix}.encoder.layers.{i}."): v for k, v in list(t.P.items()) if k.startswith(p0)})
    t.config["num_hidden_layers"] = depth
    return t


def _frontend_calls(B=8, H=512, W=384, num_vstar=16):
    from ladi_vton_b200 import CLIPTextModel, CLIPVisionModelWithProjection, encode_text_word_embedding, generate_warped_cloth, synthetic as S
    from ladi_vton_b200.inference import StandInTokenizer, clip_pixel_values, prompts_for
    from ladi_vton_b200.warp import ConvNet_TPS, UNetVanilla
    tps, ref = ConvNet_TPS(256, 192, 21, 3), UNetVanilla(24, 3, bilinear=True)
    _cpu_pack(tps, S.warp_state_dict(tps.param_shapes(), 13))
    _cpu_pack(ref, S.warp_state_dict(ref.param_shapes(), 14))
    vision, text = _cpu_tower(CLIPVisionModelWithProjection, 11), _cpu_tower(CLIPTextModel, 10)
    tok = StandInTokenizer()
    ids = tok(prompts_for(["upper_body", "lower_body", "dresses", "upper_body"] * (B // 4), num_vstar), max_length=77).input_ids
    cloth = torch.zeros((B, 3, H, W))

    def run():
        generate_warped_cloth(tps, ref, cloth, torch.zeros((B, 3, H, W)), torch.zeros((B, 18, H, W)))
        vision(clip_pixel_values(cloth, torch.device("cpu")))
        encode_text_word_embedding(text, ids, torch.zeros((B, num_vstar, 1024)), num_vstar)
    return _record(run)


def _val(a):
    return getattr(a, "value", a)


def describe(name, args, schema=None):
    """-> (kind, OrderedDict of fields) of one recorded call; raises KeyError for an entry point without a row in `schema` (default SCHEMA)."""
    kind, spec = (SCHEMA if schema is None else schema)[name]
    names = spec.split()
    assert len(names) == len(args), f"{name}: {len(args)} arguments recorded, SCHEMA names {len(names)}"
    f = OrderedDict()
    for nm, a in zip(names, args):
        if nm == "stream":
            continue
        if ":" in nm:
            assert isinstance(a, C.c_void_p), f"{name}: argument {nm} is not a pointer"
            f[nm.split(":")[0]] = 1 if a.value else 0
        else:
            assert isinstance(a, (int, float)) and not isinstance(a, bool), f"{name}: argument {nm} is not a scalar"
            f[nm] = a
    return kind, f


_GLUE = None
# warp_grid_sample with the sampling grid DOWN-scaled, up to the factor 5 its host check allows (the CLI up-scales 256x192 -> 512x384):
# the antialiased branch of the grid resize, at an integer and at a non-integer factor
GRID_DOWNSCALE = "grid down-scaled up to the host limit (synthetic)"
SYNTHETIC = [("warp_grid_sample", OrderedDict(grid=1, gh=320, gw=240, cloth=1, n=2, c=3, H=64, W=48, out=1, op=8, c_off=0)),
             ("warp_grid_sample", OrderedDict(grid=1, gh=250, gw=235, cloth=1, n=2, c=3, H=64, W=48, out=1, op=24, c_off=21))]


def collect(work):
    """work = [(workload label, () -> recorded calls)] -> (desc, calls, unknown): desc = OrderedDict key -> {kind, f, first, n} of the
    descriptors the workload census does not replay; calls = {workload: {kind: [calls, set of keys]}}; unknown = entry points recorded
    without a SCHEMA row."""
    import test_engine_trace as tt
    known = census()[0]
    desc, calls, unknown = OrderedDict(), OrderedDict(), []
    for wl, rec in work:
        cnt = calls.setdefault(wl, defaultdict(lambda: [0, set()]))
        for name, args in rec():
            if name in MODULE_ABI:
                continue
            if name in TRACED:
                op, f = parse(tt.python_trace([(name, args)])[0])
                kind, key = op, op + " " + " ".join(f"{k}={v}" for k, v in f.items())
                f = {k: (float(v) if k in ("eps", "scale") else int(v)) for k, v in f.items()}
                if key in known:
                    cnt[kind][0] += 1
                    continue
            elif name in SCHEMA:
                kind, f = describe(name, args)
                key = kind + " " + " ".join(f"{k}={v}" for k, v in f.items())
            else:
                unknown.append(name)
                continue
            cnt[kind][0] += 1
            cnt[kind][1].add(key)
            if key not in desc:
                desc[key] = dict(kind=kind, f=f, first=wl, n=0)
            desc[key]["n"] += 1
    return desc, calls, unknown


def glue_census():
    """collect() over the workloads of the module docstring, plus the SYNTHETIC descriptors (cached)."""
    global _GLUE
    if _GLUE is not None:
        return _GLUE
    import os
    for k in ("LADI_UP2X", "LADI_LN_FOLD", "LADI_CONV_2CTA"):
        assert k not in os.environ, f"census runs with library defaults; unset {k}"
    work = [(wl, functools.partial(_pipeline_calls, B, H, W, g)) for wl, B, H, W, g in PIPE_WORKLOADS] + [(FRONTEND, _frontend_calls)]
    desc, calls, unknown = collect(work)
    for kind, f in SYNTHETIC:
        desc[kind + " " + " ".join(f"{k}={v}" for k, v in f.items())] = dict(kind=kind, f=f, first=GRID_DOWNSCALE, n=1)
    _GLUE = (desc, calls, unknown)
    return _GLUE


def assert_all_known(unknown):
    assert not unknown, "entry points recorded without a SCHEMA row (add one and a replay): " + ", ".join(sorted(set(unknown)))


# ================================================================================================================ references and bounds
@functools.lru_cache(maxsize=None)
def aa_weights(n_in, n_out):
    """torch's antialiased bilinear filter (aten upsample_bilinear2d_aa, align_corners=False), restated in float64 -> (W [n_out, n_in],
    E [n_out, n_in]): W the normalised triangle weights, E a bound on the absolute error of the kernel's fp32 weights over the window
    widened by one tap on each side (a position error can move a tap across the window's truncated edge, where its weight is ~0)."""
    scale = n_in / n_out
    support = max(scale, 1.0)
    inv = 1.0 / scale if scale >= 1.0 else 1.0
    Wm, E = torch.zeros((n_out, n_in), dtype=torch.float64), torch.zeros((n_out, n_in), dtype=torch.float64)
    for o in range(n_out):
        center = scale * (o + 0.5)
        lo, hi = max(int(center - support + 0.5), 0), min(int(center + support + 0.5), n_in)  # int() truncates toward zero, as aten
        j = torch.arange(lo, hi, dtype=torch.float64)
        wt = (1.0 - ((j - center + 0.5) * inv).abs()).clamp_min(0.0)
        tot = float(wt.sum())
        Wm[o, lo:hi] = wt / tot
        d = AA_POS * (center + support + 2.0) * inv + 2.0 ** -22
        E[o, max(lo - 1, 0):min(hi + 1, n_in)] = (hi - lo + 2) * d / tot
    return Wm, E


def resample_expect(x, oh, ow, u_out):
    """x [..., h, w] float64 -> (r, bound) of the separable antialiased resize to (oh, ow), per the module docstring."""
    Wy, Ey = (t.to(x.device) for t in aa_weights(x.shape[-2], oh))
    Wx, Ex = (t.to(x.device) for t in aa_weights(x.shape[-1], ow))
    taps = int((Wy != 0).sum(1).max()) + int((Wx != 0).sum(1).max()) + 2
    r = Wy @ x @ Wx.t()
    ax = x.abs()
    err = (taps * EPS24) * (Wy @ ax @ Wx.t()) + Ey @ ax @ Wx.t() + Wy @ ax @ Ex.t() + Ey @ ax @ Ex.t()
    return r, u_out * r.abs() + err


def corr_expect(fa, fb):
    """fa, fb NHWC [n, h, w, c] float64 -> (r, bound) NHWC [n, h, w, h*w]: FeatureCorrelation of ConvNet_TPS.py as written there
    (feature_A transposed to (w, h) order, bmm, view, two transposes), seen channels-last."""
    def corr(a, b):
        n, h, w, c = a.shape
        A, B = a.permute(0, 3, 1, 2), b.permute(0, 3, 1, 2)
        feature_A = A.transpose(2, 3).contiguous().view(n, c, h * w)
        feature_B = B.contiguous().view(n, c, h * w).transpose(1, 2)
        mul = torch.bmm(feature_B, feature_A)
        return mul.view(n, h, w, h * w).transpose(2, 3).transpose(1, 2).permute(0, 2, 3, 1)
    r, m = corr(fa, fb), corr(fa.abs(), fb.abs())
    return r, U_BF16 * r.abs() + C_ACC * math.sqrt(fa.shape[3]) * EPS24 * m


def small_attn_expect(q, k, v, heads, scale, causal):
    """q [nq, C], k / v [nkv, C] float64 -> (o, bound) [nq, C]; the causal mask (key j visible to query i iff j <= i) is applied here."""
    nq, nkv, Cw = q.shape[0], k.shape[0], q.shape[1]
    hd = Cw // heads
    qh, kh, vh = (t.view(-1, heads, hd).transpose(0, 1) for t in (q, k, v))
    s = (qh @ kh.transpose(1, 2)) * scale
    if causal:
        s = s.masked_fill(torch.ones((nq, nkv), dtype=torch.bool, device=q.device).triu(1), -float("inf"))
    p = torch.exp(s - s.amax(-1, keepdim=True))
    l = p.sum(-1, keepdim=True)
    o = ((p @ vh) / l).transpose(0, 1).reshape(nq, Cw)
    sv = ((p @ vh.abs()) / l).transpose(0, 1).reshape(nq, Cw)
    return o, attn_expect(o, sv, nkv, u_p=2.0 ** -22)


def ddim_expect(x, eu, et, row, g, cfg, noise=None):
    """One DDIM step (+CFG) in float64 on [B, 4, h, w] tensors; row = the fp32 coefficient row {1/sqrt(a), sqrt(1-a), sqrt(a_prev),
    sqrt(1-a_prev-sigma^2), sigma} -> (r, bound)."""
    inv_sa, s1a, sap, s1ap, sigma = (float(v) for v in row[:5])
    e = eu + g * (et - eu) if cfg else eu
    r = sap * (x - s1a * e) * inv_sa + s1ap * e
    E = eu.abs() + (g * (et - eu).abs() + e.abs() if cfg else 0.0)
    M = abs(sap * inv_sa) * (x.abs() + abs(s1a) * E) + abs(s1ap) * E
    if noise is not None:
        r = r + sigma * noise
        M = M + abs(sigma) * noise.abs()
    return r, DDIM_ULPS * EPS24 * M + EPS24 * r.abs()


def warp_expect(low_grid, cloth, u_out=U_BF16):
    """low_grid [n, gh, gw, 2], cloth [n, c, H, W] float64 -> (r, bound) [n, c, H, W]: antialiased resize of the grid to (H, W), then
    grid_sample(bilinear, padding_mode='border', align_corners=False)."""
    n, c, H, W = cloth.shape
    g, eg = resample_expect(low_grid.permute(0, 3, 1, 2), H, W, 2.0 ** -24)  # [n, 2, H, W]; fp32 grid, no further rounding
    gx, gy = g[:, 0], g[:, 1]
    ix = (((gx + 1.0) * W - 1.0) * 0.5).clamp(0.0, W - 1.0)
    iy = (((gy + 1.0) * H - 1.0) * 0.5).clamp(0.0, H - 1.0)
    dix = eg[:, 0] * W * 0.5 + 3 * EPS24 * ((gx.abs() + 1.0) * W * 0.5 + 1.0)
    diy = eg[:, 1] * H * 0.5 + 3 * EPS24 * ((gy.abs() + 1.0) * H * 0.5 + 1.0)
    x0, y0 = ix.floor(), iy.floor()
    wx1, wy1 = ix - x0, iy - y0
    x0, y0 = x0.long(), y0.long()
    x1, y1 = (x0 + 1).clamp_max(W - 1), (y0 + 1).clamp_max(H - 1)
    flat = cloth.reshape(n, c, H * W)
    at = lambda yy, xx: torch.gather(flat, 2, (yy * W + xx).view(n, 1, -1).expand(n, c, -1)).view(n, c, H, W)  # noqa: E731
    w00, w01, w10, w11 = ((1 - wy1) * (1 - wx1))[:, None], ((1 - wy1) * wx1)[:, None], (wy1 * (1 - wx1))[:, None], (wy1 * wx1)[:, None]
    v00, v01, v10, v11 = at(y0, x0), at(y0, x1), at(y1, x0), at(y1, x1)
    r = w00 * v00 + w01 * v01 + w10 * v10 + w11 * v11
    m = w00 * v00.abs() + w01 * v01.abs() + w10 * v10.abs() + w11 * v11.abs()
    # how far the value moves per texel of position error: the largest neighbouring difference within one texel of the sample
    dX = F.max_pool2d(F.pad((cloth[..., 1:] - cloth[..., :-1]).abs(), (0, 1)), 3, 1, 1).reshape(n, c, H * W)
    dY = F.max_pool2d(F.pad((cloth[..., 1:, :] - cloth[..., :-1, :]).abs(), (0, 0, 0, 1)), 3, 1, 1).reshape(n, c, H * W)
    lx = torch.maximum(*(torch.gather(dX, 2, (yy * W + x0).view(n, 1, -1).expand(n, c, -1)) for yy in (y0, y1))).view(n, c, H, W)
    ly = torch.maximum(*(torch.gather(dY, 2, (y0 * W + xx).view(n, 1, -1).expand(n, c, -1)) for xx in (x0, x1))).view(n, c, H, W)
    return r, u_out * r.abs() + 4 * EPS24 * m + dix[:, None] * lx + diy[:, None] * ly


def upsample_ac_expect(x):
    """x NHWC [n, h, w, c] float64 -> (r, bound) NHWC [n, 2h, 2w, c] of bilinear 2x upsampling with align_corners=True."""
    n, h, w, c = x.shape

    def axis(size):
        pos = torch.arange(2 * size, dtype=torch.float64, device=x.device) * ((size - 1) / (2 * size - 1))
        i0 = pos.floor().long()
        return i0, (i0 + 1).clamp_max(size - 1), pos - i0, 2.0 ** -22 * pos + 2.0 ** -23
    y0, y1, wy, dy = axis(h)
    x0, x1, wx, dx = axis(w)
    g = lambda yy, xx: x[:, yy][:, :, xx]  # noqa: E731
    wy_, wx_ = wy.view(1, -1, 1, 1), wx.view(1, 1, -1, 1)
    v00, v01, v10, v11 = g(y0, x0), g(y0, x1), g(y1, x0), g(y1, x1)
    r = (1 - wy_) * ((1 - wx_) * v00 + wx_ * v01) + wy_ * ((1 - wx_) * v10 + wx_ * v11)
    m = (1 - wy_) * ((1 - wx_) * v00.abs() + wx_ * v01.abs()) + wy_ * ((1 - wx_) * v10.abs() + wx_ * v11.abs())
    lx = torch.maximum((v01 - v00).abs(), (v11 - v10).abs())
    ly = torch.maximum((v10 - v00).abs(), (v11 - v01).abs())
    # the position error stays below one texel, and within [i0, i0 + 1] the interpolant's slope is the neighbour difference
    return r, U_BF16 * r.abs() + 6 * EPS24 * m + dy.view(1, -1, 1, 1) * ly + dx.view(1, 1, -1, 1) * lx


# ================================================================================================================ replay (GPU)
def _buf(R, n, dtype, tail=64, fill=NAN):
    """-> (flat buffer, first n elements): a `tail` past the end shows a write beyond the operand."""
    flat = torch.full((n + tail,), fill, dtype=dtype, device=R.dev)
    return flat, flat[:n]


def _same(a, b):
    return _bitwise_equal(a, b) if a.dtype in (torch.bfloat16, torch.float32) else torch.equal(a, b)


def _tail_nan(flat, n, what):
    t = flat[n:].float()
    return [] if bool(torch.isnan(t).all()) else [f"{what}: wrote past its end at element {n + int((~torch.isnan(t)).nonzero()[0])}"]


def _exact(y, r, what):
    """bit-exact comparison (NaN allowed where the reference has it, whatever its payload) -> ([error], (0 or inf, where))."""
    if _same(y.contiguous(), r.contiguous()):
        return [], (0.0, "bit-exact")
    it = {torch.bfloat16: torch.int16, torch.float32: torch.int32}.get(y.dtype)
    bad = (y.contiguous().view(it) != r.contiguous().view(it)) if it is not None else (y != r)
    if it is not None:
        bad &= ~(torch.isnan(y) & torch.isnan(r))
        if not bool(bad.any()):
            return [], (0.0, "bit-exact, NaN where the reference has NaN")
    loc = [int(v) for v in bad.nonzero()[0]]
    msg = f"{what}: {int(bad.sum())} elements differ; first at index {loc}: got {y[tuple(loc)].item()}, ref {r[tuple(loc)].item()}"
    return [msg], (float("inf"), msg)


def _worst(q, names, extra=""):
    w = float(q.max())
    idx = [int(v) for v in torch.unravel_index(q.argmax(), q.shape)]
    where = ", ".join(f"{n} {i}" for n, i in zip(names, idx)) + extra
    return ([f"err/bound {w:.3g} at {where}"] if w > 1 else []), (w, where)


def _twice(call, fresh):
    """fresh() -> dict of buffers; call(bufs) launches; both runs are kept for the determinism check."""
    runs = []
    for _ in range(2):
        b = fresh()
        call(b)
        runs.append(b)
    torch.cuda.synchronize()
    return runs


def _determinism(runs, keys):
    return [] if all(_same(runs[0][k], runs[1][k]) for k in keys) else ["two runs differ bitwise"]


def _window(o2d, lo, hi, what):
    """The call wrote every element of columns [lo, hi) (finite) and nothing else (still NaN)."""
    errs = []
    o = o2d.float()
    if not bool(torch.isfinite(o[:, lo:hi]).all()):
        errs.append(f"{what}: non-finite in its columns [{lo}, {hi}) at (row, column - {lo}) {(~torch.isfinite(o[:, lo:hi])).nonzero()[0].tolist()}")
    outside = torch.cat([o[:, :lo], o[:, hi:]], dim=1)
    if outside.numel() and not bool(torch.isnan(outside).all()):
        errs.append(f"{what}: wrote outside its columns [{lo}, {hi}) (row, column outside) {(~torch.isnan(outside)).nonzero()[0].tolist()}")
    return errs


def _image(R, *shape):
    return R.rand(*shape) * 2 - 1


def _binary_mask(R, *shape):
    """{0, 1} with a sprinkle of exactly 0.5 (the value the `< 0.5` comparisons must send to the masked side)."""
    m = (R.rand(*shape) < 0.4).float()
    return torch.where(R.rand(*shape) < 0.02, torch.full_like(m, 0.5), m)


def replay_nchw_to_nhwc(R, f, gate_nan=False):
    from ladi_vton_b200 import lib
    n, c, h, w, fct, op, c_off = f["n"], f["c"], f["h"], f["w"], f["f"], f["op"], f["c_off"]
    H, W = h * fct, w * fct
    x = _image(R, n, c, H, W) if f["scale"] == 1.0 else R.randn(n, c, H, W)  # scale != 1: the latents the VAE decoder loads
    gate = _binary_mask(R, n, 1, H, W) if f["gate"] else None
    if gate is not None and gate_nan:  # NaN < 0.5 is false: a NaN gate masks the pixel, as `image * (mask < 0.5)` does
        gate = torch.where(R.rand(n, 1, H, W) < 0.05, NAN, gate)
    rows = n * h * w

    def fresh():
        flat, o = _buf(R, rows * op, torch.bfloat16)
        return dict(flat=flat, out=o)
    P = lambda t: C.c_void_p(t.data_ptr() if t is not None else 0)  # noqa: E731
    runs = _twice(lambda b: lib.call("ladi_nchw_f32_to_nhwc_bf16", P(x), n, c, h, w, fct, f["scale"], P(gate), P(b["out"]), op, c_off, R.stream),
                  fresh)
    out = runs[0]["out"].view(rows, op)
    errs = _window(out, c_off, c_off + c, "output") + _tail_nan(runs[0]["flat"], rows * op, "output") + _determinism(runs, ["flat"])
    # the kernel rounds the fp32 product x * scale to bf16: bit-equal to that, and (exact product when scale = 1; for the decoder's
    # 1 / scaling_factor the fp32 product carries 2^-24 before the bf16 rounding) within ROUND1 (1 + 2^-15) of float64
    xs = x[:, :, ::fct, ::fct]
    v, r = xs * f["scale"], xs.double() * float(np.float32(f["scale"]))
    if gate is not None:  # a masked pixel is +0 (`image * (mask < 0.5)` gives -0 for a negative pixel: the same value)
        keep = gate[:, :, ::fct, ::fct] < 0.5
        v, r = torch.where(keep, v, 0.0), torch.where(keep, r, 0.0)
    y = out[:, c_off:c_off + c].contiguous()
    e, res = _exact(y, v.permute(0, 2, 3, 1).reshape(rows, c).bfloat16(), "values against bf16(fp32 product)")
    r = r.permute(0, 2, 3, 1).reshape(rows, c)
    e2, res2 = _worst(ratio(y, r, ROUND1 * (1 + 2.0 ** -15) * r.abs()), ("pixel", "channel"))
    return errs + e + e2, (res if e else res2)


def replay_nhwc_to_nchw_clamp(R, f, values=None):
    from ladi_vton_b200 import lib
    n, c, h, w, xp, lo, hi = f["n"], f["c"], f["h"], f["w"], f["xp"], f["lo"], f["hi"]
    x = R.poisoned(n * h * w, xp, R.randn(n * h * w, c) * 0.8 if values is None else values, dtype=torch.float32)

    def fresh():
        flat, o = _buf(R, n * c * h * w, torch.float32)
        return dict(flat=flat, out=o)
    runs = _twice(lambda b: lib.call("ladi_nhwc_f32_to_nchw_clamp", C.c_void_p(x.data_ptr()), n, c, h, w, xp, lo, hi, C.c_void_p(b["out"].data_ptr()),
                                     R.stream), fresh)
    errs = _tail_nan(runs[0]["flat"], n * c * h * w, "output") + _determinism(runs, ["flat"])
    ref = x[:, :c].reshape(n, h, w, c).permute(0, 3, 1, 2).clamp(lo, hi).contiguous().view(-1)  # torch.clamp keeps NaN
    e, res = _exact(runs[0]["out"], ref, "values")
    return errs + e, res


def replay_inv_mask_rows(R, f):
    from ladi_vton_b200 import lib
    n, H, W, fct = f["n"], f["H"], f["W"], f["f"]
    mask = _binary_mask(R, n, 1, H, W)
    cnt = n * (H // fct) * (W // fct)

    def fresh():
        flat, o = _buf(R, cnt, torch.float32)
        return dict(flat=flat, out=o)
    runs = _twice(lambda b: lib.call("ladi_inv_mask_rows", C.c_void_p(mask.data_ptr()), n, H, W, fct, C.c_void_p(b["out"].data_ptr()), R.stream), fresh)
    errs = _tail_nan(runs[0]["flat"], cnt, "output") + _determinism(runs, ["flat"])
    e, res = _exact(runs[0]["out"], (1.0 - mask[:, 0, ::fct, ::fct]).reshape(-1), "values")
    return errs + e, res


def replay_bilinear_down8(R, f):
    from ladi_vton_b200 import lib
    n, c, H, W = f["n"], f["c"], f["H"], f["W"]
    x = R.rand(n, c, H, W) ** 4  # pose-map-like: mostly small, peaks near 1
    cnt = n * c * (H // 8) * (W // 8)

    def fresh():
        flat, o = _buf(R, cnt, torch.float32)
        return dict(flat=flat, out=o)
    runs = _twice(lambda b: lib.call("ladi_bilinear_down8", C.c_void_p(x.data_ptr()), n, c, H, W, C.c_void_p(b["out"].data_ptr()), R.stream), fresh)
    errs = _tail_nan(runs[0]["flat"], cnt, "output") + _determinism(runs, ["flat"])
    y = runs[0]["out"].view(n, c, H // 8, W // 8)
    e, _ = _exact(y, F.interpolate(x, size=(H // 8, W // 8), mode="bilinear", align_corners=False), "against fp32 F.interpolate")
    q = x.double()[:, :, 3::8, 3::8], x.double()[:, :, 3::8, 4::8], x.double()[:, :, 4::8, 3::8], x.double()[:, :, 4::8, 4::8]
    r = 0.25 * sum(q)
    errs2, res = _worst(ratio(y, r, 2.0 ** -23 * 0.25 * sum(t.abs() for t in q)), ("image", "channel", "y", "x"))
    return errs + e + errs2, res


def replay_check_binarise(R, f):
    from ladi_vton_b200 import lib
    ni, nm = f["n_image"], f["n_mask"]
    image_flat, image = _buf(R, ni, torch.float32, fill=5.0)  # a read past the end would raise the image flag
    image.copy_(_image(R, ni))
    image[::7919] = NAN  # NaN compares false: no flag, as the reference's min / max test
    m0 = R.rand(nm)
    m0[::97] = 0.5
    m0[1::97] = 0.0
    m0[2::97] = 1.0
    m0[3::1009] = NAN
    errs, cases = [], [("in range", None, None, [0, 0]), ("image 1.5 at its last element", ni - 1, None, [1, 0]),
                       ("mask -0.25 at its last element", None, nm - 1, [0, 1])]
    for what, bad_i, bad_m, want in cases:
        runs = []
        for _ in range(2 if bad_i is None and bad_m is None else 1):
            im = image_flat.clone()
            if bad_i is not None:
                im[bad_i] = 1.5
            mflat, m = _buf(R, nm, torch.float32, fill=0.3)  # must stay 0.3: the in-place binarisation stops at n_mask
            m.copy_(m0)
            if bad_m is not None:
                m[bad_m] = -0.25
            flags = torch.zeros(2, dtype=torch.int32, device=R.dev)
            lib.call("ladi_check_binarise", C.c_void_p(im.data_ptr()), ni, C.c_void_p(m.data_ptr()), nm, C.c_void_p(flags.data_ptr()), R.stream)
            runs.append(dict(m=mflat, flags=flags, src=m0 if bad_m is None else torch.where(torch.arange(nm, device=R.dev) == bad_m, -0.25, m0)))
        torch.cuda.synchronize()
        r = runs[0]
        if r["flags"].tolist() != want:
            errs.append(f"{what}: flags {r['flags'].tolist()}, expected {want}")
        if not bool((r["m"][nm:] == 0.3).all()):
            errs.append(f"{what}: mask written past n_mask")
        src = r["src"]
        ref = torch.where(src < 0.5, 0.0, torch.where(src >= 0.5, 1.0, src))
        e, _ = _exact(r["m"][:nm], ref, f"{what}: mask")
        errs += e
        if len(runs) == 2:
            errs += _determinism(runs, ["m", "flags"])
    return errs, (0.0 if not errs else float("inf"), "bit-exact mask and flags" if not errs else errs[0])


def replay_posterior_sample(R, f, logvar=None):
    """logvar: [rows, cz] values in place of the random ones (past both clamps); NaN must come out NaN, as torch.clamp keeps it."""
    from ladi_vton_b200 import lib
    mp, n, cz, h, w, scale = f["mp"], f["n"], f["cz"], f["h"], f["w"], f["scale"]
    rows = n * h * w
    lv0 = R.rand(rows, cz) * 60 - 36 if logvar is None else logvar
    mom = R.poisoned(rows, mp, torch.cat([R.randn(rows, cz) * 3, lv0], dim=1), dtype=torch.float32)  # logvar past both clamps
    noise = R.randn(n, cz, h, w)
    cnt = n * cz * h * w

    def fresh():
        flat, o = _buf(R, cnt, torch.float32)
        return dict(flat=flat, out=o)
    runs = _twice(lambda b: lib.call("ladi_posterior_sample", C.c_void_p(mom.data_ptr()), mp, C.c_void_p(noise.data_ptr()), n, cz, h, w, scale,
                                     C.c_void_p(b["out"].data_ptr()), R.stream), fresh)
    errs = _tail_nan(runs[0]["flat"], cnt, "output") + _determinism(runs, ["flat"])
    m4 = mom.view(n, h, w, mp).permute(0, 3, 1, 2).double()
    mean, lv = m4[:, :cz], m4[:, cz:2 * cz].clamp(-30.0, 20.0)
    sn = torch.exp(0.5 * lv) * noise.double()
    r = (mean + sn) * scale
    bound = abs(scale) * (2.0 ** -23 * mean.abs() + (2.0 ** -22 + 2.0 ** -23) * sn.abs()) + 2.0 ** -23 * r.abs()
    y = runs[0]["out"].view(n, cz, h, w)
    nan = torch.isnan(r)
    if not torch.equal(torch.isnan(y), nan):
        errs.append(f"NaN at {int(torch.isnan(y).sum())} outputs where the reference has {int(nan.sum())} (a NaN logvar must stay NaN)")
    e, res = _worst(ratio(y.masked_fill(nan, 0.0), r.masked_fill(nan, 0.0), bound.masked_fill(nan, 1.0)), ("image", "channel", "y", "x"))
    return errs + e, res


def _ddim_coefs(R, steps=3):
    ab = torch.tensor([0.01, 0.02, 0.03, 0.05, 0.3, 0.7, 0.95], dtype=torch.float64)[-(steps + 1):]  # alphas-cumprod, noisy to clean
    rows = torch.zeros((steps, 8), dtype=torch.float64)
    rows[:, 0], rows[:, 1] = ab[:steps].rsqrt(), (1 - ab[:steps]).sqrt()
    rows[:, 2], rows[:, 3], rows[:, 4] = ab[1:steps + 1].sqrt(), (1 - ab[1:steps + 1] - 0.01).sqrt(), 0.1
    return rows.float().to(R.dev)


def replay_ddim_cfg_step(R, f, start=0):
    """Three consecutive calls from device step index `start`: with advance, rows start, start + 1, start + 2 of the coefficient table
    and step_ptr = [s + 1, 0] after each; without, row `start` every time and step_ptr untouched."""
    from ladi_vton_b200 import lib
    ep, inp, B, h, w, cfg, g, adv = f["ep"], f["inp"], f["B"], f["h"], f["w"], f["cfg"], f["guidance"], f["advance"]
    assert f["coef"] and f["step"], "the pipeline's DDIM update reads the step counter"
    hw, Bp = h * w, (2 * B if cfg else B)
    eu = R.randn(B * hw, 4)
    eps = torch.cat([eu, eu + 0.3 * R.randn(B * hw, 4)]) if cfg else eu  # conditional = unconditional + a smaller difference
    eps = R.poisoned(Bp * hw, ep, eps, dtype=torch.float32)
    x_init = R.randn(B, 4, h, w)
    uin_init = R.randn(Bp * hw, inp).bfloat16()
    uin_init[:, :4] = NAN
    coef = _ddim_coefs(R, start + 3)
    noise = R.randn(B, 4, h, w) if f["noise"] else None
    P = lambda t: C.c_void_p(t.data_ptr() if t is not None else 0)  # noqa: E731
    g32 = float(np.float32(g))

    def run(check):
        lat, uin = x_init.clone(), uin_init.clone()
        step = torch.tensor([start, 0], dtype=torch.int32, device=R.dev)
        errs, worst = [], (0.0, "")
        for k in range(3):
            s = start + k if adv else start
            x_before = lat.clone()
            lib.call("ladi_ddim_cfg_step", P(eps), ep, P(lat), P(uin), inp, B, h, w, cfg, g, P(coef), P(step), adv, P(noise), R.stream)
            torch.cuda.synchronize()
            if not check:
                continue
            want_step = [s + 1, 0] if adv else [start, 0]
            if step.tolist() != want_step:
                errs.append(f"step {s}: step_ptr {step.tolist()}, expected {want_step} (grid-wide ticket over {-(-B * 4 * hw // 256)} CTAs)")
            e3 = eps[:, :4].double().view(Bp, h, w, 4).permute(0, 3, 1, 2)
            r, bound = ddim_expect(x_before.double(), e3[:B], e3[B:] if cfg else None, coef[s].double(), g32, cfg,
                                   noise.double() if noise is not None else None)
            q = ratio(lat, r, bound)
            e, res = _worst(q, ("image", "channel", "y", "x"), f" (step {s}; CTA {int(q.argmax()) // 256})")
            errs += e
            if res[0] > worst[0]:
                worst = res
            want = lat.permute(0, 2, 3, 1).reshape(B * hw, 4).bfloat16()
            u = uin.view(Bp * hw, inp)
            for half in range(Bp // B):
                ee, _ = _exact(u[half * B * hw:(half + 1) * B * hw, :4].contiguous(), want, f"step {s}: unet_in rows of CFG half {half}")
                errs += ee
            if not _bitwise_equal(u[:, 4:].contiguous(), uin_init[:, 4:].contiguous()):
                errs.append(f"step {s}: unet_in channels >= 4 changed")
        return errs, worst, lat, uin, step
    errs, worst, *first = run(True)
    second = run(False)[2:]
    if not all(_same(a, b) for a, b in zip(first, second)):
        errs.append("two runs differ bitwise")
    return errs, worst


def _image_out_input(R, n, h, w, xp):
    v = R.rand(n * h * w, 3) * 2.4 - 1.2  # past both clamps
    k = torch.randint(0, 255, (n * h * w, 3), device=R.dev, generator=R.g).float()
    tie = (k + 0.5) / 127.5 - 1.0  # values whose (x/2 + 0.5) * 255 lands near a rounding tie
    v = torch.where(R.rand(n * h * w, 3) < 0.2, tie, v)
    return R.poisoned(n * h * w, xp, v, dtype=torch.float32)


def replay_image_out(R, f, u8=False, values=None):
    """values: [n*h*w, 3] fp32 in place of the random ones.  NaN: image_out keeps it (torch.clamp); image_out_u8 writes 0."""
    from ladi_vton_b200 import lib
    n, h, w, xp, f32 = f["n"], f["h"], f["w"], f["xp"], f["f32"]
    x = _image_out_input(R, n, h, w, xp) if values is None else R.poisoned(n * h * w, xp, values, dtype=torch.float32)
    if not f32:
        x = x.bfloat16()
    cnt = n * h * w * 3
    dt = torch.uint8 if u8 else torch.float32

    def fresh():
        flat, o = _buf(R, cnt, dt, fill=171 if u8 else NAN)
        return dict(flat=flat, out=o)
    name = "ladi_image_out_u8" if u8 else "ladi_image_out"
    runs = _twice(lambda b: lib.call(name, C.c_void_p(x.data_ptr()), f32, n, h, w, xp, C.c_void_p(b["out"].data_ptr()), R.stream), fresh)
    tail = runs[0]["flat"][cnt:]
    errs = ([] if bool((tail == 171).all() if u8 else torch.isnan(tail).all()) else ["output: wrote past its end"]) + _determinism(runs, ["flat"])
    c = (x[:, :3].float() * 0.5 + 0.5).clamp(0.0, 1.0)
    if u8:
        v = np.rint(c.cpu().numpy() * np.float32(255.0))  # numpy: round half to even
        ref = torch.from_numpy(np.where(np.isnan(v), 0.0, v).astype(np.uint8)).to(R.dev)
    else:
        ref = c
    e, res = _exact(runs[0]["out"].view(n * h * w, 3), ref.contiguous(), "values")
    return errs + e, res


def replay_resize_aa(R, f):
    from ladi_vton_b200 import lib
    n, c, h, w, oh, ow, op, c_off = (f[k] for k in ("n", "c", "h", "w", "oh", "ow", "op", "c_off"))
    x = _image(R, n, c, h, w)
    rows = n * oh * ow

    def fresh():
        flat, o = _buf(R, rows * op, torch.bfloat16)
        return dict(flat=flat, out=o)
    runs = _twice(lambda b: lib.call("ladi_resize_aa", C.c_void_p(x.data_ptr()), n, c, h, w, oh, ow, C.c_void_p(b["out"].data_ptr()), op, c_off, R.stream),
                  fresh)
    out = runs[0]["out"].view(rows, op)
    errs = _window(out, c_off, c_off + c, "output") + _tail_nan(runs[0]["flat"], rows * op, "output") + _determinism(runs, ["flat"])
    if (oh, ow) == (h, w):  # one tap of weight exactly 1 per output: bf16(x) bit for bit
        errs += _exact(out[:, c_off:c_off + c].contiguous(), x.permute(0, 2, 3, 1).reshape(rows, c).bfloat16(), "identity resize")[0]
    worst = (0.0, "")
    for b in _pick(n, n * c * h * w, 1 << 24):
        r, bound = resample_expect(x[b].double(), oh, ow, U_BF16)
        e, res = _worst(ratio(out.view(n, oh, ow, op)[b, ..., c_off:c_off + c].permute(2, 0, 1), r, bound), ("channel", "y", "x"), f" of image {b}")
        errs += e
        worst = max(worst, res)
    return errs, worst


def replay_clip_preprocess(R, f):
    from ladi_vton_b200 import lib
    from ladi_vton_b200.inference import CLIP_MEAN, CLIP_STD
    n, c, h, w, oh, ow, qz = (f[k] for k in ("n", "c", "h", "w", "oh", "ow", "quantise"))
    x = _image(R, n, c, h, w)
    mean, std = torch.tensor(CLIP_MEAN, device=R.dev), torch.tensor(CLIP_STD, device=R.dev)
    cnt = n * c * oh * ow

    def fresh():
        flat, o = _buf(R, cnt, torch.float32)
        return dict(flat=flat, out=o)
    runs = _twice(lambda b: lib.call("ladi_clip_preprocess", C.c_void_p(x.data_ptr()), n, c, h, w, oh, ow, C.c_void_p(mean.data_ptr()),
                                     C.c_void_p(std.data_ptr()), qz, C.c_void_p(b["out"].data_ptr()), R.stream), fresh)
    errs = _tail_nan(runs[0]["flat"], cnt, "output") + _determinism(runs, ["flat"])
    y = runs[0]["out"].view(n, c, oh, ow).double()
    md, sd = mean.double().view(c, 1, 1), std.double().view(c, 1, 1)
    worst = (0.0, "")
    for b in _pick(n, n * c * h * w, 1 << 24):
        acc, eacc = resample_expect(x[b].double(), oh, ow, 0.0)
        v = (0.5 * acc + 0.5).clamp(0.0, 1.0)
        ev = 0.5 * eacc + 2.0 ** -24
        if qz:  # every level floor(255 v') with |v' - v| within the bound is a correct result
            e255 = 255.0 * ev + 255.0 * EPS24
            lo, hi = torch.floor(255.0 * v - e255), torch.floor(255.0 * v + e255)
            d = torch.full_like(v, float("inf"))
            bnd = torch.ones_like(v)
            for k in range(int((hi - lo).max()) + 1):
                lvl = ((lo + k).clamp_max(hi) / 255.0)
                rk = (lvl - md) / sd
                bk = 2.0 ** -21 * (lvl + md.abs()) / sd + 2.0 ** -24 * rk.abs()
                better = (y[b] - rk).abs() / bk < d / bnd
                d, bnd = torch.where(better, (y[b] - rk).abs(), d), torch.where(better, bk, bnd)
            q = torch.nan_to_num(d / bnd, nan=float("inf"))
        else:
            r = (v - md) / sd
            q = ratio(y[b], r, (ev + 2.0 ** -23 * (v + md.abs())) / sd + U_F32 * r.abs())
        e, res = _worst(q, ("channel", "y", "x"), f" of image {b}")
        errs += e
        worst = max(worst, res)
    return errs, worst


def _smooth_grid(R, n, gh, gw):
    """A TPS-like sampling grid: the identity lattice, a smooth displacement and a margin that reaches past +-1 (border clipping)."""
    ys, xs = torch.meshgrid(torch.linspace(-1.06, 1.06, gh, device=R.dev), torch.linspace(-1.06, 1.06, gw, device=R.dev), indexing="ij")
    a = R.randn(n, 2, 1, 1) * 0.05
    dx = a[:, 0] * torch.sin(3 * ys + 1)[None] + 0.01 * R.randn(n, gh, gw)
    dy = a[:, 1] * torch.cos(2 * xs)[None] + 0.01 * R.randn(n, gh, gw)
    return torch.stack([xs[None] + dx, ys[None] + dy], dim=3).contiguous()


def replay_warp_grid_sample(R, f, grid=None):
    """grid: fp32 [n, gh, gw, 2] in place of the smooth TPS-like one."""
    from ladi_vton_b200 import lib
    gh, gw, n, c, H, W, op, c_off = (f[k] for k in ("gh", "gw", "n", "c", "H", "W", "op", "c_off"))
    grid = _smooth_grid(R, n, gh, gw) if grid is None else grid.contiguous()
    cloth = _image(R, n, c, H, W)
    rows = n * H * W

    def fresh():
        flat, o = _buf(R, rows * op, torch.bfloat16)
        return dict(flat=flat, out=o)
    runs = _twice(lambda b: lib.call("ladi_warp_grid_sample", C.c_void_p(grid.data_ptr()), gh, gw, C.c_void_p(cloth.data_ptr()), n, c, H, W,
                                     C.c_void_p(b["out"].data_ptr()), op, c_off, R.stream), fresh)
    out = runs[0]["out"].view(rows, op)
    errs = _window(out, c_off, c_off + c, "output") + _tail_nan(runs[0]["flat"], rows * op, "output") + _determinism(runs, ["flat"])
    worst = (0.0, "")
    for b in _pick(n, n * c * H * W, 1 << 22):
        r, bound = warp_expect(grid[b:b + 1].double(), cloth[b:b + 1].double())
        e, res = _worst(ratio(out.view(n, H, W, op)[b:b + 1, ..., c_off:c_off + c].permute(0, 3, 1, 2), r, bound), ("", "channel", "y", "x"),
                        f" of image {b}")
        errs += e
        worst = max(worst, res)
    return errs, worst


def _features(R, rows, c):
    """post-ReLU activations: half zeros, the rest |N(0, 1)| with per-channel scales."""
    return (R.randn(rows, c).clamp_min(0) * torch.exp(R.randn(c, std=0.5))).bfloat16()


def replay_upsample2x_ac(R, f):
    from ladi_vton_b200 import lib
    n, h, w, c = f["n"], f["h"], f["w"], f["c"]
    x = _features(R, n * h * w, c)
    cnt = n * 4 * h * w * c

    def fresh():
        flat, o = _buf(R, cnt, torch.bfloat16)
        return dict(flat=flat, out=o)
    runs = _twice(lambda b: lib.call("ladi_upsample2x_bilinear_ac", C.c_void_p(x.data_ptr()), n, h, w, c, C.c_void_p(b["out"].data_ptr()), R.stream), fresh)
    errs = _tail_nan(runs[0]["flat"], cnt, "output") + _determinism(runs, ["flat"])
    worst = (0.0, "")
    for b in _pick(n, cnt, 1 << 26):
        r, bound = upsample_ac_expect(x.view(n, h, w, c)[b:b + 1].double())
        e, res = _worst(ratio(runs[0]["out"].view(n, 2 * h, 2 * w, c)[b:b + 1], r, bound), ("", "y", "x", "channel"), f" of image {b}")
        errs += e
        worst = max(worst, res)
    return errs, worst


def replay_space_to_depth2(R, f):
    from ladi_vton_b200 import lib
    n, h, w, c, xp, op = f["n"], f["h"], f["w"], f["c"], f["xp"], f["op"]
    x = R.poisoned(n * h * w, xp, _features(R, n * h * w, c))
    rows = n * (h // 2) * (w // 2)

    def fresh():
        flat, o = _buf(R, rows * op, torch.bfloat16)
        return dict(flat=flat, out=o)
    runs = _twice(lambda b: lib.call("ladi_space_to_depth2", C.c_void_p(x.data_ptr()), n, h, w, c, xp, C.c_void_p(b["out"].data_ptr()), op, R.stream), fresh)
    out = runs[0]["out"].view(rows, op)
    errs = _window(out, 0, 4 * c, "output") + _tail_nan(runs[0]["flat"], rows * op, "output") + _determinism(runs, ["flat"])
    ref = x[:, :c].reshape(n, h // 2, 2, w // 2, 2, c).permute(0, 1, 3, 2, 4, 5).reshape(rows, 4 * c)  # channel (sy * 2 + sx) * c + ch
    e, res = _exact(out[:, :4 * c].contiguous(), ref.contiguous(), "values")
    return errs + e, res


def replay_maxpool2(R, f, values=None):
    """values: bf16 [n*h*w, c] in place of the post-ReLU features; a window holding a NaN gives NaN, as nn.MaxPool2d does."""
    from ladi_vton_b200 import lib
    n, h, w, c = f["n"], f["h"], f["w"], f["c"]
    x = _features(R, n * h * w, c) if values is None else values.bfloat16().contiguous()
    cnt = n * (h // 2) * (w // 2) * c

    def fresh():
        flat, o = _buf(R, cnt, torch.bfloat16)
        return dict(flat=flat, out=o)
    runs = _twice(lambda b: lib.call("ladi_maxpool2_nhwc", C.c_void_p(x.data_ptr()), n, h, w, c, C.c_void_p(b["out"].data_ptr()), R.stream), fresh)
    errs = _tail_nan(runs[0]["flat"], cnt, "output") + _determinism(runs, ["flat"])
    ref = F.max_pool2d(x.view(n, h, w, c).permute(0, 3, 1, 2).float(), 2).permute(0, 2, 3, 1).bfloat16().reshape(-1)
    e, res = _exact(runs[0]["out"], ref.contiguous(), "values")
    return errs + e, res


def replay_patchify(R, f):
    from ladi_vton_b200 import lib
    n, ch, h, w, ps, kpad = f["n"], f["ch"], f["h"], f["w"], f["patch"], f["kpad"]
    px = R.randn(n, ch, h, w) * 1.2
    rows = n * (h // ps) * (w // ps)

    def fresh():
        flat, o = _buf(R, rows * kpad, torch.bfloat16)
        return dict(flat=flat, out=o)
    runs = _twice(lambda b: lib.call("ladi_patchify", C.c_void_p(px.data_ptr()), C.c_void_p(b["out"].data_ptr()), n, ch, h, w, ps, kpad, R.stream), fresh)
    errs = _tail_nan(runs[0]["flat"], rows * kpad, "output") + _determinism(runs, ["flat"])
    ref = torch.zeros((rows, kpad), device=R.dev)
    ref[:, :ch * ps * ps] = F.unfold(px, ps, stride=ps).transpose(1, 2).reshape(rows, -1)  # column (c * ps + ky) * ps + kx
    e, res = _exact(runs[0]["out"].view(rows, kpad), ref.bfloat16(), "values (zeros in the padding columns)")
    return errs + e, res


def _sum_round1(y, a, b, names):
    r = a.double() + b.double()
    return _worst(ratio(y, r, ROUND1 * r.abs()), names)


def replay_vit_assemble(R, f):
    from ladi_vton_b200 import lib
    pp, n, np_, c = f["pp"], f["n"], f["np"], f["c"]
    patch = R.poisoned(n * np_, pp, R.randn(n * np_, c))
    cls, pos = R.randn(c).bfloat16(), (R.randn(np_ + 1, c) * 0.3).bfloat16()
    cnt = n * (np_ + 1) * c

    def fresh():
        flat, o = _buf(R, cnt, torch.bfloat16)
        return dict(flat=flat, out=o)
    runs = _twice(lambda b: lib.call("ladi_vit_assemble", C.c_void_p(patch.data_ptr()), pp, C.c_void_p(cls.data_ptr()), C.c_void_p(pos.data_ptr()),
                                     C.c_void_p(b["out"].data_ptr()), n, np_, c, R.stream), fresh)
    errs = _tail_nan(runs[0]["flat"], cnt, "output") + _determinism(runs, ["flat"])
    a = torch.cat([cls.view(1, 1, c).expand(n, 1, c), patch[:, :c].view(n, np_, c)], dim=1)
    e, res = _sum_round1(runs[0]["out"].view(n, np_ + 1, c), a, pos.view(1, np_ + 1, c), ("image", "token", "channel"))
    return errs + e, res


def replay_clip_embed(R, f):
    from ladi_vton_b200 import lib
    rows, seq, c, op = f["rows"], f["seq"], f["c"], f["op"]
    B, V, nv = rows // seq, 49408, 16
    tok, pos = (R.randn(V, c) * 0.02).bfloat16(), (R.randn(seq, c) * 0.01).bfloat16()
    src = torch.randint(0, V, (B, seq), device=R.dev, generator=R.g, dtype=torch.int32)
    wemb = None
    if f["wemb"]:
        wemb = R.randn(B * nv, c).bfloat16()
        for b in range(B):  # the pseudo-words of prompt b start at a different token of each prompt, up to the last position
            s0 = seq - nv - (b * 7) % (seq - nv)
            src[b, s0:s0 + nv] = -(b * nv + torch.arange(nv, device=R.dev, dtype=torch.int32)) - 1
    src = src.view(-1).contiguous()

    def fresh():
        flat, o = _buf(R, rows * op, torch.bfloat16)
        return dict(flat=flat, out=o)
    P = lambda t: C.c_void_p(t.data_ptr() if t is not None else 0)  # noqa: E731
    runs = _twice(lambda b: lib.call("ladi_clip_embed", P(src), P(tok), P(wemb), P(pos), P(b["out"]), rows, seq, c, op, R.stream), fresh)
    out = runs[0]["out"].view(rows, op)
    errs = _window(out, 0, c, "output") + _tail_nan(runs[0]["flat"], rows * op, "output") + _determinism(runs, ["flat"])
    sl = src.long()
    e = tok[sl.clamp_min(0)]
    if wemb is not None:
        e = torch.where((sl < 0)[:, None], wemb[(-sl - 1).clamp(0, B * nv - 1)], e)
    ee, res = _sum_round1(out[:, :c], e, pos[torch.arange(rows, device=R.dev) % seq], ("row", "channel"))
    return errs + ee, res


def replay_channel_affine(R, f):
    from ladi_vton_b200 import lib
    rows, c, pitch = f["rows"], f["c"], f["pitch"]
    x0 = R.poisoned(rows, pitch, _features(R, rows, c))
    s, t = (R.rand(c) + 0.5) / (R.rand(c) + 0.5).sqrt(), R.randn(c) * 0.3

    def fresh():
        return dict(x=x0.clone())
    runs = _twice(lambda b: lib.call("ladi_channel_affine", C.c_void_p(b["x"].data_ptr()), rows, c, pitch, C.c_void_p(s.data_ptr()), C.c_void_p(t.data_ptr()),
                                     R.stream), fresh)
    errs = _layout(runs[0]["x"], c, "in-place output") + _determinism(runs, ["x"])
    r = x0[:, :c].double() * s.double() + t.double()
    e, res = _worst(ratio(runs[0]["x"][:, :c], r, (U_BF16 + EPS24) * r.abs()), ("row", "channel"))
    return errs + e, res


def replay_l2norm_channels(R, f, values=None):
    from ladi_vton_b200 import lib
    rows, c, pitch = f["rows"], f["c"], f["pitch"]
    x0 = R.poisoned(rows, pitch, _features(R, rows, c) if values is None else values)

    def fresh():
        return dict(x=x0.clone())
    runs = _twice(lambda b: lib.call("ladi_l2norm_channels", C.c_void_p(b["x"].data_ptr()), rows, c, pitch, R.stream), fresh)
    errs = _layout(runs[0]["x"], c, "in-place output") + _determinism(runs, ["x"])
    xd = x0[:, :c].double()
    r = xd / torch.sqrt((xd * xd).sum(1, keepdim=True) + 1e-6)
    e, res = _worst(ratio(runs[0]["x"][:, :c], r, (U_BF16 + 0.5 * C_ACC * math.sqrt(c) * EPS24 + 2.0 ** -22) * r.abs()), ("row", "channel"))
    return errs + e, res


def replay_feature_correlation(R, f):
    from ladi_vton_b200 import lib
    n, h, w, c, op = f["n"], f["h"], f["w"], f["c"], f["op"]
    hw = h * w

    def unit(rows):  # FeatureL2Norm outputs: post-ReLU features scaled to unit length per pixel
        a = _features(R, rows, c).float()
        return (a / a.norm(dim=1, keepdim=True).clamp_min(1e-3)).bfloat16()
    fa, fb = unit(n * hw), unit(n * hw)

    def fresh():
        flat, o = _buf(R, n * hw * op, torch.bfloat16)
        return dict(flat=flat, out=o)
    runs = _twice(lambda b: lib.call("ladi_feature_correlation", C.c_void_p(fa.data_ptr()), C.c_void_p(fb.data_ptr()), n, h, w, c,
                                     C.c_void_p(b["out"].data_ptr()), op, R.stream), fresh)
    out = runs[0]["out"].view(n * hw, op)
    errs = _window(out, 0, hw, "output") + _tail_nan(runs[0]["flat"], n * hw * op, "output") + _determinism(runs, ["flat"])
    r, bound = corr_expect(fa.view(n, h, w, c).double(), fb.view(n, h, w, c).double())
    e, res = _worst(ratio(out.view(n, h, w, op)[..., :hw], r, bound), ("image", "yB", "xB", "channel xA*h+yA"))
    return errs + e, res


def tps_expect(theta, inv, rep, n_ctrl):
    """theta [n, 2 n_ctrl], inv [K, K], rep [P, K] float64 (K = n_ctrl + 3) -> (points, points bound, grid, grid bound)."""
    n = theta.shape[0]
    pts = torch.tanh(theta).view(n, n_ctrl, 2)
    ep = 2.0 ** -22 * pts.abs()
    mapping = inv[:, :n_ctrl] @ pts  # [n, K, 2]: the 3 padding rows of the control-point matrix are zero
    em = inv[:, :n_ctrl].abs() @ (ep + C_ACC * math.sqrt(n_ctrl) * EPS24 * pts.abs())
    grid = rep @ mapping
    K = rep.shape[1]
    eg = rep.abs() @ em + C_ACC * math.sqrt(K) * EPS24 * (rep.abs() @ mapping.abs())
    return pts, ep + 2.0 ** -126, grid, eg + EPS24 * grid.abs()


def replay_tps_grid(R, f):
    from ladi_vton_b200 import lib
    from ladi_vton_b200.warp import control_points, tps_matrices
    tp, n, nc, npts = f["tp"], f["n"], f["n_ctrl"], f["npts"]
    if (nc, npts) == (25, 256 * 192):  # the ConvNet_TPS(256, 192) matrices
        inv, rep = (t.to(R.dev).contiguous() for t in tps_matrices(256, 192, control_points()))
        theta = R.poisoned(n, tp, torch.atanh(control_points().to(R.dev)).view(1, -1) + 0.2 * R.randn(n, 2 * nc), dtype=torch.float32)
    else:  # other control-point and pixel counts: matrices of the same magnitudes
        K = nc + 3
        inv, rep = R.randn(K, K) * 2, torch.cat([R.rand(npts, K - 2) * 2 - 1, R.rand(npts, 2) * 2 - 1], dim=1)
        theta = R.poisoned(n, tp, R.randn(n, 2 * nc), dtype=torch.float32)

    def fresh():
        pf, p = _buf(R, n * nc * 2, torch.float32)
        gf, g = _buf(R, n * npts * 2, torch.float32)
        return dict(pf=pf, p=p, gf=gf, g=g)
    runs = _twice(lambda b: lib.call("ladi_tps_grid", C.c_void_p(theta.data_ptr()), tp, C.c_void_p(inv.data_ptr()), C.c_void_p(rep.data_ptr()), n, nc, npts,
                                     C.c_void_p(b["p"].data_ptr()), C.c_void_p(b["g"].data_ptr()), R.stream), fresh)
    errs = (_tail_nan(runs[0]["pf"], n * nc * 2, "points") + _tail_nan(runs[0]["gf"], n * npts * 2, "grid") + _determinism(runs, ["pf", "gf"]))
    pts, bp, grid, bg = tps_expect(theta[:, :2 * nc].double(), inv.double(), rep.double(), nc)
    e1, r1 = _worst(ratio(runs[0]["p"].view(n, nc, 2), pts, bp), ("image", "control point", "coordinate"), " (points)")
    e2, r2 = _worst(ratio(runs[0]["g"].view(n, npts, 2), grid, bg), ("image", "pixel", "coordinate"), " (grid)")
    return errs + e1 + e2, max(r1, r2)


def replay_attention_small(R, f):
    B, heads, nq, nkv, hd = (f[k] for k in ("B", "heads", "nq", "nkv", "hd"))
    Cw = heads * hd
    bufs = {}
    for nm, n_, std in (("q", nq, 2 ** 0.5), ("k", nkv, 2 ** 0.5), ("v", nkv, 1.0)):
        p, bs = f[nm + "p"], f[nm + "bs"]
        t = torch.full(((B - 1) * bs + n_ * p,), NAN, dtype=torch.bfloat16, device=R.dev)
        t.as_strided((B, n_, Cw), (bs, p, 1)).copy_(R.randn(B, n_, Cw, std=std).bfloat16())
        bufs[nm] = t
    return check_attention_small(R, f, bufs)


def check_attention_small(R, f, bufs):
    """Run the descriptor f twice on the inputs bufs["q" / "k" / "v"] (bf16 tensors whose storage offset is the operand's address; they
    may be views into one buffer) into a NaN-poisoned output with a tail, then check the layout, determinism and the float64 bound of
    every query row of every image."""
    from ladi_vton_b200 import lib
    B, heads, nq, nkv, hd, causal, scale = (f[k] for k in ("B", "heads", "nq", "nkv", "hd", "causal", "scale"))
    Cw = heads * hd
    op, obs = f["op"], f["obs"]
    size = (B - 1) * obs + nq * op

    def fresh():
        flat, o = _buf(R, size, torch.bfloat16)
        return dict(flat=flat, out=o)
    P = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    runs = _twice(lambda b: lib.call("ladi_attention_small", P(bufs["q"]), P(bufs["k"]), P(bufs["v"]), P(b["out"]), B, heads, nq, nkv, hd,
                                     f["qp"], f["kp"], f["vp"], op, f["qbs"], f["kbs"], f["vbs"], obs, scale, causal, R.stream), fresh)
    flat = runs[0]["flat"]
    ov = flat.as_strided((B, nq, Cw), (obs, op, 1))
    owned = torch.zeros(flat.numel(), dtype=torch.bool, device=R.dev)  # every element of the flat buffer: row padding, gaps between images, tail
    owned.as_strided((B, nq, Cw), (obs, op, 1)).fill_(True)
    errs = _determinism(runs, ["flat"])
    fl = flat.float()
    if not bool(torch.isfinite(fl[owned]).all()):
        errs.append(f"output: non-finite at flat element {int((owned & ~torch.isfinite(fl)).nonzero()[0])} of the B x nq x heads*hd it owns")
    if not bool(torch.isnan(fl[~owned]).all()):
        errs.append(f"output: wrote flat element {int((~owned & ~torch.isnan(fl)).nonzero()[0])}, outside the rows and columns it owns")
    worst = (0.0, "")
    for b in range(B):  # every image and every query row: a causal off-by-one shows in the rows it shifts
        q, k, v = (bufs[nm].as_strided((B, n_, Cw), (f[nm + "bs"], f[nm + "p"], 1))[b].double() for nm, n_ in (("q", nq), ("k", nkv), ("v", nkv)))
        o, bound = small_attn_expect(q, k, v, heads, scale, causal)
        qq = ratio(ov[b], o, bound).view(nq, heads, hd)
        e, res = _worst(qq, ("query", "head", "column"), f" of image {b}")
        errs += e
        worst = max(worst, res)
    return errs, worst


REPLAY = {"conv": replay_conv, "ln": replay_ln, "check_binarise": replay_check_binarise, "bilinear_down8": replay_bilinear_down8,
          "nchw_to_nhwc": replay_nchw_to_nhwc, "posterior_sample": replay_posterior_sample, "inv_mask_rows": replay_inv_mask_rows,
          "ddim_cfg_step": replay_ddim_cfg_step, "image_out": replay_image_out,
          "image_out_u8": functools.partial(replay_image_out, u8=True), "resize_aa": replay_resize_aa,
          "clip_preprocess": replay_clip_preprocess, "space_to_depth2": replay_space_to_depth2, "channel_affine": replay_channel_affine,
          "l2norm_channels": replay_l2norm_channels, "feature_correlation": replay_feature_correlation, "tps_grid": replay_tps_grid,
          "warp_grid_sample": replay_warp_grid_sample, "maxpool2": replay_maxpool2, "upsample2x_ac": replay_upsample2x_ac,
          "nhwc_to_nchw_clamp": replay_nhwc_to_nchw_clamp, "attention_small": replay_attention_small, "clip_embed": replay_clip_embed,
          "patchify": replay_patchify, "vit_assemble": replay_vit_assemble}


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
    desc, calls, unknown = collect([("fake workload", lambda: [known, ("ladi_not_in_the_schema", (C.c_void_p(16), 3, C.c_void_p(0)))])])
    assert unknown == ["ladi_not_in_the_schema"] and [d["kind"] for d in desc.values()] == ["inv_mask_rows"]
    with pytest.raises(AssertionError, match="ladi_not_in_the_schema"):
        assert_all_known(unknown)


# ================================================================================================================ CPU: the bounds have teeth
def _check(y, r, bound):
    return float(ratio(y, r, bound).max())


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
    assert _check(emulate(False), r, bound) <= 1
    assert _check(emulate(True), r, bound) > 1  # 1. correlation index transposed


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
    assert _check(emulate(0), o, bound) <= 1
    assert _check(emulate(1), o, bound) > 1  # 2. the mask admits key r + 1


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
    assert _check(emulate(False), r, bound) <= 1
    assert _check(emulate(True), r, bound) > 1  # 3. CFG halves swapped


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
    assert _check(emulate(False), r, bound) <= 1
    assert _check(emulate(True), r, bound) > 1  # 4. grid_sample with align_corners=True


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
    assert _check(honest, r, bound) <= 1
    assert _check(faulty, r, bound) > 1


def test_teeth_gate_threshold():
    g = torch.Generator().manual_seed(6)
    x = torch.rand((2, 3, 16, 12), generator=g) * 2 - 1
    m = (torch.rand((2, 1, 16, 12), generator=g) < 0.4).float()
    m[:, :, ::5, ::3] = 0.5
    ref = (x * (m < 0.5)).bfloat16()
    assert _exact(ref, (x.double() * (m < 0.5)).float().bfloat16(), "")[0] == []
    assert _exact((x * (m <= 0.5)).bfloat16(), ref, "")[0] != []  # 6. gate at mask <= 0.5 instead of < 0.5


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
