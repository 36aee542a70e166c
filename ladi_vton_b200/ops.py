"""Tensor-facing wrappers over the C ABI (include/ladi_b200.h).  PyTorch is used only for device memory, streams and
dtype bookkeeping; every function below launches hand-written sm_90a kernels and nothing else.

Activation convention: NHWC bf16 tensors [N, H, W, C] whose last dim is contiguous; a channel-sliced view is fine
(pitch = stride of the W dim).  "Token" tensors [B, T, C] are the same memory viewed as [B, 1, T, C].
"""
import ctypes as C

import torch

from . import lib
from .lib import AttnDesc, ConvDesc

ACT_NONE, ACT_SILU, ACT_GEGLU, ACT_GELU, ACT_RELU = 0, 1, 2, 3, 4
BK = 64
PROFILE = None  # bench.py: set to a list to bracket every launch with CUDA events -> (name, start, end, algorithmic flops)


def _call(name, flops, *args, tag=""):
    if PROFILE is None:
        return lib.call(name, *args)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    lib.call(name, *args)
    e1.record()
    PROFILE.append((name, e0, e1, flops, tag))


def _stream():
    if lib.RECORD is not None:  # sequencing check on CPU tensors: nothing is launched
        return C.c_void_p(0)
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _nhwc(t):
    """-> (n, h, w, c, pitch) of an NHWC view; checks the layout the kernels assume."""
    assert t.dim() == 4 and t.stride(3) == 1, "expect NHWC with contiguous channels"
    n, h, w, c = t.shape
    pitch = t.stride(2)
    assert t.stride(1) == pitch * w and (n == 1 or t.stride(0) == pitch * w * h), \
        f"non-dense NHWC view: shape {tuple(t.shape)} strides {t.stride()}"
    assert pitch % 8 == 0 and t.data_ptr() % 16 == 0, "pitch must be a multiple of 8 elements and the base 16-byte aligned"
    return n, h, w, c, pitch


_SPLITK_WS = {}
SPLITK_WS_BYTES = 64 << 20


def splitk_workspace(device):
    """Persistent fp32 scratch for split-K partial sums (one per device; allocated before any graph capture)."""
    ws = _SPLITK_WS.get(device)
    if ws is None and lib.RECORD is not None:
        return torch.empty(1024, dtype=torch.float32)
    if ws is None:
        ws = _SPLITK_WS[device] = torch.empty(SPLITK_WS_BYTES // 4, dtype=torch.float32, device=device)
    return ws


def padded_k(channels):
    return (channels + BK - 1) // BK * BK


def conv2d(srcs, weight, c_out, **kw):
    """Implicit-GEMM convolution over the channel-concat of `srcs` (+ fused 1x1 over `shortcut` tensors).
    `weight`: packed bf16 [c_out, k_total] (see weights.pack_conv).  Returns the NHWC output tensor.
    rowstat: fp32 [rows, c_out/32, 2] table this call fills with per-row partial {sum, sum of squares} (LayerNorm producer side);
    ln = (stats table of the A rows, colsum fp32 [c_out], eps): LayerNorm folded into this GEMM (weights.fold_layernorm);
    up2x: `srcs` are half-resolution, `weight` = weights.pack_conv_up2x (nearest-2x upsample fused into the 3x3 conv)."""
    d, out, flops, tag = _conv_desc(srcs, weight, c_out, **kw)
    _call("ladi_conv2d_bf16", flops, C.byref(d), _stream(), tag=tag)
    return out


def conv_plan(srcs, weight, c_out, sms=0, **kw):
    """The plan (lib.ConvPlan: N tile, split-K, pair, store path, stages, tile grid) conv2d(srcs, weight, c_out, **kw) runs on a device
    with `sms` SMs (0: this one's); launches nothing."""
    return lib.conv_plan(_conv_desc(srcs, weight, c_out, **kw)[0], sms)


def _conv_desc(srcs, weight, c_out, *, ksize=3, stride=1, pad_lo=1, shortcut=(), bias=None, bias_per_row=False,
               bias_step_stride=0, step_ptr=None, residual=None, row_scale=None, act=ACT_NONE, out=None, out_fp32=False,
               force_bn=0, direct_epilogue=False, split_k=True, pair=None, rowstat=None, ln=None, up2x=False):
    """-> (ConvDesc, output tensor, algorithmic flops, profile tag) of one conv2d call."""
    assert 1 <= len(srcs) <= 2 and len(shortcut) <= 2
    d = ConvDesc()
    n, h_in, w_in, _, _ = _nhwc(srcs[0])
    if up2x:
        assert ksize == 3 and stride == 1
        h_out, w_out = 2 * h_in, 2 * w_in
    elif stride == 2:  # 3x3: padding pad_lo before, 1 after (the VAE's (0, 1, 0, 1) downsample: 0 before); 1x1: none
        pads = (2 if pad_lo == 1 else 1) if ksize == 3 else 0
        h_out, w_out = (h_in + pads - ksize) // 2 + 1, (w_in + pads - ksize) // 2 + 1
    else:
        h_out, w_out = h_in, w_in
    d.n, d.h_out, d.w_out, d.c_out = n, h_out, w_out, c_out
    d.h_in, d.w_in = h_in, w_in
    d.up2x = int(bool(up2x))
    d.ksize, d.stride, d.pad_lo = ksize, stride, pad_lo
    d.n_src = len(srcs)
    for i, s in enumerate(srcs):
        assert s.dtype == torch.bfloat16
        sn, sh, sw, sc, sp = _nhwc(s)
        assert (sn, sh, sw) == (n, h_in, w_in)
        d.src[i], d.src_c[i], d.src_pitch[i] = s.data_ptr(), sc, sp
    d.n_sc = len(shortcut)
    for i, s in enumerate(shortcut):
        assert s.dtype == torch.bfloat16
        sn, sh, sw, sc, sp = _nhwc(s)
        assert (sn, sh, sw) == (n, h_out, w_out)
        d.sc[i], d.sc_c[i], d.sc_pitch[i] = s.data_ptr(), sc, sp
    assert weight.dtype == torch.bfloat16 and weight.dim() == 2 and weight.stride(1) == 1 and weight.shape[0] >= (4 * c_out if up2x else c_out)
    d.weight, d.k_total, d.weight_pitch = weight.data_ptr(), weight.shape[1], weight.stride(0)
    if bias is not None:
        assert bias.dtype == torch.float32
    d.bias, d.bias_per_row, d.bias_step_stride = (bias.data_ptr() if bias is not None else 0), int(bias_per_row), bias_step_stride
    d.step_ptr = step_ptr.data_ptr() if step_ptr is not None else 0
    c_eff = c_out // 2 if act == ACT_GEGLU else c_out
    if out is None:
        c_alloc = c_eff if (out_fp32 or c_eff % 8 == 0) else (c_eff + 7) // 8 * 8  # bf16 rows stay 16-byte aligned (a later conv reads them by TMA)
        out = torch.empty((n, h_out, w_out, c_alloc), dtype=torch.float32 if out_fp32 else torch.bfloat16, device=srcs[0].device)[..., :c_eff]
    on, oh, ow, oc, op = (out.shape[0], out.shape[1], out.shape[2], out.shape[3], out.stride(2))
    assert (on, oh, ow) == (n, h_out, w_out) and oc >= c_eff and out.stride(3) == 1
    assert out.dtype == (torch.float32 if out_fp32 else torch.bfloat16)
    if residual is not None:
        assert residual.dtype == torch.bfloat16 and residual.shape[:3] == out.shape[:3]
        d.residual, d.residual_pitch = residual.data_ptr(), residual.stride(2)
    if row_scale is not None:
        assert row_scale.dtype == torch.float32 and row_scale.numel() == n * h_out * w_out
        d.row_scale = row_scale.data_ptr()
    d.act, d.out, d.out_pitch, d.out_fp32, d.force_bn = act, out.data_ptr(), op, int(out_fp32), force_bn
    d.force_direct_epilogue = int(direct_epilogue)
    d.pair_mode = 0 if pair is None else (1 if pair else 2)  # 2-CTA clusters sharing B: None = library default (off)
    if rowstat is not None:
        assert rowstat.dtype == torch.float32 and rowstat.is_contiguous() and rowstat.numel() == n * h_out * w_out * (c_out // 32) * 2
        d.rowstat_out = rowstat.data_ptr()
    if ln is not None:
        stats, colsum, eps = ln
        k_in = int(srcs[0].shape[3])
        assert stats.dtype == torch.float32 and stats.is_contiguous() and stats.numel() == n * h_in * w_in * (k_in // 32) * 2
        assert colsum.dtype == torch.float32 and colsum.numel() >= c_out and colsum.is_contiguous()
        d.ln_stats, d.ln_colsum, d.ln_eps = stats.data_ptr(), colsum.data_ptr(), float(eps)
    if split_k:
        ws = splitk_workspace(srcs[0].device)
        d.splitk_ws, d.splitk_ws_bytes = ws.data_ptr(), ws.numel() * 4
    # algorithmic flops: 2 * output pixels * c_out * true reduction length (padding channels excluded)
    # (a fused-upsample conv is credited with the 9 taps of the convolution it replaces: algorithmic work is implementation independent)
    k_true = ksize * ksize * sum(int(t.shape[3]) for t in srcs) + sum(int(t.shape[3]) for t in shortcut)
    return (d, out, 2.0 * n * h_out * w_out * c_out * k_true,
            f"k{ksize}s{stride}{'u' if up2x else ''} M={n * h_out * w_out} N={c_out} K={k_true} act={act}{' ln' if ln is not None else ''}{' rs' if rowstat is not None else ''}")


def _gemm_views(a, kw):
    """a [M, K] (row-strided) and the out / residual of kw as the 1 x 1 x M images conv2d takes."""
    assert a.dim() == 2 and a.stride(1) == 1
    a4 = a.as_strided((1, 1, a.shape[0], a.shape[1]), (a.stride(0) * a.shape[0], a.stride(0) * a.shape[0], a.stride(0), 1))
    kw = dict(kw)
    for key in ("out", "residual"):
        t = kw.get(key)
        if t is not None:
            kw[key] = t.as_strided((1, 1, t.shape[0], t.shape[1]), (0, 0, t.stride(0), 1))
    return a4, kw


def gemm(a, weight, n_out, **kw):
    """out[M, n_out] = epilogue(a[M, K] @ weight[n_out, K]^T); `a` may be a row-strided 2-D view."""
    a4, kw = _gemm_views(a, kw)
    o = conv2d([a4], weight, n_out, ksize=1, **kw)
    return o[0, 0]


def gemm_plan(a, weight, n_out, sms=0, **kw):
    """The plan gemm(a, weight, n_out, **kw) runs (see conv_plan)."""
    a4, kw = _gemm_views(a, kw)
    return conv_plan([a4], weight, n_out, sms=sms, ksize=1, **kw)


def attention(q, k, v, heads, scale, out=None, variant=0, trace=None):
    """q [B, Nq, >=heads*64] , k/v [B, Nkv, >=heads*64] (row-strided views of fused projections are fine) -> [B, Nq, heads*64]."""
    B, nq, nkv = q.shape[0], q.shape[1], k.shape[1]
    d, out = _attention_desc(q, k, v, heads, heads * 64, scale, out)
    d.variant = variant
    d.trace = trace.data_ptr() if trace is not None else 0
    _call("ladi_attention_bf16", 4.0 * B * heads * nq * nkv * 64, C.byref(d), _stream(), tag=f"B={B} heads={heads} nq={nq} nkv={nkv}")
    return out


def attention_d512(q, k, v, scale, out=None):
    """One head of width D = 512 (VAE mid-block AttentionBlock; 256 for the reduced-width test models): q [B, Nq, D], k/v [B, Nkv, D]
    row-strided views -> [B, Nq, D]."""
    B, nq, nkv, D = q.shape[0], q.shape[1], k.shape[1], q.shape[2]
    assert D in (256, 512), "the wide single-head attention kernel is built for head widths 512 and 256"
    for t in (q, k, v):
        assert t.shape[2] == D
    d, out = _attention_desc(q, k, v, 1, D, scale, out)
    d.head_dim = D
    _call("ladi_attention_d512_bf16", 4.0 * B * nq * nkv * D, C.byref(d), _stream(), tag=f"B={B} d{D} nq={nq} nkv={nkv}")
    return out


def attention_plan(q, k, v, heads, scale, wide=False, sms=0):
    """The launch (lib.AttnPlan: grid, tiles, work items per CTA, idle consumer warpgroups, shared memory) attention(q, k, v, heads,
    scale) -- or, with wide=True, attention_d512(q, k, v, scale) (heads 1, head width q.shape[2]) -- runs on a device with `sms` SMs (0:
    this one's); launches nothing.  Invalid -> RuntimeError."""
    D = q.shape[2] if wide else 64
    d, _ = _attention_desc(q, k, v, heads, heads * D, scale, None)
    d.head_dim = D if wide else 0
    plan = lib.AttnPlan()
    L = lib.load()
    if L.ladi_attention_plan(C.byref(d), 1 if wide else 0, sms, C.byref(plan)) != 0:
        raise RuntimeError(f"ladi_attention_plan failed: {L.ladi_last_error().decode()}")
    return plan


def _attention_desc(q, k, v, heads, width, scale, out):
    """-> (the lib.AttnDesc of q, k, v and out, the output tensor [B, Nq, width] it writes)."""
    B, nq = q.shape[0], q.shape[1]
    for t in (q, k, v):
        assert t.dtype == torch.bfloat16 and t.stride(2) == 1
    if out is None:
        out = torch.empty((B, nq, width), dtype=torch.bfloat16, device=q.device)
    d = AttnDesc()
    d.batch, d.heads, d.nq, d.nkv = B, heads, nq, k.shape[1]
    d.q, d.q_pitch, d.q_batch_stride = q.data_ptr(), q.stride(1), q.stride(0)
    d.k, d.k_pitch, d.k_batch_stride = k.data_ptr(), k.stride(1), k.stride(0)
    d.v, d.v_pitch, d.v_batch_stride = v.data_ptr(), v.stride(1), v.stride(0)
    d.out, d.out_pitch, d.out_batch_stride = out.data_ptr(), out.stride(1), out.stride(0)
    d.scale = scale
    return d, out


class GroupNormWS:
    """Per-call workspace for the two-pass GroupNorm: [n][chunks][groups][2] fp32."""

    def __init__(self, device):
        self.device, self.buf, self._retired = device, None, []

    def get(self, n, hw, groups):
        need = n * lib.load().ladi_groupnorm_chunks(hw) * groups * 2
        if lib.RECORD is not None:
            return torch.empty(need, dtype=torch.float32)
        if self.buf is None or self.buf.numel() < need:
            if self.buf is not None:
                self._retired.append(self.buf)  # an earlier, smaller session's captured graph still reads/writes this address
            self.buf = torch.empty(max(need, 1 << 20), dtype=torch.float32, device=self.device)
        return self.buf


def groupnorm(srcs, gamma, beta, groups, eps, ws, silu=False, add=None, out=None):
    """GroupNorm(+SiLU)(+add) over the channel-concat of 1-2 NHWC tensors; writes the concatenated normalised tensor."""
    x0 = srcs[0]
    n, h, w, c0, p0 = _nhwc(x0)
    if len(srcs) > 1:
        _, _, _, c1, p1 = _nhwc(srcs[1])
        x1 = srcs[1]
    else:
        x1, c1, p1 = None, 0, 0
    if out is None:
        out = torch.empty((n, h, w, c0 + c1), dtype=torch.bfloat16, device=x0.device)
    wsb = ws.get(n, h * w, groups)
    s = _stream()
    _call("ladi_groupnorm_stats", 2.0 * n * h * w * (c0 + c1), _ptr(x0), c0, p0, _ptr(x1), c1, p1, n, h * w, groups, _ptr(wsb), s)
    _call("ladi_groupnorm_apply", 4.0 * n * h * w * (c0 + c1), _ptr(x0), c0, p0, _ptr(x1), c1, p1, n, h * w, groups, _ptr(wsb), _ptr(gamma), _ptr(beta),
             eps, int(silu), _ptr(add), (add.stride(2) if add is not None else 0), _ptr(out), out.stride(2), s)
    return out


def layernorm(x, gamma, beta, eps=1e-5, out=None):
    """x [rows, C] bf16 (row-strided ok) -> [rows, C] bf16."""
    assert x.dim() == 2 and x.stride(1) == 1
    if out is None:
        out = torch.empty((x.shape[0], x.shape[1]), dtype=torch.bfloat16, device=x.device)
    _call("ladi_layernorm", 0.0, _ptr(x), x.stride(0), x.shape[0], x.shape[1], _ptr(gamma), _ptr(beta), eps, _ptr(out),
             out.stride(0), _stream())
    return out


def softmax_rows(s, scale, out=None):
    assert s.dtype == torch.float32 and s.dim() == 2 and s.stride(1) == 1
    if out is None:
        out = torch.empty(s.shape, dtype=torch.bfloat16, device=s.device)
    lib.call("ladi_softmax_rows", _ptr(s), s.shape[0], s.shape[1], s.stride(0), scale, _ptr(out), out.stride(0), _stream())
    return out


def cls_attention(q0, kv, heads, head_dim, scale):
    """q0 [B, heads*hd] bf16 (CLS query), kv [B, T, 2*heads*hd] bf16 (K | V) -> [B, heads*hd] bf16."""
    args, out = _cls_attention_args(q0, kv, heads, head_dim, scale)
    lib.call("ladi_cls_attention", *args, _stream())
    return out


def cls_attention_plan(q0, kv, heads, head_dim, scale):
    """The launch (lib.SmallAttnPlan) cls_attention(q0, kv, heads, head_dim, scale) runs; launches nothing.  Invalid -> RuntimeError."""
    args, _ = _cls_attention_args(q0, kv, heads, head_dim, scale)
    plan = lib.SmallAttnPlan()
    L = lib.load()
    if L.ladi_cls_attention_plan(*args, 0, C.byref(plan)) != 0:
        raise RuntimeError(f"ladi_cls_attention_plan failed: {L.ladi_last_error().decode()}")
    return plan


def _cls_attention_args(q0, kv, heads, head_dim, scale):
    B, T = kv.shape[0], kv.shape[1]
    assert q0.dtype == torch.bfloat16 and kv.dtype == torch.bfloat16 and kv.stride(2) == 1 and q0.stride(1) == 1
    out = torch.empty((B, heads * head_dim), dtype=torch.bfloat16, device=q0.device)
    return (_ptr(q0), q0.stride(0), _ptr(kv), kv.stride(1), B, T, heads, head_dim, scale, _ptr(out), out.stride(0)), out


def add(a, b, out=None):
    assert a.is_contiguous() and b.is_contiguous() and a.shape == b.shape and a.dtype == torch.bfloat16
    if out is None:
        out = torch.empty_like(a)
    lib.call("ladi_add_bf16", _ptr(a), _ptr(b), _ptr(out), a.numel(), _stream())
    return out


def upsample2x(x):
    n, h, w, c, p = _nhwc(x)
    assert p == c
    out = torch.empty((n, 2 * h, 2 * w, c), dtype=torch.bfloat16, device=x.device)
    _call("ladi_upsample2x_nhwc", 0.0, _ptr(x), n, h, w, c, _ptr(out), _stream())
    return out


def nchw_to_nhwc(x, out, c_off=0, scale=1.0, f=1, gate=None):
    """x NCHW fp32 (sampled every f-th pixel, optionally gated by gate<0.5) -> channels [c_off, c_off+C) of NHWC bf16 `out`."""
    assert x.dtype == torch.float32 and x.is_contiguous() and out.dtype == torch.bfloat16
    n, c, H, W = x.shape
    assert H % f == 0 and W % f == 0 and out.shape[1] == H // f and out.shape[2] == W // f and out.shape[0] == n
    if gate is not None:
        assert gate.dtype == torch.float32 and gate.is_contiguous() and gate.shape == (n, 1, H, W)
    lib.call("ladi_nchw_f32_to_nhwc_bf16", _ptr(x), n, c, H // f, W // f, f, scale, _ptr(gate), _ptr(out), out.stride(2), c_off, _stream())
    return out


def nhwc_to_nchw(x, c, c_off=0):
    n, h, w, _ = x.shape
    out = torch.empty((n, c, h, w), dtype=torch.float32, device=x.device)
    lib.call("ladi_nhwc_to_nchw_f32", _ptr(x), int(x.dtype == torch.float32), n, c, h, w, x.stride(2), c_off, _ptr(out), _stream())
    return out


def posterior_sample(moments, noise, scale):
    """moments NHWC fp32 [n,h,w,>=2cz], noise NCHW fp32 [n,cz,h,w] -> NCHW fp32 latents * scale."""
    n, cz, h, w = noise.shape
    assert moments.dtype == torch.float32 and noise.dtype == torch.float32 and noise.is_contiguous()
    out = torch.empty_like(noise)
    lib.call("ladi_posterior_sample", _ptr(moments), moments.stride(2), _ptr(noise), n, cz, h, w, scale, _ptr(out), _stream())
    return out


def inv_mask_rows(mask, f):
    n, _, H, W = mask.shape
    assert mask.dtype == torch.float32 and mask.is_contiguous()
    out = torch.empty((n, H // f, W // f), dtype=torch.float32, device=mask.device)
    lib.call("ladi_inv_mask_rows", _ptr(mask), n, H, W, f, _ptr(out), _stream())
    return out


def bilinear_down8(x):
    n, c, H, W = x.shape
    assert x.dtype == torch.float32 and x.is_contiguous()
    out = torch.empty((n, c, H // 8, W // 8), dtype=torch.float32, device=x.device)
    lib.call("ladi_bilinear_down8", _ptr(x), n, c, H, W, _ptr(out), _stream())
    return out


def ddim_cfg_step(eps, latents, unet_in, cfg, guidance, coef, step_ptr, advance=True, noise=None):
    """coef fp32 [steps, 8] (scheduler.coefficients); noise: NCHW fp32 variance noise of the eta > 0 update, or None."""
    B, _, h, w = latents.shape
    assert eps.dtype == torch.float32 and latents.dtype == torch.float32 and latents.is_contiguous()
    assert coef.dtype == torch.float32 and coef.shape[-1] == 8 and coef.is_contiguous()
    assert noise is None or (noise.dtype == torch.float32 and noise.is_contiguous() and noise.shape == latents.shape)
    lib.call("ladi_ddim_cfg_step", _ptr(eps), eps.stride(2), _ptr(latents), _ptr(unet_in), unet_in.stride(2), B, h, w, int(cfg),
             float(guidance), _ptr(coef), _ptr(step_ptr), int(advance), _ptr(noise), _stream())


def check_binarise_(image, mask, flags):
    """Range checks of prepare_mask_and_masked_image recorded in `flags` (device int32[2]) + in-place mask binarisation, no host sync."""
    assert image.dtype == torch.float32 and mask.dtype == torch.float32 and image.is_contiguous() and mask.is_contiguous()
    assert flags.dtype == torch.int32 and flags.numel() >= 2
    lib.call("ladi_check_binarise", _ptr(image), image.numel(), _ptr(mask), mask.numel(), _ptr(flags), _stream())


def image_out(x):
    n, h, w, _ = x.shape
    out = torch.empty((n, h, w, 3), dtype=torch.float32, device=x.device)
    lib.call("ladi_image_out", _ptr(x), int(x.dtype == torch.float32), n, h, w, x.stride(2), _ptr(out), _stream())
    return out


def image_out_u8(x):
    """(x/2+0.5).clamp(0,1) -> (v*255).round() as NHWC uint8 (numpy_to_pil's arithmetic on the device)."""
    n, h, w, _ = x.shape
    out = torch.empty((n, h, w, 3), dtype=torch.uint8, device=x.device)
    lib.call("ladi_image_out_u8", _ptr(x), int(x.dtype == torch.float32), n, h, w, x.stride(2), _ptr(out), _stream())
    return out


def image_save_u8(x):
    """NHWC fp32 [n,h,w,>=3] decoder output -> NHWC uint8 [n,h,w,3]: `(x+1)/2` then torchvision save_image's
    `mul(255).add_(0.5).clamp_(0,255).to(uint8)`, each step rounded in fp32 as torch does it."""
    n, h, w, _ = x.shape
    assert x.dtype == torch.float32 and x.stride(3) == 1 and x.stride(1) == w * x.stride(2) and x.stride(0) == h * x.stride(1)
    out = torch.empty((n, h, w, 3), dtype=torch.uint8, device=x.device)
    lib.call("ladi_image_save_u8", _ptr(x), n, h, w, x.stride(2), _ptr(out), _stream())
    return out


def pose_heatmaps(keypoints, h, w, sigma=9.0):
    """src/utils/posemap.py kpoint_to_heatmap for a whole batch: keypoints fp32 [..., 2] (x, y) -> fp32 [..., h, w]."""
    k = keypoints.to(torch.float32).contiguous()
    assert k.shape[-1] == 2
    out = torch.empty(tuple(k.shape[:-1]) + (h, w), dtype=torch.float32, device=k.device)
    lib.call("ladi_pose_heatmaps", _ptr(k), k.numel() // 2, h, w, float(sigma), _ptr(out), _stream())
    return out


# ---- text / vision conditioning front-end (SURVEY.md 8(f) row 1) ---------------------------------------------------------------
def attention_small(q, k, v, heads, scale, causal=False):
    """q [B, Nq, heads*hd], k/v [B, Nkv, heads*hd] bf16 views (last dim contiguous) -> [B, Nq, heads*hd] bf16.  Exact softmax,
    fp32 scores; any head width that is a multiple of 8 (the CLIP ViT-H heads are 80 wide), Nkv <= 1024, optional causal mask."""
    args, out = _attention_small_args(q, k, v, heads, scale, causal)
    B, nq, nkv, hd = args[4], args[6], args[7], args[8]
    _call("ladi_attention_small", 4.0 * B * heads * nq * nkv * hd, *args, _stream(), tag=f"B={B} heads={heads} nq={nq} nkv={nkv} hd={hd}")
    return out


def attention_small_plan(q, k, v, heads, scale, causal=False, sms=0):
    """The launch (lib.SmallAttnPlan: query-row chunks per head and image, rows per block, shared memory, opt-in) attention_small(q, k, v,
    heads, scale, causal) runs on a device with `sms` SMs (0: this one's); launches nothing.  Invalid -> RuntimeError."""
    args, _ = _attention_small_args(q, k, v, heads, scale, causal)
    plan = lib.SmallAttnPlan()
    L = lib.load()
    if L.ladi_attention_small_plan(*args, sms, C.byref(plan)) != 0:
        raise RuntimeError(f"ladi_attention_small_plan failed: {L.ladi_last_error().decode()}")
    return plan


def _attention_small_args(q, k, v, heads, scale, causal):
    """-> (the arguments of ladi_attention_small without the stream, the output tensor they write)."""
    B, nq, C = q.shape
    hd = C // heads
    for t in (q, k, v):
        assert t.dtype == torch.bfloat16 and t.stride(2) == 1
    out = torch.empty((B, nq, C), dtype=torch.bfloat16, device=q.device)
    return (_ptr(q), _ptr(k), _ptr(v), _ptr(out), B, heads, nq, k.shape[1], hd, q.stride(1), k.stride(1), v.stride(1), out.stride(1),
            q.stride(0), k.stride(0), v.stride(0), out.stride(0), float(scale), 1 if causal else 0), out


def clip_embed(src, tok, word_emb, pos, seq):
    """src int32 [rows] (>= 0: token id; < 0: -(row of word_emb) - 1), tok [V, C], word_emb [R, C] or None, pos [seq, C] bf16."""
    rows, c = src.numel(), tok.shape[1]
    assert src.dtype == torch.int32 and tok.dtype == torch.bfloat16 and pos.dtype == torch.bfloat16 and tok.is_contiguous() and pos.is_contiguous()
    assert word_emb is None or (word_emb.dtype == torch.bfloat16 and word_emb.is_contiguous() and word_emb.shape[-1] == c)
    out = torch.empty((rows, c), dtype=torch.bfloat16, device=tok.device)
    _call("ladi_clip_embed", 0.0, _ptr(src), _ptr(tok), _ptr(word_emb), _ptr(pos), _ptr(out), rows, seq, c, c, _stream())
    return out


def patchify(pixels, patch, k_pad):
    """pixels NCHW fp32 -> bf16 [n * gh * gw, k_pad] im2col rows of a patch x patch / stride patch convolution."""
    n, ch, h, w = pixels.shape
    assert pixels.dtype == torch.float32 and pixels.is_contiguous()
    out = torch.empty((n * (h // patch) * (w // patch), k_pad), dtype=torch.bfloat16, device=pixels.device)
    _call("ladi_patchify", 0.0, _ptr(pixels), _ptr(out), n, ch, h, w, patch, k_pad, _stream())
    return out


def vit_assemble(patch, cls, pos, n):
    """patch [n * np, C] bf16, cls [C], pos [np + 1, C] -> tokens [n, np + 1, C] bf16."""
    c = patch.shape[1]
    np_ = patch.shape[0] // n
    assert patch.dtype == torch.bfloat16 and patch.stride(1) == 1 and cls.is_contiguous() and pos.is_contiguous()
    out = torch.empty((n, np_ + 1, c), dtype=torch.bfloat16, device=patch.device)
    _call("ladi_vit_assemble", 0.0, _ptr(patch), patch.stride(0), _ptr(cls), _ptr(pos), _ptr(out), n, np_, c, _stream())
    return out


# ---- cloth-warping front-end (SURVEY.md 8(f) row 2) -----------------------------------------------------------------------------
def resize_aa(x, oh, ow, out=None, c_off=0):
    """torchvision resize(x, (oh, ow), BILINEAR, antialias=True): NCHW fp32 -> channels [c_off, c_off+C) of an NHWC bf16 tensor."""
    n, c, h, w = x.shape
    assert x.dtype == torch.float32 and x.is_contiguous()
    if out is None:
        out = torch.zeros((n, oh, ow, (c + 7) // 8 * 8), dtype=torch.bfloat16, device=x.device)
    assert out.dtype == torch.bfloat16 and out.is_contiguous() and out.shape[:3] == (n, oh, ow)
    _call("ladi_resize_aa", 0.0, _ptr(x), n, c, h, w, oh, ow, _ptr(out), out.shape[3], c_off, _stream())
    return out


def resize_aa_f32(x, oh, ow, out=None):
    """resize_aa's arithmetic, unrounded: NCHW fp32 -> NCHW fp32 [n, c, oh, ow] (into `out` when given)."""
    n, c, h, w = x.shape
    assert x.dtype == torch.float32 and x.is_contiguous()
    if out is None:
        out = torch.empty((n, c, oh, ow), dtype=torch.float32, device=x.device)
    assert out.dtype == torch.float32 and out.is_contiguous() and tuple(out.shape) == (n, c, oh, ow)
    _call("ladi_resize_aa_f32", 0.0, _ptr(x), n, c, h, w, oh, ow, _ptr(out), _stream())
    return out


def clip_preprocess(x, oh, ow, mean, std, quantise=False):
    """inference.py:265-271: resize((x + 1) / 2, (oh, ow), antialias=True).clamp(0, 1) -> (v - mean) / std; NCHW fp32 in and out."""
    n, c, h, w = x.shape
    assert x.dtype == torch.float32 and x.is_contiguous() and mean.numel() == c and std.numel() == c
    out = torch.empty((n, c, oh, ow), dtype=torch.float32, device=x.device)
    _call("ladi_clip_preprocess", 0.0, _ptr(x), n, c, h, w, oh, ow, _ptr(mean), _ptr(std), int(bool(quantise)), _ptr(out), _stream())
    return out


def space_to_depth2(x, c=None):
    """NHWC bf16 [n,h,w,pitch] (first c channels) -> [n,h/2,w/2,pad8(4c)] with channel (sy*2+sx)*c + ch; returns (tensor, 4c)."""
    n, h, w, cc, pitch = _nhwc(x)
    c = cc if c is None else c
    out = torch.zeros((n, h // 2, w // 2, (4 * c + 7) // 8 * 8), dtype=torch.bfloat16, device=x.device)
    _call("ladi_space_to_depth2", 0.0, _ptr(x), n, h, w, c, pitch, _ptr(out), out.shape[3], _stream())
    return out, 4 * c


def channel_affine_(x, scale, shift):
    n, h, w, c, pitch = _nhwc(x)
    _call("ladi_channel_affine", 0.0, _ptr(x), n * h * w, c, pitch, _ptr(scale), _ptr(shift), _stream())
    return x


def l2norm_channels_(x):
    n, h, w, c, pitch = _nhwc(x)
    _call("ladi_l2norm_channels", 0.0, _ptr(x), n * h * w, c, pitch, _stream())
    return x


def feature_correlation(fa, fb):
    n, h, w, c, pitch = _nhwc(fa)
    assert pitch == c and fb.shape == fa.shape and fb.is_contiguous() and fa.is_contiguous()
    hw = h * w
    out = torch.zeros((n, h, w, (hw + 7) // 8 * 8), dtype=torch.bfloat16, device=fa.device)
    _call("ladi_feature_correlation", 2.0 * n * hw * hw * c, _ptr(fa), _ptr(fb), n, h, w, c, _ptr(out), out.shape[3], _stream())
    return out[..., :hw]


def tps_grid(theta, inverse_kernel, target_coordinate_repr, n_ctrl):
    """theta fp32 [n, 2*n_ctrl] (pre-tanh) -> (points fp32 [n, n_ctrl, 2], grid fp32 [n, n_points, 2])."""
    n = theta.shape[0]
    npts = target_coordinate_repr.shape[0]
    assert theta.dtype == torch.float32 and theta.stride(1) == 1
    inverse_kernel, target_coordinate_repr = inverse_kernel.contiguous(), target_coordinate_repr.contiguous()  # torch.inverse is column-major
    points = torch.empty((n, n_ctrl, 2), dtype=torch.float32, device=theta.device)
    grid = torch.empty((n, npts, 2), dtype=torch.float32, device=theta.device)
    _call("ladi_tps_grid", 0.0, _ptr(theta), theta.stride(0), _ptr(inverse_kernel), _ptr(target_coordinate_repr), n, n_ctrl, npts, _ptr(points),
          _ptr(grid), _stream())
    return points, grid


def warp_grid_sample(low_grid, cloth, out, c_off=0):
    """low_grid fp32 [n,gh,gw,2]; cloth NCHW fp32 [n,c,H,W]; writes channels [c_off, c_off+c) of `out` NHWC bf16 [n,H,W,pitch]."""
    n, gh, gw, _ = low_grid.shape
    _, c, H, W = cloth.shape
    assert low_grid.dtype == torch.float32 and low_grid.is_contiguous() and cloth.dtype == torch.float32 and cloth.is_contiguous()
    assert out.dtype == torch.bfloat16 and out.is_contiguous() and out.shape[:3] == (n, H, W)
    _call("ladi_warp_grid_sample", 0.0, _ptr(low_grid), gh, gw, _ptr(cloth), n, c, H, W, _ptr(out), out.shape[3], c_off, _stream())
    return out


def warp_grid_sample_f32(low_grid, cloth):
    """warp_grid_sample's arithmetic, unrounded: low_grid fp32 [n,gh,gw,2], cloth NCHW fp32 [n,c,H,W] -> warped NCHW fp32 [n,c,H,W]."""
    n, gh, gw, _ = low_grid.shape
    _, c, H, W = cloth.shape
    assert low_grid.dtype == torch.float32 and low_grid.is_contiguous() and cloth.dtype == torch.float32 and cloth.is_contiguous()
    out = torch.empty((n, c, H, W), dtype=torch.float32, device=cloth.device)
    _call("ladi_warp_grid_sample_f32", 0.0, _ptr(low_grid), gh, gw, _ptr(cloth), n, c, H, W, _ptr(out), _stream())
    return out


def maxpool2(x):
    n, h, w, c, pitch = _nhwc(x)
    assert pitch == c and x.is_contiguous()
    out = torch.empty((n, h // 2, w // 2, c), dtype=torch.bfloat16, device=x.device)
    _call("ladi_maxpool2_nhwc", 0.0, _ptr(x), n, h, w, c, _ptr(out), _stream())
    return out


def upsample2x_bilinear_ac(x):
    n, h, w, c, pitch = _nhwc(x)
    assert pitch == c and x.is_contiguous()
    out = torch.empty((n, 2 * h, 2 * w, c), dtype=torch.bfloat16, device=x.device)
    _call("ladi_upsample2x_bilinear_ac", 0.0, _ptr(x), n, h, w, c, _ptr(out), _stream())
    return out


def nhwc_f32_to_nchw_clamp(x, c, lo, hi):
    n, h, w, pitch = x.shape
    assert x.dtype == torch.float32 and x.is_contiguous()
    out = torch.empty((n, c, h, w), dtype=torch.float32, device=x.device)
    _call("ladi_nhwc_f32_to_nchw_clamp", 0.0, _ptr(x), n, c, h, w, pitch, float(lo), float(hi), _ptr(out), _stream())
    return out


# ---- image-quality metrics (csrc/metrics.cu) ------------------------------------------------------------------------------------------
POOL_MAX, POOL_AVG, POOL_AVG_EXCLUDE_PAD, POOL_GLOBAL_AVG_F32 = 0, 1, 2, 3


def conv_out_size(size, k, s, p):
    return (size + 2 * p - k) // s + 1


def im2col(x, kernel, stride, padding, k_pad, shift=None, scale=None, dtype=torch.bfloat16):
    """Rows [n*oh*ow, k_pad] of `dtype` (bf16, or fp32 for the tf32 metric networks), column (ky*kw + kx)*c + ch, of a kernel=(kh, kw) /
    stride=(sh, sw) / padding=(ph, pw) convolution.  x: NHWC of the same dtype (channel-sliced views fine, c % 8 == 0), or NCHW fp32
    pixels (with shift / scale given) whose per-channel fp32 affine (x - shift) / scale is applied before the zero padding."""
    (kh, kw), (sh, sw), (ph, pw) = kernel, stride, padding
    pixels = shift is not None
    if pixels:
        assert x.dtype == torch.float32 and x.is_contiguous() and scale is not None
        n, c, h, w = x.shape
        pitch = 0
    else:
        assert x.dtype == dtype and scale is None
        n, h, w, c, pitch = _nhwc(x)
    oh, ow = conv_out_size(h, kh, sh, ph), conv_out_size(w, kw, sw, pw)
    out = torch.empty((n * oh * ow, k_pad), dtype=dtype, device=x.device)
    name = "ladi_im2col_f32" if dtype == torch.float32 else "ladi_im2col_bf16"
    _call(name, 0.0, _ptr(x), int(pixels), n, c, h, w, pitch, kh, kw, sh, sw, ph, pw, _ptr(shift), _ptr(scale), _ptr(out), k_pad, _stream())
    return out, (n, oh, ow)


_POOL = {torch.bfloat16: "ladi_pool2d_bf16", torch.float32: "ladi_pool2d_f32"}
_LPIPS = {torch.bfloat16: "ladi_lpips_layer", torch.float32: "ladi_lpips_layer_f32"}


def pool2d(x, k, s, p, mode, out=None, c_off=0):
    """torch max_pool2d / avg_pool2d on NHWC bf16 or fp32; the result (same dtype) goes to channels [c_off, c_off + C) of `out` when
    given."""
    n, h, w, c, pitch = _nhwc(x)
    oh, ow = conv_out_size(h, k, s, p), conv_out_size(w, k, s, p)
    if out is None:
        out = torch.empty((n, oh, ow, c), dtype=x.dtype, device=x.device)
    assert out.dtype == x.dtype and out.is_contiguous() and tuple(out.shape[:3]) == (n, oh, ow) and out.shape[3] >= c_off + c
    _call(_POOL[x.dtype], 0.0, _ptr(x), n, h, w, c, pitch, k, s, p, mode, _ptr(out), out.shape[3], c_off, _stream())
    return out


def global_avg_pool(x):
    """adaptive_avg_pool2d(x, 1).flatten(1): NHWC bf16 or fp32 -> fp32 [n, C]."""
    n, h, w, c, pitch = _nhwc(x)
    out = torch.empty((n, c), dtype=torch.float32, device=x.device)
    _call(_POOL[x.dtype], 0.0, _ptr(x), n, h, w, c, pitch, 0, 0, 0, POOL_GLOBAL_AVG_F32, _ptr(out), c, 0, _stream())
    return out


def lpips_layer_(fa, fb, lin, acc):
    """acc[b] += spatial mean of lin . (unit(fa) - unit(fb))^2 for NHWC bf16 or fp32 feature pairs of equal shape, dtype and pitch."""
    n, h, w, c, pitch = _nhwc(fa)
    assert fb.dtype == fa.dtype and _nhwc(fb) == (n, h, w, c, pitch) and lin.dtype == torch.float32 and lin.numel() == c and lin.is_contiguous()
    assert acc.dtype == torch.float32 and acc.numel() == n and acc.is_contiguous()
    _call(_LPIPS[fa.dtype], 0.0, _ptr(fa), _ptr(fb), n, h, w, c, pitch, _ptr(lin), _ptr(acc), _stream())
    return acc


def gemm_tf32(a, weight, n_out, out, c_off=0, bias=None, relu=False):
    """out[:, c_off:c_off + n_out] = relu?(a @ weight[:n_out, :K]^T + bias) on TF32 tensor cores (operands rounded to nearest TF32, fp32
    accumulation).  a: fp32 [M, K] (row-strided view fine), weight: fp32 [n_out, K'] with K' >= K (zero columns past the true reduction
    length), out: fp32 [M, pitch] with a contiguous last dimension."""
    assert a.dtype == weight.dtype == out.dtype == torch.float32 and a.dim() == weight.dim() == out.dim() == 2
    assert a.stride(1) == weight.stride(1) == out.stride(1) == 1 and weight.shape[0] == n_out and out.shape[0] == a.shape[0]
    assert out.shape[1] >= c_off + n_out and (bias is None or (bias.dtype == torch.float32 and bias.is_contiguous()))
    m, k = a.shape
    _call("ladi_gemm_tf32", 2.0 * m * k * n_out, _ptr(a), m, k, a.stride(0), _ptr(weight), n_out, weight.stride(0), _ptr(bias), int(relu),
          _ptr(out), out.stride(0), c_off, _stream(), tag=f"tf32 M={m} N={n_out} K={k}")
    return out


L1_MEAN_WS = 1024  # LADI_L1_MEAN_WS
_L1_WS = {}


def _rows(t):
    """A 2-D fp32 view [rows, cols] with unit column stride, or a contiguous tensor of any rank seen as [numel / last, last]."""
    if t.dim() != 2:
        assert t.is_contiguous(), "l1_mean_: a tensor of rank != 2 must be contiguous"
        t = t.reshape(-1, t.shape[-1])
    assert t.dtype == torch.float32 and t.stride(1) == 1
    return t


def l1_mean_(a, b, acc, weight=1.0):
    """acc[0] += weight * mean|a - b| (nn.L1Loss) on the device, in a fixed reduction order.  a, b: fp32 [rows, cols] views with unit column
    stride (pitches may differ and exceed cols), or contiguous tensors of equal shape; acc: a one-element fp32 device view.  The partial
    sums go to a workspace cached per device and stream, so calls issued on different streams do not share one."""
    a2, b2 = _rows(a), _rows(b)
    assert a2.shape == b2.shape and acc.dtype == torch.float32 and acc.numel() == 1
    if lib.RECORD is not None:
        ws = torch.empty(L1_MEAN_WS, dtype=torch.float32)
    else:  # the partials of one call are consumed by its own second launch: one workspace per (device, stream) keeps streams apart
        key = (a.device, torch.cuda.current_stream(a.device).cuda_stream)
        ws = _L1_WS.get(key)
        if ws is None:
            ws = _L1_WS[key] = torch.empty(L1_MEAN_WS, dtype=torch.float32, device=a.device)
    rows, cols = a2.shape
    _call("ladi_l1_mean_f32", 3.0 * rows * cols, _ptr(a2), a2.stride(0), _ptr(b2), b2.stride(0), rows, cols, float(weight), _ptr(ws), _ptr(acc),
          _stream(), tag=f"rows={rows} cols={cols}")
    return acc


def ssim(x, y):
    """Per-image SSIM (torchmetrics, data_range 1.0, gaussian 11 / 1.5) of NCHW fp32 images -> fp32 [n]."""
    assert x.dtype == torch.float32 and y.dtype == torch.float32 and x.is_contiguous() and y.is_contiguous() and x.shape == y.shape
    n, c, h, w = x.shape
    tiles = lib.load().ladi_ssim_partials(h, w) if lib.RECORD is None else 1
    if tiles < 0:
        raise ValueError(f"SSIM needs images of at least 11 x 11 pixels, got {h} x {w}")
    ws = torch.empty(n * tiles, dtype=torch.float32, device=x.device)
    out = torch.empty(n, dtype=torch.float32, device=x.device)
    _call("ladi_ssim_f32", 0.0, _ptr(x), _ptr(y), n, c, h, w, _ptr(ws), _ptr(out), _stream())
    return out


def resize_tf1_u8(x, oh, ow):
    """(x * 255).byte() + torch-fidelity's TF1 bilinear resize: NCHW fp32 in [0, 1] -> NCHW fp32 [n, c, oh, ow] in [0, 255]."""
    assert x.dtype == torch.float32 and x.is_contiguous()
    n, c, h, w = x.shape
    out = torch.empty((n, c, oh, ow), dtype=torch.float32, device=x.device)
    _call("ladi_resize_tf1_u8", 0.0, _ptr(x), n, c, h, w, oh, ow, _ptr(out), _stream())
    return out
