"""H100-native AutoencoderKL (LaDI-VTON fork semantics) and EMASC on the sm_90a kernels in ops.py.

Drop-in for src/models/AutoencoderKL.py:145-188 (`encode` returns `(obj.latent_dist, skips)`,
`decode(z, intermediate_features, int_layers)` adds the EMASC features as in src/models/vae.py:183-212) and for
src/models/emasc.py:11-40 + src/utils/data_utils.py:4-16 (`mask_features` folded into the second EMASC
conv's epilogue as a per-pixel (1-mask) row scale).  State-dict key names follow SURVEY.md Appendix A.7.

NHWC bf16 internally; NCHW fp32 at the boundary.  quant_conv (1x1) is folded algebraically into encoder.conv_out at load
time (both linear, no padding interaction); post_quant_conv stays separate because its bias meets conv_in's zero padding.
"""
import ctypes as C
import os

import torch

from . import engine as eng, lib, ops
from .module import PackedModule, _Cfg
from .weights import f32, pack_conv, pack_conv_up2x, pack_linear

SD2_VAE = dict(in_channels=3, out_channels=3, block_out_channels=(128, 256, 512, 512), layers_per_block=2,
               latent_channels=4, norm_num_groups=32, scaling_factor=0.18215, sample_size=512)


def vae_param_shapes(cfg):
    cfg = {**SD2_VAE, **cfg}
    ch, L, cz = cfg["block_out_channels"], cfg["layers_per_block"], cfg["latent_channels"]
    S = {}

    def conv(p, ci, co, k):
        S[p + ".weight"], S[p + ".bias"] = (co, ci, k, k), (co,)

    def norm(p, c):
        S[p + ".weight"], S[p + ".bias"] = (c,), (c,)

    def resnet(p, ci, co):
        norm(p + ".norm1", ci); conv(p + ".conv1", ci, co, 3); norm(p + ".norm2", co); conv(p + ".conv2", co, co, 3)
        if ci != co:
            conv(p + ".conv_shortcut", ci, co, 1)

    def mid(p, c):
        resnet(p + ".resnets.0", c, c); resnet(p + ".resnets.1", c, c)
        a = p + ".attentions.0"
        norm(a + ".group_norm", c)
        for n in ("query", "key", "value", "proj_attn"):
            S[a + f".{n}.weight"], S[a + f".{n}.bias"] = (c, c), (c,)

    conv("encoder.conv_in", cfg["in_channels"], ch[0], 3)
    out = ch[0]
    for i, c in enumerate(ch):
        prev, out = out, c
        for l in range(L):
            resnet(f"encoder.down_blocks.{i}.resnets.{l}", prev if l == 0 else out, out)
        if i < len(ch) - 1:
            conv(f"encoder.down_blocks.{i}.downsamplers.0.conv", out, out, 3)
    mid("encoder.mid_block", ch[-1]); norm("encoder.conv_norm_out", ch[-1]); conv("encoder.conv_out", ch[-1], 2 * cz, 3)
    rch = list(reversed(ch))
    conv("decoder.conv_in", cz, rch[0], 3); mid("decoder.mid_block", rch[0])
    out = rch[0]
    for i, c in enumerate(rch):
        prev, out = out, c
        for l in range(L + 1):
            resnet(f"decoder.up_blocks.{i}.resnets.{l}", prev if l == 0 else out, out)
        if i < len(ch) - 1:
            conv(f"decoder.up_blocks.{i}.upsamplers.0.conv", out, out, 3)
    norm("decoder.conv_norm_out", ch[0]); conv("decoder.conv_out", ch[0], cfg["out_channels"], 3)
    conv("quant_conv", 2 * cz, 2 * cz, 1); conv("post_quant_conv", cz, cz, 1)
    return S


class DiagonalGaussianDistribution:
    """vae.py:329-348 on device: moments NHWC fp32 [B,h,w,2cz]."""

    def __init__(self, moments, cz):
        self.moments, self.cz = moments, cz

    def sample(self, generator=None, noise=None):
        B, h, w, _ = self.moments.shape
        if noise is None:  # randn_tensor semantics (Appendix A.8): draw on the generator's device, then move
            gdev = generator.device if generator is not None else self.moments.device
            noise = torch.randn((B, self.cz, h, w), generator=generator, device=gdev, dtype=torch.float32)
        return ops.posterior_sample(self.moments, noise.to(self.moments.device, torch.float32).contiguous(), 1.0)

    def mode(self):
        return ops.nhwc_to_nchw(self.moments, self.cz)


class _Enc:
    def __init__(self, d):
        self.latent_dist = d


class _Dec:
    def __init__(self, s):
        self.sample = s


class AutoencoderKL(PackedModule):
    def __init__(self, **config):
        self.config = _Cfg({**SD2_VAE, **config})
        self.dtype = torch.bfloat16

    def param_shapes(self):
        return vae_param_shapes(self.config)

    # ------------------------------------------------------------------------------------------------------------------
    def _pack_weights(self):
        sd, dev, cfg = self._sd, self.device, self.config
        g = lambda k: sd[k].to(dev, torch.float32)
        P = {}
        ch, L, cz = cfg.block_out_channels, cfg.layers_per_block, cfg.latent_channels
        self.fuse_up = os.environ.get("LADI_UP2X", "1") != "0"

        def conv(p, ci):
            P[p + ".w"], P[p + ".b"] = pack_conv(g(p + ".weight"), [ci]), f32(g(p + ".bias"))

        def norm(p):
            P[p] = (f32(g(p + ".weight")), f32(g(p + ".bias")))

        def resnet(p, ci, co):
            norm(p + ".norm1"); norm(p + ".norm2")
            P[p + ".w1"], P[p + ".b1"] = pack_conv(g(p + ".conv1.weight"), [ci]), f32(g(p + ".conv1.bias"))
            if ci != co:
                P[p + ".w2"] = pack_conv(g(p + ".conv2.weight"), [co], g(p + ".conv_shortcut.weight"), [ci])
                P[p + ".b2"] = f32(g(p + ".conv2.bias") + g(p + ".conv_shortcut.bias"))
            else:
                P[p + ".w2"], P[p + ".b2"] = pack_conv(g(p + ".conv2.weight"), [co]), f32(g(p + ".conv2.bias"))

        def mid(p, c):
            resnet(p + ".resnets.0", c, c); resnet(p + ".resnets.1", c, c)
            a = p + ".attentions.0"
            norm(a + ".group_norm")
            P[a + ".qkv.w"] = pack_linear(torch.cat([g(a + ".query.weight"), g(a + ".key.weight"), g(a + ".value.weight")]))
            P[a + ".qkv.b"] = f32(torch.cat([g(a + ".query.bias"), g(a + ".key.bias"), g(a + ".value.bias")]))
            P[a + ".o.w"], P[a + ".o.b"] = pack_linear(g(a + ".proj_attn.weight")), f32(g(a + ".proj_attn.bias"))

        conv("encoder.conv_in", cfg.in_channels)
        out = ch[0]
        for i, c in enumerate(ch):
            prev, out = out, c
            for l in range(L):
                resnet(f"encoder.down_blocks.{i}.resnets.{l}", prev if l == 0 else out, out)
            if i < len(ch) - 1:
                conv(f"encoder.down_blocks.{i}.downsamplers.0.conv", out)
        mid("encoder.mid_block", ch[-1]); norm("encoder.conv_norm_out")
        # fold quant_conv (1x1, 2cz->2cz) into encoder.conv_out: W' = Wq . Wco, b' = Wq . bco + bq  (fp32 algebra)
        wq = g("quant_conv.weight")[:, :, 0, 0]
        wco, bco = g("encoder.conv_out.weight"), g("encoder.conv_out.bias")
        P["enc_out.w"] = pack_conv(torch.einsum("om,mikl->oikl", wq, wco), [ch[-1]])
        P["enc_out.b"] = f32(wq @ bco + g("quant_conv.bias"))
        rch = list(reversed(ch))
        P["post_quant.w"], P["post_quant.b"] = pack_linear(g("post_quant_conv.weight")[:, :, 0, 0]), f32(g("post_quant_conv.bias"))
        conv("decoder.conv_in", cz); mid("decoder.mid_block", rch[0])
        out = rch[0]
        for i, c in enumerate(rch):
            prev, out = out, c
            for l in range(L + 1):
                resnet(f"decoder.up_blocks.{i}.resnets.{l}", prev if l == 0 else out, out)
            if i < len(ch) - 1:
                p = f"decoder.up_blocks.{i}.upsamplers.0.conv"
                if self.fuse_up:
                    P[p + ".w"], P[p + ".b"] = pack_conv_up2x(g(p + ".weight"), [out]), f32(g(p + ".bias"))
                else:
                    conv(p, out)
        norm("decoder.conv_norm_out"); conv("decoder.conv_out", ch[0])
        self.P = P
        self.ws = ops.GroupNormWS(dev)

    def _make_engine(self):
        return eng.Engine(eng.flatten(self.P), **self.engine_config())

    def engine_config(self):
        cfg = self.config
        return dict(vae_channels=cfg.block_out_channels, vae_layers_per_block=cfg.layers_per_block, vae_latent_channels=cfg.latent_channels,
                    vae_in_channels=cfg.in_channels, vae_out_channels=cfg.out_channels, norm_groups=cfg.norm_num_groups,
                    fuse_upsample=int(self.fuse_up), emasc_scales=5)

    # ------------------------------------------------------------------------------------------------------------------
    def _resnet(self, p, x, co):
        P, g = self.P, self.config.norm_num_groups
        hn = ops.groupnorm([x], *P[p + ".norm1"], g, 1e-6, self.ws, silu=True)
        h = ops.conv2d([hn], P[p + ".w1"], co, bias=P[p + ".b1"])
        hn2 = ops.groupnorm([h], *P[p + ".norm2"], g, 1e-6, self.ws, silu=True)
        if x.shape[3] != co:
            return ops.conv2d([hn2], P[p + ".w2"], co, bias=P[p + ".b2"], shortcut=[x])
        return ops.conv2d([hn2], P[p + ".w2"], co, bias=P[p + ".b2"], residual=x)

    def _attn(self, a, x):
        """Single-head d=C spatial attention (diffusers 0.14 AttentionBlock, Appendix A.5; src/models/vae.py:81-90,142-150): GroupNorm ->
        one fused Q|K|V GEMM -> the flash kernel for a 512-wide head over the whole batch in ONE launch (the N x N score matrix is never
        written; the reference's baddbmm + softmax + bmm materialises it per sample) -> proj_attn GEMM with the residual in its epilogue."""
        P = self.P
        B, h, w, C = x.shape
        N = h * w
        if C not in (256, 512):
            raise NotImplementedError(f"VAE mid-block attention is built for C = 512 (256 for reduced-width test models), got {C}")
        hn = ops.groupnorm([x], *P[a + ".group_norm"], self.config.norm_num_groups, 1e-6, self.ws, silu=False)
        qkv = ops.gemm(hn.view(B * N, C), P[a + ".qkv.w"], 3 * C, bias=P[a + ".qkv.b"]).view(B, N, 3 * C)
        o = ops.attention_d512(qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:], C ** -0.5)
        return ops.gemm(o.view(B * N, C), P[a + ".o.w"], C, bias=P[a + ".o.b"], residual=x.view(B * N, C)).view(B, h, w, C)

    def _mid(self, p, x):
        c = x.shape[3]
        x = self._resnet(p + ".resnets.0", x, c)
        x = self._attn(p + ".attentions.0", x)
        return self._resnet(p + ".resnets.1", x, c)

    def encode_nhwc(self, x, nhwc=False):
        """x NCHW fp32 [B,3,H,W] (or, with nhwc=True, an already packed NHWC bf16 [B,H,W,8] buffer)
        -> (moments NHWC fp32 [B,h,w,2cz], skips[6] NHWC bf16 (entry 0 = the input itself))."""
        P, cfg = self.P, self.config
        ch, L = cfg.block_out_channels, cfg.layers_per_block
        cin = cfg.in_channels
        if nhwc:
            xin = x
            B, H, W, _ = x.shape
        else:
            B, _, H, W = x.shape
            xin = torch.zeros((B, H, W, 8), dtype=torch.bfloat16, device=self.device)
            ops.nchw_to_nhwc(x.to(self.device, torch.float32).contiguous(), xin)
        if self.use_engine():  # one ABI call (csrc/engine.cu vae_encode); the retained features are written into caller buffers
            mk = lambda c, f: torch.empty((B, H // f, W // f, c), dtype=torch.bfloat16, device=self.device)
            f1, f3, f4, f5 = mk(ch[0], 1), mk(ch[0], 2), mk(ch[1], 4), mk(ch[2], 8)
            mom = torch.empty((B, H // 8, W // 8, 2 * cfg.latent_channels), dtype=torch.float32, device=self.device)
            ws = self.engine.workspace(eng.MODULE_VAE_ENCODE, B, H, W)
            lib.call("ladi_vae_encode", self.engine.h, ops._ptr(xin), B, H, W, ops._ptr(mom), eng.ptr_array([None, f1, f1, f3, f4, f5]), ops._ptr(ws),
                     ws.numel(), ops._stream())
            return mom, [xin[..., :cin], f1, f1, f3, f4, f5]
        h = ops.conv2d([xin[..., :cin]], P["encoder.conv_in.w"], ch[0], bias=P["encoder.conv_in.b"])
        feats = [xin[..., :cin], h]
        for i, c in enumerate(ch):
            feats.append(h)
            for l in range(L):
                h = self._resnet(f"encoder.down_blocks.{i}.resnets.{l}", h, c)
            if i < len(ch) - 1:
                p = f"encoder.down_blocks.{i}.downsamplers.0.conv"
                h = ops.conv2d([h], P[p + ".w"], c, bias=P[p + ".b"], stride=2, pad_lo=0)
        h = self._mid("encoder.mid_block", h)
        hn = ops.groupnorm([h], *P["encoder.conv_norm_out"], cfg.norm_num_groups, 1e-6, self.ws, silu=True)
        mom = torch.empty((B, h.shape[1], h.shape[2], 2 * cfg.latent_channels), dtype=torch.float32, device=self.device)
        ops.conv2d([hn], P["enc_out.w"], 2 * cfg.latent_channels, bias=P["enc_out.b"], out=mom, out_fp32=True)
        return mom, feats

    def encode(self, x, return_dict=True):
        """AutoencoderKL.py:145-157: returns (object with .latent_dist, intermediate_features)."""
        mom, feats = self.encode_nhwc(x)
        return _Enc(DiagonalGaussianDistribution(mom, self.config.latent_channels)), feats

    def decode_nhwc(self, z, feats=None, int_layers=None, scale=1.0):
        """z NCHW fp32 [B,cz,h,w], multiplied by `scale` on load (the 1/scaling_factor of tryon_pipe.py:350); feats = EMASC outputs NHWC bf16 in the reference's
        list order (ascending resolution index, vae.py reverses it) -> image NHWC fp32 [B,H,W,4] (first 3 channels)."""
        P, cfg = self.P, self.config
        ch, L, cz = cfg.block_out_channels, cfg.layers_per_block, cfg.latent_channels
        rch = list(reversed(ch))
        B, _, h, w = z.shape
        zin = torch.zeros((B, h, w, 8), dtype=torch.bfloat16, device=self.device)
        ops.nchw_to_nhwc(z.to(self.device, torch.float32).contiguous(), zin, scale=scale)
        if self.use_engine():  # one ABI call (csrc/engine.cu vae_decode)
            img = torch.empty((B, 8 * h, 8 * w, 4), dtype=torch.float32, device=self.device)
            fl = list(feats) if feats else []
            lay = [int(i) for i in (int_layers or [])][:len(fl)]
            if fl and len(lay) != len(fl):
                raise ValueError("`int_layers` must name the encoder layer of every intermediate feature")
            want_c = {0: cfg.out_channels, 1: ch[0], 2: ch[1], 3: ch[2], 4: ch[3], 5: ch[3]}  # EMASC output widths per encoder layer (hubconf.py:41-42)
            want_f = {0: 1, 1: 1, 2: 1, 3: 2, 4: 4, 5: 8}
            for t, i in zip(fl, lay):
                if i not in want_c or tuple(t.shape) != (B, 8 * h // want_f[i], 8 * w // want_f[i], want_c[i]):
                    raise ValueError(f"intermediate feature of layer {i}: expected NHWC {(B, 8 * h // want_f.get(i, 1), 8 * w // want_f.get(i, 1), want_c.get(i))}, got {tuple(t.shape)}")
                assert t.dtype == torch.bfloat16 and t.stride(3) == 1 and t.stride(2) == (t.shape[3] + 7) // 8 * 8, "EMASC features: dense NHWC bf16 (pitch = channels rounded up to 8)"
            layers = (C.c_int * max(1, len(fl)))(*lay)
            ws = self.engine.workspace(eng.MODULE_VAE_DECODE, B, h, w)
            lib.call("ladi_vae_decode_emasc", self.engine.h, ops._ptr(zin), B, h, w, eng.ptr_array(fl, max(1, len(fl))), len(fl), layers, ops._ptr(img),
                     ops._ptr(ws), ws.numel(), ops._stream())
            return img
        zq = torch.zeros((B, h, w, 8), dtype=torch.bfloat16, device=self.device)
        ops.gemm(zin.view(B * h * w, 8)[:, :cz], P["post_quant.w"], cz, bias=P["post_quant.b"], out=zq.view(B * h * w, 8))
        x = ops.conv2d([zq[..., :cz]], P["decoder.conv_in.w"], rch[0], bias=P["decoder.conv_in.b"])
        x = self._mid("decoder.mid_block", x)
        rf = list(reversed(feats)) if feats else None  # vae.py:190
        for i, c in enumerate(rch):
            if rf is not None and i < len(rf):
                x = ops.add(x, rf[i])  # vae.py:193 `sample += int_feat`
            for l in range(L + 1):
                x = self._resnet(f"decoder.up_blocks.{i}.resnets.{l}", x, c)
            if i < len(ch) - 1:
                p = f"decoder.up_blocks.{i}.upsamplers.0.conv"
                x = (ops.conv2d([x], P[p + ".w"], c, bias=P[p + ".b"], up2x=True) if self.fuse_up
                     else ops.conv2d([ops.upsample2x(x)], P[p + ".w"], c, bias=P[p + ".b"]))
        last = None
        if rf is not None and int_layers and 1 in int_layers:  # vae.py:204-205, added AFTER norm + SiLU
            last = rf[len(int_layers) - 1 - int_layers.index(1)]
        hn = ops.groupnorm([x], *P["decoder.conv_norm_out"], cfg.norm_num_groups, 1e-6, self.ws, silu=True, add=last)
        img = torch.empty((B, x.shape[1], x.shape[2], 4), dtype=torch.float32, device=self.device)
        res0 = None
        if rf is not None and int_layers and 0 in int_layers:  # vae.py:209-210: image-space skip added AFTER conv_out (residual epilogue)
            res0 = rf[len(int_layers) - 1 - int_layers.index(0)][..., :cfg.out_channels]
        ops.conv2d([hn], P["decoder.conv_out.w"], cfg.out_channels, bias=P["decoder.conv_out.b"], out=img, out_fp32=True, residual=res0)
        return img

    def decode(self, z, intermediate_features=None, int_layers=None, return_dict=True):
        """AutoencoderKL.py:174-188 -> object with .sample NCHW fp32."""
        img = self.decode_nhwc(z, intermediate_features, int_layers)
        return _Dec(ops.nhwc_to_nchw(img, self.config.out_channels))


class EMASC(PackedModule):
    """emasc.py:11-40: per scale either the nonlinear form Conv(k) -> SiLU -> Conv(k) (state-dict keys conv.{i}.{0,2}.{weight,bias}; the
    hub checkpoints are k = 3) or the linear form, one Conv3x3 (keys conv.{i}.{weight,bias}; the reference's linear EMASC always builds a
    3x3 kernel and ignores `kernel_size`, emasc.py:21-24).  `mask_features` is folded into the last conv's epilogue."""

    def __init__(self, in_channels, out_channels, kernel_size=3, padding=1, stride=1, type="nonlinear"):
        if type not in ("linear", "nonlinear"):
            raise NotImplementedError(f"EMASC type {type} is not implemented.")
        k = 3 if type == "linear" else int(kernel_size)
        if stride != 1 or k % 2 == 0 or padding != (k - 1) // 2:
            raise NotImplementedError(
                f"EMASC with kernel {k}, padding {padding}, stride {stride} is not built: the output must keep the feature's resolution "
                "(a 'same' convolution), otherwise the decoder's skip add `sample += int_feat` (src/models/vae.py:193) fails in the "
                "reference itself")
        if k not in (1, 3):
            raise NotImplementedError(
                f"EMASC with a {k}x{k} kernel is not built: {k * k} taps exceed the 24 K segments (MAX_SEG) of the convolution kernel "
                "(csrc/convgemm.cu); only 3x3 and 1x1 EMASC run on it")
        self.type, self.kernel_size, self.padding = type, k, padding
        self.in_channels, self.out_channels = list(in_channels), list(out_channels)

    def param_shapes(self):
        from .synthetic import emasc_param_shapes
        return emasc_param_shapes(self.in_channels, self.out_channels, self.kernel_size, self.type)

    def _pack_weights(self):
        g = lambda k: self._sd[k].to(self.device, torch.float32)
        self.P = []
        for i, ci in enumerate(self.in_channels):
            if self.type == "linear":  # (w, b)
                self.P.append((pack_conv(g(f"conv.{i}.weight"), [ci]), f32(g(f"conv.{i}.bias"))))
            else:  # (w1, b1, w2, b2)
                self.P.append((pack_conv(g(f"conv.{i}.0.weight"), [ci]), f32(g(f"conv.{i}.0.bias")),
                               pack_conv(g(f"conv.{i}.2.weight"), [ci]), f32(g(f"conv.{i}.2.bias"))))

    def _make_engine(self):
        self._engine_weights = self.engine_weights()
        return {}  # one handle per resolution pyramid (the strides are part of the handle's config), built on first use

    def engine_weights(self):
        """Weight table of ladi_emasc_forward: emasc.<i>.w1/b1 (+ w2/b2 for the nonlinear form; the engine reads the form and the kernel
        size from the table, include/ladi_b200.h)."""
        W = {}
        for i, t in enumerate(self.P):
            for name, v in zip(("w1", "b1", "w2", "b2"), t):
                W[f"emasc.{i}.{name}"] = v
        return W

    def _engine_for(self, feats):
        H, Wd = feats[0].shape[1], feats[0].shape[2]
        strides = tuple(H // f.shape[1] for f in feats)
        e = self.engine.get(strides)
        if e is None:
            e = self.engine[strides] = eng.Engine(self._engine_weights, emasc_scales=len(feats), emasc_in=self.in_channels, emasc_out=self.out_channels,
                                                  emasc_stride=strides)
        return e, H, Wd

    def __call__(self, feats, inv_masks=None):
        """feats: list of NHWC bf16 tensors; inv_masks: optional list of fp32 (1-mask) rows per scale => mask_features fused."""
        if self.use_engine() and len(feats) == len(self.P):
            e, H, Wd = self._engine_for(feats)  # one ABI call (csrc/engine.cu emasc_forward)
            B = feats[0].shape[0]
            outs = []
            for f, co in zip(feats, self.out_channels):
                assert f.dtype == torch.bfloat16 and f.stride(3) == 1 and f.stride(2) == (f.shape[3] + 7) // 8 * 8 and H % f.shape[1] == 0
                outs.append(torch.empty((B, f.shape[1], f.shape[2], (co + 7) // 8 * 8), dtype=torch.bfloat16, device=self.device)[..., :co])
            ws = e.workspace(eng.MODULE_EMASC, B, H, Wd)
            inv = eng.ptr_array(inv_masks) if inv_masks is not None else None
            lib.call("ladi_emasc_forward", e.h, eng.ptr_array(feats), inv, B, H, Wd, eng.ptr_array(outs), ops._ptr(ws), ws.numel(), ops._stream())
            return outs
        out = []
        k, p = self.kernel_size, self.padding
        for i, f in enumerate(feats):
            rs = None if inv_masks is None else inv_masks[i]
            if self.type == "linear":
                w, b = self.P[i]
                out.append(ops.conv2d([f], w, self.out_channels[i], ksize=k, pad_lo=p, bias=b, row_scale=rs))
                continue
            w1, b1, w2, b2 = self.P[i]
            t = ops.conv2d([f], w1, self.in_channels[i], ksize=k, pad_lo=p, bias=b1, act=ops.ACT_SILU)
            out.append(ops.conv2d([t], w2, self.out_channels[i], ksize=k, pad_lo=p, bias=b2, row_scale=rs))
        return out
