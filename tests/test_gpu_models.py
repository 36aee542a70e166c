"""GPU parity of the assembled models and of the whole try-on pipeline against the fp32 CPU oracle (oracle/ladi_oracle),
same seeded weights and inputs.  The engine computes in bf16 (fp32 accumulate, fp32 latents/scheduler); the stated
tolerances are on the relative L2 error  |y - ref|_2 / |ref|_2 :
    single UNet forward        <= 2e-2      VAE moments / encoder skips  <= 2e-2
    EMASC features             <= 1.5e-2    final image (few DDIM steps) mean |diff| <= 2/255 (small config)
    VAE decode (30 convs deep, small-magnitude output): <= 1.5 x the error of the SAME oracle module executed in bf16 by
    stock PyTorch library kernels on the GPU ("what a straight port would get", SURVEY.md section 8(c) second tier), cap 5e-2.
Two engine runs with the same seed must be bit-identical (no floating-point atomics anywhere on the path).
"""
import numpy as np
import pytest
import torch

from kernel_check import rel_l2

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def small(cuda):
    from ladi_vton_b200 import synthetic as S
    from ladi_oracle.unet import UNet2DConditionModel as OU
    from ladi_oracle.vae import AutoencoderKL as OV
    from ladi_oracle.parts import EMASC as OE
    pipe, sds = S.build_pipeline(cuda, S.SMALL_UNET, S.SMALL_VAE)
    ou = OU(**S.SMALL_UNET).eval(); ou.load_state_dict(sds["unet"])
    ov = OV(**S.SMALL_VAE).eval(); ov.load_state_dict(sds["vae"])
    oe = OE(*sds["emasc_channels"]).eval(); oe.load_state_dict(sds["emasc"])
    return pipe, ou, ov, oe


def test_unet_small_forward(cuda, small):
    pipe, ou, _, _ = small
    g = torch.Generator().manual_seed(0)
    x = torch.randn((2, 31, 16, 8), generator=g)
    ctx = torch.randn((2, 77, 128), generator=g)
    with torch.no_grad():
        ref = ou(x, torch.tensor(981), ctx).sample
    y = pipe.unet(x.to(cuda), torch.tensor(981), ctx.to(cuda)).sample
    assert y.shape == ref.shape
    assert rel_l2(y, ref) < 2e-2


def test_vae_emasc_small(cuda, small):
    pipe, _, ov, oe = small
    g = torch.Generator().manual_seed(1)
    x = torch.rand((2, 3, 128, 64), generator=g) * 2 - 1
    with torch.no_grad():
        enc, feats = ov.encode(x)
        ref_m = enc.latent_dist.parameters
    mom, f = pipe.vae.encode_nhwc(x.to(cuda))
    assert rel_l2(mom.permute(0, 3, 1, 2), ref_m) < 2e-2
    for i in (1, 3, 4, 5):
        assert rel_l2(f[i].permute(0, 3, 1, 2), feats[i]) < 2e-2
    # EMASC + mask_features + decode with the skips
    from ladi_oracle.parts import mask_features
    mask = torch.zeros((2, 1, 128, 64)); mask[:, :, 30:100, 10:50] = 1
    with torch.no_grad():
        inter_ref = mask_features(oe([feats[i] for i in range(1, 6)]), mask)
        z = torch.randn((2, 4, 16, 8), generator=g)
        img_ref = ov.decode(z, list(inter_ref), [1, 2, 3, 4, 5]).sample
    from ladi_vton_b200 import ops
    md = mask.to(cuda)
    sel = [f[i] for i in range(1, 6)]
    inter = pipe.emasc(sel, [ops.inv_mask_rows(md, 128 // t.shape[1]) for t in sel])
    for a, b in zip(inter, inter_ref):
        assert rel_l2(a.permute(0, 3, 1, 2), b) < 1.5e-2
    img = pipe.vae.decode(z.to(cuda), inter, [1, 2, 3, 4, 5]).sample
    import copy
    ov_bf = copy.deepcopy(ov).to(cuda).bfloat16()
    with torch.no_grad():
        port = ov_bf.decode(z.to(cuda).bfloat16(), [t.to(cuda).bfloat16() for t in inter_ref], [1, 2, 3, 4, 5]).sample
    e_port, e_engine = rel_l2(port, img_ref), rel_l2(img, img_ref)
    print(f"VAE decode rel-L2 vs fp32 oracle: engine {e_engine:.4f}, bf16 library port {e_port:.4f}")
    assert e_engine < min(5e-2, 1.5 * e_port)


@pytest.mark.parametrize("gs,graph", [(7.5, True), (1.0, True), (7.5, False)])
def test_pipeline_small(cuda, small, gs, graph):
    from ladi_vton_b200 import synthetic as S
    from ladi_oracle.parts import DDIMScheduler
    from ladi_oracle.pipeline import OracleTryOnPipeline
    pipe, ou, ov, oe = small
    inp = S.synthetic_inputs(2, 128, 64, ctx_dim=128)
    op = OracleTryOnPipeline(ov, ou, DDIMScheduler(), oe, [1, 2, 3, 4, 5])
    ref = op(inp["image"].clone(), inp["mask_image"].clone(), inp["pose_map"], inp["warped_cloth"], inp["prompt_embeds"],
             inp["negative_prompt_embeds"], height=128, width=64, num_inference_steps=5, guidance_scale=gs,
             generator=torch.Generator().manual_seed(7))
    pipe.use_cuda_graph = graph
    out = pipe(image=inp["image"].clone(), mask_image=inp["mask_image"].clone(), pose_map=inp["pose_map"],
               warped_cloth=inp["warped_cloth"], prompt_embeds=inp["prompt_embeds"],
               negative_prompt_embeds=inp["negative_prompt_embeds"], height=128, width=64, num_inference_steps=5,
               guidance_scale=gs, generator=torch.Generator().manual_seed(7), output_type="np").images
    assert out.shape == ref.shape == (2, 128, 64, 3)
    assert np.abs(out - ref).mean() < 2.0 / 255
    print(f"pipeline gs={gs} graph={graph}: mean|engine-oracle| = {np.abs(out - ref).mean() * 255:.3f}/255")
    # second call re-uses the captured graph and must reproduce the first bit-for-bit
    out2 = pipe(image=inp["image"].clone(), mask_image=inp["mask_image"].clone(), pose_map=inp["pose_map"],
                warped_cloth=inp["warped_cloth"], prompt_embeds=inp["prompt_embeds"],
                negative_prompt_embeds=inp["negative_prompt_embeds"], height=128, width=64, num_inference_steps=5,
                guidance_scale=gs, generator=torch.Generator().manual_seed(7), output_type="np").images
    assert np.array_equal(out2, out)


def test_pipeline_errors(cuda, small):
    from ladi_vton_b200 import synthetic as S
    pipe = small[0]
    inp = S.synthetic_inputs(1, 128, 64, ctx_dim=128)
    kw = dict(image=inp["image"], mask_image=inp["mask_image"], pose_map=inp["pose_map"], warped_cloth=inp["warped_cloth"])
    with pytest.raises(ValueError, match="divisible by 8"):
        pipe(**kw, prompt_embeds=inp["prompt_embeds"], height=100, width=64)
    with pytest.raises(ValueError, match="Provide either"):
        pipe(**kw, height=128, width=64)
    with pytest.raises(ValueError, match="range"):
        pipe(**{**kw, "image": inp["image"] * 3}, prompt_embeds=inp["prompt_embeds"], negative_prompt_embeds=inp["negative_prompt_embeds"],
             height=128, width=64)
    with pytest.raises(ValueError, match="cloth_input_type"):
        pipe(**kw, prompt_embeds=inp["prompt_embeds"], negative_prompt_embeds=inp["negative_prompt_embeds"], height=128, width=64,
             cloth_input_type="bogus")


def test_unet_full_forward(cuda):
    """Full SD-2-inpaint 31-channel UNet (865,988,484 parameters), one forward at 64x48 latents, CFG batch 2."""
    from ladi_vton_b200 import UNet2DConditionModel, synthetic as S, unet_param_shapes
    from ladi_oracle.unet import UNet2DConditionModel as OU
    sd = S.random_state_dict(unet_param_shapes({}), 1234)
    ou = OU().eval(); ou.load_state_dict(sd)
    g = torch.Generator().manual_seed(0)
    x = torch.randn((2, 31, 64, 48), generator=g)
    ctx = torch.randn((2, 77, 1024), generator=g)
    with torch.no_grad():
        ref = ou(x, torch.tensor(501), ctx).sample
    unet = UNet2DConditionModel().load_state_dict(sd).to(cuda)
    y = unet(x.to(cuda), torch.tensor(501), ctx.to(cuda)).sample
    err = rel_l2(y, ref)
    print("full UNet forward rel-L2 vs fp32 oracle:", err)
    assert err < 2e-2


def test_inversion_adapter_full(cuda):
    """hubconf.py:16-27 dims (136,360,704 parameters): CLIP ViT-H features [B,257,1280] -> 16 pseudo-word tokens [B,16384]."""
    from ladi_vton_b200 import InversionAdapter, synthetic as S
    from ladi_oracle.parts import InversionAdapter as OA
    eng = InversionAdapter()
    sd = S.random_state_dict(eng.param_shapes(), 4321)
    oa = OA().eval(); oa.load_state_dict(sd)
    x = torch.randn((3, 257, 1280), generator=torch.Generator().manual_seed(5))
    with torch.no_grad():
        ref = oa(x)
    y = eng.load_state_dict(sd).to(cuda)(x)
    assert y.shape == ref.shape == (3, 16384)
    err = rel_l2(y, ref)
    print("inversion adapter rel-L2 vs fp32 oracle:", err)
    assert err < 2e-2


@pytest.mark.parametrize("opts", [dict(no_pose=True), dict(cloth_cond_rate=0.4), dict(batch=1, guidance_scale=7.5), dict(latents=True),
                                  dict(callback=True), dict(num_inference_steps=1)])
def test_pipeline_options_small(cuda, small, opts):
    """Less-travelled arguments of `__call__` (tryon_pipe.py:495-520): no_pose, cloth_cond_rate < 1 (cloth latents zeroed for the
    last steps, :718-719), batch 1, caller-supplied latents, per-step callback (disables graph replay), a single step."""
    from ladi_vton_b200 import synthetic as S
    from ladi_oracle.parts import DDIMScheduler
    from ladi_oracle.pipeline import OracleTryOnPipeline
    pipe, ou, ov, oe = small
    opts = dict(opts)
    B = opts.pop("batch", 2)
    steps = opts.pop("num_inference_steps", 5)
    gs = opts.pop("guidance_scale", 7.5)
    inp = S.synthetic_inputs(B, 128, 64, ctx_dim=128)
    kw = {k: v for k, v in opts.items() if k in ("no_pose", "cloth_cond_rate")}
    lat = torch.randn((B, 4, 16, 8), generator=torch.Generator().manual_seed(3)) if opts.get("latents") else None
    op = OracleTryOnPipeline(ov, ou, DDIMScheduler(), oe, [1, 2, 3, 4, 5])
    ref = op(inp["image"].clone(), inp["mask_image"].clone(), inp["pose_map"], inp["warped_cloth"], inp["prompt_embeds"],
             inp["negative_prompt_embeds"], height=128, width=64, num_inference_steps=steps, guidance_scale=gs,
             generator=torch.Generator().manual_seed(7), latents=None if lat is None else lat.clone(), **kw)
    seen = []
    cb = (lambda i, t, l: seen.append((i, int(t), tuple(l.shape)))) if opts.get("callback") else None
    pipe.use_cuda_graph = True
    out = pipe(image=inp["image"].clone(), mask_image=inp["mask_image"].clone(), pose_map=inp["pose_map"], warped_cloth=inp["warped_cloth"],
               prompt_embeds=inp["prompt_embeds"], negative_prompt_embeds=inp["negative_prompt_embeds"], height=128, width=64,
               num_inference_steps=steps, guidance_scale=gs, generator=torch.Generator().manual_seed(7), output_type="np",
               latents=lat, callback=cb, **kw).images
    assert out.shape == ref.shape
    mad = np.abs(out - ref).mean() * 255
    print(f"pipeline options {opts or dict(batch=B, steps=steps)}: mean|engine-oracle| = {mad:.3f}/255")
    assert mad < 2.0
    if cb is not None:
        assert [s[0] for s in seen] == list(range(steps)) and seen[0][1] == 801 and seen[0][2] == (B, 4, 16, 8)


def test_pipeline_pil_output_and_tuple(cuda, small):
    from ladi_vton_b200 import synthetic as S
    pipe = small[0]
    inp = S.synthetic_inputs(1, 128, 64, ctx_dim=128)
    res = pipe(image=inp["image"], mask_image=inp["mask_image"], pose_map=inp["pose_map"], warped_cloth=inp["warped_cloth"],
               prompt_embeds=inp["prompt_embeds"], negative_prompt_embeds=inp["negative_prompt_embeds"], height=128, width=64,
               num_inference_steps=2, generator=torch.Generator().manual_seed(7), return_dict=False)
    imgs, nsfw = res
    assert nsfw is None and len(imgs) == 1 and imgs[0].size == (64, 128) and imgs[0].mode == "RGB"  # PIL (W, H), tryon_pipe.py:759-765


def test_pipeline_full_size_config0(cuda):
    """BASELINE.json configs[0]: a single 512x384 pair, 20 DDIM steps, full-size random-init UNet/VAE/EMASC, guidance 7.5 -- the whole
    `__call__` against the fp32 CPU oracle with identical weights, inputs and noise.  Random weights + CFG 7.5 make the 20-step map
    chaotic, gate: mean |diff| <= 2/255 (measured 0.55/255, PSNR 51 dB)."""
    import ctypes
    try:  # same allocator tuning as bench.py: the fp32 oracle otherwise spends most of its time in page faults
        libc = ctypes.CDLL("libc.so.6"); libc.mallopt(-3, 1 << 30); libc.mallopt(-1, 1 << 31)
    except Exception:
        pass
    import os
    from ladi_vton_b200 import synthetic as S
    from ladi_oracle.parts import DDIMScheduler, EMASC as OE
    from ladi_oracle.pipeline import OracleTryOnPipeline
    from ladi_oracle.unet import UNet2DConditionModel as OU
    from ladi_oracle.vae import AutoencoderKL as OV
    torch.set_num_threads(min(64, os.cpu_count()))
    sds = S.build_state_dicts(seed=1234)
    with torch.device("meta"):
        ou, ov, oe = OU().eval(), OV().eval(), OE(*sds["emasc_channels"]).eval()
    ou.load_state_dict(sds["unet"], assign=True); ov.load_state_dict(sds["vae"], assign=True); oe.load_state_dict(sds["emasc"], assign=True)
    inp = S.synthetic_inputs(1, 512, 384)
    kw = dict(height=512, width=384, num_inference_steps=20, guidance_scale=7.5)
    ref = OracleTryOnPipeline(ov, ou, DDIMScheduler(), oe, [1, 2, 3, 4, 5])(
        inp["image"].clone(), inp["mask_image"].clone(), inp["pose_map"], inp["warped_cloth"], inp["prompt_embeds"],
        inp["negative_prompt_embeds"], generator=torch.Generator().manual_seed(7), **kw)
    del ou, ov, oe
    pipe, _ = S.build_pipeline(cuda, sds=sds)
    out = pipe(image=inp["image"].clone(), mask_image=inp["mask_image"].clone(), pose_map=inp["pose_map"], warped_cloth=inp["warped_cloth"],
               prompt_embeds=inp["prompt_embeds"], negative_prompt_embeds=inp["negative_prompt_embeds"],
               generator=torch.Generator().manual_seed(7), output_type="np", **kw).images
    mad = float(np.abs(out - ref).mean()) * 255
    psnr = float(10 * np.log10(1.0 / np.mean((out - ref) ** 2)))
    print(f"full-size config0 (1x512x384, 20 steps, CFG 7.5): mean|engine-oracle| = {mad:.3f}/255, PSNR {psnr:.1f} dB")
    assert out.shape == ref.shape == (1, 512, 384, 3)
    assert mad < 2.0


# ------------------------------------------------------------------------------------------------ round 2: the configs the bench runs
def _full_oracle(sds, unet=True, vae=True, emasc=True):
    import ctypes
    import os
    try:
        libc = ctypes.CDLL("libc.so.6"); libc.mallopt(-3, 1 << 30); libc.mallopt(-1, 1 << 31)
    except Exception:
        pass
    from ladi_oracle.parts import EMASC as OE
    from ladi_oracle.unet import UNet2DConditionModel as OU
    from ladi_oracle.vae import AutoencoderKL as OV
    torch.set_num_threads(min(64, os.cpu_count()))
    out = []
    with torch.device("meta"):
        mods = [OU().eval() if unet else None, OV().eval() if vae else None, OE(*sds["emasc_channels"]).eval() if emasc else None]
    for m, k in zip(mods, ("unet", "vae", "emasc")):
        if m is not None:
            m.load_state_dict(sds[k], assign=True)
        out.append(m)
    return out


def test_unet_full_forward_batch16(cuda):
    """The UNet batch bench.py runs (BASELINE configs[1]: 8 images with CFG = UNet batch 16): at this M the conv/GEMM picks other N
    tiles, CTA pairs and split-K factors than at batch 2 (csrc/convgemm.cu tile selection), so it gets its own oracle comparison.
    16 distinct samples; gate as for the batch-2 test (rel-L2 <= 2e-2 per sample and overall)."""
    from ladi_vton_b200 import UNet2DConditionModel, synthetic as S, unet_param_shapes
    sd = S.random_state_dict(unet_param_shapes({}), 1234)
    ou, _, _ = _full_oracle(dict(unet=sd), vae=False, emasc=False)
    g = torch.Generator().manual_seed(0)
    x = torch.randn((16, 31, 64, 48), generator=g)
    ctx = torch.randn((16, 77, 1024), generator=g)
    with torch.no_grad():
        ref = torch.cat([ou(x[i:i + 4], torch.tensor(501), ctx[i:i + 4]).sample for i in range(0, 16, 4)])
    del ou
    unet = UNet2DConditionModel().load_state_dict(sd).to(cuda)
    y = unet(x.to(cuda), torch.tensor(501), ctx.to(cuda)).sample
    err = rel_l2(y, ref)
    worst = max(rel_l2(y[i], ref[i]) for i in range(16))
    print(f"full UNet forward, batch 16: rel-L2 vs fp32 oracle {err:.4f}, worst sample {worst:.4f}")
    assert err < 2e-2 and worst < 2.5e-2


def test_vae_emasc_1024x768(cuda):
    """BASELINE configs[3] resolution: VAE encode (moments + skips), EMASC + mask_features and decode at 1024x768 -- the 12288-token
    mid-block attention (the flash kernel for the 512-wide head; the reference materialises a 604 MB fp32 score matrix per sample here,
    src/models/vae.py:81-90) and the full-resolution 128-channel convolutions.  Same gates as test_vae_emasc_small."""
    import copy
    from ladi_vton_b200 import ops, synthetic as S
    from ladi_oracle.parts import mask_features
    sds = S.build_state_dicts(seed=1234)
    _, ov, oe = _full_oracle(sds, unet=False)
    pipe_vae = __import__("ladi_vton_b200").AutoencoderKL().load_state_dict(sds["vae"]).to(cuda)
    emasc = __import__("ladi_vton_b200").EMASC(*sds["emasc_channels"]).load_state_dict(sds["emasc"]).to(cuda)
    g = torch.Generator().manual_seed(1)
    H, W = 1024, 768
    x = torch.rand((1, 3, H, W), generator=g) * 2 - 1
    mask = torch.zeros((1, 1, H, W)); mask[:, :, 200:800, 150:600] = 1
    with torch.no_grad():
        enc, feats = ov.encode(x)
        inter_ref = mask_features(oe([feats[i] for i in range(1, 6)]), mask)
        z = torch.randn((1, 4, H // 8, W // 8), generator=g)
        img_ref = ov.decode(z, list(inter_ref), [1, 2, 3, 4, 5]).sample
    mom, f = pipe_vae.encode_nhwc(x.to(cuda))
    assert rel_l2(mom.permute(0, 3, 1, 2), enc.latent_dist.parameters) < 2e-2
    for i in (1, 3, 4, 5):
        assert rel_l2(f[i].permute(0, 3, 1, 2), feats[i]) < 2e-2
    md = mask.to(cuda)
    sel = [f[i] for i in range(1, 6)]
    inter = emasc(sel, [ops.inv_mask_rows(md, H // t.shape[1]) for t in sel])
    for a, b in zip(inter, inter_ref):
        assert rel_l2(a.permute(0, 3, 1, 2), b) < 1.5e-2
    img = pipe_vae.decode(z.to(cuda), inter, [1, 2, 3, 4, 5]).sample
    ov_bf = copy.deepcopy(ov).to(cuda).bfloat16()
    with torch.no_grad():
        port = ov_bf.decode(z.to(cuda).bfloat16(), [t.to(cuda).bfloat16() for t in inter_ref], [1, 2, 3, 4, 5]).sample
    e_port, e_engine = rel_l2(port, img_ref), rel_l2(img, img_ref)
    print(f"VAE decode 1024x768 rel-L2 vs fp32 oracle: engine {e_engine:.4f}, bf16 library port {e_port:.4f}")
    assert e_engine < min(5e-2, 1.5 * e_port)


def test_pipeline_1024x768(cuda):
    """BASELINE configs[3] shape end to end: one 1024x768 pair, CFG 7.5, 3 DDIM steps, full-size random-init UNet/VAE/EMASC, against the
    fp32 CPU oracle with identical weights, inputs and noise (12288-token self-attention in the UNet and in the VAE, 128x96 latents;
    reference resolution handling tryon_pipe.py:584-585,632-634).  Gate: mean |diff| <= 2/255."""
    from ladi_vton_b200 import synthetic as S
    from ladi_oracle.parts import DDIMScheduler
    from ladi_oracle.pipeline import OracleTryOnPipeline
    sds = S.build_state_dicts(seed=1234)
    ou, ov, oe = _full_oracle(sds)
    inp = S.synthetic_inputs(1, 1024, 768)
    kw = dict(height=1024, width=768, num_inference_steps=3, guidance_scale=7.5)
    ref = OracleTryOnPipeline(ov, ou, DDIMScheduler(), oe, [1, 2, 3, 4, 5])(
        inp["image"].clone(), inp["mask_image"].clone(), inp["pose_map"], inp["warped_cloth"], inp["prompt_embeds"],
        inp["negative_prompt_embeds"], generator=torch.Generator().manual_seed(7), **kw)
    del ou, ov, oe
    pipe, _ = S.build_pipeline(cuda, sds=sds)
    call = lambda: pipe(image=inp["image"].clone(), mask_image=inp["mask_image"].clone(), pose_map=inp["pose_map"], warped_cloth=inp["warped_cloth"],
                        prompt_embeds=inp["prompt_embeds"], negative_prompt_embeds=inp["negative_prompt_embeds"],
                        generator=torch.Generator().manual_seed(7), output_type="np", **kw).images
    out = call()
    mad = float(np.abs(out - ref).mean()) * 255
    psnr = float(10 * np.log10(1.0 / np.mean((out - ref) ** 2)))
    print(f"1024x768 (1 image, 3 steps, CFG 7.5): mean|engine-oracle| = {mad:.3f}/255, PSNR {psnr:.1f} dB")
    assert out.shape == ref.shape == (1, 1024, 768, 3)
    assert mad < 2.0
    assert np.array_equal(call(), out)  # second call = the three captured graphs (pre / step / post): bit-identical


def test_train_emasc_forward_small(cuda, small):
    """The forward of src/train_emasc.py:388-403 (SURVEY.md section 2 row 15, the second parity scenario): posterior of the
    IMAGE, skips of the MASKED image, EMASC, mask_features, decode of the posterior SAMPLE (unscaled latents) with the skips."""
    from ladi_vton_b200 import ops
    from ladi_oracle.parts import mask_features
    pipe, _, ov, oe = small
    g = torch.Generator().manual_seed(11)
    image = torch.rand((2, 3, 128, 64), generator=g) * 2 - 1
    mask = torch.zeros((2, 1, 128, 64)); mask[:, :, 30:100, 10:50] = 1
    im_mask = image * (1 - mask)
    int_layers = [1, 2, 3, 4, 5]
    with torch.no_grad():
        post, _ = ov.encode(image)
        _, feats = ov.encode(im_mask)
        inter_ref = mask_features(oe([feats[i] for i in int_layers]), mask)
        lat_ref = post.latent_dist.sample(generator=torch.Generator().manual_seed(3))
        rec_ref = ov.decode(z=lat_ref, intermediate_features=list(inter_ref), int_layers=int_layers).sample
    post_e, _ = pipe.vae.encode(image.to(cuda))
    _, feats_e = pipe.vae.encode(im_mask.to(cuda))
    sel = [feats_e[i] for i in int_layers]
    inter = pipe.emasc(sel, [ops.inv_mask_rows(mask.to(cuda), 128 // t.shape[1]) for t in sel])
    lat = post_e.latent_dist.sample(generator=torch.Generator().manual_seed(3))
    assert rel_l2(lat, lat_ref) < 2e-2
    rec = pipe.vae.decode(z=lat, intermediate_features=inter, int_layers=int_layers).sample
    err = rel_l2(rec, rec_ref)
    print(f"train_emasc forward (small): reconstruction rel-L2 vs fp32 oracle {err:.4f}")
    assert rec.shape == rec_ref.shape == (2, 3, 128, 64)
    assert err < 5e-2
    assert (rec.float().cpu() - rec_ref).abs().mean() < 2e-2  # the L1 the training loss would see moves by < 2e-2


def test_vae_decode_int_layers_with_0(cuda, small):
    """int_layers containing 0 and 1 (src/models/vae.py:204-210): level-1 skip added after norm+SiLU, level-0 (image-space) skip added after
    conv_out.  Never used by the reference CLI (int_layers = [1..5]) but part of the decoder's surface."""
    from ladi_vton_b200 import EMASC, ops, synthetic as S
    from ladi_oracle.parts import EMASC as OE, mask_features
    pipe, _, ov, _ = small
    ein, eout = S.emasc_channels(S.SMALL_VAE["block_out_channels"])
    ein, eout = [3] + ein, [3] + eout
    sd = S.random_state_dict(S.emasc_param_shapes(ein, eout), 77)
    oe = OE(ein, eout).eval(); oe.load_state_dict(sd)
    em = EMASC(ein, eout).load_state_dict(sd).to(cuda)
    g = torch.Generator().manual_seed(2)
    x = torch.rand((2, 3, 128, 64), generator=g) * 2 - 1
    mask = torch.zeros((2, 1, 128, 64)); mask[:, :, 30:100, 10:50] = 1
    z = torch.randn((2, 4, 16, 8), generator=g)
    layers = [0, 1, 2, 3, 4, 5]
    with torch.no_grad():
        _, feats = ov.encode(x)
        inter_ref = mask_features(oe([feats[i] for i in layers]), mask)
        ref = ov.decode(z, list(inter_ref), layers).sample
    _, f = pipe.vae.encode(x.to(cuda))
    sel = [f[i] for i in layers]
    inter = em(sel, [ops.inv_mask_rows(mask.to(cuda), 128 // t.shape[1]) for t in sel])
    img = pipe.vae.decode(z.to(cuda), inter, layers).sample
    assert rel_l2(img, ref) < 5e-2


@pytest.mark.parametrize("mode", ["eta", "generator_list", "eta_generator_list"])
def test_pipeline_eta_and_generator_lists_small(cuda, small, mode):
    """`eta` > 0 (stochastic DDIM: one variance-noise draw per step after the three initial draws, tryon_pipe.py:337-345,740) and a LIST of
    per-sample generators (randn_tensor's list branch; prepare_mask_latents :445-450) -- never used by the reference CLI, part of `__call__`."""
    from ladi_vton_b200 import synthetic as S
    from ladi_oracle.parts import DDIMScheduler
    from ladi_oracle.pipeline import OracleTryOnPipeline
    pipe, ou, ov, oe = small
    inp = S.synthetic_inputs(2, 128, 64, ctx_dim=128)
    eta = 0.6 if "eta" in mode else 0.0
    gen = (lambda: [torch.Generator().manual_seed(5), torch.Generator().manual_seed(6)]) if "list" in mode else (lambda: torch.Generator().manual_seed(7))
    kw = dict(height=128, width=64, num_inference_steps=4, guidance_scale=7.5)
    ref = OracleTryOnPipeline(ov, ou, DDIMScheduler(), oe, [1, 2, 3, 4, 5])(
        inp["image"].clone(), inp["mask_image"].clone(), inp["pose_map"], inp["warped_cloth"], inp["prompt_embeds"],
        inp["negative_prompt_embeds"], generator=gen(), eta=eta, **kw)
    pipe.use_cuda_graph = True
    for _ in range(2):  # eager first call, graph replays on the second
        out = pipe(image=inp["image"].clone(), mask_image=inp["mask_image"].clone(), pose_map=inp["pose_map"], warped_cloth=inp["warped_cloth"],
                   prompt_embeds=inp["prompt_embeds"], negative_prompt_embeds=inp["negative_prompt_embeds"], generator=gen(), eta=eta,
                   output_type="np", **kw).images
        mad = np.abs(out - ref).mean() * 255
        print(f"pipeline {mode}: mean|engine-oracle| = {mad:.3f}/255")
        assert mad < 2.0


def test_pipeline_device_inputs_flags_and_shape_switch(cuda, small):
    """Device-resident inputs take the no-host-sync validation path (range flags read back with the result, caller's mask binarised in
    place); alternating between two shapes replays each shape's own captured graphs (GroupNorm workspace / weight addresses stay valid)."""
    from ladi_vton_b200 import synthetic as S
    pipe = small[0]
    pipe.use_cuda_graph = True
    outs = {}
    for rnd_ in range(3):
        for (B, H, W) in ((1, 128, 64), (2, 256, 128)):
            inp = {k: v.to(cuda) for k, v in S.synthetic_inputs(B, H, W, ctx_dim=128).items()}
            inp["mask_image"] = inp["mask_image"] * 0.8 + 0.1  # soft mask: {0.1, 0.9} -> binarised in place to {0, 1}
            m = inp["mask_image"]
            out = pipe(image=inp["image"], mask_image=m, pose_map=inp["pose_map"], warped_cloth=inp["warped_cloth"],
                       prompt_embeds=inp["prompt_embeds"], negative_prompt_embeds=inp["negative_prompt_embeds"], height=H, width=W,
                       num_inference_steps=3, generator=torch.Generator().manual_seed(7), output_type="np").images
            assert set(m.unique().tolist()) <= {0.0, 1.0}
            if (B, H, W) in outs:
                assert np.array_equal(out, outs[(B, H, W)])
            outs[(B, H, W)] = out
    bad = {k: v.to(cuda) for k, v in S.synthetic_inputs(1, 128, 64, ctx_dim=128).items()}
    with pytest.raises(ValueError, match="Image should be"):
        pipe(image=bad["image"] * 3, mask_image=bad["mask_image"], pose_map=bad["pose_map"], warped_cloth=bad["warped_cloth"],
             prompt_embeds=bad["prompt_embeds"], negative_prompt_embeds=bad["negative_prompt_embeds"], height=128, width=64,
             num_inference_steps=1, output_type="np")
    with pytest.raises(ValueError, match="num_images_per_prompt"):
        pipe(image=bad["image"], mask_image=bad["mask_image"], pose_map=bad["pose_map"], warped_cloth=bad["warped_cloth"],
             prompt_embeds=bad["prompt_embeds"], negative_prompt_embeds=bad["negative_prompt_embeds"], height=128, width=64,
             num_images_per_prompt=2)


# ------------------------------------------------------------------------------------------------ module-level C ABI (csrc/engine.cu)
def test_engine_abi_unet_forward_and_denoise_loop(cuda):
    """The module-level entry points called through ctypes with raw device pointers (what a non-Python host binds): ladi_unet_forward must
    reproduce the Python sequencing of the same kernels BIT FOR BIT (same launches, same order) and match the fp32 oracle; ladi_denoise_loop
    (N x (UNet + CFG + DDIM) enqueued by C++) must equal N replays of the pipeline's captured step."""
    import ctypes as C
    from ladi_vton_b200 import DDIMScheduler, UNet2DConditionModel, engine as eng, lib, ops, synthetic as S, unet_param_shapes
    from ladi_oracle.unet import UNet2DConditionModel as OU
    sd = S.random_state_dict(unet_param_shapes(S.SMALL_UNET), 1234)
    unet = UNet2DConditionModel(**S.SMALL_UNET).load_state_dict(sd).to(cuda)
    assert unet.engine is not None
    B, h, w = 2, 16, 8
    g = torch.Generator().manual_seed(0)
    x = torch.randn((2 * B, 31, h, w), generator=g)
    ctx = torch.randn((2 * B, 77, 128), generator=g)
    steps = unet.plan_steps([801, 601, 401])      # ladi_unet_plan_steps (sinusoid table on the device)
    kv = unet.plan_context(ctx.to(cuda))          # ladi_unet_plan_context
    ops.PROFILE = []  # the Python sequencing of the same tables (host trigonometry): equal up to the fp32 ulps of cosf / sinf
    try:
        unet._steps = unet._steps_key = None
        steps_py = unet.plan_steps([801, 601, 401]).clone()
        kv_py = unet.plan_context(ctx.to(cuda), out=torch.empty_like(kv)).clone()
    finally:
        ops.PROFILE = None
    unet._steps = unet._steps_key = None
    steps = unet.plan_steps([801, 601, 401])
    assert torch.equal(kv, kv_py)
    assert (steps - steps_py).abs().max() <= 1e-3 * steps_py.abs().max()
    xin = torch.zeros((2 * B, h, w, unet.in_pitch), dtype=torch.bfloat16, device=cuda)
    ops.nchw_to_nhwc(x.to(cuda), xin)
    step = torch.tensor([1, 0], dtype=torch.int32, device=cuda)
    l = lib.load()
    e = unet.engine
    nbytes = l.ladi_workspace_bytes(e.h, eng.MODULE_UNET, 2 * B, h, w)
    assert nbytes > 0
    ws = torch.empty(nbytes, dtype=torch.uint8, device=cuda)
    eps = torch.empty((2 * B, h, w, 4), dtype=torch.float32, device=cuda)
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    rc = l.ladi_unet_forward(e.h, C.c_void_p(xin.data_ptr()), C.c_void_p(step.data_ptr()), C.c_void_p(steps.data_ptr()), C.c_void_p(kv.data_ptr()),
                             2 * B, h, w, 77, C.c_void_p(eps.data_ptr()), C.c_void_p(ws.data_ptr()), nbytes, st)
    assert rc == 0, l.ladi_last_error()
    torch.cuda.synchronize()
    ops.PROFILE = []  # forces the Python sequencing of the same kernels
    try:
        eps_py = unet.forward_nhwc(xin, step)
    finally:
        ops.PROFILE = None
    assert torch.equal(eps, eps_py)
    ou = OU(**S.SMALL_UNET).eval(); ou.load_state_dict(sd)
    with torch.no_grad():
        ref = ou(x, torch.tensor(601), ctx).sample
    assert rel_l2(eps.permute(0, 3, 1, 2), ref) < 2e-2
    # a workspace that is too small is reported, not overrun
    rc = l.ladi_unet_forward(e.h, C.c_void_p(xin.data_ptr()), C.c_void_p(step.data_ptr()), C.c_void_p(steps.data_ptr()), C.c_void_p(kv.data_ptr()),
                             2 * B, h, w, 77, C.c_void_p(eps.data_ptr()), C.c_void_p(ws.data_ptr()), 4096, st)
    assert rc != 0 and b"workspace too small" in l.ladi_last_error()
    # ---- ladi_denoise_loop: 3 steps enqueued by C++ == 3 x (forward_nhwc + ddim_cfg_step)
    sch = DDIMScheduler(); sch.set_timesteps(3)
    coef = sch.coefficients().to(cuda)
    lat0 = torch.randn((B, 4, h, w), generator=g).to(cuda)

    def fresh():
        u = xin.clone()
        lat = lat0.clone()
        for half in (u[:B], u[B:]):
            ops.nchw_to_nhwc(lat, half, c_off=0)
        return u, lat, torch.zeros(2, dtype=torch.int32, device=cuda)
    u1, lat1, s1 = fresh()
    scratch = torch.empty((2 * B, h, w, 4), dtype=torch.float32, device=cuda)
    rc = l.ladi_denoise_loop(e.h, C.c_void_p(u1.data_ptr()), C.c_void_p(lat1.data_ptr()), C.c_void_p(s1.data_ptr()), C.c_void_p(steps.data_ptr()),
                             C.c_void_p(coef.data_ptr()), C.c_void_p(kv.data_ptr()), B, h, w, 77, 1, 7.5, 3, C.c_void_p(scratch.data_ptr()),
                             C.c_void_p(ws.data_ptr()), nbytes, st)
    assert rc == 0, l.ladi_last_error()
    u2, lat2, s2 = fresh()
    for _ in range(3):
        ops.ddim_cfg_step(unet.forward_nhwc(u2, s2), lat2, u2, True, 7.5, coef, s2)
    torch.cuda.synchronize()
    assert s1.tolist() == [3, 0] and torch.equal(lat1, lat2) and torch.equal(u1, u2)


def test_engine_abi_equals_python_sequencing_vae_emasc_adapter(cuda, small):
    """ladi_vae_encode / ladi_emasc_forward / ladi_vae_decode_emasc / ladi_inversion_adapter_forward (C++ launch sequences) against the Python
    sequencing of the same kernels: bit-identical outputs."""
    from ladi_vton_b200 import InversionAdapter, ops, synthetic as S
    pipe = small[0]
    g = torch.Generator().manual_seed(3)
    x = (torch.rand((2, 3, 128, 64), generator=g) * 2 - 1).to(cuda)
    mask = torch.zeros((2, 1, 128, 64), device=cuda); mask[:, :, 30:100, 10:50] = 1
    z = torch.randn((2, 4, 16, 8), generator=g).to(cuda)

    def run():
        mom, f = pipe.vae.encode_nhwc(x)
        sel = [f[i] for i in range(1, 6)]
        inter = pipe.emasc(sel, [ops.inv_mask_rows(mask, 128 // t.shape[1]) for t in sel])
        img = pipe.vae.decode_nhwc(z, inter, [1, 2, 3, 4, 5])
        return [mom] + [t.clone() for t in f[1:]] + [t.clone() for t in inter] + [img[..., :3].clone()]  # (channel 3 of the image buffer is padding)
    assert pipe.vae.engine is not None and pipe.emasc.engine is not None
    a = run()
    ops.PROFILE = []
    try:
        b = run()
    finally:
        ops.PROFILE = None
    for i, (s, t) in enumerate(zip(a, b)):
        assert torch.equal(s, t), f"output {i} of the C++ sequence differs from the Python sequencing"
    ad = InversionAdapter(input_dim=128, hidden_dim=256, output_dim=512, heads=2, mlp_dim=256)
    ad.load_state_dict(S.random_state_dict(ad.param_shapes(), 4)).to(cuda)
    feats = torch.randn((3, 17, 128), generator=g)
    y = ad(feats)
    ops.PROFILE = []
    try:
        y2 = ad(feats)
    finally:
        ops.PROFILE = None
    assert ad.engine is not None and torch.equal(y, y2)
