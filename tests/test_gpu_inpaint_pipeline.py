"""GPU tests of the SD-2 inpainting path (9-channel UNet input latents4 | mask1 | masked4) and of the inversion-adapter validation built
on it (eval.generate_images_inversion_adapter, python -m ladi_vton_b200.eval_inversion_adapter):

  * conv_in with 9 input channels at input pitch 16 against float64 with the census's per-element bound (kernel_check.conv_expect), at
    the pipeline's shape (batch 16, 64x48 latents -> 320 channels) and a ragged one;
  * the full-size 9-channel UNet at batch 2, 64x48 latents, against the fp32 oracle (the gate of test_unet_full_forward, rel-L2 < 2e-2),
    and `ladi_unet_forward` bit-identical to the Python sequencing of the same kernels;
  * `StableDiffusionInpaintPipeline` with reduced-width models against its fp32 CPU restatement (oracle/ladi_oracle/inpaint_pipeline.py),
    final images mean |diff| <= 2/255 (the try-on pipeline's gate), over guidance, num_images_per_prompt, image broadcast, a generator
    list, eta > 0, string prompts, a callback and the output types; a second call (graph replay) is bit-identical to the first (eager);
  * the `generate_images_inversion_adapter` body against oracle/ladi_oracle/adapter_val_body.py (mean |diff| <= 2/255);
  * the CLI end to end: the output tree, identical files from two runs, and the metrics JSON of `--compute_metrics --random_init`."""
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from kernel_check import conv_expect, cpu_gen, max_ratio, rel_l2
from model_pairs import NV, cli_models

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("n,h,w", [(16, 64, 48), (3, 13, 7)], ids=["pipeline", "ragged"])
def test_conv_in_nine_channels(cuda, n, h, w):
    """conv_in reads the first 9 channels of the pitch-16 UNet input (K = 81) and writes 320."""
    from ladi_vton_b200 import ops, weights
    g = cpu_gen(31)
    x = torch.zeros((n, h, w, 16), dtype=torch.bfloat16)
    x[..., :9] = torch.randn((n, h, w, 9), generator=g).bfloat16()
    wt = (torch.randn((320, 9, 3, 3), generator=g) * 81 ** -0.5).bfloat16().float()
    b = torch.randn((320,), generator=g)
    xin = x.to(cuda)
    y = ops.conv2d([xin[..., :9]], weights.pack_conv(wt.to(cuda), [9]), 320, bias=b.to(cuda))
    torch.cuda.synchronize()
    assert y.shape[:3] == (n, h, w) and bool(torch.isfinite(y[..., :320].float()).all())
    xd, wd = x[..., :9].double().permute(0, 3, 1, 2), wt.double()
    acc = F.conv2d(xd, wd, padding=1).permute(0, 2, 3, 1) + b.double()
    m = F.conv2d(xd.abs(), wd.abs(), padding=1).permute(0, 2, 3, 1) + b.double().abs()
    r, bound = conv_expect(acc, m, 81, ops.ACT_NONE)
    worst = max_ratio(y[..., :320].cpu().reshape(-1, 320), r.reshape(-1, 320), bound.reshape(-1, 320))
    print(f"conv_in 9 -> 320 at {n}x{h}x{w}: worst err/bound {worst:.3f}")
    assert worst <= 1.0


def test_unet9_full_forward(cuda):
    """Full-size SD-2 inpainting UNet (in_channels=9), one forward at 64x48 latents, batch 2."""
    from ladi_oracle.unet import UNet2DConditionModel as OU
    from ladi_vton_b200 import UNet2DConditionModel, ops, synthetic as S, unet_param_shapes
    sd = S.random_state_dict(unet_param_shapes({"in_channels": 9}), 1234)
    ou = OU(in_channels=9).eval(); ou.load_state_dict(sd)
    g = torch.Generator().manual_seed(0)
    x = torch.randn((2, 9, 64, 48), generator=g)
    ctx = torch.randn((2, 77, 1024), generator=g)
    with torch.no_grad():
        ref = ou(x, torch.tensor(501), ctx).sample
    del ou
    unet = UNet2DConditionModel(in_channels=9).load_state_dict(sd).to(cuda)
    y = unet(x.to(cuda), torch.tensor(501), ctx.to(cuda)).sample
    assert unet.engine is not None and unet.in_pitch == 16
    err = rel_l2(y, ref)
    print("full 9-channel UNet forward rel-L2 vs fp32 oracle:", err)
    assert err < 2e-2
    xin = torch.zeros((2, 64, 48, 16), dtype=torch.bfloat16, device=cuda)
    ops.nchw_to_nhwc(x.to(cuda).contiguous(), xin)
    step = torch.zeros(2, dtype=torch.int32, device=cuda)
    eps = unet.forward_nhwc(xin, step).clone()  # ladi_unet_forward, on the tables the call above planned
    ops.PROFILE = []  # forces the Python sequencing of the same kernels
    try:
        eps_py = unet.forward_nhwc(xin, step)
    finally:
        ops.PROFILE = None
    assert torch.equal(eps, eps_py), "ladi_unet_forward differs from the Python sequencing at 9 input channels"


# ---- the pipeline with reduced-width models ---------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def models(cuda):
    """model_pairs.cli_models (text / vision towers, adapter, VAE on shared seeded weights) plus a reduced-width 9-channel UNet pair."""
    from ladi_oracle.unet import UNet2DConditionModel as OU
    from ladi_vton_b200 import UNet2DConditionModel, synthetic as S
    from ladi_vton_b200.unet import unet_param_shapes
    eng, orc = cli_models(cuda)
    cfg9 = {**S.SMALL_UNET, "in_channels": 9}
    sd = S.random_state_dict(unet_param_shapes(cfg9), 71)
    ou = OU(**cfg9).eval(); ou.load_state_dict(sd)
    eng["unet9"], orc["unet9"] = UNet2DConditionModel(**cfg9).load_state_dict(sd).to(cuda), ou
    return eng, orc


def _pipes(eng, orc):
    from ladi_oracle.inpaint_pipeline import OracleInpaintPipeline
    from ladi_oracle.parts import DDIMScheduler as ODDIM
    from ladi_vton_b200 import DDIMScheduler, StableDiffusionInpaintPipeline
    pipe = StableDiffusionInpaintPipeline(vae=eng["vae"], text_encoder=eng["text_encoder"], tokenizer=eng["tokenizer"], unet=eng["unet9"],
                                          scheduler=DDIMScheduler(), safety_checker=None, feature_extractor=None,
                                          requires_safety_checker=False)
    return pipe, OracleInpaintPipeline(orc["pipe"].vae, orc["unet9"], ODDIM())


H, W = 128, 64
CASES = {
    "cfg1": dict(guidance=1.0),
    "cfg7.5": dict(),
    "n2": dict(n=2),
    "broadcast": dict(images=1),
    "generator_list": dict(gen_list=True),
    "eta": dict(eta=0.5),
    "strings": dict(strings=True),
    "strings_n2_cfg1": dict(strings=True, n=2, guidance=1.0),
    "callback": dict(callback=True),
}


def _images(n, seed=3):
    g = torch.Generator().manual_seed(seed)
    image = torch.rand((n, 3, H, W), generator=g) * 2 - 1
    mask = torch.zeros((n, 1, H, W))
    for i in range(n):
        mask[i, :, 20 + 8 * i:100, 8 + 4 * i:52] = 1
    return image, mask


@pytest.mark.parametrize("case", list(CASES))
def test_pipeline_vs_oracle(cuda, models, case):
    """Two prompts; 3 DDIM steps; engine vs fp32 oracle on the same CPU-generator draws; then the same call again (graphs replayed)."""
    from ladi_oracle.eval_body import _encode
    eng, orc = models
    o = CASES[case]
    guidance, n, eta = o.get("guidance", 7.5), o.get("n", 1), o.get("eta", 0.0)
    image, mask = _images(o.get("images", 2))
    g = torch.Generator().manual_seed(4)
    pe, ne = torch.randn((2, 77, 128), generator=g), torch.randn((2, 77, 128), generator=g)
    prompts = ["a photo of a model wearing a dress", "an upper body garment"]
    if o.get("strings"):
        pe = _encode(orc["tokenizer"], orc["text_encoder"], prompts, 77)
        ne = _encode(orc["tokenizer"], orc["text_encoder"], ["", ""], 77)
    gens = lambda: [torch.Generator().manual_seed(10 + i) for i in range(2 * n)] if o.get("gen_list") else torch.Generator().manual_seed(7)  # noqa: E731
    pipe, opipe = _pipes(eng, orc)
    pipe.to(cuda)
    o_steps = []
    want = opipe(image.clone(), mask.clone(), pe, ne if guidance > 1 else None, height=H, width=W, num_inference_steps=3,
                 guidance_scale=guidance, num_images_per_prompt=n, generator=gens(), eta=eta,
                 callback=(lambda i, t, lat: o_steps.append(lat.clone())) if o.get("callback") else None)
    text = dict(prompt=prompts) if o.get("strings") else dict(prompt_embeds=pe.to(cuda), negative_prompt_embeds=ne.to(cuda))
    outs = []
    for _ in range(2):
        steps = []
        cb = (lambda i, t, lat: steps.append(lat.clone())) if o.get("callback") else None
        out = pipe(image=image.to(cuda), mask_image=mask.to(cuda), height=H, width=W, num_inference_steps=3, guidance_scale=guidance,
                   num_images_per_prompt=n, eta=eta, generator=gens(), output_type="np", callback=cb, **text)
        assert out.nsfw_content_detected is None
        outs.append(out.images)
        if cb is not None:
            assert len(steps) == len(o_steps) == 3
            assert rel_l2(steps[-1], o_steps[-1]) < 3e-2
    got = outs[0]
    assert got.shape == want.shape == (2 * n, H, W, 3)
    mad = float(np.abs(got - want).mean())
    print(f"inpaint pipeline {case}: mean|engine - oracle| = {mad * 255:.3f}/255")
    assert mad < 2.0 / 255
    assert np.array_equal(outs[0], outs[1]), "the replayed call differs from the eager one"


def test_pipeline_output_types_and_tiling(cuda, models):
    """2 prompts x 2 images per prompt: the pt / np / pil outputs of one workload agree, and rows 0 and 2 (the same image, different
    initial latents) differ."""
    eng, orc = models
    pipe, _ = _pipes(eng, orc)
    pipe.to(cuda)
    image, mask = _images(2)
    g = torch.Generator().manual_seed(4)
    pe, ne = torch.randn((2, 77, 128), generator=g).to(cuda), torch.randn((2, 77, 128), generator=g).to(cuda)
    kw = dict(image=image.to(cuda), mask_image=mask.to(cuda), prompt_embeds=pe, negative_prompt_embeds=ne, height=H, width=W,
              num_inference_steps=2, num_images_per_prompt=2)
    pt = pipe(generator=torch.Generator().manual_seed(1), output_type="pt", **kw).images
    npy = pipe(generator=torch.Generator().manual_seed(1), output_type="np", **kw).images
    pil, nsfw = pipe(generator=torch.Generator().manual_seed(1), return_dict=False, **kw)
    assert nsfw is None and pt.is_cuda and pt.shape == (4, H, W, 3) and len(pil) == 4 and pil[0].size == (W, H)
    assert np.array_equal(pt.cpu().numpy(), npy)
    assert np.array_equal(np.stack([np.asarray(p) for p in pil]), (npy * 255).round().astype(np.uint8))
    assert not np.array_equal(npy[0], npy[2])


# ---- the validation body and the CLI ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pre", [False, True], ids=["vision_tower", "clip_cloth_features"])
def test_adapter_val_body_vs_oracle(cuda, models, pre):
    from ladi_oracle import adapter_val_body as ob
    from ladi_vton_b200.eval import adapter_val_batch
    from ladi_vton_b200.eval_inversion_adapter import outputlist_for, parse_args
    from ladi_vton_b200.inference import SyntheticTryOnDataset
    eng, orc = models
    argv = ["--dataset", "vitonhd", "--output_dir", "o"] + (["--use_clip_cloth_features"] if pre else [])
    ds = SyntheticTryOnDataset(2, (512, 384), ["upper_body", "dresses"], seed=9, outputlist=outputlist_for(parse_args(argv)), clip_dim=160)
    batch = next(iter(torch.utils.data.DataLoader(ds, batch_size=2)))
    pipe, opipe = _pipes(eng, orc)
    pipe.to(cuda)
    want = ob.run_batch({k: (v.clone() if torch.is_tensor(v) else v) for k, v in batch.items()}, opipe, orc["inversion_adapter"],
                        orc["vision_encoder"], orc["tokenizer"], orc["text_encoder"], NV, 7.5, 2, torch.Generator().manual_seed(3))
    got = adapter_val_batch(pipe, eng["inversion_adapter"], eng["vision_encoder"], None, batch, NV, torch.Generator().manual_seed(3), 2, 7.5)
    got = np.stack([np.asarray(im, dtype=np.float32) / 255 for im in got])
    assert got.shape == want.shape == (2, 512, 384, 3)
    mad = float(np.abs(got - want).mean())
    print(f"adapter validation body (pre={pre}): mean|engine - oracle| = {mad * 255:.3f}/255")
    assert mad < 2.0 / 255


def test_cli_random_init_end_to_end(cuda, tmp_path):
    """Full-size random-init models through main(): the reference's tree, identical files from two runs."""
    from PIL import Image
    from ladi_vton_b200.eval_inversion_adapter import main
    argv = ["--dataset", "vitonhd", "--synthetic_samples", "3", "--test_batch_size", "2", "--num_inference_steps", "2", "--random_init"]
    w1 = main(argv + ["--output_dir", str(tmp_path / "a")])
    w2 = main(argv + ["--output_dir", str(tmp_path / "b")])
    d = os.path.join(tmp_path, "a", "imgs_step_random_init_paired", "upper_body")
    assert sorted(os.listdir(d)) == ["00000_00.jpg", "00001_00.jpg", "00002_00.jpg"] and len(w1) == 3
    im = Image.open(os.path.join(d, "00001_00.jpg"))
    assert im.size == (384, 512) and im.format == "JPEG"
    for a, b in zip(w1, w2):
        assert np.array_equal(np.asarray(Image.open(a)), np.asarray(Image.open(b)))


def _gt_tree(root, n):
    from PIL import Image
    rs = np.random.RandomState(15)
    names = [f"{i:05d}_00.jpg" for i in range(n)]
    os.makedirs(os.path.join(root, "test", "image"))
    with open(os.path.join(root, "test_pairs.txt"), "w") as f:
        f.write("".join(f"{a} {a}\n" for a in names))
    for nm in names:
        Image.fromarray(rs.randint(0, 256, size=(8, 6, 3)).astype(np.uint8)).resize((384, 512)).save(os.path.join(root, "test", "image", nm))


def test_cli_compute_metrics(cuda, models, tmp_path, monkeypatch):
    """--compute_metrics --random_init: the engine's metrics over the written folder, into metrics_<save_name>_<order>_all.json."""
    from ladi_vton_b200.eval_inversion_adapter import main
    monkeypatch.setenv("HOME", str(tmp_path))  # the ground-truth statistics cache (~/.cache/ladi_vton_b200/metrics)
    eng, _ = models
    root = str(tmp_path / "vitonhd")
    _gt_tree(root, 6)
    m = dict(scheduler=eng["scheduler"], text_encoder=eng["text_encoder"], vae=eng["vae"], tokenizer=eng["tokenizer"], unet=eng["unet9"],
             inversion_adapter=eng["inversion_adapter"], vision_encoder=eng["vision_encoder"])
    argv = ["--dataset", "vitonhd", "--vitonhd_dataroot", root, "--output_dir", str(tmp_path / "out"), "--synthetic_samples", "6",
            "--test_batch_size", "3", "--num_inference_steps", "2", "--num_vstar", str(NV), "--random_init", "--compute_metrics",
            "--save_name", "imgs_step_7"]
    written = main(argv, models=m)
    assert len(written) == 6 and all(p.startswith(str(tmp_path / "out" / "imgs_step_7_paired")) for p in written)
    out = json.load(open(tmp_path / "out" / "metrics_imgs_step_7_paired_all.json"))
    assert list(out) == ['ssim_score', 'lpips_score', 'fid_score', 'kid_score', 'is_score'], out
    assert all(np.isfinite(v) for v in out.values()), out
    print(f"\n[adapter validation] metrics: {out}")
