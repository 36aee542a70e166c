"""GPU tests of the CLI mirror (ladi_vton_b200/inference.py <- src/inference.py:225-324): the fused CLIP image
preprocessing kernel, the whole batch body against its fp32 CPU restatement (oracle/ladi_oracle/inference_body.py) on shared seeded
weights, and `main()` writing the reference's output tree.  Reduced-width models keep the CPU oracle to seconds; the image size is the
CLI's hard-coded 512x384 and the warping module is the hub configuration (ConvNet_TPS(256,192,21,3), UNetVanilla(24,3)).
Tolerances (engine bf16 vs oracle fp32): pixel values 1e-5 abs; warped cloth rel-L2 3e-2; CLIP features / pseudo-words / text states
rel-L2 3e-2; final image mean |diff| <= 2/255 (the stated pipeline tolerance)."""
import os

import numpy as np
import pytest
import torch

from kernel_check import rel_l2
from model_pairs import NV, cli_models

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("quantise", [False, True])
def test_clip_preprocess(cuda, quantise):
    from ladi_oracle.inference_body import CLIP_MEAN, CLIP_STD, clip_pixel_values
    from ladi_vton_b200 import ops, synthetic as S
    cloth = S.warp_inputs(2, 512, 384, seed=3)["cloth"] * 1.2  # exceeds [-1,1] in places: exercises the clamp
    ref = clip_pixel_values(cloth, "uint8" if quantise else "float")
    mean, std = torch.tensor(CLIP_MEAN, device=cuda), torch.tensor(CLIP_STD, device=cuda)
    out = ops.clip_preprocess(cloth.to(cuda).contiguous(), 224, 224, mean, std, quantise).cpu()
    assert out.shape == ref.shape == (2, 3, 224, 224)
    d = (out - ref).abs()
    if not quantise:
        assert float(d.max()) < 1e-5, float(d.max())
    else:  # floor() may flip one level where the fused and the separable filter differ in the last ulp
        assert float((d > 1e-5).float().mean()) < 1e-3 and float(d.max()) < 1.01 / 255 / min(CLIP_STD)
    with pytest.raises(RuntimeError, match="down-scale"):
        ops.clip_preprocess(torch.zeros((1, 3, 2048, 64), device=cuda), 224, 224, mean, std)


@pytest.fixture(scope="module")
def models(cuda):
    return cli_models(cuda)


ARGV = ["--test_order", "paired", "--dataset", "vitonhd", "--synthetic_samples", "3", "--batch_size", "2", "--num_inference_steps", "2",
        "--num_vstar", str(NV)]


def test_loop_body_vs_oracle(cuda, models):
    """src/inference.py:226-312 end to end: engine (bf16 kernels) vs the fp32 CPU restatement, same weights, same CPU generator seed."""
    from ladi_oracle import inference_body as ob
    from ladi_vton_b200 import StableDiffusionTryOnePipeline, encode_text_word_embedding, generate_warped_cloth
    from ladi_vton_b200.inference import SyntheticTryOnDataset, clip_pixel_values, parse_args, prompts_for, run_batch
    eng, orc = models
    args = parse_args(ARGV + ["--output_dir", "unused"])
    ds = SyntheticTryOnDataset(2, (512, 384), ["upper_body"], seed=9)
    batch = next(iter(torch.utils.data.DataLoader(ds, batch_size=2)))
    want, o_warp, o_feats, o_word, o_ctx = ob.run_batch({k: (v.clone() if torch.is_tensor(v) else v) for k, v in batch.items()}, num_vstar=NV,
                                                        guidance_scale=7.5, num_inference_steps=2,
                                                        generator=torch.Generator().manual_seed(3), return_all=True, **orc)
    assert prompts_for(batch["category"], NV) == ob.prompts_for(batch["category"], NV)
    # stages
    warped = generate_warped_cloth(eng["tps"], eng["refinement"], batch["cloth"], batch["im_mask"], batch["pose_map"])
    feats = eng["vision_encoder"](clip_pixel_values(batch["cloth"], cuda)).last_hidden_state
    word = eng["inversion_adapter"](feats).reshape(2, NV, -1)
    ids = eng["tokenizer"](prompts_for(batch["category"], NV)).input_ids
    ctx = encode_text_word_embedding(eng["text_encoder"], ids, word, NV).last_hidden_state
    errs = dict(warped=rel_l2(warped, o_warp), feats=rel_l2(feats, o_feats), word=rel_l2(word, o_word), ctx=rel_l2(ctx, o_ctx))
    print("loop-body stage rel-L2:", errs)
    assert all(e < 3e-2 for e in errs.values()), errs
    # whole body
    pipe = StableDiffusionTryOnePipeline(text_encoder=eng["text_encoder"], vae=eng["vae"], tokenizer=eng["tokenizer"], unet=eng["unet"],
                                         scheduler=eng["scheduler"], emasc=eng["emasc"], emasc_int_layers=[1, 2, 3, 4, 5]).to(cuda)
    got = run_batch(batch, eng, pipe, args, torch.Generator().manual_seed(3), cuda)
    got = np.stack([np.asarray(im, dtype=np.float32) / 255 for im in got])
    assert got.shape == want.shape == (2, 512, 384, 3)
    mad = float(np.abs(got - want).mean())
    print(f"loop body: mean|engine - oracle| = {mad * 255:.3f}/255 (uint8-quantised engine output)")
    assert mad < 2.0 / 255


def test_main_writes_reference_tree(cuda, models, tmp_path):
    from PIL import Image
    from ladi_vton_b200.inference import main
    eng, _ = models
    out1, out2 = str(tmp_path / "a"), str(tmp_path / "b")
    w1 = main(ARGV + ["--output_dir", out1, "--use_png"], models=eng)
    w2 = main(ARGV + ["--output_dir", out2, "--use_png"], models=eng)
    d = os.path.join(out1, "paired", "upper_body")
    assert sorted(os.listdir(d)) == ["00000_00.png", "00001_00.png", "00002_00.png"] and len(w1) == 3
    im = Image.open(os.path.join(d, "00002_00.png"))
    assert im.size == (384, 512) and im.mode == "RGB"
    for a, b in zip(w1, w2):  # same seed -> same files (cuda generator, deterministic kernels)
        assert np.array_equal(np.asarray(Image.open(a)), np.asarray(Image.open(b)))
    w3 = main(ARGV + ["--output_dir", str(tmp_path / "c")], models=eng)
    assert w3[0].endswith(os.path.join("paired", "upper_body", "00000_00.jpg")) and Image.open(w3[0]).format == "JPEG"
