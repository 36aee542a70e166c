"""GPU tests of the forms src/eval.py and the training scripts build, and of the evaluation CLI mirror (ladi_vton_b200/eval.py):

  * linear and 1x1 EMASC through `ladi_emasc_forward` at full width (hub channel plan) and 512x384, with mask_features fused: the EMASC
    gate of test_gpu_models.py against the fp32 oracle (rel-L2 <= 1.5e-2), and bit-identical to the Python sequencing of the same kernels;
  * the full-size inversion adapter with 2 encoder layers: the gate of test_inversion_adapter_full (rel-L2 < 2e-2) and engine == Python
    sequencing bit for bit;
  * the `generate_images_from_tryon_pipe` body (eval.eval_batch) with reduced-width models, as tests/test_gpu_cli.py does, against its
    fp32 CPU restatement oracle/ladi_oracle/eval_body.py, final images mean |diff| <= 2/255, over the text_usage / cloth_input_type /
    emasc_type combinations;
  * `main()` writing `<output_dir>/<save_name>_<order>/<category>/`, identical files from two runs, and the feature cache written by
    compute_cloth_clip_features driving a `--use_clip_cloth_features` run."""
import os
import pickle

import numpy as np
import pytest
import torch

from kernel_check import rel_l2
from model_pairs import CTX, NV, cli_models

pytestmark = pytest.mark.gpu
EIN, EOUT = [128, 128, 128, 256, 512], [128, 256, 512, 512, 512]


@pytest.mark.parametrize("kw", [dict(type="linear", padding=1), dict(kernel_size=1, padding=0)], ids=["linear", "k1"])
def test_emasc_forms_full_width(cuda, kw):
    from ladi_oracle.emasc_forms import EMASC as OE
    from ladi_oracle.parts import mask_features
    from ladi_vton_b200 import EMASC, ops, synthetic as S
    em = EMASC(EIN, EOUT, **kw)
    sd = S.random_state_dict(em.param_shapes(), 91)
    em.load_state_dict(sd).to(cuda)
    oe = OE(EIN, EOUT, **kw).eval()
    oe.load_state_dict(sd)
    H, W = 512, 384
    g = torch.Generator().manual_seed(5)
    strides = [1, 1, 2, 4, 8]
    x = [torch.randn((2, c, H // s, W // s), generator=g) for c, s in zip(EIN, strides)]
    mask = torch.zeros((2, 1, H, W)); mask[:, :, 100:400, 80:300] = 1
    with torch.no_grad():
        ref = mask_features(oe([t.clone() for t in x]), mask)
    feats = []
    for t in x:
        f = torch.zeros((2, t.shape[2], t.shape[3], (t.shape[1] + 7) // 8 * 8), dtype=torch.bfloat16, device=cuda)[..., :t.shape[1]]
        f.copy_(t.permute(0, 2, 3, 1).to(cuda))
        feats.append(f)
    inv = [ops.inv_mask_rows(mask.to(cuda), s) for s in strides]
    got = em(feats, inv)
    assert em.engine is not None
    errs = [rel_l2(a.permute(0, 3, 1, 2), b) for a, b in zip(got, ref)]
    print(f"EMASC {kw} rel-L2 per scale vs fp32 oracle:", errs)
    assert all(e <= 1.5e-2 for e in errs), errs
    ops.PROFILE = []
    try:
        py = em(feats, inv)  # the Python sequencing of the same kernels
    finally:
        ops.PROFILE = None
    for i, (a, b) in enumerate(zip(got, py)):
        assert torch.equal(a, b), f"scale {i}: ladi_emasc_forward differs from the Python sequencing"


def test_inversion_adapter_two_layers_full(cuda):
    from ladi_oracle.parts import InversionAdapter as OA
    from ladi_vton_b200 import InversionAdapter, ops, synthetic as S
    eng = InversionAdapter(num_encoder_layers=2)
    sd = S.random_state_dict(eng.param_shapes(), 4321)
    oa = OA(num_encoder_layers=2).eval(); oa.load_state_dict(sd)
    x = torch.randn((3, 257, 1280), generator=torch.Generator().manual_seed(5))
    with torch.no_grad():
        ref = oa(x)
    eng.load_state_dict(sd).to(cuda)
    y = eng(x)
    assert eng.engine is not None and y.shape == ref.shape == (3, 16384)
    err = rel_l2(y, ref)
    print("inversion adapter (2 encoder layers) rel-L2 vs fp32 oracle:", err)
    assert err < 2e-2
    ops.PROFILE = []
    try:
        y2 = eng(x)
    finally:
        ops.PROFILE = None
    assert torch.equal(y, y2), "ladi_inversion_adapter_forward differs from the Python sequencing"


# ---- the generate_images_from_tryon_pipe body with reduced-width models -------------------------------------------------------------


@pytest.fixture(scope="module")
def models(cuda):
    """The CLI tests' engine / oracle pairs (model_pairs.cli_models, same seeded weights), plus a 27-channel UNet, linear and 1x1 EMASC and a 2-layer adapter."""
    from ladi_oracle.emasc_forms import EMASC as OE
    from ladi_oracle.parts import InversionAdapter as OA
    from ladi_oracle.unet import UNet2DConditionModel as OU
    from ladi_vton_b200 import EMASC, InversionAdapter, UNet2DConditionModel, synthetic as S
    from ladi_vton_b200.unet import unet_param_shapes
    eng, orc = cli_models(cuda)
    ein, eout = S.emasc_channels(S.SMALL_VAE["block_out_channels"])
    for name, kw, seed in (("linear", dict(type="linear", padding=1), 61), ("k1", dict(kernel_size=1, padding=0), 62)):
        e = EMASC(ein, eout, **kw)
        sd = S.random_state_dict(e.param_shapes(), seed)
        o = OE(ein, eout, **kw).eval(); o.load_state_dict(sd)
        eng[f"emasc_{name}"], orc[f"emasc_{name}"] = e.load_state_dict(sd).to(cuda), o
    cfg27 = {**S.SMALL_UNET, "in_channels": 27}
    sd = S.random_state_dict(unet_param_shapes(cfg27), 63)
    ou = OU(**cfg27).eval(); ou.load_state_dict(sd)
    eng["unet27"], orc["unet27"] = UNet2DConditionModel(**cfg27).load_state_dict(sd).to(cuda), ou
    ad = InversionAdapter(input_dim=160, hidden_dim=256, output_dim=CTX * NV, heads=2, mlp_dim=320, num_encoder_layers=2)
    sd = S.random_state_dict(ad.param_shapes(), 64)
    oa = OA(input_dim=160, hidden_dim=256, output_dim=CTX * NV, heads=2, mlp_dim=320, num_encoder_layers=2).eval(); oa.load_state_dict(sd)
    eng["adapter2"], orc["adapter2"] = ad.load_state_dict(sd).to(cuda), oa
    return eng, orc


def _pipes(eng, orc, cloth_input_type, emasc_type):
    from ladi_oracle.parts import DDIMScheduler as ODDIM
    from ladi_oracle.pipeline import OracleTryOnPipeline
    from ladi_vton_b200 import StableDiffusionTryOnePipeline
    ukey = "unet27" if cloth_input_type == "none" else "unet"
    ekey = {"none": None, "nonlinear": "emasc", "linear": "emasc_linear", "k1": "emasc_k1"}[emasc_type]
    layers = [1, 2, 3, 4, 5] if ekey else None
    pipe = StableDiffusionTryOnePipeline(text_encoder=eng["text_encoder"], vae=eng["vae"], tokenizer=eng["tokenizer"], unet=eng[ukey],
                                         scheduler=eng["scheduler"], emasc=eng[ekey] if ekey else None, emasc_int_layers=layers)
    opipe = OracleTryOnPipeline(orc["pipe"].vae, orc[ukey] if ukey == "unet27" else orc["pipe"].unet, ODDIM(),
                                (orc[ekey] if ekey != "emasc" else orc["pipe"].emasc) if ekey else None, layers)
    return pipe, opipe


CASES = [  # (text_usage, precomputed features, cloth_input_type, emasc_type, adapter)
    ("inversion_adapter", False, "warped", "nonlinear", "inversion_adapter"),
    ("inversion_adapter", True, "warped", "linear", "adapter2"),
    ("noun_chunks", False, "warped", "none", None),
    ("none", False, "none", "nonlinear", None),
    ("noun_chunks", False, "none", "k1", None),
    ("inversion_adapter", False, "none", "linear", "adapter2"),
]


@pytest.mark.parametrize("text_usage,pre,cloth_input_type,emasc_type,adapter", CASES)
def test_eval_body_vs_oracle(cuda, models, text_usage, pre, cloth_input_type, emasc_type, adapter):
    from ladi_oracle import eval_body as ob
    from ladi_vton_b200.eval import eval_batch, outputlist_for, parse_args
    from ladi_vton_b200.inference import SyntheticTryOnDataset
    eng, orc = models
    argv = ["--dataset", "vitonhd", "--output_dir", "o", "--save_name", "s", "--test_order", "paired", "--unet_dir", "u",
            "--text_usage", text_usage, "--cloth_input_type", cloth_input_type] + (["--use_clip_cloth_features"] if pre else [])
    ds = SyntheticTryOnDataset(2, (512, 384), ["upper_body", "dresses"], seed=9, outputlist=outputlist_for(parse_args(argv)), clip_dim=160)
    batch = next(iter(torch.utils.data.DataLoader(ds, batch_size=2)))
    pipe, opipe = _pipes(eng, orc, cloth_input_type, emasc_type)
    pipe.to(cuda)
    kw = dict(text_usage=text_usage, cloth_input_type=cloth_input_type, num_vstar=NV, guidance_scale=7.5, num_inference_steps=2)
    want = ob.run_batch({k: (v.clone() if torch.is_tensor(v) else v) for k, v in batch.items()}, opipe, orc.get(adapter),
                        orc["vision_encoder"], orc["tokenizer"], orc["text_encoder"], generator=torch.Generator().manual_seed(3), **kw)
    got = eval_batch(pipe, eng.get(adapter), batch, text_usage, eng["vision_encoder"], None, cloth_input_type, 1, NV,
                     torch.Generator().manual_seed(3), 2, 7.5)
    got = np.stack([np.asarray(im, dtype=np.float32) / 255 for im in got])
    assert got.shape == want.shape == (2, 512, 384, 3)
    mad = float(np.abs(got - want).mean())
    print(f"eval body {text_usage} pre={pre} cloth={cloth_input_type} emasc={emasc_type}: mean|engine - oracle| = {mad * 255:.3f}/255")
    assert mad < 2.0 / 255


def _eval_models(eng, emasc="emasc", adapter="inversion_adapter"):
    return dict(scheduler=eng["scheduler"], text_encoder=eng["text_encoder"], vae=eng["vae"], tokenizer=eng["tokenizer"], unet=eng["unet"],
                emasc=eng[emasc], inversion_adapter=eng[adapter], vision_encoder=eng["vision_encoder"])


ARGV = ["--dataset", "vitonhd", "--save_name", "run", "--test_order", "unpaired", "--unet_dir", "unused", "--synthetic_samples", "3",
        "--batch_size", "2", "--num_inference_steps", "2", "--num_vstar", str(NV), "--random_init"]


def test_main_writes_reference_tree(cuda, models, tmp_path):
    from PIL import Image
    from ladi_vton_b200.eval import main
    eng, _ = models
    w1 = main(ARGV + ["--output_dir", str(tmp_path / "a"), "--use_png"], models=_eval_models(eng))
    w2 = main(ARGV + ["--output_dir", str(tmp_path / "b"), "--use_png"], models=_eval_models(eng))
    d = os.path.join(tmp_path, "a", "run_unpaired", "upper_body")
    assert sorted(os.listdir(d)) == ["00000_00.png", "00001_00.png", "00002_00.png"] and len(w1) == 3
    assert Image.open(os.path.join(d, "00001_00.png")).size == (384, 512)
    for a, b in zip(w1, w2):
        assert np.array_equal(np.asarray(Image.open(a)), np.asarray(Image.open(b)))
    w3 = main(ARGV + ["--output_dir", str(tmp_path / "c"), "--emasc_type", "linear"], models=_eval_models(eng, "emasc_linear"))
    assert w3[0].endswith(os.path.join("run_unpaired", "upper_body", "00000_00.jpg")) and Image.open(w3[0]).format == "JPEG"


class _WithNames(torch.utils.data.Dataset):
    """The synthetic samples with `c_name` (the keys compute_cloth_clip_features reads), or with `clip_cloth_features` looked up by
    name in a written cache (what vitonhd.py:100-107,121-122 does)."""

    def __init__(self, base, cache=None):
        self.base, self.cache = base, cache

    def __len__(self):
        return len(self.base)

    def __getitem__(self, i):
        s = dict(self.base[i])
        name = f"{i:05d}_00.jpg"
        if self.cache is None:
            return dict(cloth=s["cloth"], c_name=name)
        feats, names = self.cache
        s["clip_cloth_features"] = feats[names.index(name)].float()
        return s


def test_feature_cache_drives_eval_run(cuda, models, tmp_path):
    from PIL import Image
    from ladi_vton_b200 import compute_cloth_clip_features as ccf
    from ladi_vton_b200.eval import main, outputlist_for, parse_args
    from ladi_vton_b200.inference import SyntheticTryOnDataset
    eng, _ = models
    base = SyntheticTryOnDataset(3, (512, 384), ["upper_body"], seed=1234)
    paths = ccf.main(["--dataset", "vitonhd", "--save_dir", str(tmp_path / "cache"), "--batch_size", "2"], vision_encoder=eng["vision_encoder"],
                     datasets=(_WithNames(base), _WithNames(base)))
    feats = torch.load(os.path.join(tmp_path, "cache", "test_last_hidden_state_features.pt"))
    names = pickle.load(open(os.path.join(tmp_path, "cache", "test_features_names.pkl"), "rb"))
    assert len(paths) == 4 and feats.dtype == torch.float16 and feats.shape == (3, 257, 160) and names == [f"{i:05d}_00.jpg" for i in range(3)]
    argv = ARGV + ["--use_png", "--use_clip_cloth_features"]
    ol = outputlist_for(parse_args(argv + ["--output_dir", "x"]))
    cached = _WithNames(SyntheticTryOnDataset(3, (512, 384), ["upper_body"], seed=1234, outputlist=[k for k in ol if k != "clip_cloth_features"]),
                        (feats, names))
    m = _eval_models(eng)
    m["vision_encoder"] = None  # src/eval.py:273-275: with precomputed features the vision tower is not built
    w_cached = main(argv + ["--output_dir", str(tmp_path / "cached")], models=m, dataset=cached)
    w_live = main(ARGV + ["--use_png", "--output_dir", str(tmp_path / "live")], models=_eval_models(eng))
    assert len(w_cached) == len(w_live) == 3
    mad = np.mean([np.abs(np.asarray(Image.open(a), dtype=np.float32) - np.asarray(Image.open(b), dtype=np.float32)).mean()
                   for a, b in zip(w_cached, w_live)])
    print(f"cached (fp16) vs on-the-fly CLIP features: mean|diff| = {mad:.3f}/255")
    assert mad < 2.0
