"""Host-side tests of the SD-2 inpainting pipeline (`StableDiffusionInpaintPipeline`, pipeline.py) and of the inversion-adapter
validation CLI (ladi_vton_b200/eval_inversion_adapter.py <- src/train_inversion_adapter.py:544-569): flag-for-flag parity with the
trainer's parser (golden read from the reference source by tests/golden/make_adapter_val_golden.py), the validation function's
signature, prompt template, outputlist and folder name; the fp32 oracle pinned to the try-on oracle and its `num_images_per_prompt`
tiling; the C++ UNet launch sequence at 9 input channels; and the errors.  No GPU needed."""
import inspect
import json
import os

import numpy as np
import pytest
import torch

from kernel_check import compare, record  # noqa: F401  (record: a fixture)

GOLD = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "adapter_val_flags.json")))
BASE = ["--dataset", "vitonhd", "--output_dir", "o"]
ENGINE = {"--inversion_adapter_dir", "--inversion_adapter_name", "--save_name", "--num_inference_steps", "--guidance_scale",
          "--vision_model_name_or_path", "--reference_src", "--random_init", "--synthetic_samples", "--compute_metrics", "--metrics_weights_dir"}
SHARED = {"--dataset", "--dresscode_dataroot", "--vitonhd_dataroot", "--output_dir", "--pretrained_model_name_or_path", "--seed",
          "--test_batch_size", "--num_workers_test", "--test_order", "--num_vstar", "--num_encoder_layers", "--use_clip_cloth_features",
          "--enable_xformers_memory_efficient_attention"}


def test_flags_match_reference_trainer():
    from ladi_vton_b200.eval_inversion_adapter import build_parser
    parser = build_parser()
    acts = {a.option_strings[0]: a for a in parser._actions if a.option_strings and a.option_strings[0] != "-h"}
    engine = {a.option_strings[0] for g in parser._action_groups if g.title == "engine" for a in g._group_actions}
    assert engine == ENGINE and set(acts) - engine == SHARED
    ref = {f["flags"][0]: f for f in GOLD["flags"]}
    assert len(ref) == 33 and SHARED <= set(ref) and not (engine & set(ref))
    for name in SHARED:
        f, a = ref[name], acts[name]
        assert a.option_strings == f["flags"]
        if f.get("action") == "store_true":
            assert a.nargs == 0 and a.const is True and a.default is False
        else:
            assert a.type.__name__ == f["type"], f
            assert a.default == f.get("default"), f
        assert bool(a.required) == bool(f.get("required", False)), f
        assert (list(a.choices) if a.choices else None) == f.get("choices"), f


def test_validation_function_and_dataset_surface():
    """image_from_pipe.py:139-143 signature and defaults, the :173-180 prompt template, the :281-285 outputlist and the :562 folder name."""
    from ladi_vton_b200.eval import generate_images_inversion_adapter
    from ladi_vton_b200.eval_inversion_adapter import OUTPUTLIST, SAVE_NAME, outputlist_for, parse_args
    from ladi_vton_b200.inference import CATEGORY_TEXT, prompts_for
    sig = inspect.signature(generate_images_inversion_adapter)
    assert list(sig.parameters) == GOLD["function_params"]
    assert {k: p.default for k, p in sig.parameters.items() if p.default is not inspect.Parameter.empty} == GOLD["function_defaults"]
    assert CATEGORY_TEXT == GOLD["category_text"]
    assert prompts_for(["dresses"], 2) == ['a photo of a model wearing a dress  $  $ ']
    assert OUTPUTLIST == GOLD["outputlist"] and outputlist_for(parse_args(BASE)) == GOLD["outputlist"]
    assert GOLD["outputlist_append"] == {"flag": "--use_clip_cloth_features", "appends": "clip_cloth_features"}
    assert outputlist_for(parse_args(BASE + ["--use_clip_cloth_features"])) == GOLD["outputlist"] + ["clip_cloth_features"]
    assert SAVE_NAME.format(1500) == GOLD["save_name"].format(global_step=1500)


def _touch(d, names):
    for n in names:
        open(os.path.join(d, n), "wb").close()


def test_checkpoint_and_save_name(tmp_path):
    """`latest` takes the highest step among `inversion_adapter_*` in --inversion_adapter_dir (default --output_dir), and the folder is
    named after that step."""
    from ladi_vton_b200.eval_inversion_adapter import default_save_name, parse_args
    d = str(tmp_path)
    _touch(d, ["inversion_adapter_500.pth", "inversion_adapter_40000.pth", "inversion_adapter_9000.pth", "unet_99999.pth", "notes.txt"])
    assert default_save_name(parse_args(["--dataset", "vitonhd", "--output_dir", d])) == "imgs_step_40000"
    other = ["--dataset", "vitonhd", "--output_dir", "elsewhere", "--inversion_adapter_dir", d]
    assert default_save_name(parse_args(other)) == "imgs_step_40000"
    assert default_save_name(parse_args(other + ["--inversion_adapter_name", "inversion_adapter_500.pth"])) == "imgs_step_500"
    with pytest.raises(ValueError, match="--save_name"):
        default_save_name(parse_args(other + ["--inversion_adapter_name", "adapter_final.pth"]))
    assert parse_args(["--dataset", "vitonhd", "--output_dir", d]).inversion_adapter_dir == d


def test_argument_errors(tmp_path):
    from ladi_vton_b200.eval_inversion_adapter import check_args, check_base_unet, parse_args
    with pytest.raises(ValueError, match="VitonHD dataroot must be provided"):
        check_args(parse_args(BASE))
    with pytest.raises(ValueError, match="DressCode dataroot must be provided"):
        check_args(parse_args(["--dataset", "dresscode", "--output_dir", "o"]))
    with pytest.raises(NotImplementedError, match="1.5 inpainting base"):
        check_args(parse_args(BASE + ["--synthetic_samples", "1", "--random_init", "--pretrained_model_name_or_path",
                                      "runwayml/stable-diffusion-inpainting"]))
    root = tmp_path / "sd2"
    os.makedirs(root / "unet")
    with pytest.raises(FileNotFoundError, match="config.json"):
        check_base_unet(str(tmp_path))
    for cin in (31, 4):
        json.dump({"in_channels": cin}, open(root / "unet" / "config.json", "w"))
        with pytest.raises(ValueError, match=f"in_channels={cin}"):
            check_args(parse_args(BASE + ["--synthetic_samples", "1", "--pretrained_model_name_or_path", str(root)]))
    json.dump({"in_channels": 9}, open(root / "unet" / "config.json", "w"))
    check_args(parse_args(BASE + ["--synthetic_samples", "1", "--pretrained_model_name_or_path", str(root)]))
    check_args(parse_args(BASE + ["--synthetic_samples", "1", "--random_init"]))  # with random weights no folder is read


@pytest.mark.skipif(torch.cuda.is_available(), reason="CPU-only check")
def test_cli_has_no_cpu_path(tmp_path):
    from ladi_vton_b200.eval_inversion_adapter import main
    with pytest.raises(RuntimeError, match="no CPU path"):
        main(["--dataset", "vitonhd", "--output_dir", str(tmp_path), "--synthetic_samples", "2", "--random_init"])
    assert os.listdir(tmp_path) == []


# ---- pipeline call errors (raised on the host before any device work) -------------------------------------------------------------------
class _Cfg:
    def __init__(self, **kw):
        self.__dict__.update(kw)


def _stub_pipe(in_channels=9):
    from ladi_vton_b200 import StableDiffusionInpaintPipeline
    vae = type("V", (), {"config": _Cfg(block_out_channels=(1, 2, 3, 4), latent_channels=4)})()
    unet = type("U", (), {"config": _Cfg(in_channels=in_channels, sample_size=8)})()
    pipe = StableDiffusionInpaintPipeline(vae=vae, text_encoder=None, tokenizer=None, unet=unet, scheduler=None, safety_checker=None,
                                          feature_extractor=None, requires_safety_checker=False)
    pipe.device = torch.device("cuda")  # the checks below run before anything touches the device
    return pipe


def test_pipeline_surface():
    from ladi_vton_b200 import StableDiffusionInpaintPipeline
    assert list(inspect.signature(StableDiffusionInpaintPipeline.__init__).parameters)[1:] == [
        "vae", "text_encoder", "tokenizer", "unet", "scheduler", "safety_checker", "feature_extractor", "requires_safety_checker"]
    assert list(inspect.signature(StableDiffusionInpaintPipeline.__call__).parameters)[1:] == [
        "prompt", "image", "mask_image", "height", "width", "num_inference_steps", "guidance_scale", "negative_prompt",
        "num_images_per_prompt", "eta", "generator", "latents", "prompt_embeds", "negative_prompt_embeds", "output_type", "return_dict",
        "callback", "callback_steps"]
    with pytest.raises(RuntimeError, match="CUDA"):
        _stub_pipe().to("cpu")


def test_pipeline_errors():
    from ladi_vton_b200.pipeline import _check_tiling
    img, mask, pe = torch.zeros((2, 3, 64, 64)), torch.zeros((2, 1, 64, 64)), torch.zeros((1, 77, 8))
    with pytest.raises(ValueError, match=r"expects 31 input channels .* = 9"):
        _stub_pipe(31)(prompt_embeds=pe, image=img, mask_image=mask, height=64, width=64)
    with pytest.raises(ValueError, match="The passed mask and the required batch size don't match"):  # 2 images, 3 samples
        _stub_pipe()(prompt_embeds=torch.zeros((3, 77, 8)), image=img, mask_image=mask, height=64, width=64)
    with pytest.raises(ValueError, match="The passed images and the required batch size don't match"):
        _check_tiling(1, 2, 3)
    with pytest.raises(ValueError, match="The passed mask and the required batch size don't match"):
        _check_tiling(2, 2, 5)
    _check_tiling(2, 2, 4), _check_tiling(1, 1, 3), _check_tiling(3, 3, 3)
    with pytest.raises(ValueError, match="at most one image per sample"):  # 2 images for 1 sample
        _stub_pipe()(prompt_embeds=pe, image=img, mask_image=mask, height=64, width=64)
    gens = [torch.Generator().manual_seed(i) for i in range(4)]
    with pytest.raises(ValueError, match="one masked-image latent per sample, but only 2 images"):  # 2 prompts x 2 images per prompt
        _stub_pipe()(prompt_embeds=torch.zeros((2, 77, 8)), image=img, mask_image=mask, height=64, width=64, num_images_per_prompt=2,
                     generator=gens)
    with pytest.raises(ValueError, match="list of generators of length 3"):
        _stub_pipe()(prompt_embeds=torch.zeros((2, 77, 8)), image=img, mask_image=mask, height=64, width=64, generator=gens[:3])


# ---- oracle ----------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def small_oracle():
    from ladi_oracle.unet import UNet2DConditionModel as OU
    from ladi_oracle.vae import AutoencoderKL as OV
    from ladi_vton_b200 import synthetic as S
    from ladi_vton_b200.unet import unet_param_shapes
    cfg = {**S.SMALL_UNET, "in_channels": 9}
    sds = S.build_state_dicts(cfg, S.SMALL_VAE, seed=8)
    ou = OU(**cfg).eval(); ou.load_state_dict(sds["unet"])
    ov = OV(**S.SMALL_VAE).eval(); ov.load_state_dict(sds["vae"])
    assert unet_param_shapes(cfg)["conv_in.weight"][1] == 9
    return ou, ov


class _First9:
    """The 9-channel UNet behind a wider input: drops the try-on pipeline's (zero) pose channel."""

    def __init__(self, unet):
        self.unet, self.config, self.dtype = unet, unet.config, unet.dtype

    def __call__(self, x, t, encoder_hidden_states):
        return self.unet(x[:, :9], t, encoder_hidden_states=encoder_hidden_states)


def _inputs(n, H=128, W=64, seed=3):
    g = torch.Generator().manual_seed(seed)
    image = torch.rand((n, 3, H, W), generator=g) * 2 - 1
    mask = torch.zeros((n, 1, H, W))
    for i in range(n):
        mask[i, :, 16 + 8 * i:96, 8:48 + 4 * i] = 1
    return image, mask


@pytest.mark.parametrize("guidance", [1.0, 7.5])
def test_oracle_pinned_to_tryon_oracle(small_oracle, guidance):
    """num_images_per_prompt=1, one image per prompt: the inpainting oracle is the try-on oracle with cloth_input_type 'none', no EMASC
    and no pose (one zero pose channel the wrapped UNet drops), bit for bit."""
    from ladi_oracle.inpaint_pipeline import OracleInpaintPipeline
    from ladi_oracle.parts import DDIMScheduler
    from ladi_oracle.pipeline import OracleTryOnPipeline
    ou, ov = small_oracle
    image, mask = _inputs(2)
    g = torch.Generator().manual_seed(4)
    pe, ne = torch.randn((2, 77, 128), generator=g), torch.randn((2, 77, 128), generator=g)
    kw = dict(height=128, width=64, num_inference_steps=2, guidance_scale=guidance, eta=0.3)
    got = OracleInpaintPipeline(ov, ou, DDIMScheduler())(image.clone(), mask.clone(), pe, ne, generator=torch.Generator().manual_seed(5), **kw)
    want = OracleTryOnPipeline(ov, _First9(ou), DDIMScheduler())(image.clone(), mask.clone(), torch.zeros((2, 1, 128, 64)), None, pe, ne,
                                                                   generator=torch.Generator().manual_seed(5), no_pose=True,
                                                                   cloth_input_type="none", **kw)
    assert got.shape == (2, 128, 64, 3) and np.array_equal(got, want)


class _Recorder:
    """A UNet stand-in that records its inputs and predicts zero noise."""

    def __init__(self):
        self.config, self.dtype, self.calls = _Cfg(sample_size=16), torch.float32, []

    def __call__(self, x, t, encoder_hidden_states):
        self.calls.append((x.clone(), encoder_hidden_states.clone()))
        return _Cfg(sample=torch.zeros((x.shape[0], 4) + tuple(x.shape[2:])))


def test_oracle_tiling_known_answer(small_oracle):
    """2 prompts x 2 images per prompt, one image per prompt: prompt rows [a, a, b, b]; mask and masked-image latent rows [a, b, a, b]."""
    from ladi_oracle.inpaint_pipeline import OracleInpaintPipeline
    from ladi_oracle.parts import DDIMScheduler
    _, ov = small_oracle
    image, mask = _inputs(2)
    g = torch.Generator().manual_seed(4)
    pe, ne = torch.randn((2, 77, 128), generator=g), torch.randn((2, 77, 128), generator=g)
    rec = _Recorder()
    pipe = OracleInpaintPipeline(ov, rec, DDIMScheduler())
    pipe.trace = {}
    pipe(image, mask, pe, ne, height=128, width=64, num_inference_steps=1, guidance_scale=7.5, num_images_per_prompt=2,
         generator=torch.Generator().manual_seed(5))
    x, ctx = rec.calls[0]
    assert x.shape == (8, 9, 16, 8) and ctx.shape == (8, 77, 128)
    for r, p in enumerate([0, 0, 1, 1]):  # [uncond x4, cond x4], each grouped per prompt
        assert torch.equal(ctx[r], ne[p]) and torch.equal(ctx[4 + r], pe[p])
    m, ml = pipe.trace["mask_latents"], pipe.trace["masked_latents"]
    for r, i in enumerate([0, 1, 0, 1]):
        assert torch.equal(m[r], m[i]) and torch.equal(ml[r], ml[i])
        assert torch.equal(x[r, 4:5], m[r]) and torch.equal(x[4 + r, 5:9], ml[r])
    assert not torch.equal(m[0], m[1]) and not torch.equal(ml[0], ml[1])
    lat = x[:4, :4]
    assert all(not torch.equal(lat[i], lat[j]) for i in range(4) for j in range(i))  # one initial-latent draw per sample
    assert torch.equal(x[:4, :4], x[4:, :4])


# ---- the C++ UNet launch sequence at 9 input channels -----------------------------------------------------------------------------------
@pytest.mark.parametrize("B,h,w", [(2, 16, 8), (4, 8, 16)])
def test_unet9_sequence_matches_python(record, B, h, w):
    """As test_engine_trace.py does for 31 channels: the input pitch is 16 (9 channels rounded up to 8), conv_in reads K = 81."""
    from ladi_vton_b200 import UNet2DConditionModel, engine as eng, synthetic as S, unet_param_shapes
    cfg = {**S.SMALL_UNET, "in_channels": 9}
    unet = UNet2DConditionModel(**cfg)
    unet._sd = S.random_state_dict(unet_param_shapes(cfg), 1)
    unet.device = torch.device("cpu")
    unet._pack()
    assert unet.in_pitch == 16
    e = eng.Engine(eng.flatten(unet.P), plan_only=True, **unet.engine_config())
    assert e.query(eng.Q_IN_PITCH) == 16 and e.query(eng.Q_TEMB_TOTAL) == unet.temb_total and e.query(eng.Q_KV_TOTAL) == unet.kv_total
    unet._steps = torch.zeros((4, unet.temb_total))
    unet._ctx = torch.zeros((B, 77, unet.kv_total), dtype=torch.bfloat16)
    unet.forward_nhwc(torch.zeros((B, h, w, 16), dtype=torch.bfloat16), torch.zeros(2, dtype=torch.int32))
    assert compare(record.RECORD, e.trace(eng.MODULE_UNET, B, h, w), "UNet forward, 9 input channels") > 300
    assert e.workspace_bytes(eng.MODULE_UNET, B, h, w) > 0
