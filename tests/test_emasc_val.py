"""Host-side tests of the EMASC trainer's validation on the engine (`eval.extract_save_vae_images`, `python -m ladi_vton_b200.eval_emasc`
<- src/train_emasc.py:431-472, src/utils/image_from_pipe.py:221-258): flag-for-flag parity with the trainer's parser and the function's
parameters (golden read from the reference source by tests/golden/make_emasc_val_golden.py), checkpoint discovery and the folder name,
the errors (each raised before the GPU is touched), the fp32 oracle body pinned to what the reference's own function hands to
torchvision.utils.save_image (tests/golden/emasc_val_small.npz), and the host image writer byte for byte against torchvision's.
No GPU needed."""
import importlib.util
import inspect
import json
import os

import numpy as np
import pytest
import torch

HERE = os.path.dirname(__file__)
GOLD = json.load(open(os.path.join(HERE, "golden", "emasc_val_flags.json")))
SMALL = np.load(os.path.join(HERE, "golden", "emasc_val_small.npz"))
BASE = ["--dataset", "vitonhd", "--output_dir", "o"]
ENGINE = {"--emasc_dir", "--emasc_name", "--save_name", "--reference_src", "--random_init", "--synthetic_samples", "--compute_metrics",
          "--metrics_weights_dir"}
SHARED = {"--dataset", "--dresscode_dataroot", "--vitonhd_dataroot", "--output_dir", "--pretrained_model_name_or_path", "--seed",
          "--test_batch_size", "--num_workers_test", "--test_order", "--emasc_type", "--emasc_kernel", "--emasc_padding"}


def _generator():
    """tests/golden/make_emasc_val_golden.py, for the inputs, weights and forms the golden was written with."""
    spec = importlib.util.spec_from_file_location("make_emasc_val_golden", os.path.join(HERE, "golden", "make_emasc_val_golden.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_flags_match_reference_trainer():
    from ladi_vton_b200.eval_emasc import TRAINING_ONLY, build_parser
    parser = build_parser()
    acts = {a.option_strings[0]: a for a in parser._actions if a.option_strings and a.option_strings[0] != "-h"}
    engine = {a.option_strings[0] for g in parser._action_groups if g.title == "engine" for a in g._group_actions}
    assert engine == ENGINE and set(acts) - engine == SHARED
    ref = {f["flags"][0]: f for f in GOLD["flags"]}
    assert len(ref) == 32 and not (engine & set(ref))
    assert set(ref) - SHARED == set(TRAINING_ONLY) and len(TRAINING_ONLY) == len(set(TRAINING_ONLY))
    for name in SHARED:
        f, a = ref[name], acts[name]
        assert a.option_strings == f["flags"]
        assert a.type.__name__ == f["type"], f
        assert a.default == f.get("default"), f
        assert bool(a.required) == bool(f.get("required", False)), f
        assert (list(a.choices) if a.choices else None) == f.get("choices"), f


def test_validation_function_and_dataset_surface():
    """image_from_pipe.py:221-224 parameters, the trainer's test outputlist and categories, and the :446 folder name."""
    from ladi_vton_b200.eval import extract_save_vae_images
    from ladi_vton_b200.eval_emasc import CATEGORIES, OUTPUTLIST
    from ladi_vton_b200.eval_inversion_adapter import SAVE_NAME
    assert list(inspect.signature(extract_save_vae_images).parameters) == GOLD["function_params"]
    assert OUTPUTLIST == GOLD["outputlist"] and CATEGORIES == GOLD["category"]
    assert SAVE_NAME.format(1500) == GOLD["save_name"].format(global_step=1500)


def _touch(d, names):
    for n in names:
        open(os.path.join(d, n), "wb").close()


def test_checkpoint_and_save_name(tmp_path):
    """`latest` takes the highest step among `emasc_*` in --emasc_dir (default --output_dir), the folder is named after that step, and
    the inversion adapter's discovery, which shares the function, is unchanged."""
    from ladi_vton_b200 import eval_inversion_adapter as A
    from ladi_vton_b200.eval_emasc import check_args, parse_args
    d = str(tmp_path)
    _touch(d, ["emasc_500.pth", "emasc_40000.pth", "emasc_9000.pth", "inversion_adapter_70000.pth", "unet_99999.pth", "notes.txt"])
    assert A.default_save_name(parse_args(["--dataset", "vitonhd", "--output_dir", d]), "emasc") == "imgs_step_40000"
    other = ["--dataset", "vitonhd", "--output_dir", "elsewhere", "--emasc_dir", d, "--synthetic_samples", "1"]
    assert check_args(parse_args(other + ["--random_init"]))[1] == "imgs_step_random_init"
    args = parse_args(other)
    args.pretrained_model_name_or_path = _vae_root(tmp_path)
    assert check_args(args)[1] == "imgs_step_40000"
    args.emasc_name = "emasc_500.pth"
    assert check_args(args)[1] == "imgs_step_500"
    args.save_name = "mine"
    assert check_args(args)[1] == "mine"
    assert parse_args(["--dataset", "vitonhd", "--output_dir", d]).emasc_dir == d
    ia = A.parse_args(["--dataset", "vitonhd", "--output_dir", d])
    assert A.default_save_name(ia) == A.default_save_name(ia, "inversion_adapter") == "imgs_step_70000"


def _vae_root(tmp_path, **over):
    from ladi_vton_b200.vae import SD2_VAE
    root = tmp_path / "sd"
    os.makedirs(root / "vae", exist_ok=True)
    cfg = {"_class_name": "AutoencoderKL", "act_fn": "silu", "sample_size": 512, **{k: v for k, v in SD2_VAE.items() if k != "sample_size"}}
    cfg["block_out_channels"] = list(cfg["block_out_channels"])
    json.dump({**cfg, **over}, open(root / "vae" / "config.json", "w"))
    return str(root)


@pytest.fixture
def no_cuda(monkeypatch):
    """Any step towards the GPU fails the test: the errors below must come first."""
    from ladi_vton_b200 import lib

    def touched(*a, **k):
        raise AssertionError("the GPU was touched before the argument error")
    monkeypatch.setattr(lib, "load", touched)
    monkeypatch.setattr(torch.cuda, "is_available", touched)
    monkeypatch.setattr(torch.cuda, "current_device", touched)


def test_argument_errors_before_the_gpu(tmp_path, no_cuda):
    from ladi_vton_b200.eval_emasc import main
    out = str(tmp_path / "run")
    with pytest.raises(ValueError, match="VitonHD dataroot must be provided"):
        main(["--dataset", "vitonhd", "--output_dir", out])
    with pytest.raises(ValueError, match="DressCode dataroot must be provided"):
        main(["--dataset", "dresscode", "--output_dir", out])
    syn = ["--dataset", "vitonhd", "--output_dir", out, "--synthetic_samples", "2"]
    with pytest.raises(NotImplementedError, match="MAX_SEG"):  # vae.EMASC's message for a 5x5 kernel
        main(syn + ["--random_init", "--emasc_kernel", "5", "--emasc_padding", "2"])
    with pytest.raises(FileNotFoundError, match="config.json"):
        main(syn + ["--pretrained_model_name_or_path", str(tmp_path / "nothing")])
    with pytest.raises(ValueError, match="latent_channels"):
        main(syn + ["--pretrained_model_name_or_path", _vae_root(tmp_path, latent_channels=16)])
    with pytest.raises(ValueError, match="block_out_channels"):
        main(syn + ["--pretrained_model_name_or_path", _vae_root(tmp_path, block_out_channels=[64, 128, 256, 256])])
    ck = tmp_path / "ck"
    os.makedirs(ck)
    _touch(str(ck), ["emasc_final.pth"])
    with pytest.raises(ValueError, match="--save_name"):
        main(syn + ["--pretrained_model_name_or_path", _vae_root(tmp_path), "--emasc_dir", str(ck), "--emasc_name", "emasc_final.pth"])
    assert not os.path.exists(out)


def test_sd15_vae_is_accepted(tmp_path):
    """Only the VAE is read, and SD-1.5 inpainting's VAE is the same architecture: no text encoder, tokenizer or base-model name check."""
    from ladi_vton_b200.eval_emasc import check_args, parse_args
    root = _vae_root(tmp_path, scaling_factor=0.18215, sample_size=256)
    args = parse_args(BASE + ["--synthetic_samples", "1", "--pretrained_model_name_or_path", root, "--save_name", "s"])
    assert check_args(args)[1] == "s"
    check_args(parse_args(BASE + ["--synthetic_samples", "1", "--random_init", "--pretrained_model_name_or_path",
                                  "runwayml/stable-diffusion-inpainting"]))


@pytest.mark.skipif(torch.cuda.is_available(), reason="CPU-only check")
def test_cli_has_no_cpu_path(tmp_path):
    from ladi_vton_b200.eval_emasc import main
    with pytest.raises(RuntimeError, match="no CPU path"):
        main(["--dataset", "vitonhd", "--output_dir", str(tmp_path), "--synthetic_samples", "2", "--random_init"])
    assert os.listdir(tmp_path) == []


def _oracle(form, vsd, esd, ein, eout, forms):
    from ladi_oracle.emasc_forms import EMASC as OE
    from ladi_oracle.vae import AutoencoderKL as OV
    from ladi_vton_b200 import synthetic as S
    ov = OV(**S.SMALL_VAE).eval()
    ov.load_state_dict(vsd)
    kw = dict(forms[form][0])
    oe = OE(ein, eout, kernel_size=kw["kernel_size"], padding=kw["padding"], type=kw["type"]).eval()
    oe.load_state_dict(esd[form])
    return ov, oe


@pytest.mark.parametrize("form", ["nonlinear_k3", "nonlinear_k1", "linear"])
def test_oracle_body_matches_reference_function(form):
    """The fp32 oracle body, with the global RNG seeded as the generator seeded it, reproduces the tensors the reference's own
    extract_save_vae_images passed to save_image (the bound of the train_emasc pin)."""
    from ladi_oracle.vae_val_body import run_batch
    g = _generator()
    vsd, esd, (ein, eout) = g.state_dicts()
    ov, oe = _oracle(form, vsd, esd, ein, eout, g.FORMS)
    torch.manual_seed(g.SEED)
    out = run_batch(g.inputs(), ov, oe, g.INT_LAYERS, g.FORMS[form][0]["type"])
    ref = SMALL[f"{form}/images"]
    assert out.shape == ref.shape == (2, 3, g.H, g.W)
    err = np.abs(out.numpy() - ref).max()
    print(f"{form}: max |oracle - reference| = {err:.2e}")
    assert err < 1e-4
    assert list(SMALL[f"{form}/names"]) == ["upper_body/00001_00.jpg", "lower_body/00002_00.jpg"]


@pytest.mark.parametrize("ext", ["jpg", "png"])
def test_host_writer_matches_torchvision(tmp_path, ext):
    """The golden tensors, quantised by save_image's own expression and written by eval.write_image, give the same bytes as
    torchvision.utils.save_image(t, path) called without `quality` (what the reference's call amounts to)."""
    import torchvision
    from ladi_oracle.vae_val_body import save_image_u8
    from ladi_vton_b200.eval import write_image
    for form in ("nonlinear_k3", "nonlinear_k1", "linear"):
        for i, t in enumerate(torch.from_numpy(SMALL[f"{form}/images"])):
            a, b = tmp_path / f"{form}_{i}_engine.{ext}", tmp_path / f"{form}_{i}_tv.{ext}"
            write_image(save_image_u8(t).numpy(), str(a))
            torchvision.utils.save_image(t, str(b))
            assert a.read_bytes() == b.read_bytes(), (form, i, ext)


def test_quantisation_expression_is_save_images():
    """save_image_u8 is torchvision's `mul(255).add_(0.5).clamp_(0, 255)` + uint8 cast, including at the rounding ties, where it differs
    from numpy_to_pil's round-half-to-even (image_out_u8)."""
    from ladi_oracle.vae_val_body import save_image_u8
    k = torch.arange(256, dtype=torch.float32)
    t = ((k + 0.5) / 255).reshape(1, 1, 256).expand(3, 1, 256).contiguous()
    u = save_image_u8(t)[0, :, 0].long()
    assert torch.equal(u, t[0, 0].mul(255).add(0.5).clamp(0, 255).to(torch.uint8).long())
    assert (u != t[0, 0].mul(255).round().clamp(0, 255).long()).any()
