"""Host-side tests of the warping trainer's validation on the engine (`eval_tps.compute_metric`, `python -m ladi_vton_b200.eval_tps`
<- src/train_tps.py:29-92, :283-515): flag-for-flag parity with the trainer's parser (tests/golden/tps_val_flags.json, read from the
reference source by tests/golden/make_tps_val_golden.py), the stage the trainer validated a checkpoint's epoch in, the errors (each raised
before the GPU is touched), the VGG-19 oracle tap for tap against torchvision's own `vgg19().features`, and the fp32 oracle body against
what the reference's own compute_metric returned (tests/golden/tps_val_small.npz).  No GPU needed."""
import importlib.util
import inspect
import json
import os

import numpy as np
import pytest
import torch

HERE = os.path.dirname(__file__)
GOLD = json.load(open(os.path.join(HERE, "golden", "tps_val_flags.json")))
SMALL = np.load(os.path.join(HERE, "golden", "tps_val_small.npz"))
ENGINE = {"--reference_src", "--vgg_weights", "--random_init", "--synthetic_samples", "--stage", "--output_json"}
SHARED = {"--dataset", "--dresscode_dataroot", "--checkpoints_dir", "--vitonhd_dataroot", "--exp_name", "-b", "-j", "--height", "--width",
          "--dense", "--vgg_weight", "--epochs_tps"}


def _generator():
    spec = importlib.util.spec_from_file_location("make_tps_val_golden", os.path.join(HERE, "golden", "make_tps_val_golden.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_flags_match_reference_trainer():
    from ladi_vton_b200.eval_tps import TRAINING_ONLY, build_parser
    parser = build_parser()
    acts = {a.option_strings[0]: a for a in parser._actions if a.option_strings and a.option_strings[0] != "-h"}
    engine = {a.option_strings[0] for g in parser._action_groups if g.title == "engine" for a in g._group_actions}
    assert engine == ENGINE and set(acts) - engine == SHARED
    ref = {f["flags"][0]: f for f in GOLD["flags"]}
    assert len(ref) == 21 and not (engine & set(ref))
    assert set(ref) - SHARED == set(TRAINING_ONLY) and len(TRAINING_ONLY) == len(set(TRAINING_ONLY))
    for name in SHARED:
        f, a = ref[name], acts[name]
        assert a.option_strings == f["flags"]
        if "action" in f:
            assert f["action"] == "store_true" and a.const is True and a.nargs == 0, f
        else:
            assert a.type.__name__ == f["type"], f
        assert a.dest == f.get("dest", a.dest)
        if "default_src" in f:  # PROJECT_ROOT / "TPS_checkpoints": resolved from --reference_src (checkpoints_dir below)
            assert f["default_src"] == "str(PROJECT_ROOT / 'TPS_checkpoints')" and a.default is None
        else:
            assert a.default == f.get("default"), f
        assert bool(a.required) == bool(f.get("required", False)), f
        assert (list(a.choices) if a.choices else None) == f.get("choices"), f


def test_validation_function_and_dataset_surface():
    from ladi_vton_b200.eval_tps import OUTPUTLIST, compute_metric
    assert list(inspect.signature(compute_metric).parameters) == GOLD["compute_metric_params"]
    sig = inspect.signature(compute_metric).parameters
    assert sig["refinement"].default is None and sig["height"].default == 512 and sig["width"].default == 384
    assert OUTPUTLIST == GOLD["outputlist"]


@pytest.mark.parametrize("epoch,stage", [(50, "tps"), (51, "refinement"), (1, "tps"), (100, "refinement")])
def test_stage_follows_the_trainers_epochs(epoch, stage):
    from ladi_vton_b200.eval_tps import infer_stage
    assert infer_stage("auto", epoch, 50) == stage
    assert infer_stage("tps", epoch, 50) == "tps" and infer_stage("refinement", epoch, 50) == "refinement"


def _checkpoint(path, epoch):
    os.makedirs(os.path.dirname(path), exist_ok=True)
    torch.save({"epoch": epoch, "tps": {}, "refinement": {}, "optimizer_tps": {"state": {}}, "optimizer_ref": {"state": {}}}, path)


def test_checkpoint_resolution_and_stage(tmp_path):
    from ladi_vton_b200.eval_tps import check_args, checkpoint_file, parse_args
    src = tmp_path / "ladi-vton" / "src"
    os.makedirs(src)
    base = ["--dataset", "vitonhd", "--exp_name", "e", "--synthetic_samples", "2", "--vgg_weight", "0"]
    args = parse_args(base + ["--reference_src", str(src)])
    assert checkpoint_file(args) == str(tmp_path / "ladi-vton" / "TPS_checkpoints" / "e" / "checkpoint_last.pth")
    _checkpoint(checkpoint_file(args), 50)
    assert check_args(args)[1:] == (50, "tps")
    _checkpoint(checkpoint_file(args), 51)
    assert check_args(args)[1:] == (51, "refinement")
    args = parse_args(base + ["--checkpoints_dir", str(tmp_path / "ladi-vton" / "TPS_checkpoints"), "--epochs_tps", "60"])
    assert check_args(args)[1:] == (51, "tps")


@pytest.fixture
def no_cuda(monkeypatch):
    from ladi_vton_b200 import lib

    def touched(*a, **k):
        raise AssertionError("the GPU was touched before the argument error")
    monkeypatch.setattr(lib, "load", touched)
    monkeypatch.setattr(torch.cuda, "is_available", touched)
    monkeypatch.setattr(torch.cuda, "current_device", touched)


def test_argument_errors_before_the_gpu(tmp_path, no_cuda):
    from ladi_vton_b200.eval_tps import main
    with pytest.raises(ValueError, match="VitonHD dataroot must be provided"):
        main(["--dataset", "vitonhd", "--exp_name", "e"])
    with pytest.raises(ValueError, match="DressCode dataroot must be provided"):
        main(["--dataset", "dresscode", "--exp_name", "e"])
    syn = ["--dataset", "vitonhd", "--exp_name", "e", "--synthetic_samples", "2"]
    with pytest.raises(ValueError, match="--reference_src"):
        main(syn)
    missing = str(tmp_path / "ck" / "e" / "checkpoint_last.pth")
    with pytest.raises(FileNotFoundError, match=missing.replace("\\", "\\\\")):
        main(syn + ["--checkpoints_dir", str(tmp_path / "ck")])
    _checkpoint(missing, 3)
    with pytest.raises(FileNotFoundError, match="--vgg_weights"):
        main(syn + ["--checkpoints_dir", str(tmp_path / "ck")])


def test_random_init_is_epoch_zero():
    from ladi_vton_b200.eval_tps import check_args, parse_args
    base = ["--dataset", "vitonhd", "--exp_name", "e", "--synthetic_samples", "2", "--random_init"]
    assert check_args(parse_args(base))[1:] == (0, "tps")
    assert check_args(parse_args(base + ["--stage", "refinement"]))[1:] == (0, "refinement")


def test_compute_metric_refuses_other_criteria():
    """Losses accumulate on the device: torch.nn.L1Loss() (mean) is taken as vgg.L1Loss(); other callables raise before any work."""
    from ladi_vton_b200.eval_tps import compute_metric
    with pytest.raises(TypeError, match="criterion_l1"):
        compute_metric([], None, lambda a, b: (a - b).abs().mean(), None)
    with pytest.raises(TypeError, match="criterion_l1"):
        compute_metric([], None, torch.nn.L1Loss(reduction="sum"), None)
    with pytest.raises(TypeError, match="criterion_vgg"):
        compute_metric([], None, torch.nn.L1Loss(), object())


@pytest.mark.skipif(torch.cuda.is_available(), reason="CPU-only check")
def test_cli_has_no_cpu_path(tmp_path):
    from ladi_vton_b200.eval_tps import main
    with pytest.raises(RuntimeError, match="no CPU path"):
        main(["--dataset", "vitonhd", "--exp_name", "e", "--synthetic_samples", "2", "--random_init"])


def test_synthetic_samples_have_the_trainers_keys():
    from ladi_vton_b200.eval_tps import OUTPUTLIST
    from ladi_vton_b200.inference import SyntheticTryOnDataset
    s = SyntheticTryOnDataset(2, (64, 48), outputlist=OUTPUTLIST + ["dense_uv"])[1]
    assert list(s) == OUTPUTLIST + ["dense_uv"]
    assert s["c_name"] == "00001_00.jpg" and s["im_cloth"].shape == (3, 64, 48) and s["dense_uv"].shape == (2, 64, 48)
    assert float(s["im_cloth"].min()) >= -1 and float(s["im_cloth"].max()) <= 1 and float(s["dense_uv"].abs().max()) <= 1


def test_oracle_vgg_taps_bit_exact_against_torchvision():
    import torchvision
    from ladi_oracle.vgg import VGG19
    g = _generator()
    tv = torchvision.models.vgg19(weights=None).eval()
    tv.load_state_dict(g.vgg_state_dict(), strict=False)
    sd = tv.state_dict()
    ov = VGG19().load_torchvision(sd).eval()
    x = torch.randn((2, 3, 40, 32), generator=torch.Generator().manual_seed(3))
    f = tv.features
    with torch.no_grad():
        taps, h = [], x
        for lo, hi in ((0, 2), (2, 7), (7, 12), (12, 21), (21, 30)):
            h = f[lo:hi](h)
            taps.append(h.clone())
        mine = ov(x)
    assert len(mine) == 5
    for a, b in zip(mine, taps):
        assert torch.equal(a, b)


def test_engine_vgg_key_contract():
    import torchvision
    from ladi_vton_b200.vgg import VGG19, resized_size
    sd = torchvision.models.vgg19(weights=None).state_dict()
    m = VGG19()
    want = m.param_shapes()
    assert set(want) == {k for k in sd if k.startswith("features.") and int(k.split(".")[1]) < 30}
    assert all(tuple(sd[k].shape) == want[k] for k in want)
    m.load_state_dict(sd)  # classifier.* and features.30+ are accepted and dropped
    assert resized_size(512, 384) == (341, 256) and resized_size(256, 192) == (341, 256) and resized_size(384, 512) == (256, 341)


@pytest.mark.parametrize("case", ["tps", "refinement", "refinement_dense", "refinement_no_vgg"])
def test_oracle_body_matches_reference_function(case):
    from ladi_oracle.tps_val_body import compute_metric
    from ladi_oracle.vgg import VGG19, VGGLoss
    from ladi_oracle.warp import ConvNet_TPS, UNetVanilla
    g = _generator()
    dense, with_ref, with_vgg = g.CASES[case]
    tsd, rsd = g.warp_state_dicts(dense)
    tps = ConvNet_TPS(256, 192, 5 if dense else 21, 3).eval()
    tps.load_state_dict(tsd, strict=False)
    ref = UNetVanilla(8 if dense else 24, 3).eval()
    ref.load_state_dict(rsd)
    vgg = VGGLoss(VGG19().load_torchvision(g.vgg_state_dict())) if with_vgg else None
    loss, vgg_loss, _ = compute_metric(g.batches(dense), tps, vgg, ref if with_ref else None, g.H, g.W)
    want = SMALL[case]
    print(f"{case}: oracle {loss:.7f} {vgg_loss:.7f}  reference {want[0]:.7f} {want[1]:.7f}")
    assert abs(loss - want[0]) <= 1e-5 * abs(want[0])
    assert abs(vgg_loss - want[1]) <= 1e-5 * abs(want[1]) if with_vgg else vgg_loss == 0 == want[1]
