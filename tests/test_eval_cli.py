"""Host-side tests of the evaluation CLI mirror (ladi_vton_b200/eval.py <- src/eval.py) and of the CLIP cloth-feature cache writer
(ladi_vton_b200/compute_cloth_clip_features.py <- src/utils/compute_cloth_clip_features.py): flag-for-flag parity with the reference
parser (golden read from the reference source by tests/golden/make_eval_golden.py), `latest` checkpoint discovery, the reference's error
texts, the UNet width rule, and the cache files' names, dtype, shape and pickled name list.  No GPU needed."""
import json
import os
import pickle

import pytest
import torch

GOLD = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "eval_flags.json")))
BASE = ["--dataset", "vitonhd", "--output_dir", "o", "--save_name", "s", "--test_order", "paired", "--unet_dir", "u"]


def test_flags_match_reference_parser():
    from ladi_vton_b200.eval import build_parser
    parser = build_parser()
    acts = {a.option_strings[0]: a for a in parser._actions if a.option_strings and a.option_strings[0] != "-h"}
    engine = {a.option_strings[0] for g in parser._action_groups if g.title == "engine" for a in g._group_actions}
    assert engine == {"--vision_model_name_or_path", "--reference_src", "--random_init", "--synthetic_samples"}
    ref_names = [f["flags"][0] for f in GOLD["flags"]]
    assert len(ref_names) == 31
    assert sorted(set(acts) - engine) == sorted(ref_names)
    for f in GOLD["flags"]:
        a = acts[f["flags"][0]]
        assert a.option_strings == f["flags"]
        if f.get("action") == "store_true":
            assert a.nargs == 0 and a.const is True and a.default is False
        else:
            assert a.type.__name__ == f["type"], f
            assert a.default == f.get("default"), f
        assert bool(a.required) == bool(f.get("required", False)), f
        assert (list(a.choices) if a.choices else None) == f.get("choices"), f


def _touch(d, names):
    for n in names:
        open(os.path.join(d, n), "wb").close()


def test_latest_checkpoint_discovery(tmp_path):
    """src/eval.py:187-195 (and the emasc / inversion adapter twins): highest numeric suffix among the files with the prefix."""
    from ladi_vton_b200.eval import checkpoint_path
    assert GOLD["latest_prefixes"] == ["unet", "emasc", "inversion_adapter"]
    d = str(tmp_path)
    _touch(d, ["unet_9000.pth", "unet_40000.pth", "unet_500.pth", "emasc_12.pth", "emasc_3.pth", "inversion_adapter_7.pth",
               "inversion_adapter_70.pth", "optimizer_99999.pth", "notes.txt"])
    assert checkpoint_path(d, "latest", "unet") == os.path.join(d, "unet_40000.pth")
    assert checkpoint_path(d, "latest", "emasc") == os.path.join(d, "emasc_12.pth")
    assert checkpoint_path(d, "latest", "inversion_adapter") == os.path.join(d, "inversion_adapter_70.pth")
    assert checkpoint_path(d, "unet_9000.pth", "unet") == os.path.join(d, "unet_9000.pth")  # an explicit name is used as given
    assert checkpoint_path(d, "anything.bin", "unet") == os.path.join(d, "anything.bin")


def test_reference_errors():
    from ladi_vton_b200.eval import check_args, parse_args
    with pytest.raises(ValueError, match="VitonHD dataroot must be provided"):
        check_args(parse_args(BASE))
    dc = ["--dataset", "dresscode"] + BASE[2:]
    with pytest.raises(ValueError, match="DressCode dataroot must be provided"):
        check_args(parse_args(dc))
    ok = BASE + ["--vitonhd_dataroot", "/data"]
    with pytest.raises(ValueError, match=r"No EMASC checkpoint found. Make sure to specify --emasc_dir"):
        check_args(parse_args(ok + ["--inversion_adapter_dir", "a"]))
    with pytest.raises(ValueError, match=r"No inversion adapter checkpoint found. Make sure to specify --inversion_adapter_dir"):
        check_args(parse_args(ok + ["--emasc_dir", "e"]))
    check_args(parse_args(ok + ["--emasc_dir", "e", "--inversion_adapter_dir", "a"]))
    check_args(parse_args(ok + ["--emasc_type", "none", "--text_usage", "noun_chunks"]))
    check_args(parse_args(BASE + ["--synthetic_samples", "2", "--random_init"]))
    with pytest.raises(NotImplementedError, match="1.5 inpainting base"):
        check_args(parse_args(ok + ["--emasc_dir", "e", "--inversion_adapter_dir", "a", "--pretrained_model_name_or_path",
                                    "runwayml/stable-diffusion-inpainting"]))


def test_sd15_local_folder_is_refused(tmp_path):
    from ladi_vton_b200.eval import check_args, parse_args
    os.makedirs(tmp_path / "text_encoder")
    json.dump({"hidden_size": 768}, open(tmp_path / "text_encoder" / "config.json", "w"))
    with pytest.raises(NotImplementedError, match="not built"):
        check_args(parse_args(BASE + ["--synthetic_samples", "1", "--random_init", "--pretrained_model_name_or_path", str(tmp_path)]))


def test_outputlist_and_unet_width():
    """src/eval.py:166 and :235-277."""
    from ladi_vton_b200.eval import outputlist_for, parse_args
    a = parse_args(BASE)
    assert outputlist_for(a) == ['image', 'pose_map', 'captions', 'inpaint_mask', 'im_mask', 'category', 'im_name', 'warped_cloth', 'cloth']
    a = parse_args(BASE + ["--cloth_input_type", "none", "--use_clip_cloth_features"])
    assert outputlist_for(a)[-1] == 'clip_cloth_features' and 'warped_cloth' not in outputlist_for(a)
    assert 'cloth' not in outputlist_for(parse_args(BASE + ["--text_usage", "none"]))
    from ladi_vton_b200 import UNet2DConditionModel
    from ladi_vton_b200.unet import unet_param_shapes
    for cit, c in (("none", 27), ("warped", 31)):
        u = UNet2DConditionModel(in_channels=27 if cit == "none" else 31)
        assert unet_param_shapes(dict(u.config))["conv_in.weight"][1] == c


def test_synthetic_dataset_eval_keys():
    from ladi_vton_b200.eval import outputlist_for, parse_args
    from ladi_vton_b200.inference import SyntheticTryOnDataset
    ol = outputlist_for(parse_args(BASE + ["--use_clip_cloth_features"]))
    ds = SyntheticTryOnDataset(3, size=(64, 48), outputlist=ol, clip_dim=32)
    b = next(iter(torch.utils.data.DataLoader(ds, batch_size=2)))
    assert sorted(b) == sorted(ol)
    assert b["warped_cloth"].shape == (2, 3, 64, 48) and b["clip_cloth_features"].shape == (2, 257, 32)
    assert b["clip_cloth_features"].dtype == torch.float16 and isinstance(b["captions"][0], str)


@pytest.mark.skipif(torch.cuda.is_available(), reason="CPU-only check")
def test_eval_cli_has_no_cpu_path(tmp_path):
    from ladi_vton_b200.eval import main
    with pytest.raises(RuntimeError, match="no CPU path"):
        main(BASE[:2] + ["--output_dir", str(tmp_path)] + BASE[4:] + ["--synthetic_samples", "2", "--random_init"])
    assert os.listdir(tmp_path) == []


class _FakeVision:
    """Stands in for the CLIP vision tower: last_hidden_state [B, 257, 1280] derived from the pixel values."""

    def __call__(self, pixel_values):
        class _O:
            pass
        o = _O()
        B = pixel_values.shape[0]
        o.last_hidden_state = pixel_values.mean(dim=(1, 2, 3)).view(B, 1, 1).expand(B, 257, 1280) + torch.arange(1280.0) / 1280
        return o


class _FakeProcessor:
    def __call__(self, images, return_tensors="pt"):
        class _O:
            pass
        o = _O()
        o.pixel_values = images * 2 - 1
        return o


class _Clothes(torch.utils.data.Dataset):
    def __init__(self, n, seed):
        self.x = torch.rand((n, 3, 64, 48), generator=torch.Generator().manual_seed(seed)) * 2 - 1
        self.n = n

    def __len__(self):
        return self.n

    def __getitem__(self, i):
        return dict(cloth=self.x[i], c_name=f"{i:05d}_00.jpg")


def test_feature_cache_writer(tmp_path):
    """src/utils/compute_cloth_clip_features.py:143-166: per split, fp16 [N, 257, 1280] last_hidden_state features and the pickled list of
    cloth names, under the names the reference dataset classes read (vitonhd.py:100-107)."""
    from ladi_vton_b200.compute_cloth_clip_features import default_save_dir, save_cloth_features
    assert default_save_dir("/x/ladi-vton/src/", "vitonhd") == os.path.join("/x/ladi-vton", "data", "clip_cloth_embeddings", "vitonhd")
    with pytest.raises(ValueError, match="--save_dir"):
        default_save_dir(None, "vitonhd")
    loader = torch.utils.data.DataLoader(_Clothes(5, 1), batch_size=2, shuffle=False)
    fp, npath = save_cloth_features(loader, _FakeVision(), "test", str(tmp_path / "cache"), torch.device("cpu"), _FakeProcessor())
    assert os.path.basename(fp) == "test_last_hidden_state_features.pt" and os.path.basename(npath) == "test_features_names.pkl"
    feats = torch.load(fp)
    assert feats.dtype == torch.float16 and feats.shape == (5, 257, 1280)
    names = pickle.load(open(npath, "rb"))
    assert names == [f"{i:05d}_00.jpg" for i in range(5)]
    # what vitonhd.py:121-122 does with them
    assert torch.equal(feats[names.index("00003_00.jpg")], feats[3])


def test_feature_cache_cli_args():
    from ladi_vton_b200.compute_cloth_clip_features import build_parser, main
    a = build_parser().parse_args(["--dataset", "dresscode"])
    assert (a.batch_size, a.num_workers, a.pretrained_model_name_or_path) == (16, 8, "stabilityai/stable-diffusion-2-inpainting")
    with pytest.raises(ValueError, match="DressCode dataroot must be provided"):
        main(["--dataset", "dresscode"])
    with pytest.raises(NotImplementedError, match="SD-2"):
        main(["--dataset", "vitonhd", "--vitonhd_dataroot", "/d", "--pretrained_model_name_or_path", "runwayml/stable-diffusion-inpainting"])
