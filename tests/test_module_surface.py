"""CPU tests (no GPU needed): every engine model class shares one reference-facing surface (ladi_vton_b200/module.py) -- a state dict
is checked against `param_shapes()` whatever `strict` says, `.to("cpu")` raises, and the weights are packed once per device and
state dict, with the packing step replaced by a counter so that no kernel runs."""
import pytest
import torch


def _models():
    from ladi_vton_b200 import (EMASC, AutoencoderKL, CLIPTextModel, CLIPVisionModelWithProjection, ConvNet_TPS, InversionAdapter,
                                UNet2DConditionModel, UNetVanilla, synthetic as S)
    from ladi_vton_b200.metrics import FIDInceptionV3, LPIPSAlex
    return {
        "unet": lambda: UNet2DConditionModel(**S.SMALL_UNET),
        "vae": lambda: AutoencoderKL(**S.SMALL_VAE),
        "emasc": lambda: EMASC(*S.emasc_channels(S.SMALL_VAE["block_out_channels"])),
        "adapter": lambda: InversionAdapter(input_dim=128, hidden_dim=256, output_dim=512, heads=2, mlp_dim=256),
        "clip_text": lambda: CLIPTextModel(vocab_size=1000, hidden_size=128, intermediate_size=256, num_hidden_layers=2, num_attention_heads=2),
        "clip_vision": lambda: CLIPVisionModelWithProjection(hidden_size=160, intermediate_size=320, num_hidden_layers=2, num_attention_heads=2),
        "tps": lambda: ConvNet_TPS(32, 32, 6, 1),
        "refinement": lambda: UNetVanilla(24, 3, True, widths=(8, 16, 32, 64, 128)),
        "inception": FIDInceptionV3,
        "lpips": LPIPSAlex,
    }


NAMES = ["unet", "vae", "emasc", "adapter", "clip_text", "clip_vision", "tps", "refinement", "inception", "lpips"]


def _model_and_sd(name):
    m = _models()[name]()
    return m, {k: torch.empty(s) for k, s in m.param_shapes().items()}  # the values are never read: packing is not run here


@pytest.mark.parametrize("strict", [True, False])
@pytest.mark.parametrize("name", NAMES)
def test_missing_or_misshaped_key_raises(name, strict):
    m, sd = _model_and_sd(name)
    k = next(k for k in sd if not m.optional(k))
    with pytest.raises(RuntimeError, match="state_dict mismatch"):
        m.load_state_dict({j: v for j, v in sd.items() if j != k}, strict=strict)
    with pytest.raises(RuntimeError, match="state_dict mismatch"):
        m.load_state_dict({**sd, k: torch.empty(tuple(sd[k].shape) + (2,))}, strict=strict)
    assert m._sd is None


@pytest.mark.parametrize("name", NAMES)
def test_unexpected_key_raises_only_when_strict(name):
    m, sd = _model_and_sd(name)
    sd["not_a_parameter.weight"] = torch.empty(1)
    with pytest.raises(RuntimeError, match="state_dict mismatch"):
        m.load_state_dict(sd)
    assert m.load_state_dict(sd, strict=False) is m
    assert "not_a_parameter.weight" not in m._sd


@pytest.mark.parametrize("name", NAMES)
def test_no_cpu_path(name):
    m, sd = _model_and_sd(name)
    with pytest.raises(RuntimeError, match="no CPU path"):
        m.load_state_dict(sd).to("cpu")


@pytest.mark.parametrize("name", NAMES)
def test_packs_once_per_device_and_state_dict(name, monkeypatch):
    m, sd = _model_and_sd(name)
    packs = []
    monkeypatch.setattr(m, "_pack_weights", lambda: packs.append(m.device))
    monkeypatch.setattr(torch.cuda, "current_device", lambda: 0)
    monkeypatch.setenv("LADI_ENGINE", "0")
    assert m.eval() is m and m.requires_grad_(False) is m
    m.load_state_dict(sd)
    assert packs == [] and m.device.type == "cpu"
    assert m.to("cuda") is m and packs == [torch.device("cuda", 0)] and m.pack_gen == 1
    # the same device again (also spelt with its index, or as a dtype only): nothing is packed again
    for again in ("cuda", "cuda:0", torch.device("cuda")):
        assert m.to(again) is m
    assert m.to(torch.bfloat16) is m and m.to(dtype=torch.float16) is m
    assert len(packs) == 1 and m.pack_gen == 1
    assert m._sd is not None  # host-resident sources are kept
    m.load_state_dict(sd)
    assert len(packs) == 2 and m.pack_gen == 2 and m.engine is None and not m.use_engine()
    m._sd = None  # what packing from device-resident sources leaves
    with pytest.raises(RuntimeError, match="released after packing"):
        m.to("cuda:1")
    assert m.device == torch.device("cuda", 0) and m.to("cuda") is m and len(packs) == 2
