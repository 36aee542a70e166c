"""CPU tests of the EMASC forms (linear; nonlinear 3x3 and 1x1) and of the inversion adapter with L encoder layers that src/eval.py and the
training scripts build: state-dict keys and shapes equal the reference classes' (golden written by tests/golden/make_forms_golden.py from
the reference's own emasc.py / inversion_adapter.py), unsupported EMASC forms are refused with their reason, the oracle's linear and 1x1
EMASC equal the reference class outputs bit for bit, and the oracle's L-layer adapter equals stacked `transformers` CLIPEncoderLayers."""
import json
import os

import numpy as np
import pytest
import torch

GOLD = os.path.join(os.path.dirname(__file__), "golden")
SHAPES = json.load(open(os.path.join(GOLD, "forms_state_dicts.json")))
CIN, COUT = [128, 128, 128, 256, 512], [128, 256, 512, 512, 512]


@pytest.mark.parametrize("tag,kw", [("emasc_linear", dict(type="linear", kernel_size=3, padding=1)),
                                    ("emasc_linear", dict(type="linear", kernel_size=1, padding=1)),  # the reference ignores kernel_size
                                    ("emasc_nonlinear_k3", dict(kernel_size=3, padding=1)),
                                    ("emasc_nonlinear_k1", dict(kernel_size=1, padding=0))])
def test_emasc_state_dict_matches_reference(tag, kw):
    from ladi_vton_b200 import EMASC
    em = EMASC(CIN, COUT, stride=1, **kw)
    assert {k: list(v) for k, v in em.param_shapes().items()} == SHAPES[tag]
    sd = {k: torch.zeros(v) for k, v in SHAPES[tag].items()}
    em.load_state_dict(sd)  # strict
    bad = dict(sd)
    bad.pop(next(iter(bad)))
    with pytest.raises(RuntimeError, match="state_dict mismatch"):
        em.load_state_dict(bad)


@pytest.mark.parametrize("kw,reason", [(dict(kernel_size=5, padding=2), "MAX_SEG"), (dict(kernel_size=7, padding=3), "MAX_SEG"),
                                       (dict(kernel_size=3, padding=0), "skip add"), (dict(kernel_size=1, padding=1), "skip add"),
                                       (dict(kernel_size=2, padding=1), "skip add"), (dict(kernel_size=3, padding=1, stride=2), "skip add"),
                                       (dict(type="linear", padding=0), "skip add"), (dict(type="gated"), "not implemented")])
def test_unsupported_emasc_forms_are_refused(kw, reason):
    from ladi_vton_b200 import EMASC
    with pytest.raises(NotImplementedError, match=reason):
        EMASC(CIN, COUT, **kw)


@pytest.mark.parametrize("L", [2, 3])
def test_adapter_state_dict_matches_reference(L):
    from ladi_vton_b200 import InversionAdapter
    from ladi_vton_b200.clip import VIT_H_14, _Cfg
    ad = InversionAdapter(input_dim=1280, hidden_dim=1280 * 4, output_dim=1024 * 16, num_encoder_layers=L, config=_Cfg(VIT_H_14))
    assert {k: list(v) for k, v in ad.param_shapes().items()} == SHAPES[f"adapter_L{L}"]


def test_adapter_rejects_zero_layers():
    from ladi_vton_b200 import InversionAdapter
    with pytest.raises(ValueError, match="num_encoder_layers"):
        InversionAdapter(num_encoder_layers=0)


@pytest.mark.parametrize("form,kw", [("linear", dict(type="linear", kernel_size=3, padding=1)), ("k1", dict(kernel_size=1, padding=0))])
def test_oracle_emasc_forms_equal_reference_golden(form, kw):
    """emasc_forms.npz holds the reference EMASC's own outputs (make_forms_golden.py): the oracle must reproduce them bit for bit."""
    from ladi_oracle.emasc_forms import EMASC as OE
    g = np.load(os.path.join(GOLD, "emasc_forms.npz"))
    sd = {k.split("/sd/", 1)[1]: torch.from_numpy(g[k]) for k in g.files if k.startswith(f"{form}/sd/")}
    oe = OE([8, 16], [16, 24], **kw).eval()
    oe.load_state_dict(sd)
    with torch.no_grad():
        y = oe([torch.from_numpy(g[f"{form}/x{i}"]) for i in range(2)])
    for i in range(2):
        assert torch.equal(y[i], torch.from_numpy(g[f"{form}/y{i}"])), f"{form} scale {i}"
    from ladi_vton_b200 import EMASC  # the engine model accepts the same state dict
    EMASC([8, 16], [16, 24], **kw).load_state_dict(sd)


@pytest.mark.parametrize("L", [2, 3])
def test_oracle_adapter_equals_stacked_transformers_layers(L):
    """oracle InversionAdapter(num_encoder_layers=L) == inversion_adapter.py:22-28 with transformers' CLIPEncoderLayer (the class the
    reference instantiates at :9), same weights."""
    from transformers import CLIPVisionConfig
    from transformers.models.clip.modeling_clip import CLIPEncoderLayer
    from ladi_oracle.parts import InversionAdapter as OA
    from ladi_vton_b200 import synthetic as S
    d, heads, mlp = 64, 4, 128
    oa = OA(input_dim=d, hidden_dim=96, output_dim=80, heads=heads, mlp_dim=mlp, num_encoder_layers=L).eval()
    sd = S.random_state_dict({k: tuple(v.shape) for k, v in oa.state_dict().items()}, 11)
    for k in sd:
        if "layer_norm" in k or "post_layernorm" in k:  # non-trivial LayerNorm affine
            sd[k] = sd[k] + 0.1 * torch.randn(sd[k].shape, generator=torch.Generator().manual_seed(len(k)))
    oa.load_state_dict(sd)
    cfg = CLIPVisionConfig(hidden_size=d, intermediate_size=mlp, num_attention_heads=heads, hidden_act="gelu", layer_norm_eps=1e-5,
                           attention_dropout=0.0)
    cfg._attn_implementation = "eager"
    layers = torch.nn.ModuleList([CLIPEncoderLayer(cfg) for _ in range(L)]).eval()
    layers.load_state_dict({k.split(".", 1)[1]: v for k, v in sd.items() if k.startswith("encoder_layers.")})
    x = torch.randn((2, 19, d), generator=torch.Generator().manual_seed(3))
    with torch.no_grad():
        h = x
        for layer in layers:
            h = layer(h, None)  # (hidden_states, attention_mask); the installed transformers has no causal-mask argument
            h = h[0] if isinstance(h, tuple) else h
        ln = torch.nn.functional.layer_norm(h[:, 0], (d,), sd["post_layernorm.weight"], sd["post_layernorm.bias"], 1e-5)
        ref = oa.layers(ln)
        got = oa(x)
    assert torch.allclose(got, ref, rtol=1e-5, atol=1e-5), float((got - ref).abs().max())


def test_hub_constructors_pass_forms_through():
    from ladi_vton_b200 import hub
    sd = {k: torch.zeros(v) for k, v in SHAPES["emasc_linear"].items()}
    em = hub.emasc("vitonhd", state_dict=sd, type="linear")
    assert em.type == "linear" and em.kernel_size == 3
    em = hub.emasc("vitonhd", state_dict={k: torch.zeros(v) for k, v in SHAPES["emasc_nonlinear_k1"].items()}, kernel_size=1, padding=0)
    assert em.kernel_size == 1
    ad = hub.inversion_adapter("vitonhd", state_dict={k: torch.zeros(v) for k, v in SHAPES["adapter_L2"].items()}, num_encoder_layers=2)
    assert ad.num_encoder_layers == 2
