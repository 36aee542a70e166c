"""Writes two goldens from the reference's own model classes (LADI_REFERENCE = a checkout of the reference; src/models/emasc.py needs
only torch.nn, src/models/inversion_adapter.py the installed transformers' CLIPEncoderLayer, both run on the CPU):

  * tests/golden/emasc_forms.npz -- the EMASC 'linear' form and the nonlinear form with kernel_size=1, padding=0 (`--emasc_type linear`,
    `--emasc_kernel 1 --emasc_padding 0` of src/eval.py / train_emasc.py), each with seeded weights on seeded two-scale inputs.  Stored:
    the state dict (key -> array), the inputs and the outputs, under `<form>/...`.
  * tests/golden/forms_state_dicts.json -- state-dict key -> shape of the reference classes as src/eval.py builds them: EMASC linear,
    nonlinear 3x3 and nonlinear 1x1 over the hub channel plan, and InversionAdapter with 2 and 3 encoder layers built with a
    `transformers` CLIPVisionConfig of CLIP ViT-H/14 (hidden 1280, 16 heads, MLP 5120) and output 1024 * 16.

    python tests/golden/make_forms_golden.py
"""
import importlib.util
import json
import os

import numpy as np
import torch

REF = os.environ["LADI_REFERENCE"]
HERE = os.path.dirname(os.path.abspath(__file__))
OUT, SHAPES = os.path.join(HERE, "emasc_forms.npz"), os.path.join(HERE, "forms_state_dicts.json")
IN_CH, OUT_CH, SIZES = [8, 16], [16, 24], [(12, 10), (6, 5)]
FORMS = {"linear": dict(kernel_size=3, padding=1, type="linear"), "k1": dict(kernel_size=1, padding=0, type="nonlinear")}


def _load(name):
    spec = importlib.util.spec_from_file_location(f"ref_{name}", os.path.join(REF, "src", "models", f"{name}.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def shapes():
    from transformers import CLIPVisionConfig
    emasc, adapter = _load("emasc"), _load("inversion_adapter")
    cin, cout = [128, 128, 128, 256, 512], [128, 256, 512, 512, 512]  # src/eval.py:200-201
    sd = lambda m: {k: list(v.shape) for k, v in m.state_dict().items()}  # noqa: E731
    out = {"emasc_linear": sd(emasc.EMASC(cin, cout, kernel_size=3, padding=1, stride=1, type="linear")),
           "emasc_nonlinear_k3": sd(emasc.EMASC(cin, cout, kernel_size=3, padding=1, stride=1, type="nonlinear")),
           "emasc_nonlinear_k1": sd(emasc.EMASC(cin, cout, kernel_size=1, padding=0, stride=1, type="nonlinear"))}
    cfg = CLIPVisionConfig(hidden_size=1280, intermediate_size=5120, num_attention_heads=16, num_hidden_layers=32, image_size=224, patch_size=14)
    for L in (2, 3):  # src/eval.py:253-257
        out[f"adapter_L{L}"] = sd(adapter.InversionAdapter(input_dim=1280, hidden_dim=1280 * 4, output_dim=1024 * 16, config=cfg,
                                                           num_encoder_layers=L))
    json.dump(out, open(SHAPES, "w"), indent=0)


def main():
    shapes()
    mod = _load("emasc")
    out = {}
    for seed, (tag, kw) in enumerate(FORMS.items()):
        torch.manual_seed(100 + seed)
        m = mod.EMASC(IN_CH, OUT_CH, stride=1, **kw).eval()
        g = torch.Generator().manual_seed(200 + seed)
        sd = {k: torch.randn(v.shape, generator=g) * 0.2 for k, v in m.state_dict().items()}
        m.load_state_dict(sd)
        x = [torch.randn((2, c, h, w), generator=g) for c, (h, w) in zip(IN_CH, SIZES)]
        with torch.no_grad():
            y = m([t.clone() for t in x])
        for k, v in sd.items():
            out[f"{tag}/sd/{k}"] = v.numpy()
        for i, (a, b) in enumerate(zip(x, y)):
            out[f"{tag}/x{i}"], out[f"{tag}/y{i}"] = a.numpy(), b.numpy()
    np.savez_compressed(OUT, **out)
    print(f"{len(out)} arrays -> {OUT}")


if __name__ == "__main__":
    main()
