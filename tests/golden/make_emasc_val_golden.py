"""Writes two goldens for the EMASC trainer's validation (LADI_REFERENCE = a checkout of the reference):

  * tests/golden/emasc_val_flags.json, read from the AST as make_adapter_val_golden.py does (the trainer cannot be imported here:
    accelerate is not installed): every `parser.add_argument(...)` of src/train_emasc.py as (flags, type, default, required, choices,
    action); the test datasets' `outputlist` and `category`; the `save_name=` it passes to `extract_save_vae_images` (an f-string over the
    global step, kept as its format string); and the parameter names of `extract_save_vae_images` (src/utils/image_from_pipe.py).
  * tests/golden/emasc_val_small.npz: what the reference's own `extract_save_vae_images` hands to `torchvision.utils.save_image`,
    captured by replacing that function.  The reference module runs unmodified on the diffusers shim (oracle/shim; its
    `StableDiffusionInpaintPipeline` import gets a placeholder, the function does not use it), CPU fp32, with the small VAE config
    (synthetic.SMALL_VAE) and `inputs()`: two 128x96 images in one batch, the global RNG seeded by `torch.manual_seed(SEED)` before each
    call.  One entry per EMASC form of FORMS: `<form>/images` [2,3,128,96] fp32 and `<form>/names` (the paths' last two parts).

    python tests/golden/make_emasc_val_golden.py
"""
import ast
import json
import os
import shutil
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT_FLAGS, OUT_NPZ = os.path.join(HERE, "emasc_val_flags.json"), os.path.join(HERE, "emasc_val_small.npz")
SEED, H, W = 5, 128, 96
INT_LAYERS = [1, 2, 3, 4, 5]
# form -> (EMASC constructor keywords of src/models/emasc.py, state-dict seed)
FORMS = {"nonlinear_k3": (dict(kernel_size=3, padding=1, type="nonlinear"), 1236),
         "nonlinear_k1": (dict(kernel_size=1, padding=0, type="nonlinear"), 1237),
         "linear": (dict(kernel_size=3, padding=1, type="linear"), 1238)}


def inputs():
    """One batch of the trainer's test loader at 128x96: image in [-1, 1], a rectangular inpaint_mask, im_mask = image * (1 - mask)."""
    g = torch.Generator().manual_seed(31)
    image = torch.rand((2, 3, H, W), generator=g) * 2 - 1
    mask = torch.zeros((2, 1, H, W))
    mask[0, :, 24:104, 16:80] = 1
    mask[1, :, 40:120, 8:64] = 1
    return dict(image=image, im_mask=image * (1 - mask), inpaint_mask=mask, category=["upper_body", "lower_body"],
                im_name=["00001_00.jpg", "00002_00.jpg"])


def state_dicts():
    """Seeded small-config VAE weights and, per form, the EMASC weights (synthetic.random_state_dict)."""
    from ladi_vton_b200 import synthetic as S
    from ladi_vton_b200.vae import vae_param_shapes
    ein, eout = S.emasc_channels(S.SMALL_VAE["block_out_channels"])
    em = {f: S.random_state_dict(S.emasc_param_shapes(ein, eout, kw["kernel_size"], kw["type"]), seed) for f, (kw, seed) in FORMS.items()}
    return S.random_state_dict(vae_param_shapes(S.SMALL_VAE), 1235), em, (ein, eout)


def _fstring(node):
    return "".join(v.value if isinstance(v, ast.Constant) else "{" + ast.unparse(v.value) + "}" for v in node.values)


def flags(ref):
    tree = ast.parse(open(os.path.join(ref, "src", "train_emasc.py")).read())
    out, outputlist, category, save_name = [], set(), set(), None
    for node in ast.walk(tree):
        if isinstance(node, ast.Call) and isinstance(node.func, ast.Attribute) and node.func.attr == "add_argument":
            kw = {k.arg: (k.value.id if isinstance(k.value, ast.Name) else ast.literal_eval(k.value)) for k in node.keywords if k.arg != "help"}
            out.append(dict(flags=[ast.literal_eval(a) for a in node.args], line=node.lineno, **kw))
        if isinstance(node, ast.Call) and isinstance(node.func, ast.Name) and node.func.id in ("DressCodeDataset", "VitonHDDataset"):
            kw = {k.arg: k.value for k in node.keywords}
            if ast.literal_eval(kw["phase"]) == "test":
                outputlist.add(tuple(ast.literal_eval(kw["outputlist"])))
                if "category" in kw:
                    category.add(tuple(ast.literal_eval(kw["category"])))
        if isinstance(node, ast.Call) and isinstance(node.func, ast.Name) and node.func.id == "extract_save_vae_images":
            save_name = next(_fstring(k.value) for k in node.keywords if k.arg == "save_name")
    assert len(outputlist) == 1 and len(category) == 1, (outputlist, category)
    out.sort(key=lambda f: f["line"])
    fn = next(n for n in ast.walk(ast.parse(open(os.path.join(ref, "src", "utils", "image_from_pipe.py")).read()))
              if isinstance(n, ast.FunctionDef) and n.name == "extract_save_vae_images")
    return dict(source=["src/train_emasc.py", "src/utils/image_from_pipe.py"], flags=out, outputlist=list(outputlist.pop()),
                category=list(category.pop()), save_name=save_name, function_params=[a.arg for a in fn.args.args])


def run_reference(ref):
    for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "oracle", "shim"), ref):
        sys.path.insert(0, p)
    import diffusers
    diffusers.StableDiffusionInpaintPipeline = object  # imported by image_from_pipe.py, not used by extract_save_vae_images
    import torchvision
    from src.models.AutoencoderKL import AutoencoderKL as RefVAE
    from src.models.emasc import EMASC as RefEMASC
    from src.utils import image_from_pipe
    from ladi_vton_b200 import synthetic as S
    vsd, esd, (ein, eout) = state_dicts()
    vae = RefVAE(in_channels=3, out_channels=3, down_block_types=("DownEncoderBlock2D",) * 4, up_block_types=("UpDecoderBlock2D",) * 4,
                 block_out_channels=S.SMALL_VAE["block_out_channels"], layers_per_block=2, latent_channels=4, norm_num_groups=32,
                 sample_size=H).eval()
    vae.load_state_dict(vsd)
    captured = []
    torchvision.utils.save_image = lambda t, fp, **kw: captured.append((t.detach().clone(), fp, kw))
    out, tmp = {}, tempfile.mkdtemp()
    for form, (kw, _) in FORMS.items():
        emasc = RefEMASC(ein, eout, stride=1, **kw).eval()
        emasc.load_state_dict(esd[form])
        captured.clear()
        torch.manual_seed(SEED)
        image_from_pipe.extract_save_vae_images(vae, emasc, [inputs()], INT_LAYERS, tmp, "paired", "imgs_step_1", kw["type"])
        assert all(k == dict(quality=95) for _, _, k in captured)
        out[f"{form}/images"] = torch.stack([t for t, _, _ in captured]).numpy()
        out[f"{form}/names"] = np.array(["/".join(fp.split(os.sep)[-2:]) for _, fp, _ in captured])
    shutil.rmtree(tmp)
    return out


def main():
    ref = os.environ["LADI_REFERENCE"]
    json.dump(flags(ref), open(OUT_FLAGS, "w"), indent=1)
    torch.set_num_threads(4)
    out = run_reference(ref)
    np.savez_compressed(OUT_NPZ, **out)
    print(f"-> {OUT_FLAGS}, {OUT_NPZ}: " + ", ".join(f"{k} {v.shape}" for k, v in out.items()))


if __name__ == "__main__":
    main()
