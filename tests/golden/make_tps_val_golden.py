"""Writes two goldens for the warping trainer's validation (LADI_REFERENCE = a checkout of the reference):

  * tests/golden/tps_val_flags.json, read from the AST (src/train_tps.py imports wandb and the dataset classes): every
    `parser.add_argument(...)` of src/train_tps.py as (flags, type, default, required, choices, action, dest); a default that is not a
    literal is kept as its source text under `default_src`; the test `outputlist` (`dataset_output_list`) and the parameter names of
    `compute_metric`.
  * tests/golden/tps_val_small.npz: the (loss, vgg_loss) that the reference's own `compute_metric` returns, with its own VGGLoss, ConvNet_TPS
    and UNetVanilla, on CPU fp32 at 256x192 for two batches of B = 2 (`batches(dense)`), in the four cases of CASES.  The module is
    imported unmodified with stand-ins for wandb and the dataset classes (not called), `torch.Tensor.cuda` patched to a no-op (ConvNet_TPS's
    forward calls it), and `torchvision.models.vgg19` patched to build without downloading and load `vgg_state_dict()`.

    python tests/golden/make_tps_val_golden.py
"""
import ast
import json
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT_FLAGS, OUT_NPZ = os.path.join(HERE, "tps_val_flags.json"), os.path.join(HERE, "tps_val_small.npz")
H, W, B = 256, 192, 2
# case -> (dense, with refinement, with the VGG loss)
CASES = {"tps": (False, False, True), "refinement": (False, True, True), "refinement_dense": (True, True, True),
         "refinement_no_vgg": (False, True, False)}


def batches(dense):
    """Two batches of the trainer's test keys at 256x192: smooth cloth, im_mask, pose heat-maps (or a 2-channel dense UV map), im_cloth."""
    from ladi_vton_b200 import synthetic as S
    out = []
    for k in range(2):
        w = S.warp_inputs(B, H, W, seed=41 + k)
        g = torch.Generator().manual_seed(51 + k)
        im_cloth = torch.rand((B, 3, H, W), generator=g) * 2 - 1
        im_cloth[:, :, :H // 4] = -1
        b = dict(cloth=w["cloth"], im_mask=w["im_mask"], pose_map=w["pose_map"], im_cloth=im_cloth, image=torch.zeros((B, 3, H, W)))
        if dense:
            b["dense_uv"] = w["pose_map"][:, :2] * 2 - 1
        out.append(b)
    return out


def warp_state_dicts(dense):
    from ladi_vton_b200 import synthetic as S
    from ladi_vton_b200.warp import ConvNet_TPS, UNetVanilla, control_points
    tps = ConvNet_TPS(256, 192, 5 if dense else 21, 3)
    ref = UNetVanilla(8 if dense else 24, 3, bilinear=True)
    return (S.warp_state_dict(tps.param_shapes(), 61 + dense, ctrl_bias=torch.atanh(control_points()).view(-1)),
            S.warp_state_dict(ref.param_shapes(), 71 + dense))


def vgg_state_dict(seed=81):
    """Seeded weights for torchvision's vgg19 `features`: He-normal convolutions (metrics.random_state_dict) and non-zero biases
    U(-0.1, 0.1), so that a bias dropped or attached to the wrong layer changes every tap."""
    from ladi_vton_b200.metrics import random_state_dict
    from ladi_vton_b200.vgg import VGG19
    sd = random_state_dict(VGG19().param_shapes(), seed)
    g = torch.Generator().manual_seed(seed + 1)
    for k in sorted(sd):
        if k.endswith(".bias"):
            sd[k] = torch.rand(sd[k].shape, generator=g) * 0.2 - 0.1
    return sd


def flags(ref):
    src = open(os.path.join(ref, "src", "train_tps.py")).read()
    tree = ast.parse(src)
    out, outputlist, params = [], None, None
    for node in ast.walk(tree):
        if isinstance(node, ast.Call) and isinstance(node.func, ast.Attribute) and node.func.attr == "add_argument":
            kw = {}
            for k in node.keywords:
                if k.arg == "help":
                    continue
                if isinstance(k.value, ast.Name):
                    kw[k.arg] = k.value.id
                else:
                    try:
                        kw[k.arg] = ast.literal_eval(k.value)
                    except ValueError:
                        kw[k.arg + "_src"] = ast.unparse(k.value)
            out.append(dict(flags=[ast.literal_eval(a) for a in node.args], line=node.lineno, **kw))
        if isinstance(node, ast.Assign) and any(isinstance(t, ast.Name) and t.id == "dataset_output_list" for t in node.targets):
            outputlist = ast.literal_eval(node.value)
        if isinstance(node, ast.FunctionDef) and node.name == "compute_metric":
            params = [a.arg for a in node.args.args]
    out.sort(key=lambda f: f["line"])
    return dict(source=["src/train_tps.py"], flags=out, outputlist=outputlist, compute_metric_params=params)


def run_reference(ref):
    for p in (ROOT, os.path.join(ref, "src")):
        sys.path.insert(0, p)
    sys.modules["wandb"] = types.ModuleType("wandb")
    for name, cls in (("dataset.dresscode", "DressCodeDataset"), ("dataset.vitonhd", "VitonHDDataset")):
        m = types.ModuleType(name)
        setattr(m, cls, object)
        sys.modules[name] = m
    sys.modules.setdefault("dataset", types.ModuleType("dataset"))
    torch.Tensor.cuda = lambda self, *a, **k: self
    import torchvision
    orig = torchvision.models.vgg19
    vsd = vgg_state_dict()

    def vgg19(*a, **k):
        m = orig(weights=None)
        m.load_state_dict(vsd, strict=False)
        return m
    torchvision.models.vgg19 = vgg19
    import train_tps as T  # the reference module, unmodified
    from models.ConvNet_TPS import ConvNet_TPS
    from models.UNet import UNetVanilla
    from utils.vgg_loss import VGGLoss
    assert T.device.type == "cpu"
    out = {}
    for case, (dense, with_ref, with_vgg) in CASES.items():
        tsd, rsd = warp_state_dicts(dense)
        tps = ConvNet_TPS(256, 192, 5 if dense else 21, 3)
        tps.load_state_dict(tsd, strict=False)  # the gridGen buffers are the reference's own
        refinement = UNetVanilla(n_channels=8 if dense else 24, n_classes=3, bilinear=True)
        refinement.load_state_dict(rsd)
        vgg = VGGLoss() if with_vgg else None
        loss, vgg_loss, _ = T.compute_metric(batches(dense), tps, torch.nn.L1Loss(), vgg, refinement=refinement if with_ref else None,
                                             height=H, width=W)
        out[case] = np.array([loss, vgg_loss], dtype=np.float64)
        print(case, out[case])
    return out


def main():
    ref = os.environ["LADI_REFERENCE"]
    json.dump(flags(ref), open(OUT_FLAGS, "w"), indent=1)
    torch.set_num_threads(8)
    out = run_reference(ref)
    np.savez_compressed(OUT_NPZ, **out)
    print(f"-> {OUT_FLAGS}, {OUT_NPZ}")


if __name__ == "__main__":
    main()
