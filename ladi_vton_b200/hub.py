"""Hub constructors -- the same names, argument and returned-object roles as hubconf.py:16-66
(`inversion_adapter`, `extended_unet`, `emasc`, `warping_module`), returning the H100-native modules.

The reference fetches configs and checkpoints over the network (`torch.hub.load_state_dict_from_url`, hubconf.py:25-26,35-36,
50-51).  There is no network on the target boxes, so checkpoints are read from local files with the reference's release file names
(`unet_vitonhd.pth`, `emasc_dresscode.pth`, ...) in `checkpoint_dir` (argument, or $LADI_CHECKPOINT_DIR).  The architecture constants
that the reference reads from the hub configs are written out here: SD-2-inpainting UNet with `in_channels=31` (hubconf.py:31-33),
EMASC channel plan (hubconf.py:41-42), CLIP ViT-H-14 vision width 1280 / MLP 5120 / 16 heads and text width 1024 (hubconf.py:17-23).
"""
import os

import torch

from .adapter import InversionAdapter
from .unet import UNet2DConditionModel
from .vae import EMASC
from .warp import ConvNet_TPS, UNetVanilla

DATASETS = ("dresscode", "vitonhd")
RELEASE_URL = "https://github.com/miccunifi/ladi-vton/releases/download/weights/"


def _checkpoint(name, dataset, checkpoint_dir):
    if dataset not in DATASETS:
        raise ValueError(f"dataset must be one of {DATASETS}, got {dataset!r}")
    d = checkpoint_dir or os.environ.get("LADI_CHECKPOINT_DIR")
    fname = f"{name}_{dataset}.pth"
    if d is None:
        raise FileNotFoundError(f"no checkpoint directory given: pass checkpoint_dir= or set LADI_CHECKPOINT_DIR to a folder holding "
                                f"{fname} (the reference downloads it from {RELEASE_URL}{fname})")
    path = os.path.join(d, fname)
    if not os.path.isfile(path):
        raise FileNotFoundError(f"{path} not found (the reference downloads it from {RELEASE_URL}{fname})")
    return torch.load(path, map_location="cpu")


def inversion_adapter(dataset, checkpoint_dir=None, state_dict=None, num_encoder_layers=1):
    """hubconf.py:16-27.  `state_dict=` bypasses the file read (tests, synthetic weights); `num_encoder_layers` > 1 builds the adapters
    the training scripts make with `--num_encoder_layers` (the release checkpoints have 1)."""
    m = InversionAdapter(input_dim=1280, hidden_dim=1280 * 4, output_dim=1024 * 16, num_encoder_layers=num_encoder_layers, heads=16, mlp_dim=5120)
    return m.load_state_dict(state_dict if state_dict is not None else _checkpoint("inversion_adapter", dataset, checkpoint_dir))


def extended_unet(dataset, checkpoint_dir=None, state_dict=None):
    """hubconf.py:30-37: the SD-2-inpainting UNet with the input convolution widened to 31 channels."""
    m = UNet2DConditionModel(in_channels=31)
    return m.load_state_dict(state_dict if state_dict is not None else _checkpoint("unet", dataset, checkpoint_dir))


def emasc(dataset, checkpoint_dir=None, state_dict=None, kernel_size=3, padding=1, type="nonlinear"):
    """hubconf.py:40-53 (the release checkpoints are nonlinear 3x3; `kernel_size` / `padding` / `type` select the forms train_emasc.py
    can make, see vae.EMASC)."""
    m = EMASC([128, 128, 128, 256, 512], [128, 256, 512, 512, 512], kernel_size=kernel_size, padding=padding, stride=1, type=type)
    return m.load_state_dict(state_dict if state_dict is not None else _checkpoint("emasc", dataset, checkpoint_dir))


def warping_module(dataset, checkpoint_dir=None, state_dict=None):
    """hubconf.py:56-66: (ConvNet_TPS(256, 192, 21, 3), UNetVanilla(24, 3, bilinear=True)) from `warping_<dataset>.pth`, a dict with
    the two state dicts under 'tps' and 'refinement'."""
    ck = state_dict if state_dict is not None else _checkpoint("warping", dataset, checkpoint_dir)
    tps = ConvNet_TPS(256, 192, 21, 3).load_state_dict(ck["tps"])
    refinement = UNetVanilla(n_channels=24, n_classes=3, bilinear=True).load_state_dict(ck["refinement"])
    return tps, refinement
