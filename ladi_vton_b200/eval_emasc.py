"""`python -m ladi_vton_b200.eval_emasc` -- validate a trained EMASC checkpoint on the engine, as the reference's trainer does at each
checkpoint (src/train_emasc.py:431-472): every test image is encoded, its masked copy's encoder skips go through EMASC with
`mask_features`, and the posterior sample is decoded with them, by `extract_save_vae_images` (eval.py <- src/utils/image_from_pipe.py:221-258)
into `<output_dir>/<save_name>_<test_order>/<category>/<im_name>`; with `--compute_metrics` the folder is scored by the engine's metrics
(val_metrics.compute_metrics(..., 'all', ['all'], ...)) into `<output_dir>/metrics_<save_name>_<test_order>_all.json`.

The flags the validation uses are the trainer's own (src/train_emasc.py:41-168: same names, types, defaults, choices and required-ness),
so a training command line works once the training-only flags (TRAINING_ONLY) are dropped.  The `engine` group adds:
  * `--emasc_dir` (default `--output_dir`, where the trainer writes `emasc_<step>.pth`) and `--emasc_name` (default `latest`: the highest
    step, as eval.checkpoint_path finds it);
  * `--save_name`, default `imgs_step_<step>` from the checkpoint's step, the folder name the trainer validates into;
  * `--reference_src` for the real datasets, `--random_init` and `--synthetic_samples` (as in eval.py);
  * `--compute_metrics` / `--metrics_weights_dir`: the metric networks' local weight files (or seeded random ones with `--random_init`).
Only the VAE of `--pretrained_model_name_or_path` is read (`<root>/vae`), and its config must be the SD-2 VAE's architecture, which the
SD-1.5 inpainting model shares.  One process: the reference validates on its main process only.  The engine computes in bf16 with fp32
accumulation; the reference validates under fp16 autocast.
"""
import argparse
import json
import os

import torch

from .eval import EMASC_IN, EMASC_OUT, INT_LAYERS, SD2_INPAINT, _load, _load_folder_state_dict, _random_init, checkpoint_path
from .eval_inversion_adapter import default_save_name
from .inference import build_dataset, check_args as check_dataroots

OUTPUTLIST = ['image', 'pose_map', 'inpaint_mask', 'im_mask', 'category', 'im_name']  # src/train_emasc.py:259, :277 (the test datasets)
CATEGORIES = ['dresses', 'upper_body', 'lower_body']  # :257 (Dress Code)
# src/train_emasc.py flags that only training reads
TRAINING_ONLY = ['--train_batch_size', '--num_train_epochs', '--max_train_steps', '--gradient_accumulation_steps', '--learning_rate',
                 '--lr_scheduler', '--lr_warmup_steps', '--allow_tf32', '--adam_beta1', '--adam_beta2', '--adam_weight_decay',
                 '--adam_epsilon', '--max_grad_norm', '--mixed_precision', '--report_to', '--local_rank', '--checkpointing_steps',
                 '--resume_from_checkpoint', '--num_workers', '--vgg_weight']
VAE_ARCH_KEYS = ("in_channels", "out_channels", "block_out_channels", "layers_per_block", "latent_channels", "norm_num_groups")


def build_parser():
    """The validation flags of src/train_emasc.py:41-168, plus an `engine` group."""
    parser = argparse.ArgumentParser(description="Validation of a trained EMASC checkpoint: VAE reconstruction with EMASC skips")
    parser.add_argument("--dataset", type=str, required=True, choices=["dresscode", "vitonhd"], help="dataset to use")
    parser.add_argument('--dresscode_dataroot', type=str, help='DressCode dataroot')
    parser.add_argument('--vitonhd_dataroot', type=str, help='VitonHD dataroot')
    parser.add_argument("--output_dir", type=str, required=True,
                        help="The trainer's output directory: the images (and the metrics) are written here")
    parser.add_argument("--pretrained_model_name_or_path", type=str, default=SD2_INPAINT,
                        help="Local folder of the Stable Diffusion inpainting model; only its vae/ is read.")
    parser.add_argument("--seed", type=int, default=1234, help="A seed for reproducible validation.")
    parser.add_argument("--test_batch_size", type=int, default=16, help="Batch size for the testing dataloader.")
    parser.add_argument("--num_workers_test", type=int, default=8, help="Test DataLoader number of workers.")
    parser.add_argument("--test_order", type=str, default="paired", choices=["unpaired", "paired"],
                        help="Whether to use paired or unpaired test data.")
    parser.add_argument("--emasc_type", type=str, default='nonlinear', choices=["linear", "nonlinear"],
                        help="Whether to use linear or nonlinear EMASC.")
    parser.add_argument("--emasc_kernel", type=int, default=3, help="EMASC kernel size.")
    parser.add_argument("--emasc_padding", type=int, default=1, help="EMASC padding size.")
    eng = parser.add_argument_group("engine", "checkpoint selection, and options for machines without network access")
    eng.add_argument("--emasc_dir", type=str, default=None,
                     help="Directory of the EMASC checkpoints (default: --output_dir, where the trainer writes them)")
    eng.add_argument("--emasc_name", type=str, default="latest", help="Checkpoint file in --emasc_dir; `latest` takes the highest step")
    eng.add_argument("--save_name", type=str, default=None,
                     help="Name of the image folder inside output_dir (default imgs_step_<step of the checkpoint>)")
    eng.add_argument("--reference_src", type=str, default=None, help="`src/` folder of a miccunifi/ladi-vton checkout (dataset classes)")
    eng.add_argument("--random_init", action="store_true", help="seeded random weights for the VAE and EMASC (synthetic workload)")
    eng.add_argument("--synthetic_samples", type=int, default=0, help="use N synthetic samples instead of a dataset")
    eng.add_argument("--compute_metrics", action="store_true", help="score the written images (src/train_emasc.py:452-456)")
    eng.add_argument("--metrics_weights_dir", type=str, default=None, help="local weight files of the metric networks (val_metrics.py)")
    return parser


def parse_args(argv=None):
    args = build_parser().parse_args(argv)
    args.emasc_dir = args.emasc_dir or args.output_dir
    return args


def check_vae_config(root):
    """`<root>/vae/config.json` must describe the SD-2 VAE (vae.SD2_VAE; the SD-1.5 inpainting VAE has the same architecture)."""
    from .vae import SD2_VAE
    p = os.path.join(root, "vae", "config.json")
    if not os.path.isfile(p):
        raise FileNotFoundError(f"no {p}: --pretrained_model_name_or_path must be a local folder of a Stable Diffusion inpainting model")
    cfg = json.load(open(p))
    diff = {k: cfg.get(k) for k in VAE_ARCH_KEYS if k in cfg and (list(cfg[k]) if k == "block_out_channels" else cfg[k])
            != (list(SD2_VAE[k]) if k == "block_out_channels" else SD2_VAE[k])}
    if diff:
        raise ValueError(f"{root}/vae has {diff}: EMASC validation runs the Stable Diffusion VAE "
                         f"({ {k: SD2_VAE[k] for k in VAE_ARCH_KEYS} }), whose encoder skips the EMASC channel plan is built for")


def build_emasc(args):
    """The EMASC of src/train_emasc.py:206-217, not yet loaded: its constructor refuses the forms that are not built."""
    from . import EMASC
    return EMASC(EMASC_IN, EMASC_OUT, kernel_size=args.emasc_kernel, padding=args.emasc_padding, stride=1, type=args.emasc_type)


def check_args(args):
    """Everything that can fail before the GPU is touched: the dataroot errors of the reference, the EMASC form, the VAE's config, the
    checkpoint file and the step in its name.  Returns (EMASC module, save_name)."""
    check_dataroots(args)
    emasc = build_emasc(args)
    if not args.random_init:
        check_vae_config(args.pretrained_model_name_or_path)
    return emasc, args.save_name or default_save_name(args, "emasc")


def build_models(args, emasc, device):
    """dict(vae, emasc): the VAE from `<root>/vae` and the EMASC checkpoint (or seeded random weights), engine objects on `device`."""
    from . import AutoencoderKL, synthetic as S
    from .vae import vae_param_shapes
    if args.random_init:
        vae = AutoencoderKL().load_state_dict(S.random_state_dict(vae_param_shapes({}), args.seed + 1, device="cuda", fast=True))
        emasc = _random_init(emasc, args.seed + 2)
    else:
        vae = AutoencoderKL().load_state_dict(_load_folder_state_dict(os.path.join(args.pretrained_model_name_or_path, "vae")))
        emasc = emasc.load_state_dict(_load(checkpoint_path(args.emasc_dir, args.emasc_name, "emasc")))
    return dict(vae=vae.to(device), emasc=emasc.to(device))


@torch.no_grad()
def main(argv=None, models=None, dataset=None):
    """`models=` / `dataset=` inject prebuilt engine objects (dict(vae, emasc)) / any dataset with the reference's batch keys.
    Returns the written image paths."""
    args = parse_args(argv)
    emasc, save_name = check_args(args)
    from . import lib
    from .eval import extract_save_vae_images
    lib.load()  # fail before any work if the CUDA extension is missing: there is no CPU path
    if not torch.cuda.is_available():
        raise RuntimeError("ladi_vton_b200.eval_emasc needs a CUDA device (sm_90a); there is no CPU path")
    device = torch.device("cuda", torch.cuda.current_device())
    if args.seed is not None:  # utils/set_seeds.py
        import random
        import numpy as np
        random.seed(args.seed), np.random.seed(args.seed), torch.manual_seed(args.seed), torch.cuda.manual_seed_all(args.seed)
    models = models or build_models(args, emasc, device)
    test_dataset = dataset if dataset is not None else build_dataset(args, CATEGORIES, OUTPUTLIST)
    loader = torch.utils.data.DataLoader(test_dataset, shuffle=False, batch_size=args.test_batch_size,
                                         num_workers=args.num_workers_test if dataset is None and args.synthetic_samples <= 0 else 0)
    written = extract_save_vae_images(models["vae"], models["emasc"], loader, INT_LAYERS, args.output_dir, args.test_order,
                                      save_name=save_name, emasc_type=args.emasc_type)
    torch.cuda.empty_cache()
    if args.compute_metrics:  # :452-456
        from .val_metrics import compute_metrics
        metrics = compute_metrics(os.path.join(args.output_dir, f"{save_name}_{args.test_order}"), args.test_order, args.dataset, 'all',
                                  ['all'], args.dresscode_dataroot, args.vitonhd_dataroot, weights_dir=args.metrics_weights_dir,
                                  random_init=args.random_init)
        print(metrics, flush=True)
        with open(os.path.join(args.output_dir, f"metrics_{save_name}_{args.test_order}_all.json"), "w+") as f:
            json.dump(metrics, f, indent=4)
    return written


if __name__ == "__main__":
    main()
