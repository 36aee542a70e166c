"""`python -m ladi_vton_b200.eval_inversion_adapter` -- validate a trained inversion adapter checkpoint on the engine, as the reference's
trainer does at each checkpoint (src/train_inversion_adapter.py:544-569): the stock SD-2 inpainting model (9-channel UNet input
latents4 | mask1 | masked4, `StableDiffusionInpaintPipeline`) with the adapter's pseudo-words in the prompt, images written by
`generate_images_inversion_adapter` (eval.py <- src/utils/image_from_pipe.py:139-218) to
`<output_dir>/<save_name>_<test_order>/<category>/<im_name>`, and with `--compute_metrics` scored by the engine's metrics
(val_metrics.compute_metrics(..., 'all', ['all'], ...)) into `<output_dir>/metrics_<save_name>_<test_order>_all.json`.

The flags the validation uses are the trainer's own (src/train_inversion_adapter.py:41-184: same names, types, defaults, choices and
required-ness), so a training command line works once the training-only flags are dropped.  The `engine` group adds:
  * `--inversion_adapter_dir` (default `--output_dir`, where the trainer writes `inversion_adapter_<step>.pth`) and
    `--inversion_adapter_name` (default `latest`: the highest step, as eval.checkpoint_path finds it);
  * `--save_name`, default `imgs_step_<step>` from the checkpoint's step, the folder name the trainer validates into;
  * `--num_inference_steps` / `--guidance_scale` (the validation function's defaults, 50 and 7.5);
  * the offline options of eval.py: local model folders, `--reference_src` for the real datasets, `--random_init`, `--synthetic_samples`;
  * `--compute_metrics` / `--metrics_weights_dir`: the metric networks' local weight files (or seeded random ones with `--random_init`).
One process: the reference validates on its main process only.  `--enable_xformers_memory_efficient_attention` is accepted (the
engine's attention is already fused).  The engine computes in bf16 with fp32 accumulation; the reference validates under fp16 autocast.
"""
import argparse
import json
import os

import torch

from .eval import SD2_INPAINT, _load_folder_state_dict, _random_init, adapter_models, base_models, check_base_model, checkpoint_path
from .inference import build_dataset, check_args as check_dataroots

OUTPUTLIST = ['image', 'inpaint_mask', 'im_mask', 'category', 'im_name', 'cloth']  # src/train_inversion_adapter.py:281
CATEGORIES = ['dresses', 'upper_body', 'lower_body']  # :296-305
SAVE_NAME = "imgs_step_{}"  # :562


def build_parser():
    """The validation flags of src/train_inversion_adapter.py:41-184, plus an `engine` group."""
    parser = argparse.ArgumentParser(description="Validation of a trained inversion adapter on the SD-2 inpainting pipeline")
    parser.add_argument("--dataset", type=str, required=True, choices=["dresscode", "vitonhd"], help="dataset to use")
    parser.add_argument('--dresscode_dataroot', type=str, help='DressCode dataroot')
    parser.add_argument('--vitonhd_dataroot', type=str, help='VitonHD dataroot')
    parser.add_argument("--output_dir", type=str, required=True,
                        help="The trainer's output directory: the images (and the metrics) are written here")
    parser.add_argument("--pretrained_model_name_or_path", type=str, default=SD2_INPAINT,
                        help="Local folder of the SD-2 inpainting model (unet/, vae/, text_encoder/, tokenizer/).")
    parser.add_argument("--seed", type=int, default=1234, help="A seed for reproducible validation.")
    parser.add_argument("--test_batch_size", type=int, default=16, help="Batch size for the testing dataloader.")
    parser.add_argument("--enable_xformers_memory_efficient_attention", action="store_true",
                        help="Accepted for compatibility (attention is already a fused kernel).")
    parser.add_argument("--num_workers_test", type=int, default=8, help="Number of workers to use in the test dataloaders.")
    parser.add_argument("--test_order", type=str, default="paired", choices=["unpaired", "paired"],
                        help="Whether to use paired or unpaired test data.")
    parser.add_argument("--num_vstar", default=16, type=int, help="Number of predicted v* per image to use")
    parser.add_argument("--num_encoder_layers", default=1, type=int, help="Number of ViT layer to use in inversion adapter")
    parser.add_argument("--use_clip_cloth_features", action="store_true", help="Whether to use precomputed clip cloth features")
    eng = parser.add_argument_group("engine", "checkpoint selection, and options for machines without network access")
    eng.add_argument("--inversion_adapter_dir", type=str, default=None,
                     help="Directory of the inversion adapter checkpoints (default: --output_dir, where the trainer writes them)")
    eng.add_argument("--inversion_adapter_name", type=str, default="latest",
                     help="Checkpoint file in --inversion_adapter_dir; `latest` takes the highest step")
    eng.add_argument("--save_name", type=str, default=None,
                     help="Name of the image folder inside output_dir (default imgs_step_<step of the checkpoint>)")
    eng.add_argument("--num_inference_steps", default=50, type=int, help="Number of diffusion steps")
    eng.add_argument("--guidance_scale", default=7.5, type=float, help="Guidance scale for the diffusion")
    eng.add_argument("--vision_model_name_or_path", type=str, default="laion/CLIP-ViT-H-14-laion2B-s32B-b79K",
                     help="local folder of the CLIP ViT-H vision tower (src/train_inversion_adapter.py:235)")
    eng.add_argument("--reference_src", type=str, default=None, help="`src/` folder of a miccunifi/ladi-vton checkout (dataset classes)")
    eng.add_argument("--random_init", action="store_true", help="seeded random weights for every model (synthetic workload)")
    eng.add_argument("--synthetic_samples", type=int, default=0, help="use N synthetic samples instead of a dataset")
    eng.add_argument("--compute_metrics", action="store_true", help="score the written images (src/train_inversion_adapter.py:565-569)")
    eng.add_argument("--metrics_weights_dir", type=str, default=None, help="local weight files of the metric networks (val_metrics.py)")
    return parser


def parse_args(argv=None):
    args = build_parser().parse_args(argv)
    args.inversion_adapter_dir = args.inversion_adapter_dir or args.output_dir
    return args


def check_args(args):
    """The dataroot errors of the reference, the one base model that is built, and its UNet."""
    check_dataroots(args)
    check_base_model(args.pretrained_model_name_or_path)
    if not args.random_init:
        check_base_unet(args.pretrained_model_name_or_path)


def check_base_unet(root):
    """The validation runs the base model's own UNet: `<root>/unet/config.json` must declare the 9 input channels of SD-2 inpainting."""
    p = os.path.join(root, "unet", "config.json")
    if not os.path.isfile(p):
        raise FileNotFoundError(f"no {p}: --pretrained_model_name_or_path must be a local folder of the SD-2 inpainting model")
    cin = json.load(open(p)).get("in_channels")
    if cin != 9:
        raise ValueError(f"{root}/unet has in_channels={cin}: inversion-adapter validation runs the stock SD-2 inpainting UNet, "
                         "in_channels=9 (latents 4 + mask 1 + masked image 4); a try-on UNet is evaluated with ladi_vton_b200.eval")


def default_save_name(args, prefix="inversion_adapter"):
    """`imgs_step_<step>` (src/train_inversion_adapter.py:562, src/train_emasc.py:446) with the step of the checkpoint file
    `<prefix>_<step>.pth`, found from `args.<prefix>_dir` and `args.<prefix>_name` (`latest`: the highest step)."""
    if args.random_init:
        return SAVE_NAME.format("random_init")
    name = os.path.basename(checkpoint_path(getattr(args, f"{prefix}_dir"), getattr(args, f"{prefix}_name"), prefix))
    step = os.path.splitext(name)[0].split("_")[-1]
    if not step.isdigit():
        raise ValueError(f"{name} does not end in a training step ({prefix}_<step>.pth): pass --save_name")
    return SAVE_NAME.format(int(step))


def outputlist_for(args):
    return OUTPUTLIST + (['clip_cloth_features'] if args.use_clip_cloth_features else [])  # :281-285


def build_models(args, device):
    """The base model (UNet from `<root>/unet`, VAE, text encoder, tokenizer; eval.base_models), the adapter and the vision tower
    (eval.adapter_models), every module an engine object on `device`."""
    from . import UNet2DConditionModel
    m = base_models(args)
    unet = UNet2DConditionModel(in_channels=9)
    if args.random_init:
        m["unet"] = _random_init(unet, args.seed)
    else:
        m["unet"] = unet.load_state_dict(_load_folder_state_dict(os.path.join(args.pretrained_model_name_or_path, "unet")))
    m["inversion_adapter"], m["vision_encoder"] = adapter_models(args, m["text_encoder"])
    for k, v in m.items():
        if v is not None and k not in ("scheduler", "tokenizer"):
            v.to(device)
    return m


@torch.no_grad()
def main(argv=None, models=None, dataset=None):
    """`models=` / `dataset=` inject prebuilt engine objects (the dict of build_models) / any dataset with the reference's batch keys.
    Returns the written image paths."""
    args = parse_args(argv)
    check_args(args)
    from . import StableDiffusionInpaintPipeline, lib
    from .eval import generate_images_inversion_adapter
    lib.load()  # fail before any work if the CUDA extension is missing: there is no CPU path
    if not torch.cuda.is_available():
        raise RuntimeError("ladi_vton_b200.eval_inversion_adapter needs a CUDA device (sm_90a); there is no CPU path")
    device = torch.device("cuda", torch.cuda.current_device())
    save_name = args.save_name or default_save_name(args)
    if args.seed is not None:  # utils/set_seeds.py
        import random
        import numpy as np
        random.seed(args.seed), np.random.seed(args.seed), torch.manual_seed(args.seed), torch.cuda.manual_seed_all(args.seed)
    models = models or build_models(args, device)
    test_dataset = dataset if dataset is not None else build_dataset(args, CATEGORIES, outputlist_for(args))
    loader = torch.utils.data.DataLoader(test_dataset, shuffle=False, batch_size=args.test_batch_size,
                                         num_workers=args.num_workers_test if dataset is None and args.synthetic_samples <= 0 else 0)
    val_pipe = StableDiffusionInpaintPipeline(text_encoder=models["text_encoder"], vae=models["vae"], unet=models["unet"],
                                              tokenizer=models["tokenizer"], scheduler=models["scheduler"], safety_checker=None,
                                              requires_safety_checker=False, feature_extractor=None).to(device)
    written = generate_images_inversion_adapter(val_pipe, models["inversion_adapter"], models["vision_encoder"], models.get("processor"),
                                                loader, args.output_dir, args.test_order, save_name=save_name, num_vstar=args.num_vstar,
                                                seed=args.seed, num_inference_steps=args.num_inference_steps,
                                                guidance_scale=args.guidance_scale)
    del val_pipe
    torch.cuda.empty_cache()
    if args.compute_metrics:  # :565-569
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
