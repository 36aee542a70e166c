"""`python -m ladi_vton_b200.eval` -- the reference's evaluation CLI for user-trained checkpoints (src/eval.py, README "Inference with the
trained models") on the H100 engine.

Same flags, types, defaults, choices and required-ness as its `parse_args` (src/eval.py:32-132), the same dataroot and missing-checkpoint
errors, the same `latest` checkpoint discovery (:187-195, :212-220, :258-266: the file with the highest numeric suffix among the files
named `unet*`, `emasc*`, `inversion_adapter*`), a 27- or 31-channel UNet from `--cloth_input_type` (:166), EMASC of type `--emasc_type`
with `--emasc_kernel` / `--emasc_padding` (linear, or nonlinear 3x3 / 1x1; vae.EMASC says why other forms are not built), an inversion
adapter with `--num_encoder_layers` layers, and the batch body of src/utils/image_from_pipe.py:26-130 (`generate_images_from_tryon_pipe`,
also what train_vto.py calls for validation) with its three `--text_usage` branches.  Output tree:
`<output_dir>/<save_name>_<test_order>/<category>/<im_name>` (jpg quality 95, or png with --use_png).

The engine computes in bf16 with fp32 accumulation; the reference's eval.py runs its models in fp16 under autocast (:319-335, :350).

What differs, because the target boxes have no network (the reference downloads the base model and the vision tower, :158-163, :241-246):
  * `--pretrained_model_name_or_path` is a local diffusers folder of the SD-2 inpainting model (text_encoder/, vae/, tokenizer/) and the
    CLIP ViT-H vision tower is read from `--vision_model_name_or_path`; the SD-1.5 inpainting base is not built and is refused;
  * `--random_init` builds every model with seeded random weights and `--synthetic_samples N` replaces the dataset by N synthetic samples
    with the batch keys of src/dataset/vitonhd.py (with it the checkpoint folders are not read);
  * the real datasets and `--compute_metrics` are the reference's own code, imported from `--reference_src` (a checkout's `src/` folder);
    with `--use_clip_cloth_features` its dataset classes read the cache that `python -m ladi_vton_b200.compute_cloth_clip_features`
    writes;
  * `--allow_tf32`, `--enable_xformers_memory_efficient_attention` are accepted: the engine always computes in bf16 and its attention is
    already fused.
`generate_images_inversion_adapter` (src/utils/image_from_pipe.py:139-218, the inversion-adapter trainer's validation) is here too; its CLI
is `python -m ladi_vton_b200.eval_inversion_adapter`, and so is `extract_save_vae_images` (src/utils/image_from_pipe.py:221-258, the EMASC
trainer's reconstruction check), whose CLI is `python -m ladi_vton_b200.eval_emasc`.
Scoring on the engine (instead of `--compute_metrics`, which runs the reference's own val_metrics.py from `--reference_src`):
`python -m ladi_vton_b200.val_metrics --gen_folder <output_dir>/<save_name>_<test_order> --test_order <order> --dataset ... --metrics_weights_dir W`.
"""
import argparse
import json
import os
import sys

import torch

from .inference import (StandInTokenizer, _load_folder_state_dict, _try_tokenizer, batches_for_rank, build_dataset, clip_pixel_values,
                        prompts_for, save_images)

SD2_INPAINT, SD15_INPAINT = "stabilityai/stable-diffusion-2-inpainting", "runwayml/stable-diffusion-inpainting"
EMASC_IN, EMASC_OUT, INT_LAYERS = [128, 128, 128, 256, 512], [128, 256, 512, 512, 512], [1, 2, 3, 4, 5]  # src/eval.py:200-202


def build_parser():
    """The reference's parser (src/eval.py:32-124) flag for flag, plus an `engine` group for the local-file / synthetic options."""
    parser = argparse.ArgumentParser(description="Evaluation of trained LaDI-VTON models")
    parser.add_argument("--dataset", type=str, required=True, choices=["dresscode", "vitonhd"], help="dataset to use")
    parser.add_argument('--dresscode_dataroot', type=str, help='DressCode dataroot')
    parser.add_argument('--vitonhd_dataroot', type=str, help='VitonHD dataroot')
    parser.add_argument("--output_dir", type=str, required=True, help="Path to the output directory")
    parser.add_argument("--save_name", type=str, required=True, help="Name of the saving folder inside output_dir")
    parser.add_argument("--test_order", type=str, required=True, choices=["unpaired", "paired"])
    parser.add_argument("--unet_dir", required=True, type=str, help="Directory where to load the trained unet from")
    parser.add_argument("--unet_name", type=str, default="latest",
                        help="Name of the unet to load from the directory specified by `--unet_dir`. To load the latest checkpoint, use `latest`.")
    parser.add_argument("--inversion_adapter_dir", type=str, default=None,
                        help="Directory where to load the trained inversion adapter from. Required when using --text_usage=inversion_adapter")
    parser.add_argument("--inversion_adapter_name", type=str, default="latest",
                        help="Name of the inversion adapter to load from the directory specified by `--inversion_adapter_dir`. "
                             "To load the latest checkpoint, use `latest`.")
    parser.add_argument("--emasc_dir", type=str, default=None,
                        help="Directory where to load the trained EMASC from. Required when --emasc_type!=none")
    parser.add_argument("--emasc_name", type=str, default="latest",
                        help="Name of the EMASC to load from the directory specified by `--emasc_dir`. To load the latest checkpoint, use `latest`.")
    parser.add_argument("--pretrained_model_name_or_path", type=str, default=SD2_INPAINT,
                        help="Local folder of the SD-2 inpainting model (text_encoder/, vae/, tokenizer/).")
    parser.add_argument("--seed", type=int, default=1234, help="A seed for reproducible inference.")
    parser.add_argument("--batch_size", type=int, default=8, help="Batch size (per device) for the dataloader.")
    parser.add_argument("--allow_tf32", action="store_true", help="Accepted for compatibility (the engine computes in bf16).")
    parser.add_argument("--enable_xformers_memory_efficient_attention", action="store_true",
                        help="Accepted for compatibility (attention is already a fused kernel).")
    parser.add_argument("--num_workers", type=int, default=8, help="Number of workers for the dataloader")
    parser.add_argument("--category", type=str, choices=['all', 'lower_body', 'upper_body', 'dresses'], default='all')
    parser.add_argument("--emasc_type", type=str, default='nonlinear', choices=["none", "linear", "nonlinear"],
                        help="Whether to use linear or nonlinear EMASC.")
    parser.add_argument("--emasc_kernel", type=int, default=3, help="EMASC kernel size.")
    parser.add_argument("--emasc_padding", type=int, default=1, help="EMASC padding size.")
    parser.add_argument("--text_usage", type=str, default='inversion_adapter', choices=["none", "noun_chunks", "inversion_adapter"],
                        help="if 'none' do not use the text, if 'noun_chunks' use the coarse noun chunks, if "
                             "'inversion_adapter' use the features obtained trough the inversion adapter net")
    parser.add_argument("--cloth_input_type", type=str, choices=["warped", "none"], default='warped',
                        help="cloth input type. If 'warped' use the warped cloth, if none do not use the cloth as input of the unet")
    parser.add_argument("--num_vstar", default=16, type=int, help="Number of predicted v* images to use")
    parser.add_argument("--num_encoder_layers", default=1, type=int, help="Number of ViT layer to use in inversion adapter")
    parser.add_argument("--use_png", default=False, action="store_true", help="Use png instead of jpg")
    parser.add_argument("--num_inference_steps", default=50, type=int, help="Number of diffusion steps")
    parser.add_argument("--guidance_scale", default=7.5, type=float, help="Guidance scale for the diffusion")
    parser.add_argument("--use_clip_cloth_features", action="store_true", help="Whether to use precomputed clip cloth features")
    parser.add_argument("--compute_metrics", default=False, action="store_true", help="Compute metrics after generation")
    eng = parser.add_argument_group("engine", "options for machines without network access")
    eng.add_argument("--vision_model_name_or_path", type=str, default="laion/CLIP-ViT-H-14-laion2B-s32B-b79K",
                     help="local folder of the CLIP ViT-H vision tower (src/eval.py:245)")
    eng.add_argument("--reference_src", type=str, default=None, help="`src/` folder of a miccunifi/ladi-vton checkout (dataset classes, metrics)")
    eng.add_argument("--random_init", action="store_true", help="seeded random weights for every model (synthetic workload)")
    eng.add_argument("--synthetic_samples", type=int, default=0, help="use N synthetic samples instead of a dataset")
    return parser


def parse_args(argv=None):
    return build_parser().parse_args(argv)


def check_args(args):
    """src/eval.py:138-142 (dataroots), :223 and :269 (checkpoint folders), and the one base model that is built."""
    if args.synthetic_samples <= 0:
        if args.dataset == "vitonhd" and args.vitonhd_dataroot is None:
            raise ValueError("VitonHD dataroot must be provided")
        if args.dataset == "dresscode" and args.dresscode_dataroot is None:
            raise ValueError("DressCode dataroot must be provided")
    check_base_model(args.pretrained_model_name_or_path)
    if not args.random_init:
        if args.emasc_type != 'none' and args.emasc_dir is None:
            raise ValueError("No EMASC checkpoint found. Make sure to specify --emasc_dir")
        if args.text_usage == 'inversion_adapter' and args.inversion_adapter_dir is None:
            raise ValueError("No inversion adapter checkpoint found. Make sure to specify --inversion_adapter_dir")


def check_base_model(path):
    """The one base model that is built: SD-2 inpainting (by name, or a local folder with a 1024-wide text encoder)."""
    if path == SD15_INPAINT or _text_width(path) not in (None, 1024):
        raise NotImplementedError(f"{path}: the Stable Diffusion 1.5 inpainting base (CLIP ViT-L/14, 768-wide text "
                                  "states, attention heads 40/80/160 wide) is not built; this engine runs the SD-2 inpainting base "
                                  f"({SD2_INPAINT})")


def _text_width(folder):
    p = os.path.join(folder, "text_encoder", "config.json")
    return json.load(open(p)).get("hidden_size") if os.path.isfile(p) else None


def checkpoint_path(directory, name, prefix):
    """src/eval.py:187-195: `name` as given, or with name == "latest" the file starting with `prefix` whose name ends in the highest
    number (`<prefix>_<step>.<ext>`)."""
    if name != "latest":
        return os.path.join(directory, name)
    dirs = [d for d in os.listdir(directory) if d.startswith(prefix)]
    dirs = sorted(dirs, key=lambda x: int(os.path.splitext(x.split("_")[-1])[0]))
    return os.path.join(directory, dirs[-1])


def outputlist_for(args):
    """src/eval.py:235-277."""
    out = ['image', 'pose_map', 'captions', 'inpaint_mask', 'im_mask', 'category', 'im_name']
    if args.cloth_input_type == 'warped':
        out.append('warped_cloth')
    if args.text_usage == 'inversion_adapter':
        out.append('clip_cloth_features' if args.use_clip_cloth_features else 'cloth')
    return out


def build_models(args, device):
    """src/eval.py:158-277 -> dict(scheduler, text_encoder, vae, tokenizer, unet, emasc, inversion_adapter, vision_encoder); emasc is None
    with --emasc_type none, inversion_adapter / vision_encoder are None unless --text_usage inversion_adapter (vision_encoder also with
    --use_clip_cloth_features, :273-275).  Every module is an engine object already on `device`."""
    from . import EMASC, UNet2DConditionModel
    m = base_models(args)
    unet = UNet2DConditionModel(in_channels=27 if args.cloth_input_type == "none" else 31)  # :172
    if args.random_init:
        m["unet"] = _random_init(unet, args.seed)
    else:
        m["unet"] = unet.load_state_dict(_load(checkpoint_path(args.unet_dir, args.unet_name, "unet")))
    m["emasc"] = None
    if args.emasc_type != 'none':  # :198-226
        em = EMASC(EMASC_IN, EMASC_OUT, kernel_size=args.emasc_kernel, padding=args.emasc_padding, stride=1, type=args.emasc_type)
        m["emasc"] = _random_init(em, args.seed + 2) if args.random_init else em.load_state_dict(_load(checkpoint_path(args.emasc_dir, args.emasc_name, "emasc")))
    m["inversion_adapter"] = m["vision_encoder"] = None
    if args.text_usage == 'inversion_adapter':  # :240-278
        m["inversion_adapter"], m["vision_encoder"] = adapter_models(args, m["text_encoder"])
    for k, v in m.items():
        if v is not None and hasattr(v, "to") and k not in ("scheduler", "tokenizer"):
            v.to(device)
    return m


def _load(path):
    return torch.load(path, map_location="cpu")


def _random_init(mod, seed):
    from . import synthetic as S
    return mod.load_state_dict(S.random_state_dict(mod.param_shapes(), seed, device="cuda", fast=True))


def base_models(args):
    """The parts of the SD-2 inpainting base every validation runs (src/eval.py:158-163): dict(scheduler, text_encoder, vae, tokenizer)
    from `--pretrained_model_name_or_path`, or seeded random weights (and the stand-in tokenizer when no tokenizer files are there)."""
    from . import AutoencoderKL, CLIPTextModel, DDIMScheduler, synthetic as S
    from .vae import vae_param_shapes
    m = dict(scheduler=DDIMScheduler())
    if args.random_init:
        m["text_encoder"] = _random_init(CLIPTextModel(), args.seed + 10)
        m["vae"] = AutoencoderKL().load_state_dict(S.random_state_dict(vae_param_shapes({}), args.seed + 1, device="cuda", fast=True))
        m["tokenizer"] = _try_tokenizer(args) or StandInTokenizer()
    else:
        root = args.pretrained_model_name_or_path
        m["text_encoder"] = CLIPTextModel().load_state_dict(_load_folder_state_dict(os.path.join(root, "text_encoder")))
        m["vae"] = AutoencoderKL().load_state_dict(_load_folder_state_dict(os.path.join(root, "vae")))
        m["tokenizer"] = _try_tokenizer(args)
        if m["tokenizer"] is None:
            raise FileNotFoundError(f"no tokenizer files under {root}/tokenizer")
    return m


def adapter_models(args, text_encoder):
    """src/eval.py:240-278 (and src/train_inversion_adapter.py:230-260): the inversion adapter with `--num_encoder_layers` layers from
    `--inversion_adapter_dir` / `--inversion_adapter_name`, and the CLIP vision tower (None with --use_clip_cloth_features)."""
    from . import CLIPVisionModelWithProjection, InversionAdapter
    vis = CLIPVisionModelWithProjection()
    ia = InversionAdapter(input_dim=vis.config.hidden_size, hidden_dim=vis.config.hidden_size * 4,
                          output_dim=text_encoder.config.hidden_size * args.num_vstar, num_encoder_layers=args.num_encoder_layers,
                          config=vis.config)
    if args.random_init:
        ia = _random_init(ia, args.seed + 12)
    else:
        ia = ia.load_state_dict(_load(checkpoint_path(args.inversion_adapter_dir, args.inversion_adapter_name, "inversion_adapter")))
    vision = None
    if not args.use_clip_cloth_features:
        vision = (_random_init(vis, args.seed + 11) if args.random_init
                  else vis.load_state_dict(_load_folder_state_dict(args.vision_model_name_or_path), strict=False))
    return ia, vision


def _pseudo_word_states(pipe, inversion_adapter, batch, vision_encoder, processor, num_vstar):
    """image_from_pipe.py:62-83 (and :160-190): CLIP features of the cloth (the batch's `clip_cloth_features` when present) -> inversion
    adapter -> the category prompt with `num_vstar` pseudo-words -> text encoder states."""
    from . import encode_text_word_embedding
    device = pipe.device
    clip_cloth_features = batch.get("clip_cloth_features")
    if clip_cloth_features is None:
        clip_cloth_features = vision_encoder(clip_pixel_values(batch["cloth"], device, processor)).last_hidden_state
    word_embeddings = inversion_adapter(clip_cloth_features.to(device))
    word_embeddings = word_embeddings.reshape((word_embeddings.shape[0], num_vstar, -1))
    tok = pipe.tokenizer
    tokenized_text = tok(prompts_for(batch["category"], num_vstar), max_length=tok.model_max_length, padding="max_length", truncation=True,
                         return_tensors="pt").input_ids
    return encode_text_word_embedding(pipe.text_encoder, tokenized_text, word_embeddings, num_vstar).last_hidden_state


@torch.no_grad()
def eval_batch(pipe, inversion_adapter, batch, text_usage, vision_encoder, processor, cloth_input_type, cloth_cond_rate, num_vstar, generator,
               num_inference_steps, guidance_scale):
    """The loop body of src/utils/image_from_pipe.py:42-117 -> list of PIL images.  `warped_cloth` is the dataset's (the warping module
    does not run here); the CLIP features are the batch's `clip_cloth_features` when present, else CLIP preprocessing + the vision tower."""
    model_img = batch.get("image")
    mask_img = batch.get("inpaint_mask")
    if mask_img is not None:
        mask_img = mask_img.type(torch.float32)
    pose_map, warped_cloth = batch.get("pose_map"), batch.get("warped_cloth")
    if text_usage == "noun_chunks":
        prompts = batch["captions"]
    elif text_usage == "none":
        prompts = [""] * len(batch["captions"])
    elif text_usage == "inversion_adapter":
        encoder_hidden_states = _pseudo_word_states(pipe, inversion_adapter, batch, vision_encoder, processor, num_vstar)
    else:
        raise ValueError(f"Unknown text usage {text_usage}")
    kw = dict(image=model_img, mask_image=mask_img, pose_map=pose_map, warped_cloth=warped_cloth, height=512, width=384,
              guidance_scale=guidance_scale, num_images_per_prompt=1, generator=generator, cloth_input_type=cloth_input_type,
              cloth_cond_rate=cloth_cond_rate, num_inference_steps=num_inference_steps)
    if text_usage == "inversion_adapter":
        return pipe(prompt_embeds=encoder_hidden_states, **kw).images
    return pipe(prompt=prompts, **kw).images


@torch.no_grad()
def generate_images_from_tryon_pipe(pipe, inversion_adapter, test_dataloader, output_dir: str, order: str, save_name: str, text_usage: str,
                                    vision_encoder, processor, cloth_input_type: str, cloth_cond_rate: int = 1, num_vstar: int = 1,
                                    seed: int = 1234, num_inference_steps: int = 50, guidance_scale: int = 7.5, use_png: bool = False):
    """src/utils/image_from_pipe.py:26-130 (same signature): every batch of `test_dataloader` through `eval_batch`, images written to
    `<output_dir>/<save_name>_<order>/<category>/<im_name>`.  Returns the written paths."""
    save_path = os.path.join(output_dir, f"{save_name}_{order}")
    os.makedirs(save_path, exist_ok=True)
    generator = torch.Generator("cuda").manual_seed(seed)
    written = []
    for batch in test_dataloader:
        images = eval_batch(pipe, inversion_adapter, batch, text_usage, vision_encoder, processor, cloth_input_type, cloth_cond_rate, num_vstar,
                            generator, num_inference_steps, guidance_scale)
        written += save_images(images, batch["category"], batch["im_name"], save_path, use_png)
    return written


@torch.no_grad()
def adapter_val_batch(pipe, inversion_adapter, vision_encoder, processor, batch, num_vstar, generator, num_inference_steps, guidance_scale):
    """The loop body of src/utils/image_from_pipe.py:154-203 -> list of PIL images: pseudo-word text states from the cloth, then the
    inpainting pipeline on the person image and its inpainting mask at 512x384, one image per prompt."""
    encoder_hidden_states = _pseudo_word_states(pipe, inversion_adapter, batch, vision_encoder, processor, num_vstar)
    return pipe(image=batch["image"], mask_image=batch["inpaint_mask"].type(torch.float32), prompt_embeds=encoder_hidden_states, height=512,
                width=384, guidance_scale=guidance_scale, num_images_per_prompt=1, generator=generator,
                num_inference_steps=num_inference_steps).images


@torch.no_grad()
def generate_images_inversion_adapter(pipe, inversion_adapter, vision_encoder, processor, test_dataloader, output_dir, order: str,
                                      save_name: str, num_vstar=1, seed=1234, num_inference_steps=50, guidance_scale=7.5, use_png=False):
    """src/utils/image_from_pipe.py:139-218 (same signature): every batch of `test_dataloader` through `adapter_val_batch` with one CUDA
    generator seeded once, images written to `<output_dir>/<save_name>_<order>/<category>/<im_name>`.  Returns the written paths."""
    save_path = os.path.join(output_dir, f"{save_name}_{order}")
    os.makedirs(save_path, exist_ok=True)
    generator = torch.Generator("cuda").manual_seed(seed)
    written = []
    for batch in test_dataloader:
        images = adapter_val_batch(pipe, inversion_adapter, vision_encoder, processor, batch, num_vstar, generator, num_inference_steps,
                                   guidance_scale)
        written += save_images(images, batch["category"], batch["im_name"], save_path, use_png)
    return written


def write_image(u8, path):
    """The tail of torchvision.utils.save_image for one image already quantised by its rule (ops.image_save_u8): `Image.fromarray(ndarr)
    .save(fp)` with the format taken from the file name and no other argument.  The reference passes `quality=95`, which never reaches
    PIL (DESIGN.md section 7), so a `.jpg` is written at PIL's default quality, as it is here."""
    from PIL import Image
    Image.fromarray(u8).save(path)


@torch.no_grad()
def vae_recon_batch(vae, emasc, batch, int_layers, emasc_type):
    """The loop body of src/utils/image_from_pipe.py:234-249 on the device -> the decoded images, NHWC fp32 [B,H,W,4] (first 3 channels):
    the posterior of `image`, the skips `int_layers` of `im_mask` through EMASC with `mask_features` by `inpaint_mask` fused, one
    posterior draw from the global CUDA RNG ([B,4,h,w], as randn_tensor without a generator), and the decode with the skips.
    With emasc_type "none": encode, sample and decode without skips (the reference's branch reads `.latent_dist` off the
    tuple `encode` returns and cannot run; this is what it means to do, the VAE-only reconstruction)."""
    from . import ops
    from .vae import DiagonalGaussianDistribution
    device = vae.device
    image = batch["image"].to(device, torch.float32)
    mom, _ = vae.encode_nhwc(image)
    feats = None
    if emasc_type != "none":
        _, skips = vae.encode_nhwc(batch["im_mask"].to(device, torch.float32))
        sel = [skips[i] for i in int_layers]
        mask = batch["inpaint_mask"].to(device, torch.float32).contiguous()
        feats = emasc(sel, [ops.inv_mask_rows(mask, image.shape[2] // f.shape[1]) for f in sel])
    latents = DiagonalGaussianDistribution(mom, vae.config.latent_channels).sample()
    return vae.decode_nhwc(latents, feats, list(int_layers) if feats is not None else None)


@torch.no_grad()
def extract_save_vae_images(vae, emasc, test_dataloader, int_layers, output_dir: str, order: str, save_name: str, emasc_type: str):
    """src/utils/image_from_pipe.py:221-258 (same signature), the EMASC trainer's validation: every batch of `test_dataloader` through
    `vae_recon_batch`, save_image's quantisation of `(x + 1) / 2` on the device (ops.image_save_u8), one device-to-host copy of the uint8
    images, each written by `write_image` to `<output_dir>/<save_name>_<order>/<category>/<im_name>`.  Returns the written paths."""
    from . import ops
    save_path = os.path.join(output_dir, f"{save_name}_{order}")
    os.makedirs(save_path, exist_ok=True)
    written = []
    for batch in test_dataloader:
        u8 = ops.image_save_u8(vae_recon_batch(vae, emasc, batch, int_layers, emasc_type)).cpu().numpy()
        for img, cat, name in zip(u8, batch["category"], batch["im_name"]):
            os.makedirs(os.path.join(save_path, cat), exist_ok=True)
            write_image(img, os.path.join(save_path, cat, name))
            written.append(os.path.join(save_path, cat, name))
    return written


class _RankShard:
    """Every world-th batch of a dataloader, like the sharded dataloader `accelerator.prepare` returns (src/eval.py:317)."""

    def __init__(self, loader, rank, world):
        self.loader, self.mine = loader, set(batches_for_rank(len(loader), rank, world))

    def __iter__(self):
        return (b for i, b in enumerate(self.loader) if i in self.mine)

    def __len__(self):
        return len(self.mine)


@torch.no_grad()
def main(argv=None, models=None, dataset=None):
    """`models=` / `dataset=` inject prebuilt engine objects (the dict of build_models) / any dataset with the reference's batch keys."""
    args = parse_args(argv)
    check_args(args)
    from . import StableDiffusionTryOnePipeline, lib
    lib.load()  # fail before any work if the CUDA extension is missing: there is no CPU path
    if not torch.cuda.is_available():
        raise RuntimeError("ladi_vton_b200.eval needs a CUDA device (sm_90a); there is no CPU path")
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    device = torch.device("cuda", int(os.environ.get("LOCAL_RANK", 0)))
    torch.cuda.set_device(device)
    if args.seed is not None:  # utils/set_seeds.py
        import random
        import numpy as np
        random.seed(args.seed), np.random.seed(args.seed), torch.manual_seed(args.seed), torch.cuda.manual_seed_all(args.seed)
    models = models or build_models(args, device)
    category = [args.category] if args.category != 'all' else ['dresses', 'upper_body', 'lower_body']
    test_dataset = dataset if dataset is not None else build_dataset(args, category, outputlist_for(args))
    loader = torch.utils.data.DataLoader(test_dataset, shuffle=False, batch_size=args.batch_size,
                                         num_workers=args.num_workers if dataset is None and args.synthetic_samples <= 0 else 0)
    val_pipe = StableDiffusionTryOnePipeline(text_encoder=models["text_encoder"], vae=models["vae"], tokenizer=models["tokenizer"],
                                             unet=models["unet"], scheduler=models["scheduler"], emasc=models["emasc"],
                                             emasc_int_layers=INT_LAYERS if models["emasc"] is not None else None).to(device)
    written = generate_images_from_tryon_pipe(val_pipe, models["inversion_adapter"], _RankShard(loader, rank, world), args.output_dir,
                                              args.test_order, args.save_name, args.text_usage, models["vision_encoder"], models.get("processor"),
                                              args.cloth_input_type, 1, args.num_vstar, args.seed, args.num_inference_steps, args.guidance_scale,
                                              args.use_png)
    del val_pipe
    torch.cuda.empty_cache()
    if args.compute_metrics:  # :357-364 -- the metric networks are the reference's own code
        if args.reference_src and args.reference_src not in sys.path:
            sys.path.insert(0, args.reference_src)
        try:
            from utils.val_metrics import compute_metrics
        except ImportError as e:
            raise ImportError(f"--compute_metrics runs the reference's src/utils/val_metrics.py: pass --reference_src ({e})") from e
        metrics = compute_metrics(os.path.join(args.output_dir, f"{args.save_name}_{args.test_order}"), args.test_order, args.dataset,
                                  args.category, ['all'], args.dresscode_dataroot, args.vitonhd_dataroot)
        with open(os.path.join(args.output_dir, f"metrics_{args.save_name}_{args.test_order}_{args.category}.json"), "w+") as f:
            json.dump(metrics, f, indent=4)
    return written


if __name__ == "__main__":
    main()
