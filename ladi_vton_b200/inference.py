"""`python -m ladi_vton_b200.inference` -- the reference's full inference CLI (src/inference.py) on the H100 engine.

Same flags, defaults, choices and required-ness as `parse_args` (src/inference.py:31-96), same dataroot checks (:104-108), same batch body
(:225-324: warp the cloth -> CLIP vision features -> inversion adapter -> pseudo-word text encoding -> try-on pipeline -> save), same output
tree `output_dir/<test_order>/<category>/<im_name>` (jpg quality 95, or png with --use_png).  Every arithmetic stage of the body runs on
the engine's sm_90a kernels; tokenizer, dataset tensorisation and image files stay on the host, as in the reference.

What differs, because the target boxes have no network (the reference downloads everything, :123-138):
  * checkpoints are local files -- `--checkpoint_dir` (or $LADI_CHECKPOINT_DIR) holds the release files `unet_<dataset>.pth`,
    `emasc_<dataset>.pth`, `inversion_adapter_<dataset>.pth`, `warping_<dataset>.pth` (hub.py) and `--pretrained_model_name_or_path` /
    `--vision_model_name_or_path` are local diffusers / transformers folders (state dicts are read with torch.load or safetensors);
  * `--random_init` builds every model with seeded random weights (the synthetic workload of BASELINE.json) and `--synthetic_samples N`
    replaces the dataset by N synthetic samples with the batch keys of src/dataset/vitonhd.py;
  * the real datasets are the reference's own classes (`dataset.vitonhd.VitonHDDataset`, `dataset.dresscode.DressCodeDataset`), imported
    from `--reference_src` (a checkout's `src/` folder) -- dataset code is out of this engine's scope (SURVEY.md 8(f) row 3);
  * multi-process: under torchrun each rank takes every world_size-th batch (what `accelerator.prepare(dataloader)` does at :221) and
    writes its own files; there is no collective.  (`parse_args` of the reference reads a non-existent `args.local_rank` when
    LOCAL_RANK is set, :91-93; here LOCAL_RANK just selects the device.)
  * `--mixed_precision`, `--allow_tf32`, `--enable_xformers_memory_efficient_attention` are accepted: the engine always computes in bf16
    with fp32 accumulation and its attention is already fused.
  * `--compute_metrics` runs the reference's own src/utils/val_metrics.py from `--reference_src`; to score the written images on the
    engine instead: `python -m ladi_vton_b200.val_metrics --gen_folder <output_dir> --test_order <order> --dataset ... --metrics_weights_dir W`.
"""
import argparse
import json
import os
import sys

import torch

CATEGORY_TEXT = {  # src/inference.py:279-283
    'dresses': 'a dress',
    'upper_body': 'an upper body garment',
    'lower_body': 'a lower body garment',
}
CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)  # preprocessor_config.json of laion/CLIP-ViT-H-14-laion2B-s32B-b79K
CLIP_STD = (0.26862954, 0.26130258, 0.27577711)
OUTPUTLIST = ['image', 'pose_map', 'inpaint_mask', 'im_mask', 'category', 'im_name', 'cloth']  # :156


def build_parser():
    """The reference's parser (src/inference.py:32-89) flag for flag, plus an `engine` group for the local-file / synthetic options."""
    parser = argparse.ArgumentParser(description="Full inference script")
    parser.add_argument("--pretrained_model_name_or_path", type=str, default="stabilityai/stable-diffusion-2-inpainting",
                        help="Path to pretrained model or model identifier from huggingface.co/models.")
    parser.add_argument("--output_dir", type=str, required=True, help="Path to the output directory")
    parser.add_argument("--allow_tf32", action="store_true", help="Accepted for compatibility (the engine computes in bf16).")
    parser.add_argument("--seed", type=int, default=1234, help="A seed for reproducible training.")
    parser.add_argument("--batch_size", type=int, default=8, help="Batch size to use.")
    parser.add_argument("--mixed_precision", type=str, default=None, choices=["no", "fp16", "bf16"],
                        help="Accepted for compatibility (the engine computes in bf16 with fp32 accumulation).")
    parser.add_argument("--enable_xformers_memory_efficient_attention", action="store_true",
                        help="Accepted for compatibility (attention is already a fused kernel).")
    parser.add_argument('--dresscode_dataroot', type=str, help='DressCode dataroot')
    parser.add_argument('--vitonhd_dataroot', type=str, help='VitonHD dataroot')
    parser.add_argument("--num_workers", type=int, default=8, help="Number of workers for the dataloader")
    parser.add_argument("--num_vstar", default=16, type=int, help="Number of predicted v* images to use")
    parser.add_argument("--test_order", type=str, required=True, choices=["unpaired", "paired"])
    parser.add_argument("--dataset", type=str, required=True, choices=["dresscode", "vitonhd"], help="dataset to use")
    parser.add_argument("--category", type=str, choices=['all', 'lower_body', 'upper_body', 'dresses'], default='all')
    parser.add_argument("--use_png", default=False, action="store_true", help="Whether to use png or jpg for saving")
    parser.add_argument("--num_inference_steps", default=50, type=int, help="Number of diffusion steps")
    parser.add_argument("--guidance_scale", default=7.5, type=float, help="Guidance scale")
    parser.add_argument("--compute_metrics", default=False, action="store_true", help="Compute metrics after generation")
    eng = parser.add_argument_group("engine", "options for machines without network access")
    eng.add_argument("--checkpoint_dir", type=str, default=None, help="folder with the release .pth files (default $LADI_CHECKPOINT_DIR)")
    eng.add_argument("--vision_model_name_or_path", type=str, default="laion/CLIP-ViT-H-14-laion2B-s32B-b79K",
                     help="local folder of the CLIP ViT-H vision tower (src/inference.py:127-128)")
    eng.add_argument("--reference_src", type=str, default=None, help="`src/` folder of a miccunifi/ladi-vton checkout (dataset classes, metrics)")
    eng.add_argument("--random_init", action="store_true", help="seeded random weights for every model (synthetic workload)")
    eng.add_argument("--synthetic_samples", type=int, default=0, help="use N synthetic samples instead of a dataset")
    return parser


def parse_args(argv=None):
    return build_parser().parse_args(argv)


def check_args(args):
    """src/inference.py:104-108 (synthetic runs need no dataroot)."""
    if args.synthetic_samples <= 0:
        if args.dataset == "vitonhd" and args.vitonhd_dataroot is None:
            raise ValueError("VitonHD dataroot must be provided")
        if args.dataset == "dresscode" and args.dresscode_dataroot is None:
            raise ValueError("DressCode dataroot must be provided")


# ---- data ---------------------------------------------------------------------------------------------------------------------------
class SyntheticTryOnDataset(torch.utils.data.Dataset):
    """N samples with the keys, shapes and value ranges the reference datasets return for `outputlist` (src/dataset/vitonhd.py:109-375):
    image / cloth [3,H,W] in [-1,1], im_mask [3,H,W] (the agnostic person image), pose_map [18,H,W] Gaussian heat-maps,
    inpaint_mask [1,H,W] binary, category str, im_name '<index>.jpg'; for src/eval.py also warped_cloth [3,H,W] in [-1,1], captions
    (a noun-chunk string) and clip_cloth_features (fp16 [257, clip_dim], the cache of src/utils/compute_cloth_clip_features.py); for
    src/train_tps.py also c_name (the cloth's file name), im_cloth [3,H,W] (the person image inside the mask, -1 outside: the garment
    cut from the person) and dense_uv [2,H,W] in [-1,1] (Dress Code's dense UV map, smooth here)."""

    def __init__(self, n, size=(512, 384), categories=('upper_body',), seed=1234, outputlist=None, clip_dim=1280):
        from . import synthetic as S
        self.n, self.size, self.categories = n, size, list(categories)
        self.outputlist = list(outputlist) if outputlist is not None else OUTPUTLIST
        H, W = size
        self.a = S.synthetic_inputs(n, H, W, seed=seed, ctx_dim=8)
        self.w = S.warp_inputs(n, H, W, seed=seed + 1)
        if "clip_cloth_features" in self.outputlist:
            self.clip = torch.randn((n, 257, clip_dim), generator=torch.Generator().manual_seed(seed + 2)).half()

    def __len__(self):
        return self.n

    def __getitem__(self, i):
        mask = self.a["mask_image"][i]
        cat = self.categories[i % len(self.categories)]
        get = dict(image=lambda: self.a["image"][i], cloth=lambda: self.w["cloth"][i], im_mask=lambda: self.a["image"][i] * (mask < 0.5),
                   pose_map=lambda: self.a["pose_map"][i], inpaint_mask=lambda: mask, category=lambda: cat, im_name=lambda: f"{i:05d}_00.jpg",
                   warped_cloth=lambda: self.a["warped_cloth"][i], captions=lambda: f"{CATEGORY_TEXT[cat].split(' ', 1)[1]}, sample {i}",
                   clip_cloth_features=lambda: self.clip[i], c_name=lambda: f"{i:05d}_00.jpg",
                   im_cloth=lambda: torch.where(mask >= 0.5, self.a["image"][i], torch.full_like(self.a["image"][i], -1.0)),
                   dense_uv=lambda: self.w["pose_map"][i][:2] * 2 - 1)
        return {k: get[k]() for k in self.outputlist}


def build_dataset(args, category, outputlist=OUTPUTLIST):
    """src/inference.py:149-180 (src/eval.py:289-310 with its own `outputlist`)."""
    if args.synthetic_samples > 0:
        cats = category if args.dataset == "dresscode" else ['upper_body']
        return SyntheticTryOnDataset(args.synthetic_samples, (512, 384), cats, args.seed, outputlist)
    if args.reference_src and args.reference_src not in sys.path:
        sys.path.insert(0, args.reference_src)
    try:
        if args.dataset == "dresscode":
            from dataset.dresscode import DressCodeDataset
            return DressCodeDataset(dataroot_path=args.dresscode_dataroot, phase='test', order=args.test_order, radius=5,
                                    outputlist=outputlist, category=category, size=(512, 384))
        from dataset.vitonhd import VitonHDDataset
        return VitonHDDataset(dataroot_path=args.vitonhd_dataroot, phase='test', order=args.test_order, radius=5, outputlist=outputlist,
                              size=(512, 384))
    except ImportError as e:
        raise ImportError("the dataset classes are the reference's own (src/dataset/*.py, out of this engine's scope): pass "
                          f"--reference_src <ladi-vton>/src or use --synthetic_samples N ({e})") from e


class StandInTokenizer:
    """Used only with --random_init when no tokenizer files are available: the CLIPTokenizer call surface (`model_max_length`,
    `__call__(text, max_length, padding, truncation, return_tensors).input_ids`) with the ids that matter kept exact -- BOS 49406, EOS/pad
    49407 and '$' -> 259 (the placeholder id src/utils/encode_text_word_embedding.py:20 searches for); every other word hashes to a
    stable id.  Random-weight runs carry no semantics, so only the token pattern matters."""
    model_max_length = 77
    bos_token_id, eos_token_id = 49406, 49407

    def __call__(self, text, max_length=None, padding="max_length", truncation=True, return_tensors="pt"):
        L = max_length or self.model_max_length
        rows = []
        for t in ([text] if isinstance(text, str) else text):
            ids = [self.bos_token_id]
            for wd in t.split():
                ids.append(259 if wd == "$" else 1000 + sum((i + 1) * ord(ch) for i, ch in enumerate(wd)) % 40000)
            ids = ids[:L - 1] + [self.eos_token_id]
            rows.append(ids + [self.eos_token_id] * (L - len(ids)))

        class _Out:
            input_ids = torch.tensor(rows, dtype=torch.long)
        return _Out()


def _load_folder_state_dict(folder):
    for name in ("model.safetensors", "diffusion_pytorch_model.safetensors"):
        p = os.path.join(folder, name)
        if os.path.isfile(p):
            from safetensors.torch import load_file
            return load_file(p)
    for name in ("pytorch_model.bin", "diffusion_pytorch_model.bin"):
        p = os.path.join(folder, name)
        if os.path.isfile(p):
            return torch.load(p, map_location="cpu")
    raise FileNotFoundError(f"no model.safetensors / pytorch_model.bin / diffusion_pytorch_model.* in {folder} (no network: "
                            "--pretrained_model_name_or_path and --vision_model_name_or_path must be local folders, or use --random_init)")


def build_models(args, device):
    """src/inference.py:123-138 -> dict(scheduler, text_encoder, vae, vision_encoder, tokenizer, unet, emasc, inversion_adapter, tps,
    refinement), every module an engine object already on `device`."""
    from . import AutoencoderKL, CLIPTextModel, CLIPVisionModelWithProjection, DDIMScheduler, hub, synthetic as S
    from .warp import ConvNet_TPS, UNetVanilla, control_points
    m = dict(scheduler=DDIMScheduler())
    if args.random_init:
        rnd = lambda mod, seed: mod.load_state_dict(S.random_state_dict(mod.param_shapes(), seed, device="cuda", fast=True))  # noqa: E731
        sds = S.build_state_dicts(seed=args.seed, device="cuda")
        m["text_encoder"] = rnd(CLIPTextModel(), args.seed + 10)
        m["vision_encoder"] = rnd(CLIPVisionModelWithProjection(), args.seed + 11)
        m["vae"] = AutoencoderKL().load_state_dict(sds["vae"])
        m["unet"] = hub.extended_unet(args.dataset, state_dict=sds["unet"])
        m["emasc"] = hub.emasc(args.dataset, state_dict=sds["emasc"])
        ia = hub.InversionAdapter(input_dim=1280, hidden_dim=5120, output_dim=1024 * args.num_vstar, num_encoder_layers=1, heads=16, mlp_dim=5120)
        m["inversion_adapter"] = rnd(ia, args.seed + 12)
        tps, ref = ConvNet_TPS(256, 192, 21, 3), UNetVanilla(n_channels=24, n_classes=3, bilinear=True)
        bias = torch.atanh(control_points()).view(-1)  # regression head starts at the identity lattice, ConvNet_TPS.py:199-203
        m["tps"] = tps.load_state_dict(S.warp_state_dict(tps.param_shapes(), args.seed + 13, ctrl_bias=bias))
        m["refinement"] = ref.load_state_dict(S.warp_state_dict(ref.param_shapes(), args.seed + 14))
        m["tokenizer"] = _try_tokenizer(args) or StandInTokenizer()
    else:
        root = args.pretrained_model_name_or_path
        m["text_encoder"] = CLIPTextModel().load_state_dict(_load_folder_state_dict(os.path.join(root, "text_encoder")))
        m["vae"] = AutoencoderKL().load_state_dict(_load_folder_state_dict(os.path.join(root, "vae")))
        m["vision_encoder"] = CLIPVisionModelWithProjection().load_state_dict(_load_folder_state_dict(args.vision_model_name_or_path), strict=False)
        m["tokenizer"] = _try_tokenizer(args)
        if m["tokenizer"] is None:
            raise FileNotFoundError(f"no tokenizer files under {root}/tokenizer")
        m["unet"] = hub.extended_unet(args.dataset, checkpoint_dir=args.checkpoint_dir)
        m["emasc"] = hub.emasc(args.dataset, checkpoint_dir=args.checkpoint_dir)
        m["inversion_adapter"] = hub.inversion_adapter(args.dataset, checkpoint_dir=args.checkpoint_dir)
        m["tps"], m["refinement"] = hub.warping_module(args.dataset, checkpoint_dir=args.checkpoint_dir)
    for k, v in m.items():
        if hasattr(v, "to") and k not in ("scheduler", "tokenizer"):
            v.to(device)
            if hasattr(v, "eval"):
                v.eval()
    return m


def _try_tokenizer(args):
    folder = os.path.join(args.pretrained_model_name_or_path, "tokenizer")
    if not os.path.isdir(folder):
        return None
    from transformers import CLIPTokenizer
    return CLIPTokenizer.from_pretrained(folder)


def clip_pixel_values(cloth, device, processor=None, mode="uint8"):
    """src/inference.py:265-268: resize((cloth + 1) / 2, (224, 224), antialias=True).clamp(0, 1) -> processor(...).pixel_values.
    With a `processor` object (the reference's `AutoProcessor`, when its files are available locally) the host path of the reference is
    kept byte for byte; otherwise the resize, the clamp and the CLIP normalisation run as one kernel (ops.clip_preprocess).  What
    CLIPImageProcessor does to [0,1] floats is version behaviour (DESIGN.md section 7): `mode` = "uint8" (default, the
    pinned transformers 4.27.3: floats round-trip through uint8), "double_rescale" ((v/255 - mean)/std, transformers >= 4.28 incl. the
    installed 5.5) or "float" ((v - mean)/std)."""
    from . import ops
    if processor is not None:
        import torchvision
        x = torchvision.transforms.functional.resize((cloth + 1) / 2, (224, 224), antialias=True).clamp(0, 1)
        return processor(images=x, return_tensors="pt").pixel_values.to(device)
    if mode not in ("uint8", "double_rescale", "float"):
        raise ValueError(f"unknown CLIP preprocessing mode {mode!r}")
    k = 255.0 if mode == "double_rescale" else 1.0  # (v/255 - mean)/std == (v - 255 mean)/(255 std)
    mean = torch.tensor(CLIP_MEAN, dtype=torch.float32, device=device) * k
    std = torch.tensor(CLIP_STD, dtype=torch.float32, device=device) * k
    return ops.clip_preprocess(cloth.to(device, torch.float32).contiguous(), 224, 224, mean, std, quantise=(mode == "uint8"))


def prompts_for(categories, num_vstar):
    """src/inference.py:279-286 (the exact string, spacing included: the tokenizer sees `num_vstar` '$' words)."""
    return [f'a photo of a model wearing {CATEGORY_TEXT[c]} {" $ " * num_vstar}' for c in categories]


def run_batch(batch, models, pipe, args, generator, device, processor=None, size=(512, 384)):
    """The loop body src/inference.py:226-312 -> list of PIL images."""
    from . import encode_text_word_embedding, generate_warped_cloth
    model_img, mask_img, pose_map = batch["image"].float(), batch["inpaint_mask"].float(), batch["pose_map"].float()
    cloth, im_mask = batch["cloth"].float(), batch["im_mask"].float()
    warped_cloth = generate_warped_cloth(models["tps"], models["refinement"], cloth, im_mask, pose_map)  # :236-263
    pixel_values = clip_pixel_values(cloth, device, processor)  # :265-268
    clip_cloth_features = models["vision_encoder"](pixel_values).last_hidden_state  # :269-273
    word_embeddings = models["inversion_adapter"](clip_cloth_features)  # :276
    word_embeddings = word_embeddings.reshape((word_embeddings.shape[0], args.num_vstar, -1))  # :277
    tok = models["tokenizer"]
    tokenized_text = tok(prompts_for(batch["category"], args.num_vstar), max_length=tok.model_max_length, padding="max_length",
                         truncation=True, return_tensors="pt").input_ids  # :289-291
    encoder_hidden_states = encode_text_word_embedding(models["text_encoder"], tokenized_text, word_embeddings,
                                                       args.num_vstar).last_hidden_state  # :294-295
    return pipe(image=model_img, mask_image=mask_img, pose_map=pose_map, warped_cloth=warped_cloth, prompt_embeds=encoder_hidden_states,
                height=size[0], width=size[1], guidance_scale=args.guidance_scale, num_images_per_prompt=1, generator=generator,
                cloth_input_type='warped', num_inference_steps=args.num_inference_steps).images  # :298-311


def save_images(images, categories, names, save_dir, use_png):
    """src/inference.py:314-324."""
    paths = []
    for gen_image, cat, name in zip(images, categories, names):
        os.makedirs(os.path.join(save_dir, cat), exist_ok=True)
        if use_png:
            name = name.replace(".jpg", ".png")
            gen_image.save(os.path.join(save_dir, cat, name))
        else:
            gen_image.save(os.path.join(save_dir, cat, name), quality=95)
        paths.append(os.path.join(save_dir, cat, name))
    return paths


def batches_for_rank(n_batches, rank, world):
    """Which batch indices a rank processes: every world-th batch, like the sharded dataloader `accelerator.prepare` returns (:221)."""
    return [i for i in range(n_batches) if i % world == rank]


@torch.no_grad()
def main(argv=None, models=None, dataset=None, size=(512, 384)):
    """`models=` / `dataset=` inject prebuilt engine objects / any dataset with the reference's batch keys (used by the tests)."""
    args = parse_args(argv)
    check_args(args)
    from . import StableDiffusionTryOnePipeline, lib
    lib.load()  # fail before any work if the CUDA extension is missing: there is no CPU path
    if not torch.cuda.is_available():
        raise RuntimeError("ladi_vton_b200.inference needs a CUDA device (sm_90a); there is no CPU path")
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    device = torch.device("cuda", int(os.environ.get("LOCAL_RANK", 0)))
    torch.cuda.set_device(device)
    if args.seed is not None:  # utils/set_seeds.py
        import random
        import numpy as np
        random.seed(args.seed), np.random.seed(args.seed), torch.manual_seed(args.seed), torch.cuda.manual_seed_all(args.seed)
    models = models or build_models(args, device)
    if args.enable_xformers_memory_efficient_attention:
        models["unet"].enable_xformers_memory_efficient_attention()
    category = [args.category] if args.category != 'all' else ['dresses', 'upper_body', 'lower_body']
    test_dataset = dataset if dataset is not None else build_dataset(args, category)
    test_dataloader = torch.utils.data.DataLoader(test_dataset, shuffle=False, batch_size=args.batch_size,
                                                  num_workers=args.num_workers if dataset is None and args.synthetic_samples <= 0 else 0)
    val_pipe = StableDiffusionTryOnePipeline(text_encoder=models["text_encoder"], vae=models["vae"], tokenizer=models["tokenizer"],
                                             unet=models["unet"], scheduler=models["scheduler"], emasc=models["emasc"],
                                             emasc_int_layers=[1, 2, 3, 4, 5]).to(device)
    save_dir = os.path.join(args.output_dir, args.test_order)
    os.makedirs(save_dir, exist_ok=True)
    generator = torch.Generator("cuda").manual_seed(args.seed)
    written = []
    try:
        from tqdm import tqdm
        it = tqdm(test_dataloader, disable=rank != 0)
    except ImportError:
        it = test_dataloader
    mine = set(batches_for_rank(len(test_dataloader), rank, world))
    for idx, batch in enumerate(it):
        if idx not in mine:
            continue
        images = run_batch(batch, models, val_pipe, args, generator, device, processor=models.get("processor"), size=size)
        written += save_images(images, batch["category"], batch["im_name"], save_dir, args.use_png)
    del val_pipe
    torch.cuda.empty_cache()
    if args.compute_metrics:  # :338-343 -- the metric code (FID/KID/LPIPS networks) is the reference's own and needs its dependencies
        if args.reference_src and args.reference_src not in sys.path:
            sys.path.insert(0, args.reference_src)
        try:
            from utils.val_metrics import compute_metrics
        except ImportError as e:
            raise ImportError(f"--compute_metrics runs the reference's src/utils/val_metrics.py: pass --reference_src ({e})") from e
        metrics = compute_metrics(save_dir, args.test_order, args.dataset, args.category, ['all'], args.dresscode_dataroot, args.vitonhd_dataroot)
        with open(os.path.join(save_dir, f"metrics_{args.test_order}_{args.category}.json"), "w+") as f:
            json.dump(metrics, f, indent=4)
    return written


if __name__ == "__main__":
    main()
