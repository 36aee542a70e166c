"""`python -m ladi_vton_b200.compute_cloth_clip_features` -- the reference's CLIP cloth-feature cache (src/utils/compute_cloth_clip_features.py,
README step 2.5) on the H100 engine: the `last_hidden_state` of the CLIP ViT-H vision tower for every in-shop cloth of the train and test
splits, which `--use_clip_cloth_features` of the training scripts and of `python -m ladi_vton_b200.eval` then read instead of running the
vision tower.

Same flags as its `parse_args` (:30-50), the same splits and dataset arguments (:82-129: order 'paired', radius 5, size 512x384,
outputlist ('cloth', 'c_name')), the same files: `{split}_last_hidden_state_features.pt` (fp16 [N, 257, 1280], the reference's
`.half()`) and `{split}_features_names.pkl` (the pickled list of cloth names in dataset order), under
`<reference checkout>/data/clip_cloth_embeddings/<dataset>/` -- where the reference dataset classes read them (vitonhd.py:100-107) --
or under `--save_dir`.  The CLIP preprocessing and the vision tower run on the engine's kernels (inference.clip_pixel_values,
clip.CLIPVisionModelWithProjection) and compute in bf16 with fp32 accumulation; the reference runs the tower in fp16 under autocast
(:152-158).  The dataset classes are the reference's own, imported from `--reference_src`.
"""
import argparse
import os
import pickle
import sys

import torch


def build_parser():
    parser = argparse.ArgumentParser(description="Precompute the CLIP features of the in-shop cloths")
    parser.add_argument("--dataset", type=str, required=True, choices=["dresscode", "vitonhd"], help="dataset to use")
    parser.add_argument('--dresscode_dataroot', type=str, help='DressCode dataroot')
    parser.add_argument('--vitonhd_dataroot', type=str, help='VitonHD dataroot')
    parser.add_argument("--pretrained_model_name_or_path", type=str, default="stabilityai/stable-diffusion-2-inpainting",
                        help="Base model the features are for; only the SD-2 inpainting base (CLIP ViT-H/14) is built.")
    parser.add_argument("--batch_size", type=int, default=16, help="Batch size (per device) for the testing dataloader.")
    parser.add_argument("--num_workers", type=int, default=8, help="Number of workers for the testing dataloader.")
    eng = parser.add_argument_group("engine", "options for machines without network access")
    eng.add_argument("--vision_model_name_or_path", type=str, default="laion/CLIP-ViT-H-14-laion2B-s32B-b79K",
                     help="local folder of the CLIP ViT-H vision tower")
    eng.add_argument("--reference_src", type=str, default=None, help="`src/` folder of a miccunifi/ladi-vton checkout (dataset classes)")
    eng.add_argument("--save_dir", type=str, default=None,
                     help="output folder (default: <reference checkout>/data/clip_cloth_embeddings/<dataset>, next to --reference_src)")
    return parser


def default_save_dir(reference_src, dataset):
    """PROJECT_ROOT / 'data' / 'clip_cloth_embeddings' / dataset of the reference (:161), PROJECT_ROOT being the parent of `src/`."""
    if reference_src is None:
        raise ValueError("pass --save_dir, or --reference_src so that the cache lands where the reference dataset classes read it")
    return os.path.join(os.path.dirname(os.path.abspath(reference_src.rstrip("/"))), "data", "clip_cloth_embeddings", dataset)


@torch.no_grad()
def save_cloth_features(loader, vision_encoder, split, save_dir, device, processor=None):
    """:143-166: every batch's cloth -> CLIP pixel values -> vision tower last_hidden_state (stored fp16 on the host) and its `c_name`s;
    writes `{split}_last_hidden_state_features.pt` and `{split}_features_names.pkl` into `save_dir`.  Returns the two paths."""
    from .inference import clip_pixel_values
    feats, names = [], []
    for batch in loader:
        pixel_values = clip_pixel_values(batch["cloth"].float(), device, processor)
        feats.append(vision_encoder(pixel_values).last_hidden_state.cpu().half())
        names.extend(batch["c_name"])
    os.makedirs(save_dir, exist_ok=True)
    fp, npath = os.path.join(save_dir, f"{split}_last_hidden_state_features.pt"), os.path.join(save_dir, f"{split}_features_names.pkl")
    torch.save(torch.cat(feats, dim=0), fp)
    with open(npath, "wb") as f:
        pickle.dump(names, f)
    return fp, npath


def build_datasets(args):
    """:82-129: the train and test splits of the reference dataset classes with outputlist ('cloth', 'c_name')."""
    if args.reference_src and args.reference_src not in sys.path:
        sys.path.insert(0, args.reference_src)
    outputlist = ('cloth', 'c_name')
    try:
        if args.dataset == "dresscode":
            from dataset.dresscode import DressCodeDataset
            return [DressCodeDataset(dataroot_path=args.dresscode_dataroot, phase=phase, order='paired', radius=5,
                                     category=['dresses', 'upper_body', 'lower_body'], size=(512, 384), outputlist=outputlist)
                    for phase in ("train", "test")]
        from dataset.vitonhd import VitonHDDataset
        return [VitonHDDataset(dataroot_path=args.vitonhd_dataroot, phase=phase, order='paired', radius=5, size=(512, 384), outputlist=outputlist)
                for phase in ("train", "test")]
    except ImportError as e:
        raise ImportError(f"the dataset classes are the reference's own (src/dataset/*.py): pass --reference_src <ladi-vton>/src ({e})") from e


@torch.no_grad()
def main(argv=None, vision_encoder=None, datasets=None, processor=None):
    """`vision_encoder=` / `datasets=` (train, test) / `processor=` (a CLIP image processor, see inference.clip_pixel_values) inject
    prebuilt objects (used by the tests)."""
    args = build_parser().parse_args(argv)
    if args.dataset == "vitonhd" and args.vitonhd_dataroot is None and datasets is None:  # :60-63
        raise ValueError("VitonHD dataroot must be provided")
    if args.dataset == "dresscode" and args.dresscode_dataroot is None and datasets is None:
        raise ValueError("DressCode dataroot must be provided")
    if args.pretrained_model_name_or_path != "stabilityai/stable-diffusion-2-inpainting" and not os.path.isdir(args.pretrained_model_name_or_path):
        raise NotImplementedError(f"{args.pretrained_model_name_or_path}: only the SD-2 inpainting base (CLIP ViT-H/14 cloth features) is built")
    save_dir = args.save_dir or default_save_dir(args.reference_src, args.dataset)
    device = torch.device("cuda", int(os.environ.get("LOCAL_RANK", 0)))
    if vision_encoder is None:
        from . import CLIPVisionModelWithProjection, lib
        from .inference import _load_folder_state_dict
        lib.load()
        if not torch.cuda.is_available():
            raise RuntimeError("ladi_vton_b200.compute_cloth_clip_features needs a CUDA device (sm_90a); there is no CPU path")
        vision_encoder = CLIPVisionModelWithProjection().load_state_dict(_load_folder_state_dict(args.vision_model_name_or_path), strict=False)
        vision_encoder.to(device)
    train_ds, test_ds = datasets if datasets is not None else build_datasets(args)
    out = []
    for ds, split in ((train_ds, "train"), (test_ds, "test")):
        loader = torch.utils.data.DataLoader(ds, shuffle=False, batch_size=args.batch_size, num_workers=args.num_workers if datasets is None else 0)
        out += save_cloth_features(loader, vision_encoder, split, save_dir, device, processor)
    return out


if __name__ == "__main__":
    main()
