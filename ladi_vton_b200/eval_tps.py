"""`python -m ladi_vton_b200.eval_tps` -- validate a trained warping checkpoint on the engine, as the reference's warping trainer does after
each epoch (src/train_tps.py:463-505): `compute_metric` scores `checkpoint_last.pth` on the paired and the unpaired test split with the
L1 loss and the VGG-19 perceptual loss between the warped cloth and the cloth cut from the person image (`im_cloth`).

  * `compute_metric(dataloader, tps, criterion_l1, criterion_vgg, refinement=None, height=512, width=384)` is train_tps.py:29-92 on
    engine objects: the warp of warp.py (the TPS-only stage reads the sampled cloth itself, fp32; with `refinement` the refinement
    network's unclamped output), `vgg.L1Loss` / `vgg.VGGLoss` accumulating on the device (one read-back per split), and the reference's
    `running_loss / (step + 1)`: the mean of the per-batch losses, summed in float64 on the host.  `criterion_vgg=None` gives 0.
    `visual` is the last batch's [[image, cloth, im_cloth, warped_cloth.clamp(-1, 1)]] on the host; the wandb image grids are not built.
    `criterion_l1` may be the reference's `torch.nn.L1Loss()` (mean reduction) or `vgg.L1Loss()`; other callables raise TypeError.
  * The CLI keeps the trainer's flags that the validation reads (train_tps.py:283-310: same names, types, defaults and required-ness)
    and drops TRAINING_ONLY.  `--checkpoints_dir` defaults, as in the reference, to `TPS_checkpoints` in the reference checkout, so it is
    resolved from `--reference_src` (the checkout's `src/`); without either the run refuses.  The checkpoint's `tps`, `refinement` and
    `epoch` entries are read, its optimizer states ignored.  `--stage auto` validates as the trainer did for the epoch that wrote the
    checkpoint: epoch <= --epochs_tps is the TPS-only stage (:452-486), any later epoch the refinement stage (:523-565).
  * The test loaders are the trainer's (:373-381): shuffle=True, drop_last=True, with the global RNG seeded by `torch.manual_seed(1234)`,
    which the reference module runs at import.  `--random_init` has no checkpoint and stands for epoch 0.  The reference's shuffle has also consumed the training epochs' draws by then, so when
    the number of test samples is not a multiple of the batch size, WHICH samples are dropped differs from a given training run (on
    VITON-HD, 2032 test pairs at batch 16, nothing is dropped and the losses do not depend on the order).
  * The results are printed and written as JSON (`--output_json`) under the trainer's wandb keys, plus `epoch` and `stage`.

The VGG-19 weights are torchvision's local file (`--vgg_weights`, vgg.VGG_FILE); `--random_init` draws seeded random weights for every
network and `--synthetic_samples N` replaces the datasets.  The TPS and the refinement network compute in bf16 with fp32 accumulation,
the VGG loss in TF32 (vgg.py).
"""
import argparse
import json
import os
import sys

import torch

OUTPUTLIST = ['c_name', 'im_name', 'cloth', 'image', 'im_cloth', 'im_mask', 'pose_map', 'category']  # src/train_tps.py:326
# src/train_tps.py flags that only training (or the --only_extraction path, out of scope) reads
TRAINING_ONLY = ['--const_weight', '--lr', '--wandb_log', '--wandb_project', '--wandb_entity', '--only_extraction', '--l1_weight',
                 '--save_path', '--epochs_refinement']
STAGES = ("auto", "tps", "refinement")
SEED = 1234  # src/train_tps.py:22-24


def build_parser():
    """The validation flags of src/train_tps.py:283-310, plus an `engine` group."""
    parser = argparse.ArgumentParser(description="Validation of a trained warping checkpoint: L1 and VGG losses of the warped cloth")
    parser.add_argument("--dataset", type=str, required=True, choices=["dresscode", "vitonhd"], help="dataset to use")
    parser.add_argument('--dresscode_dataroot', type=str, help='DressCode dataroot')
    parser.add_argument('--checkpoints_dir', type=str, default=None,
                        help="the trainer's checkpoint directory (default: TPS_checkpoints in the checkout of --reference_src)")
    parser.add_argument('--vitonhd_dataroot', type=str, help='VitonHD dataroot')
    parser.add_argument('--exp_name', type=str, required=True, help='experiment name')
    parser.add_argument('-b', '--batch_size', type=int, default=16, help='train/test batch size')
    parser.add_argument('-j', '--workers', type=int, default=10, help='number of data loading workers')
    parser.add_argument("--height", type=int, default=512)
    parser.add_argument("--width", type=int, default=384)
    parser.add_argument('--dense', dest='dense', default=False, action='store_true', help='use dense uv map')
    parser.add_argument('--vgg_weight', type=float, default=0.25, help='weight for the VGG loss (refinement network)')
    parser.add_argument('--epochs_tps', type=int, default=50, help='number of epochs to train the TPS network')
    eng = parser.add_argument_group("engine", "stage selection, and options for machines without network access")
    eng.add_argument("--reference_src", type=str, default=None,
                     help="`src/` folder of a miccunifi/ladi-vton checkout (dataset classes, default --checkpoints_dir)")
    eng.add_argument("--vgg_weights", type=str, default=None, help=f"torchvision's VGG-19 weight file ({'vgg19-dcbb9e9d.pth'})")
    eng.add_argument("--random_init", action="store_true",
                     help="seeded random weights for every network (synthetic workload); epoch 0, so `--stage auto` is TPS-only")
    eng.add_argument("--synthetic_samples", type=int, default=0, help="use N synthetic samples per split instead of a dataset")
    eng.add_argument("--stage", type=str, default="auto", choices=list(STAGES),
                     help="auto: the stage the trainer validated the checkpoint's epoch in (TPS-only up to --epochs_tps)")
    eng.add_argument("--output_json", type=str, default=None, help="write the results here as JSON")
    return parser


def parse_args(argv=None):
    return build_parser().parse_args(argv)


def checkpoints_dir(args):
    """--checkpoints_dir, or the reference's default PROJECT_ROOT/TPS_checkpoints (train_tps.py:25,287) of the --reference_src checkout."""
    if args.checkpoints_dir is not None:
        return args.checkpoints_dir
    if args.reference_src is None:
        raise ValueError("--checkpoints_dir is not given and its default (TPS_checkpoints in the reference checkout) cannot be resolved "
                         "without --reference_src")
    return os.path.join(os.path.dirname(os.path.abspath(args.reference_src.rstrip("/\\"))), "TPS_checkpoints")


def checkpoint_file(args):
    return os.path.join(checkpoints_dir(args), args.exp_name, "checkpoint_last.pth")


def infer_stage(stage, epoch, epochs_tps):
    """The stage the trainer validated `epoch` in: it saves epoch e + 1 after TPS epoch e < epochs_tps (:452-515)."""
    if stage != "auto":
        return stage
    return "tps" if epoch <= epochs_tps else "refinement"


def check_args(args):
    """Everything that can fail before the GPU is touched: the dataroots (:317-320), the checkpoint and the VGG weight file.  Returns
    (checkpoint dict or None with --random_init, epoch, stage)."""
    if args.synthetic_samples <= 0:
        if args.dataset == "vitonhd" and args.vitonhd_dataroot is None:
            raise ValueError("VitonHD dataroot must be provided")
        if args.dataset == "dresscode" and args.dresscode_dataroot is None:
            raise ValueError("DressCode dataroot must be provided")
    if args.random_init:  # no checkpoint: epoch 0, which `auto` validates as the TPS-only stage, like any epoch <= --epochs_tps
        return None, 0, infer_stage(args.stage, 0, args.epochs_tps)
    path = checkpoint_file(args)
    if not os.path.isfile(path):
        raise FileNotFoundError(f"no warping checkpoint at {path}")
    if args.vgg_weight > 0 and not (args.vgg_weights and os.path.isfile(args.vgg_weights)):
        raise FileNotFoundError(f"--vgg_weight {args.vgg_weight} > 0 needs torchvision's VGG-19 file (--vgg_weights, got {args.vgg_weights})")
    ck = torch.load(path, map_location="cpu")
    epoch = int(ck["epoch"])
    return ck, epoch, infer_stage(args.stage, epoch, args.epochs_tps)


def build_models(args, ck, device):
    """dict(tps, refinement, vgg): src/train_tps.py:384-403 on the engine (vgg None when --vgg_weight <= 0)."""
    from . import synthetic as S
    from .metrics import random_state_dict
    from .vgg import VGG19, VGGLoss
    from .warp import ConvNet_TPS, UNetVanilla, control_points
    tps = ConvNet_TPS(256, 192, 5 if args.dense else 21, 3)
    ref = UNetVanilla(n_channels=8 if args.dense else 24, n_classes=3, bilinear=True)
    vgg = VGGLoss() if args.vgg_weight > 0 else None
    if ck is None:
        tps.load_state_dict(S.warp_state_dict(tps.param_shapes(), SEED + 13, ctrl_bias=torch.atanh(control_points()).view(-1)))
        ref.load_state_dict(S.warp_state_dict(ref.param_shapes(), SEED + 14))
        if vgg is not None:
            vgg.load_state_dict(random_state_dict(VGG19().param_shapes(), SEED + 15))
    else:
        tps.load_state_dict(ck["tps"])
        ref.load_state_dict(ck["refinement"])
        if vgg is not None:
            vgg.load_state_dict(torch.load(args.vgg_weights, map_location="cpu"))
    return dict(tps=tps.to(device), refinement=ref.to(device), vgg=vgg.to(device) if vgg is not None else None)


def build_datasets(args):
    """(paired, unpaired) test datasets of src/train_tps.py:350-368, or synthetic ones."""
    outputlist = OUTPUTLIST + (['dense_uv'] if args.dense else [])
    size = (args.height, args.width)
    if args.synthetic_samples > 0:
        from .inference import SyntheticTryOnDataset
        cats = ['dresses', 'upper_body', 'lower_body'] if args.dataset == "dresscode" else ['upper_body']
        return tuple(SyntheticTryOnDataset(args.synthetic_samples, size, cats, SEED + k, outputlist) for k in (0, 1))
    if args.reference_src and args.reference_src not in sys.path:
        sys.path.insert(0, args.reference_src)
    try:
        if args.dataset == "vitonhd":
            from dataset.vitonhd import VitonHDDataset
            return tuple(VitonHDDataset(phase='test', order=o, dataroot_path=args.vitonhd_dataroot, outputlist=outputlist, size=size)
                         for o in ('paired', 'unpaired'))
        from dataset.dresscode import DressCodeDataset
        return tuple(DressCodeDataset(dataroot_path=args.dresscode_dataroot, phase='test', order=o, outputlist=outputlist, size=size)
                     for o in ('paired', 'unpaired'))
    except ImportError as e:
        raise ImportError("the dataset classes are the reference's own (src/dataset/*.py): pass --reference_src <ladi-vton>/src or use "
                          f"--synthetic_samples N ({e})") from e


@torch.no_grad()
def compute_metric(dataloader, tps, criterion_l1, criterion_vgg, refinement=None, height=512, width=384):
    """src/train_tps.py:29-92 on the engine -> (loss, vgg_loss, visual).  criterion_l1: `vgg.L1Loss()`, or `torch.nn.L1Loss()` with its
    mean reduction (the reference's object; it is computed by the same kernel); criterion_vgg: `vgg.VGGLoss` or None.  Anything else is
    refused with TypeError: both losses accumulate on the device, which a plain callable cannot do."""
    from .vgg import L1Loss, VGGLoss
    from .warp import refine_warped_cloth, tps_warped_cloth
    if isinstance(criterion_l1, torch.nn.L1Loss) and criterion_l1.reduction == "mean":
        criterion_l1 = L1Loss()
    if not isinstance(criterion_l1, L1Loss):
        raise TypeError(f"compute_metric: criterion_l1 must be vgg.L1Loss() or torch.nn.L1Loss(), got {type(criterion_l1).__name__}")
    if criterion_vgg is not None and not isinstance(criterion_vgg, VGGLoss):
        raise TypeError(f"compute_metric: criterion_vgg must be vgg.VGGLoss or None, got {type(criterion_vgg).__name__}")
    dev = tps.device
    accs, last = [], None
    for step, inputs in enumerate(dataloader):
        cloth, im_cloth, im_mask = inputs['cloth'], inputs['im_cloth'], inputs['im_mask']
        pose_map = inputs.get('dense_uv')
        if pose_map is None:
            pose_map = inputs['pose_map']
        if tuple(cloth.shape[-2:]) != (height, width):
            raise ValueError(f"compute_metric: the batch is {tuple(cloth.shape[-2:])}, height x width is {(height, width)}: the engine warps "
                             "at the dataset's resolution")
        if refinement:
            warped = refine_warped_cloth(tps, refinement, cloth, im_mask, pose_map)
        else:
            warped = tps_warped_cloth(tps, cloth, im_mask, pose_map)
        target = im_cloth.to(dev, torch.float32).contiguous()
        acc = torch.zeros(2, dtype=torch.float32, device=dev)  # [L1, VGG] of this batch
        criterion_l1(warped, target, acc=acc[0:1])
        if criterion_vgg:
            criterion_vgg(warped, target, acc=acc[1:2])
        accs.append(acc)
        last = (inputs['image'], cloth, im_cloth, warped)
    if last is None:
        raise ValueError("compute_metric: the dataloader yielded no batch")
    per_batch = torch.stack(accs).cpu().double()  # the one device-to-host read of the split
    running_loss = vgg_running_loss = 0.0
    for l1, vg in per_batch.tolist():
        running_loss += l1
        if criterion_vgg:
            vgg_running_loss += vg
    image, cloth, im_cloth, warped = last
    visual = [[image, cloth, im_cloth, warped.cpu().clamp(-1, 1)]]
    return running_loss / (step + 1), vgg_running_loss / (step + 1), visual


@torch.no_grad()
def main(argv=None, models=None, datasets=None):
    """`models=` (dict(tps, refinement, vgg)) / `datasets=` ((paired, unpaired), the reference's batch keys) inject prebuilt objects.
    Returns the results dict."""
    args = parse_args(argv)
    ck, epoch, stage = check_args(args)
    from . import lib
    from .vgg import L1Loss
    lib.load()
    if not torch.cuda.is_available():
        raise RuntimeError("ladi_vton_b200.eval_tps needs a CUDA device (sm_90a); there is no CPU path")
    device = torch.device("cuda", torch.cuda.current_device())
    models = models or build_models(args, ck, device)
    paired, unpaired = datasets if datasets is not None else build_datasets(args)
    torch.manual_seed(SEED)
    workers = args.workers if datasets is None and args.synthetic_samples <= 0 else 0
    refinement = models["refinement"] if stage == "refinement" else None
    out = dict(epoch=epoch, stage=stage)
    for split, ds in (("paired", paired), ("unpaired", unpaired)):
        loader = torch.utils.data.DataLoader(batch_size=args.batch_size, dataset=ds, shuffle=True, num_workers=workers, drop_last=True)
        loss, vgg_loss, _ = compute_metric(loader, models["tps"], L1Loss(), models["vgg"], refinement=refinement, height=args.height,
                                           width=args.width)
        out[f"eval/eval_loss_{split}"], out[f"eval/eval_vgg_loss_{split}"] = loss, vgg_loss
    print(json.dumps(out), flush=True)
    if args.output_json:
        with open(args.output_json, "w") as f:
            json.dump(out, f, indent=4)
    return out


if __name__ == "__main__":
    main()
