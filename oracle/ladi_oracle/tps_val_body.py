"""TEST INFRASTRUCTURE ONLY (see oracle/ladi_oracle/__init__.py) -- fp32 restatement of the warping trainer's validation,
src/train_tps.py:29-92 (`compute_metric`), on the warping oracle (warp.py) and the VGG-loss oracle (vgg.py).  Pinned to what the
reference's own function returns through tests/golden/tps_val_small.npz."""
import torch
import torch.nn.functional as F

from .warp import _resize


def warped_cloth(inputs, tps, refinement=None, height=512, width=384, low=(256, 192)):
    """train_tps.py:44-80: the TPS-only sampled cloth, or the refinement network's (unclamped) output when `refinement` is given."""
    cloth, im_mask = inputs["cloth"].float(), inputs["im_mask"].float()
    pose_map = inputs.get("dense_uv")
    if pose_map is None:
        pose_map = inputs["pose_map"]
    pose_map = pose_map.float()
    agnostic = torch.cat([_resize(im_mask, low), _resize(pose_map, low)], 1)
    low_grid, _ = tps(_resize(cloth, low), agnostic)
    grid = _resize(low_grid.permute(0, 3, 1, 2), (height, width)).permute(0, 2, 3, 1)
    warped = F.grid_sample(cloth, grid, padding_mode="border", align_corners=False)
    if refinement is not None:
        warped = refinement(torch.cat([im_mask, pose_map, warped], 1))
    return warped


@torch.no_grad()
def compute_metric(batches, tps, criterion_vgg=None, refinement=None, height=512, width=384):
    """-> (loss, vgg_loss, per-batch [(l1, vgg)]): the means of the per-batch losses, as running_loss / (step + 1)."""
    per = []
    for inputs in batches:
        warped = warped_cloth(inputs, tps, refinement, height, width)
        target = inputs["im_cloth"].float().to(warped.device)
        l1 = F.l1_loss(warped, target).item()
        vg = criterion_vgg(warped, target).item() if criterion_vgg is not None else 0.0
        per.append((l1, vg))
    n = len(per)
    return sum(p[0] for p in per) / n, (sum(p[1] for p in per) / n if criterion_vgg is not None else 0), per
