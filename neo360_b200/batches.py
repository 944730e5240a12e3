"""Training-batch assembly on the device: the dict the reference's dataset hands to `training_step`
(datasets/nerds360_ae.py:513-764; SURVEY.md section 8 row f3).

The reference's `__getitem__` builds, on the host, every ray of the 20 target views (20 x H x W x 3 floats for each of rays_o, rays_d,
viewdirs), stacks them, and keeps `ray_batch_size` = 500 rows chosen by one `torch.randint(0, T*H*W)` (nerds360_ae.py:730-748).  Here the
target views stay resident in HBM as (T,3,4) poses and (T,H,W,3) images, and only the kept rays are computed (`neo_sample_rays`, bit-identical per
ray to the whole-frame generator).  `pix_inds` is drawn exactly as the reference draws it (CPU `torch.randint`, same generator stream), so a
seeded run picks the same pixels; it is the only per-step host-to-device copy (8 bytes per ray).

Disk I/O, PIL/cv2 decoding and scene bookkeeping are out of scope (SURVEY.md section 2 row 19: OUT); callers hand in decoded tensors."""
from __future__ import annotations

from typing import Dict, Optional

import numpy as np
import torch

from . import ops

RAY_BATCH_SIZE = 500      # nerds360_ae.py:535-538
NUM_TARGET_VIEWS = 20     # nerds360_ae.py dest views per item (SURVEY.md section 8 f3)
PATCH = 30                # LPIPS fine-tuning patch side (nerds360_ae.py:638-664)


class TargetViews:
    """Decoded target views of one scene, resident on the device: what `read_data` returns per view (nerds360_ae.py:277-487), minus the rays."""

    def __init__(self, poses: torch.Tensor, images: torch.Tensor, focal: float, instance_masks: Optional[torch.Tensor] = None,
                 nocs_2d: Optional[torch.Tensor] = None):
        if not poses.is_cuda:
            raise RuntimeError("neo360_b200 needs CUDA tensors (no CPU fallback)")
        T, H, W, _ = images.shape
        if poses.shape[0] != T:
            raise ValueError(f"{poses.shape[0]} poses for {T} images")
        self.poses = poses[:, :3, :4].contiguous().float()
        self.images = images.contiguous().float()          # (T,H,W,3) in [0,1]: ToTensor()(img).permute(1,2,0)  (nerds360_ae.py:706-708)
        self.masks = None if instance_masks is None else instance_masks.reshape(-1, 1).float()
        self.nocs = None if nocs_2d is None else nocs_2d.reshape(-1, 3).float()
        self.focal, self.T, self.H, self.W = float(focal), T, H, W


def draw_pix_inds(n_views: int, H: int, W: int, ray_batch_size: int = RAY_BATCH_SIZE, generator: Optional[torch.Generator] = None) -> torch.Tensor:
    """`torch.randint(0, len(dest_view_nums) * H * W, (ray_batch_size,))` on the host, as nerds360_ae.py:730-732 draws it."""
    return torch.randint(0, n_views * H * W, (ray_batch_size,), generator=generator)


def train_batch(views: TargetViews, src: Dict[str, torch.Tensor], pix_inds: Optional[torch.Tensor] = None, ray_batch_size: int = RAY_BATCH_SIZE,
                generator: Optional[torch.Generator] = None) -> Dict[str, torch.Tensor]:
    """One training sample with the reference's keys (nerds360_ae.py:750-764).  `src` carries the source-view entries as the dataset
    produces them: src_imgs (NV,3,H,W) normalised, src_poses, src_focal, src_c."""
    dev = views.poses.device
    if pix_inds is None:
        pix_inds = draw_pix_inds(views.T, views.H, views.W, ray_batch_size, generator)
    pix = pix_inds.to(dev, non_blocking=True)
    o, vd, rd, radii, tgt = ops.sample_rays(pix, views.H, views.W, views.focal, views.poses, views.images)
    n = o.shape[0]
    sample = {k: src[k] for k in ("src_imgs", "src_poses", "src_focal", "src_c")}
    sample["instance_mask"] = views.masks[pix] if views.masks is not None else torch.zeros(n, 1, device=dev)
    sample["rays_o"], sample["rays_d"], sample["viewdirs"] = o, rd, vd
    sample["target"] = tgt
    sample["nocs_2d"] = views.nocs[pix] if views.nocs is not None else torch.zeros(n, 3, device=dev)
    sample["radii"] = radii
    sample["multloss"] = torch.zeros(n, 1, device=dev)
    sample["normals"] = torch.zeros_like(o)
    return sample


def patch_pix_inds(view: int, x: int, y: int, H: int, W: int) -> torch.Tensor:
    """The flat indices into the (T,H,W) stack of the 30x30 patch at row x, column y of target view `view`, in the reference's order
    (`view(H, W)[x:x+30, y:y+30].reshape(-1)`, nerds360_ae.py:638-664): row-major over the patch."""
    if not (0 <= x <= H - PATCH and 0 <= y <= W - PATCH):
        raise ValueError(f"patch at ({x}, {y}) does not fit a {H}x{W} view")
    r = torch.arange(PATCH, dtype=torch.int64)
    return (view * H * W + (x + r)[:, None] * W + (y + r)[None, :]).reshape(-1)


def patch_batch(views: TargetViews, src: Dict[str, torch.Tensor], view: int, x: Optional[int] = None, y: Optional[int] = None) -> Dict[str, torch.Tensor]:
    """The LPIPS fine-tuning sample (nerds360_ae.py:598-664): the 900 rays of one 30x30 patch of target view `view`, with the keys of
    train_batch.  x (row) and y (column) not given are drawn as the reference draws them: np.random.randint(0, H - 30 + 1), then
    np.random.randint(0, W - 30 + 1), from numpy's global generator."""
    if not 0 <= view < views.T:
        raise ValueError(f"view {view} of {views.T}")
    if x is None:
        x = np.random.randint(0, views.H - PATCH + 1)
    if y is None:
        y = np.random.randint(0, views.W - PATCH + 1)
    return train_batch(views, src, pix_inds=patch_pix_inds(view, int(x), int(y), views.H, views.W))
