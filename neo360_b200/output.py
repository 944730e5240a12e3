"""Output side of the render path (SURVEY.md section 8(f4)): the step AFTER `render_rays*` in the reference's Lightning systems.

    reference                                              here
    --------------------------------------------------     ------------------------------------------------------------
    LitModel.alter_gather_cat  models/interface.py:30-50    gather_images(): NCCL all-gather of every rank's ray range into frames
    LitModel.psnr_each         models/interface.py:53-61    psnr_each(): clipped squared error reduced on the GPU (neo_clipped_sq_err)
    LitModel.ssim_each         models/interface.py:101-111  ssim_each() / ssim(): piqa's SSIM() in CUDA (neo_ssim, csrc/metrics.cu)
    get_obj_rgbs_from_segmap + psnr_each  models/utils.py:102-109
                                                           psnr_obj_each(): the same reduction over the masked pixels (neo_clipped_sq_err_masked)
    LitModel.lpips_each        models/interface.py:113-122  lpips_each() / lpips(): piqa's LPIPS(network="vgg") with the user's weight files
                                                           (lpips.LPIPS.from_files): VGG-16 trunk as framework convolutions, scaling and
                                                           the distance head in CUDA (neo_lpips_prepare, neo_lpips_head, csrc/lpips.cu)
    LitModel.psnr / .ssim / .lpips  models/interface.py:124-172
                                                           stat(): the {"name", "mean", "test"} dicts write_stats takes
    store_image / store_depth_img / store_depth_raw  models/utils.py:21-53
                                                           store_image() / store_depth_img() / store_depth_raw() (same file naming)
    write_stats                models/utils.py:62-73        write_stats(): results.json, byte for byte
results.json has an LPIPS entry when the caller passes stat("LPIPS", lpips_each(...)) to write_stats; without an LPIPS model nothing
changes.
"""
from __future__ import annotations

import json
import math
import os
from typing import List, Sequence, Tuple

import numpy as np
import torch

from . import _lib as L
from . import sharding


def psnr(pred: torch.Tensor, gt: torch.Tensor) -> float:
    """-10 log10(mean((clip(pred) - clip(gt))^2)); the reduction runs in the library's CUDA kernel (no CPU fallback)."""
    if not (pred.is_cuda and gt.is_cuda):
        raise RuntimeError("neo360_b200 needs CUDA tensors (no CPU fallback)")
    a, b = pred.contiguous().float(), gt.contiguous().float()
    if a.shape != b.shape:
        raise ValueError(f"shape mismatch {tuple(a.shape)} vs {tuple(b.shape)}")
    out = torch.zeros(1, dtype=torch.float64, device=a.device)
    with torch.cuda.device(a.device):
        L.check(L.load().neo_clipped_sq_err(a.data_ptr(), b.data_ptr(), a.numel(), out.data_ptr(), torch.cuda.current_stream().cuda_stream))
    mse = float(out.item()) / a.numel()
    return float("inf") if mse == 0 else -10.0 * math.log10(mse)


def psnr_each(preds: Sequence[torch.Tensor], gts: Sequence[torch.Tensor]) -> torch.Tensor:
    """models/interface.py:53-61"""
    return torch.tensor([psnr(p, g) for p, g in zip(preds, gts)])


def psnr_obj_each(preds: Sequence[torch.Tensor], gts: Sequence[torch.Tensor], masks: Sequence[torch.Tensor]) -> torch.Tensor:
    """get_obj_rgbs_from_segmap (models/utils.py:102-109) followed by psnr_each: the PSNR of each frame's (h,w,3) values over the pixels
    where its (h,w) bool / uint8 mask is non-zero.  An empty mask gives NaN (the reference's mean of an empty tensor).  One launch per
    frame and one device-to-host copy for all of them."""
    preds, gts, masks = list(preds), list(gts), list(masks)
    if not len(preds) == len(gts) == len(masks):
        raise ValueError(f"{len(preds)} preds, {len(gts)} gts and {len(masks)} masks")
    if not preds:
        return torch.tensor([])
    dev = preds[0].device
    sums = torch.zeros(len(preds), dtype=torch.float64, device=dev) if dev.type == "cuda" else None
    counts = torch.zeros(len(preds), dtype=torch.int64, device=dev) if dev.type == "cuda" else None
    keep = []
    for i, (p, g, m) in enumerate(zip(preds, gts, masks)):
        if not (p.is_cuda and g.is_cuda and m.is_cuda and p.device == g.device == m.device == dev):
            raise RuntimeError("neo360_b200 needs CUDA tensors on one device (no CPU fallback)")
        if p.shape != g.shape or p.dim() != 3 or p.shape[-1] != 3 or tuple(m.shape) != tuple(p.shape[:2]):
            raise ValueError(f"frame {i}: pred {tuple(p.shape)}, gt {tuple(g.shape)}, mask {tuple(m.shape)}; expected (h,w,3), (h,w,3), (h,w)")
        if m.dtype not in (torch.bool, torch.uint8):
            raise ValueError(f"frame {i}: the mask must be bool or uint8, not {m.dtype}")
        a, b, mk = p.contiguous().float(), g.contiguous().float(), m.contiguous().view(torch.uint8)
        keep.append((a, b, mk))
        with torch.cuda.device(dev):
            L.check(L.load().neo_clipped_sq_err_masked(a.data_ptr(), b.data_ptr(), mk.data_ptr(), mk.numel(), sums[i:].data_ptr(),
                                                       counts[i:].data_ptr(), torch.cuda.current_stream().cuda_stream))
    out = []
    for s, c in zip(sums.tolist(), counts.tolist()):
        mse = s / c if c else float("nan")
        out.append(float("inf") if mse == 0 else -10.0 * math.log10(mse))
    return torch.tensor(out)


def ssim_batch(pred: torch.Tensor, gt: torch.Tensor, return_map: bool = False):
    """SSIM of (n,H,W,3) frames on the GPU (neo_ssim): float64 (n,) on the frames' device, and with `return_map` the fp32 ss map
    (n,H-10,W-10,3) as well.  The definition is piqa's SSIM() at its defaults, inputs clipped to [0, 1] (csrc/metrics.cu)."""
    if not (pred.is_cuda and gt.is_cuda and pred.device == gt.device):
        raise RuntimeError("neo360_b200 needs CUDA tensors on one device (no CPU fallback)")
    if pred.shape != gt.shape or pred.dim() != 4 or pred.shape[-1] != 3:
        raise ValueError(f"expected two (n,H,W,3) tensors, got {tuple(pred.shape)} and {tuple(gt.shape)}")
    n, H, W, _ = pred.shape
    a, b = pred.contiguous().float(), gt.contiguous().float()
    lib = L.load()
    nbytes = lib.neo_ssim_workspace_bytes(n, H, W)
    if nbytes == 0:
        raise ValueError(f"SSIM needs n >= 1 frames of at least 11x11 pixels, got {tuple(pred.shape)}")
    ws = torch.empty(nbytes // 8, dtype=torch.float64, device=a.device)
    out = torch.empty(n, dtype=torch.float64, device=a.device)
    ss_map = torch.empty(n, H - 10, W - 10, 3, dtype=torch.float32, device=a.device) if return_map else None
    with torch.cuda.device(a.device):
        L.check(lib.neo_ssim(a.data_ptr(), b.data_ptr(), n, H, W, out.data_ptr(), None if ss_map is None else ss_map.data_ptr(),
                             ws.data_ptr(), nbytes, torch.cuda.current_stream().cuda_stream))
    return (out, ss_map) if return_map else out


def ssim(pred: torch.Tensor, gt: torch.Tensor) -> float:
    """SSIM of one (h,w,3) frame, as LitModel.ssim_each computes it per frame (models/interface.py:101-111)."""
    return float(ssim_batch(pred.unsqueeze(0), gt.unsqueeze(0))[0])


def ssim_each(preds: Sequence[torch.Tensor], gts: Sequence[torch.Tensor]) -> torch.Tensor:
    """models/interface.py:101-111: one SSIM per frame, a float32 tensor like psnr_each's.  Frames of equal size go to the GPU in one call;
    each frame's value does not depend on which other frames share its call."""
    preds, gts = list(preds), list(gts)
    if len(preds) != len(gts):
        raise ValueError(f"{len(preds)} preds and {len(gts)} gts")
    groups = {}
    for i, (p, g) in enumerate(zip(preds, gts)):
        if p.shape != g.shape:
            raise ValueError(f"frame {i}: shape mismatch {tuple(p.shape)} vs {tuple(g.shape)}")
        groups.setdefault((tuple(p.shape), p.device, g.device), []).append(i)
    vals = torch.empty(len(preds), dtype=torch.float64)
    for idx in groups.values():
        vals[idx] = ssim_batch(torch.stack([preds[i] for i in idx]), torch.stack([gts[i] for i in idx])).cpu()
    return vals.float()


def lpips(pred: torch.Tensor, gt: torch.Tensor, model) -> float:
    """LPIPS of one (h,w,3) frame with an `neo360_b200.lpips.LPIPS` model on the frame's device: inputs clipped to [0, 1] and scaled as
    piqa scales them (csrc/lpips.cu)."""
    with torch.no_grad():
        return float(model(pred.unsqueeze(0), gt.unsqueeze(0))[0])


def lpips_each(preds: Sequence[torch.Tensor], gts: Sequence[torch.Tensor], model) -> torch.Tensor:
    """models/interface.py:113-122: one LPIPS per frame, one frame at a time as the reference runs them, a float32 tensor like
    ssim_each's."""
    preds, gts = list(preds), list(gts)
    if len(preds) != len(gts):
        raise ValueError(f"{len(preds)} preds and {len(gts)} gts")
    return torch.tensor([lpips(p, g, model) for p, g in zip(preds, gts)], dtype=torch.float64).float()


def stat(name: str, values: torch.Tensor) -> dict:
    """The dict LitModel.psnr / .ssim build from a `*_each` result (models/interface.py:124-155), the input of write_stats."""
    m = values.mean().item()
    return {"name": name, "mean": m, "test": m}


def write_stats(fpath: str, *stats: dict) -> None:
    """models/utils.py:62-73, byte for byte: {name: {key: float}} without "name" / "scene_wise", indent 4, keys sorted.  Stats of the same
    name overwrite each other in call order: the reference's Mip-NeRF 360 call passes psnr and then psnr_obj, both named "PSNR", so its
    results.json holds the object PSNR under "PSNR" (DESIGN.md quirk Q20)."""
    d = {}
    for s in stats:
        d[s["name"]] = {k: float(w) for (k, w) in s.items() if k != "name" and k != "scene_wise"}
    with open(fpath, "w") as fp:
        json.dump(d, fp, indent=4, sort_keys=True)


def gather_images(local: torch.Tensor, image_sizes: Sequence[Tuple[int, int]], world: int, chunk: int, group=None) -> List[torch.Tensor]:
    """alter_gather_cat (models/interface.py:30-50): `local` holds this rank's rays (rows) of the concatenated frames, sharded with
    sharding.shard_range; returns the frames [(h,w,3) | (h,w)] on every rank.  world == 1 needs no process group."""
    n = sum(h * w for h, w in image_sizes)
    allr = local if world == 1 else sharding.gather_rays(local, n, world, chunk, group)
    if allr.dim() == 2 and allr.shape[-1] == 1:
        allr = allr.squeeze(-1)
    ret, cur = [], 0
    for (h, w) in image_sizes:
        ret.append(allr[cur:cur + h * w].reshape(h, w, 3) if allr.dim() == 2 else allr[cur:cur + h * w].reshape(h, w))
        cur += h * w
    return ret


def _to8b(x: np.ndarray) -> np.ndarray:
    return (255 * np.clip(x, 0, 1)).astype(np.uint8)


def store_image(dirpath: str, rgbs: Sequence[torch.Tensor], name: str) -> List[str]:
    """models/utils.py:21-27: one `<name><idx:03d>.jpg` per frame (PPM when PIL is unavailable)."""
    os.makedirs(dirpath, exist_ok=True)
    paths = []
    for i, rgb in enumerate(rgbs):
        img = _to8b(rgb.detach().cpu().numpy())
        try:
            from PIL import Image
            path = os.path.join(dirpath, f"{name}{str(i).zfill(3)}.jpg")
            Image.fromarray(img).save(path)
        except ImportError:
            path = os.path.join(dirpath, f"{name}{str(i).zfill(3)}.ppm")
            with open(path, "wb") as f:
                f.write(b"P6 %d %d 255\n" % (img.shape[1], img.shape[0]))
                f.write(img.tobytes())
        paths.append(path)
    return paths


def depth_images(depths: Sequence[torch.Tensor]) -> List[np.ndarray]:
    """The uint8 (h,w,3) arrays store_depth_img saves (models/utils.py:29-37): depths normalised by the min and max over ALL frames
    together (the range guarded by 1e-8), scaled by 255 and truncated to uint8, then cv2.applyColorMap(COLORMAP_JET), whose output is
    BGR.  The reference hands that BGR array to PIL, which saves it as RGB: red and blue are exchanged in its files (quirk Q19)."""
    try:
        import cv2
    except ImportError as e:
        raise RuntimeError("store_depth_img needs OpenCV (the cv2 module) for the reference's COLORMAP_JET colouring") from e
    depth_maps = [d.detach().cpu().numpy() for d in depths]
    depth_imgs = (depth_maps - np.min(depth_maps)) / (max(np.max(depth_maps) - np.min(depth_maps), 1e-8))
    return [cv2.applyColorMap((img * 255).astype(np.uint8), cv2.COLORMAP_JET) for img in depth_imgs]


def store_depth_img(dirpath: str, depths: Sequence[torch.Tensor], name: str) -> List[str]:
    """models/utils.py:29-43: one `<name><idx:03d>.jpg` per frame of depth_images(depths), saved through PIL as the reference does."""
    from PIL import Image
    os.makedirs(dirpath, exist_ok=True)
    paths = []
    for i, img in enumerate(depth_images(depths)):
        path = os.path.join(dirpath, f"{name}{str(i).zfill(3)}.jpg")
        Image.fromarray(img).save(path)
        paths.append(path)
    return paths


def store_depth_raw(dirpath: str, depths: Sequence[torch.Tensor], name: str) -> List[str]:
    """models/utils.py:45-53: compressed npz per frame."""
    os.makedirs(dirpath, exist_ok=True)
    paths = []
    for i, d in enumerate(depths):
        path = os.path.join(dirpath, f"{name}{str(i).zfill(3)}.npz")
        np.savez_compressed(path, d.detach().cpu().numpy())
        paths.append(path)
    return paths
