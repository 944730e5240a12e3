"""TEST INFRASTRUCTURE ONLY -- the training step of the reference's Mip-NeRF 360 (LitMipNeRF360.training_step,
models/mipnerf360/model.py:427-456) restated on top of `mip_oracle`'s stages.

* `render` is `mip_oracle.render` as training runs it: sdist is detached after `sample_intervals` (stop_level_grad, model.py:309-310), so
  under autograd the outputs are differentiable w.r.t. the MLP parameters exactly as the reference's are; the initial sdist / weights follow
  the rays' dtype and device, so it runs in float64 and on the GPU (the eager baseline of tools/bench_mip_train.py).  Forward values are
  `mip_oracle.render`'s.
* `searchsorted`, `lossfun_outer`, `lossfun_distortion`: the reference's own mask / O(N^2) forms (helper.py:108-152).
* `training_loss_terms`: the data, interlevel and distortion terms of the training loss (model.py:442-449, 725-741).

Pinned to the unmodified reference by oracle/make_golden_mip_train.py (tests/golden/mip360_train_vectors.npz).  Nothing under
`neo360_b200/` imports this file.
"""
from __future__ import annotations

from typing import Dict, List, Optional

import torch

from .mip_oracle import EPS, alpha_weights, cast_cone, contract, ipe_features, max_dilate_weights, mlp, sample_intervals

Tensor = torch.Tensor


def render(batch: Dict[str, Tensor], P: Dict[str, Tensor], basis: Tensor, n_prop: int, n_nerf: int, near: float, far: float,
           train_frac: float = 1.0, rand: Optional[List[Tensor]] = None):
    """MipNeRF360.forward (model.py:236-365) in training: 3 levels, defaults, sdist detached.  rand = per-level (B,1) jitters."""
    o, d, vd, radii = batch["rays_o"], batch["rays_d"], batch["viewdirs"], batch["radii"]
    B = o.shape[0]
    s_to_t = lambda s: 1 / (s * (1 / far) + (1 - s) * (1 / near))
    sdist = torch.cat([torch.zeros(B, 1, dtype=o.dtype, device=o.device), torch.ones(B, 1, dtype=o.dtype, device=o.device)], -1)
    weights = torch.ones(B, 1, dtype=o.dtype, device=o.device)
    prod = 1
    renderings, history = [], []
    for lvl in range(3):
        is_prop = lvl < 2
        n = n_prop if is_prop else n_nerf
        dilation = 0.0025 + 0.5 * 1.0 / prod
        prod *= n
        if lvl > 0:
            sdist, weights = max_dilate_weights(sdist, weights, dilation)
            sdist, weights = sdist[..., 1:-1], weights[..., 1:-1]
        anneal = (10 * train_frac) / (9 * train_frac + 1)
        logits = torch.where(sdist[..., 1:] > sdist[..., :-1], anneal * torch.log(weights + 0.0), torch.full_like(weights, -torch.inf))
        sdist = sample_intervals(sdist, logits, n, None if rand is None else rand[lvl]).detach()     # stop_level_grad
        tdist = s_to_t(sdist)
        z, zc = contract(*cast_cone(tdist, o, d, radii))
        density, rgb = mlp(P, f"mlps.{lvl}.", ipe_features(z, zc, basis), vd, 4 if is_prop else 8, is_prop)
        weights = alpha_weights(density, tdist, d)
        acc = weights.sum(-1)
        renderings.append({"rgb": (weights[..., None] * rgb).sum(-2) + torch.clip(1 - acc[..., None], min=0) * 1.0})
        history.append({"density": density, "rgb": rgb, "sdist": sdist, "weights": weights})
    return renderings, history


def searchsorted(a, v):
    """helper.py:108-113 (mask form)."""
    i = torch.arange(a.shape[-1], device=a.device)
    v_ge_a = v[..., None, :] >= a[..., :, None]
    idx_lo = torch.where(v_ge_a, i[..., :, None], i[..., :1, None]).max(dim=-2).values
    idx_hi = torch.where(~v_ge_a, i[..., :, None], i[..., -1:, None]).min(dim=-2).values
    return idx_lo, idx_hi


def lossfun_outer(t, w, t_env, w_env):
    """helper.py:117-141: the outer half of inner_outer, then clip(w - w_outer, 0)^2 / (w + eps)."""
    cy1 = torch.cat([torch.zeros_like(w_env[..., :1]), torch.cumsum(w_env, dim=-1)], dim=-1)
    idx_lo, idx_hi = searchsorted(t_env, t)
    w_outer = torch.take_along_dim(cy1, idx_hi, dim=-1)[..., 1:] - torch.take_along_dim(cy1, idx_lo, dim=-1)[..., :-1]
    return torch.clip(w - w_outer, min=0) ** 2 / (w + EPS)


def lossfun_distortion(t, w):
    """helper.py:145-152, the O(N^2) form."""
    ut = (t[..., 1:] + t[..., :-1]) / 2
    dut = torch.abs(ut[..., :, None] - ut[..., None, :])
    loss_inter = torch.sum(w * torch.sum(w[..., None, :] * dut, dim=-1), dim=-1)
    loss_intra = torch.sum(w ** 2 * (t[..., 1:] - t[..., :-1]), dim=-1) / 3
    return loss_inter + loss_intra


def training_loss_terms(renderings, history, target, charb_padding=0.001):
    """LitMipNeRF360.training_step's loss terms (model.py:442-449, 725-741): data, interlevel, distortion (unweighted)."""
    data = torch.sqrt(((renderings[-1]["rgb"] - target) ** 2).mean() + charb_padding ** 2)
    c, w = history[-1]["sdist"].detach(), history[-1]["weights"].detach()
    inter = sum(torch.mean(lossfun_outer(c, w, h["sdist"], h["weights"])) for h in history[:-1])
    dist = torch.mean(lossfun_distortion(history[-1]["sdist"], history[-1]["weights"]))
    return data, inter, dist
