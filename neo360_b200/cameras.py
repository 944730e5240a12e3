"""Learnable corrections of camera poses, for refining noisy poses by photometric gradient (BARF, NeRF--, CamP style).

`PoseCorrection(n_views)` holds, per view, an axis-angle rotation w and a translation tau, both zero at the start, and maps a stack of
camera-to-world matrices [R | t] to [R exp([w]x) | t + tau].  Feed its output to `ops.sample_rays` / `ops.get_rays`, whose rays are then
differentiable w.r.t. the corrected poses, and those rays to `NeRF.forward` (neo360_b200.vanilla), which then differentiates w.r.t. the rays
even with its MLPs frozen.  The correction is a few framework ops per view; the ray generation and the model stay CUDA."""
from __future__ import annotations

import torch
import torch.nn as nn

Tensor = torch.Tensor

# below this squared angle, sin(th)/th and (1 - cos th)/th^2 come from their Taylor series: the closed forms divide by zero at w = 0 and
# lose digits near it, and sqrt(w . w) has an infinite derivative at zero
_SMALL_ANGLE_SQ = 1e-6


def skew(w: Tensor) -> Tensor:
    """[w]x for w (..., 3): the matrix with [w]x v = w x v."""
    z = torch.zeros_like(w[..., 0])
    return torch.stack([torch.stack([z, -w[..., 2], w[..., 1]], -1),
                        torch.stack([w[..., 2], z, -w[..., 0]], -1),
                        torch.stack([-w[..., 1], w[..., 0], z], -1)], -2)


def so3_exp(w: Tensor) -> Tensor:
    """Rodrigues' formula exp([w]x) = I + A [w]x + B [w]x^2, A = sin th / th, B = (1 - cos th) / th^2, th = |w|, for w (..., 3).  Near
    th = 0 A and B are their series 1 - th^2/6 + th^4/120 and 1/2 - th^2/24 + th^4/720, so the value and the gradient stay finite at 0."""
    th2 = (w * w).sum(-1)
    small = th2 < _SMALL_ANGLE_SQ
    th = torch.sqrt(torch.where(small, torch.ones_like(th2), th2))
    a = torch.where(small, 1 - th2 / 6 + th2 * th2 / 120, torch.sin(th) / th)
    b = torch.where(small, 0.5 - th2 / 24 + th2 * th2 / 720, (1 - torch.cos(th)) / (th * th))
    K = skew(w)
    eye = torch.eye(3, dtype=w.dtype, device=w.device).expand(K.shape)
    return eye + a[..., None, None] * K + b[..., None, None] * (K @ K)


class PoseCorrection(nn.Module):
    """Per-view pose correction: `omega` (n_views, 3) axis-angle and `tau` (n_views, 3) translation, initialised to zero (the identity).
    forward(c2w (n_views, 3, 4) or (n_views, 4, 4)) -> the corrected poses, same shape: R exp([omega]x) and t + tau."""

    def __init__(self, n_views: int):
        super().__init__()
        self.omega = nn.Parameter(torch.zeros(n_views, 3))
        self.tau = nn.Parameter(torch.zeros(n_views, 3))

    def forward(self, c2w: Tensor) -> Tensor:
        if c2w.dim() != 3 or c2w.shape[0] != self.omega.shape[0] or c2w.shape[1] not in (3, 4) or c2w.shape[2] != 4:
            raise ValueError(f"PoseCorrection({self.omega.shape[0]}) takes c2w ({self.omega.shape[0]}, 3|4, 4), got {tuple(c2w.shape)}")
        w, tau = self.omega.to(c2w.dtype), self.tau.to(c2w.dtype)
        R = c2w[:, :3, :3] @ so3_exp(w)
        t = c2w[:, :3, 3] + tau
        out = torch.cat([R, t[..., None]], -1)
        return torch.cat([out, c2w[:, 3:]], 1) if c2w.shape[1] == 4 else out
