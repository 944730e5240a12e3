"""TEST INFRASTRUCTURE ONLY -- CPU restatement (oracle) of the Mip-NeRF 360 renderer of the reference
(models/mipnerf360/model.py:30-365, models/mipnerf360/helper.py), SURVEY.md section 8(a) row a18 / Appendix A.6.

Pinned to the unmodified reference by oracle/make_golden.py (tests/golden/mip360_reference_vectors.npz).  The scene
contraction uses the closed-form Jacobian J = f I + ((2-2r)/r^4) x x^T, f = (2r-1)/r^2 for r > 1 (identity inside the unit
ball) instead of functorch.jacrev (helper.py:33-66)."""
from __future__ import annotations

import math
from typing import Dict, List, Optional

import torch
import torch.nn.functional as F

Tensor = torch.Tensor
EPS = 1.1920929e-07


def sorted_interp(x, xp, fp):
    """helper.py:207-222: piecewise-linear interp of fp over sorted xp at x (value max/min under the compare mask)."""
    mask = x[..., None, :] >= xp[..., :, None]
    fp0 = torch.max(torch.where(mask, fp[..., None], fp[..., :1, None]), dim=-2).values
    fp1 = torch.min(torch.where(~mask, fp[..., None], fp[..., -1:, None]), dim=-2).values
    xp0 = torch.max(torch.where(mask, xp[..., None], xp[..., :1, None]), dim=-2).values
    xp1 = torch.min(torch.where(~mask, xp[..., None], xp[..., -1:, None]), dim=-2).values
    off = torch.clip(torch.nan_to_num((x - xp0) / (xp1 - xp0), 0), 0, 1)
    return fp0 + off * (fp1 - fp0)


def max_dilate_weights(t, w, dilation, domain=(0.0, 1.0)):
    """helper.py:152-192 with renormalize=True."""
    p = w / torch.clip(t[..., 1:] - t[..., :-1], min=EPS)
    t0 = t[..., :-1] - dilation
    t1 = t[..., 1:] + dilation
    td = torch.sort(torch.cat([t, t0, t1], -1), -1).values
    td = torch.clip(td, domain[0], domain[1])
    mask = (t0[..., None, :] <= td[..., None]) & (t1[..., None, :] > td[..., None])
    pd = torch.where(mask, p[..., None, :], torch.zeros_like(p[..., None, :])).max(-1).values[..., :-1]
    wd = pd * (td[..., 1:] - td[..., :-1])
    wd = wd / torch.clip(wd.sum(-1, keepdim=True), min=EPS)
    return td, wd


def sample_intervals(t, w_logits, n, u_jitter: Optional[Tensor] = None, domain=(0.0, 1.0)):
    """helper.py:343-396 (single_jitter=True).  u_jitter (B,1) replaces torch.rand when randomized."""
    if u_jitter is None:
        pad = 1 / (2 * n)
        u = torch.linspace(pad, 1 - pad - EPS, n, device=t.device)
        u = torch.broadcast_to(u, t.shape[:-1] + (n,))
    else:
        u_max = EPS + (1 - EPS) / n
        max_jitter = (1 - u_max) / (n - 1) - EPS
        u = torch.linspace(0, 1 - u_max, n, device=t.device) + u_jitter * max_jitter
    u = u.type_as(t)
    w = F.softmax(w_logits, dim=-1)
    cw = torch.cumsum(w[..., :-1], -1).clip(max=1.0)
    one = cw.shape[:-1] + (1,)
    cw = torch.cat([torch.zeros(one).type_as(cw), cw, torch.ones(one).type_as(cw)], -1)
    centers = sorted_interp(u, cw, t)
    mid = (centers[..., 1:] + centers[..., :-1]) / 2
    first = torch.clip(2 * centers[..., :1] - mid[..., :1], min=domain[0])
    last = torch.clip(2 * centers[..., -1:] - mid[..., -1:], max=domain[1])
    return torch.cat([first, mid, last], -1)


def cast_cone(tdist, o, d, radii):
    """helper.py:278-339 (ray_shape='cone', diag=False) -> means (B,n,3), covs (B,n,3,3)."""
    t0, t1 = tdist[..., :-1], tdist[..., 1:]
    mu, hw = (t0 + t1) / 2, (t1 - t0) / 2
    denom = (3 * mu ** 2 + hw ** 2).clip(min=EPS)
    t_mean = mu + (2 * mu * hw ** 2) / denom
    t_var = (hw ** 2) / 3 - (4 / 15) * hw ** 4 * (12 * mu ** 2 - hw ** 2) / denom ** 2
    r_var = ((mu ** 2) / 4 + (5 / 12) * hw ** 2 - (4 / 15) * (hw ** 4) / denom) * radii ** 2
    mean = d[..., None, :] * t_mean[..., None]
    dmag = torch.sum(d ** 2, -1, keepdim=True).clip(min=1e-10)
    d_outer = d[..., :, None] * d[..., None, :]
    null_outer = torch.eye(3, dtype=d.dtype, device=d.device) - d[..., :, None] * (d / dmag)[..., None, :]
    cov = t_var[..., None, None] * d_outer[..., None, :, :] + r_var[..., None, None] * null_outer[..., None, :, :]
    return mean + o[..., None, :], cov


def contract(mean, cov):
    """helper.py:33-66, closed-form Jacobian."""
    r2 = torch.sum(mean ** 2, -1, keepdim=True).clip(min=1e-32)
    r = torch.sqrt(r2)
    inside = r2 <= 1
    f = (2 * r - 1) / r2
    z = torch.where(inside, mean, f * mean)
    g = (2 - 2 * r) / (r2 * r2)
    eye = torch.eye(3, dtype=mean.dtype, device=mean.device)
    J = f[..., None] * eye + g[..., None] * mean[..., :, None] * mean[..., None, :]
    J = torch.where(inside[..., None], eye.expand_as(J), J)
    return z, J @ cov @ J.transpose(-1, -2)


def ipe_features(mean, cov, basis, min_deg=0, max_deg=12):
    """lift_and_diagonalize + integrated_pos_enc (helper.py:70-88): -> (..., 504)."""
    m = mean @ basis
    v = torch.sum(basis[None, None] * (cov @ basis), dim=-2)
    scales = 2.0 ** torch.arange(min_deg, max_deg, dtype=mean.dtype, device=mean.device)
    sm = (m[..., None, :] * scales[:, None]).reshape(*m.shape[:-1], -1)
    sv = (v[..., None, :] * scales[:, None] ** 2).reshape(*v.shape[:-1], -1)
    return torch.exp(-0.5 * torch.cat([sv, sv], -1)) * torch.sin(torch.cat([sm, sm + 0.5 * math.pi], -1))


def dir_enc(x, deg=4):
    scales = 2.0 ** torch.arange(0, deg, dtype=x.dtype, device=x.device)
    xb = (x[..., None, :] * scales[:, None]).reshape(*x.shape[:-1], -1)
    return torch.cat([x, torch.sin(torch.cat([xb, xb + 0.5 * math.pi], -1))], -1)


def mlp(P: Dict[str, Tensor], pre: str, feats: Tensor, viewdirs: Tensor, depth: int, disable_rgb: bool):
    """MipNeRF360MLP.forward (model.py:111-173).  feats (B,n,504)."""
    lin = lambda name, x: F.linear(x, P[pre + name + ".weight"], P[pre + name + ".bias"])
    x = feats
    for i in range(depth):
        x = torch.relu(lin(f"pts_linear.{i}", x))
        if i % 4 == 0 and i > 0:
            x = torch.cat([x, feats], -1)
    density = F.softplus(lin("density_layer", x)[..., 0] - 1.0)
    if disable_rgb:
        return density, torch.zeros(*feats.shape[:-1], 3, dtype=feats.dtype, device=feats.device)
    beta = lin("bottleneck_layer", x)
    de = dir_enc(viewdirs)
    y = torch.relu(lin("views_linear.0", torch.cat([beta, torch.broadcast_to(de[..., None, :], beta.shape[:-1] + (de.shape[-1],))], -1)))
    rgb = torch.sigmoid(lin("rgb_layer", y)) * (1 + 2 * 0.001) - 0.001
    return density, rgb


def alpha_weights(density, tdist, d):
    """helper.py:234-260 (opaque_background=True)."""
    dd = density * (tdist[..., 1:] - tdist[..., :-1]) * torch.norm(d[..., None, :], dim=-1)
    dd = torch.cat([dd[..., :-1], torch.full_like(dd[..., -1:], torch.inf)], -1)
    alpha = 1 - torch.exp(-dd)
    trans = torch.exp(-torch.cat([torch.zeros_like(dd[..., :1]), torch.cumsum(dd[..., :-1], -1)], -1))
    return alpha * trans


def render(batch: Dict[str, Tensor], P: Dict[str, Tensor], basis: Tensor, n_prop: int, n_nerf: int, near: float, far: float,
           train_frac: float = 1.0, rand: Optional[List[Tensor]] = None):
    """MipNeRF360.forward (model.py:236-365), 3 levels, defaults.  rand = per-level (B,1) jitters (randomized=True)."""
    o, d, vd, radii = batch["rays_o"], batch["rays_d"], batch["viewdirs"], batch["radii"]
    B = o.shape[0]
    s_to_t = lambda s: 1 / (s * (1 / far) + (1 - s) * (1 / near))
    sdist = torch.cat([torch.zeros(B, 1), torch.ones(B, 1)], -1)
    weights = torch.ones(B, 1)
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
        sdist = sample_intervals(sdist, logits, n, None if rand is None else rand[lvl])
        tdist = s_to_t(sdist)
        mean, cov = cast_cone(tdist, o, d, radii)
        z, zc = contract(mean, cov)
        feats = ipe_features(z, zc, basis)
        density, rgb = mlp(P, f"mlps.{lvl}.", feats, vd, 4 if is_prop else 8, is_prop)
        weights = alpha_weights(density, tdist, d)
        acc = weights.sum(-1)
        out = (weights[..., None] * rgb).sum(-2) + torch.clip(1 - acc[..., None], min=0) * 1.0
        renderings.append({"rgb": out})
        history.append({"density": density, "rgb": rgb, "sdist": sdist, "weights": weights})
    return renderings, history
