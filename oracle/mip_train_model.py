"""TEST INFRASTRUCTURE ONLY -- float64 restatement of the Mip-NeRF 360 compositing backward, `composite_bwd_kernel` (csrc/mip.cu, entry
point `neo_mip_composite_bwd`), and of its forward, `composite_kernel` (entry point `neo_mip_composite`).

The stage is the head activations + compute_alpha_weights(opaque_background) + volumetric_rendering with a white background
(models/mipnerf360/helper.py:234-274, model.py:142-173) of raw density r (n,N) and raw rgb q (n,N,3) at tdist (n,N+1):
    x_k = softplus(r_k - 1) delta_k,  delta_k = (t_{k+1} - t_k) |d|,  x_{N-1} = inf,  T_k = exp(-sum_{j<k} x_j),  w_k = (1 - e^{-x_k}) T_k,
    c_k = sigmoid(q_k) 1.002 - 0.001,  rgb = sum_k w_k c_k + clip(1 - acc, min=0),  acc = sum_k w_k.
Backward, with m = [1 - acc >= 0] (the gradient of the clip):
    G_k = g_w_k + g_rgb . c_k - m sum(g_rgb),   dL/dx_k = G_k e^{-x_k} T_k - sum_{j>k} G_j w_j  (0 for k = N-1),
    d_r_k = (delta_k dL/dx_k + g_density_k) softplus'(r_k - 1),   d_q_k = (w_k g_rgb + g_rgb_s_k) 1.002 s_k (1 - s_k).
With `fp32=True` the values the kernel rounds are rounded the same way: delta = fp32(fp32(t_{k+1} - t_k) * fp32 |d|), x = fp32(density
delta) with the density rounded to fp32, the exclusive scan of x in fp32 in the kernel's order (a Hillis-Steele warp scan per chunk of
32, then the carry), and s (1 - s) in the kernel's form q / (1 + q)^2, q = exp(-|raw rgb|), which keeps its value where the sigmoid
saturates (float64 1 - s cancels to 0 beyond |raw rgb| ~ 37).  With `fp32=False` everything is float64 of the inputs (x as the
reference's (density * (t_{k+1} - t_k)) * |d|, s (1 - s) as autograd's sigmoid backward), and the backward equals torch.autograd
through `mip_oracle`'s activations + `alpha_weights` + rendering (tests/test_mip_train_model.py).

Every output element also gets a MAGNITUDE, the unit the GPU bounds are stated in (2^-24 N magnitude): the same expression with every term
in absolute value, T counted as T (1 + sum_{j<k} x_j) and e^{-x} as e^{-x} (1 + x) (the relative error of an exponential grows with its
argument), alpha T as alpha T (1 + excl) + e (1 + x) T (the absolute rounding of 1 - e), and the m sum(g_rgb) term always counted.  Under
the opaque background sum w = 1, so that term cancels in dL/dx in exact arithmetic and the kernel's m (decided on its own fp32 acc) may differ
from this model's without leaving the unit.  Nothing under `neo360_b200/` imports this file.
"""
from __future__ import annotations

from typing import Dict, Optional

import torch
import torch.nn.functional as F

from .train_stage_model import _rev_excl_cumsum

Tensor = torch.Tensor


def _warp_excl_scan_fp32(x: Tensor) -> Tensor:
    """Exclusive prefix sum of x (n,N) float32 in composite_kernel's order: per chunk of 32 lanes a Hillis-Steele scan (lane l adds lane
    l - o for o = 1, 2, 4, 8, 16), then the chunk's inclusive values plus the carry; the carry is lane 31's."""
    n, N = x.shape
    out = torch.empty_like(x)
    carry = torch.zeros(n, dtype=torch.float32, device=x.device)
    for base in range(0, N, 32):
        w = min(32, N - base)
        v = torch.zeros(n, 32, dtype=torch.float32, device=x.device)
        v[:, :w] = x[:, base:base + w]
        for o in (1, 2, 4, 8, 16):
            v = torch.cat([v[:, :o], v[:, o:] + v[:, :-o]], 1)
        incl = v + carry[:, None]
        out[:, base:base + w] = torch.cat([carry[:, None], incl[:, :-1]], 1)[:, :w]
        carry = incl[:, 31]
    return out


def composite_terms(raw_density: Tensor, tdist: Tensor, d: Tensor, fp32: bool = True) -> Dict[str, Tensor]:
    """Per sample (float64): z = r - 1, density, delta, x (inf for the last sample), exclusive scan, e = exp(-x), T, alpha, w."""
    n, N = raw_density.shape
    if fp32:
        z = (raw_density.float() - 1.0).double()
        dens = F.softplus(z).float().double()
        d32, t32 = d.float(), tdist.float()
        dn = torch.sqrt((d32[:, 0] * d32[:, 0] + d32[:, 1] * d32[:, 1]) + d32[:, 2] * d32[:, 2])
        delta = ((t32[:, 1:] - t32[:, :-1]) * dn[:, None]).double()
        x = (dens * delta).float()
        excl = _warp_excl_scan_fp32(torch.cat([x[:, :-1], torch.zeros_like(x[:, :1])], 1)).double()
        x = x.double()
    else:
        z = raw_density.double() - 1.0
        dens = F.softplus(z)
        t64 = tdist.double()
        dn = torch.linalg.norm(d.double(), dim=-1)
        delta = (t64[:, 1:] - t64[:, :-1]) * dn[:, None]
        x = (dens * (t64[:, 1:] - t64[:, :-1])) * dn[:, None]
        excl = torch.cat([torch.zeros_like(x[:, :1]), torch.cumsum(x[:, :-1], 1)], 1)
    x = torch.cat([x[:, :-1], torch.full_like(x[:, :1], float("inf"))], 1)
    e = torch.exp(-x)
    T = torch.exp(-excl)
    alpha = 1.0 - e
    return dict(z=z, dens=dens, delta=delta, x=x, excl=excl, e=e, T=T, alpha=alpha, w=alpha * T)


def _rgb(raw_rgb: Optional[Tensor], like: Tensor) -> Tensor:
    if raw_rgb is None:
        return torch.zeros(*like.shape, 3, dtype=torch.float64, device=like.device)
    return torch.sigmoid(raw_rgb.double()) * (1 + 2 * 0.001) - 0.001


def composite_fwd(raw_density: Tensor, raw_rgb: Optional[Tensor], tdist: Tensor, d: Tensor, fp32: bool = True) -> Dict[str, Tensor]:
    """rgb (n,3), weights (n,N), density (n,N), rgb_s (n,N,3) (zeros for a proposal level) and acc (n), float64."""
    k = composite_terms(raw_density, tdist, d, fp32)
    c = _rgb(raw_rgb, k["w"])
    acc = k["w"].sum(1)
    rgb = (k["w"][..., None] * c).sum(1) + torch.clip(1.0 - acc, min=0)[:, None]
    return dict(rgb=rgb, w=k["w"], density=k["dens"], rgb_s=c, acc=acc)


def composite_bwd(raw_density: Tensor, raw_rgb: Optional[Tensor], tdist: Tensor, d: Tensor, g_rgb=None, g_w=None, g_density=None, g_rgb_s=None,
                  fp32: bool = True, m: Optional[Tensor] = None) -> Dict[str, Tensor]:
    """d_raw_density (n,N), d_raw_rgb (n,N,3) (None for a proposal level) and their magnitudes; None upstream gradients are zero.  `m`
    (n) overrides the clip's gradient mask, which is otherwise [1 - acc >= 0] of this model's acc."""
    k = composite_terms(raw_density, tdist, d, fp32)
    n, N = raw_density.shape
    z = lambda *s: torch.zeros(*s, dtype=torch.float64, device=raw_density.device)
    gc = g_rgb.double() if g_rgb is not None else z(n, 3)
    gw = g_w.double() if g_w is not None else z(n, N)
    gdn = g_density.double() if g_density is not None else z(n, N)
    grs = g_rgb_s.double() if (g_rgb_s is not None and raw_rgb is not None) else z(n, N, 3)
    w, e, T = k["w"], k["e"], k["T"]
    if m is None:
        m = (1.0 - w.sum(1) >= 0).double()
    c = _rgb(raw_rgb, w)
    G = gw + (c * gc[:, None, :]).sum(-1) - (m * gc.sum(-1))[:, None]
    Gm = gw.abs() + (c.abs() * gc.abs()[:, None, :]).sum(-1) + gc.abs().sum(-1)[:, None]
    last = torch.zeros_like(w, dtype=torch.bool)
    last[:, -1] = True
    dx = torch.where(last, 0.0, G * e * T - _rev_excl_cumsum(G * w))
    em = torch.where(e > 0, e * (1.0 + torch.where(last, 0.0, k["x"])), 0.0)
    Tm = T * (1.0 + k["excl"])
    wm = k["alpha"] * Tm + em * T
    dxm = torch.where(last, 0.0, Gm * (em * T + e * Tm) + _rev_excl_cumsum(Gm * wm))
    sp = torch.where(k["z"] > 20, torch.ones_like(k["z"]), torch.sigmoid(k["z"]))
    out = dict(d_raw_density=(k["delta"] * dx + gdn) * sp, d_raw_density_mag=(k["delta"] * dxm + gdn.abs()) * sp, d_raw_rgb=None,
               d_raw_rgb_mag=None, m=m, w=w)
    if raw_rgb is not None:
        if fp32:    # the kernel's s (1 - s) = q / (1 + q)^2, q = exp(-|x|): no cancellation where the sigmoid saturates
            qe = torch.exp(-raw_rgb.double().abs())
            ds = 1.002 * qe / (1 + qe) ** 2
        else:       # autograd's sigmoid backward
            s = torch.sigmoid(raw_rgb.double())
            ds = 1.002 * s * (1 - s)
        out["d_raw_rgb"] = (w[..., None] * gc[:, None, :] + grs) * ds
        out["d_raw_rgb_mag"] = (wm[..., None] * gc.abs()[:, None, :] + grs.abs()) * ds
    return out
