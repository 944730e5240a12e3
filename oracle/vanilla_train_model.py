"""TEST INFRASTRUCTURE ONLY -- float64 restatement of the vanilla-NeRF compositing backward, `composite_bwd_kernel` in mode 2
(csrc/sampling.cu, entry point `neo_vanilla_composite_bwd`), and of its forward, `composite_kernel` in mode 2.

Mode 2 is models/vanilla_nerf/helper.py:521-559: ascending t, delta_k = (t_{k+1} - t_k) |d| with the last interval 1e10 |d|,
T_k = prod_{j<k} (1 - alpha_j + 1e-10) (quirk Q9), white background adds 1 - acc, depth = clamp(nan_to_num(sum w t, inf), min, max)
over the chunk (quirk Q10).  The backward uses the same formulas as the NeO-360 model (oracle/train_stage_model.py):
    G_i = g_comp . c_i + g_w_i + g_acc - white sum(g_comp) + g_depth' t_i,   S_i = sum_{j>i} G_j w_j,
    dalpha_i = G_i T_i - S_i / a_i,   dsigma_i = dalpha_i delta_i e_i,   dc_i = w_i g_comp,
where g_depth' = g_depth where sum w t is finite and 0 elsewhere (the gradient of nan_to_num, and of clamp(x, min(x), max(x)), which
passes everywhere).  With `fp32=True` the values the kernel rounds before any decision are rounded the same way: delta = fp32
(fp32(t_{k+1} - t_k) * fp32 |d|) (the last one fp32(1e10f |d|)), sigma delta in fp32, alpha = fp32(1 - e), the 1e-10 as its fp32 value.
The magnitude of every output element and the alpha-rounding allowance are those of `train_stage_model.composite_bwd`.  With
`fp32=False` the backward equals torch.autograd through `vanilla_oracle.composite` in float64 (tests/test_vanilla_train_model.py).
Nothing under `neo360_b200/` imports this file.
"""
from __future__ import annotations

from typing import Dict

import torch

from .train_stage_model import EPS32, U, _rev_excl_cumsum

Tensor = torch.Tensor


def composite_terms(sigma: Tensor, t: Tensor, d: Tensor, fp32: bool = True) -> Dict[str, Tensor]:
    """Per sample of mode 2: delta, e = exp(-sigma delta), alpha, a = 1 - alpha + 1e-10, exclusive T, and the kernel's alpha allowance."""
    t64, s64 = t.double(), sigma.double()
    if fp32:    # __fsqrt_rn(dot3_(d, d)); mul_(sub_(t[k+1], t[k]), dn); mul_(1e10f, dn)
        d32 = d.float()
        dn = torch.sqrt((d32[:, 0] * d32[:, 0] + d32[:, 1] * d32[:, 1]) + d32[:, 2] * d32[:, 2]).double()[:, None]
        gap = torch.cat([(t.float()[:, 1:] - t.float()[:, :-1]).double(), torch.full_like(t64[:, :1], float(torch.tensor(1e10, dtype=torch.float32)))], 1)
        dist = (gap * dn).float().double()
        sd = (s64 * dist).float().double()
    else:
        gap = torch.cat([t64[:, 1:] - t64[:, :-1], torch.full_like(t64[:, :1], 1e10)], 1)
        dist = gap * torch.linalg.norm(d.double(), dim=-1, keepdim=True)
        sd = s64 * dist
    e = torch.exp(-sd)
    alpha = (1.0 - e).float().double() if fp32 else 1.0 - e
    a = 1.0 - alpha + (EPS32 if fp32 else 1e-10)
    incl = torch.cumprod(a, 1)
    T = torch.cat([torch.ones_like(incl[:, :1]), incl[:, :-1]], 1)
    dalpha = torch.zeros_like(alpha)
    if fp32:    # the same allowance as train_stage_model.composite_terms: the kernel's expf is within 2 ulp of e
        a32 = alpha.float()
        up = (torch.nextafter(a32, torch.full_like(a32, 2.0)) - a32).double()
        down = (a32 - torch.nextafter(a32, torch.zeros_like(a32))).double()
        margin = torch.minimum(up, down) / 2 - (1.0 - e - alpha).abs()
        flip = margin <= 4 * U * e
        dalpha = torch.where(alpha < 0.5, 4 * U * e + U * alpha, torch.where(flip, torch.maximum(up, down), torch.zeros_like(alpha)))
    return dict(dist=dist, e=e, alpha=alpha, a=a, T=T, dalpha=dalpha)


def composite_fwd(rgb: Tensor, sigma: Tensor, t: Tensor, d: Tensor, white: bool, fp32: bool = True) -> Dict[str, Tensor]:
    """comp (n,3), acc (n), w (n,N), depth (n) in float64 (depth before nan_to_num / clamp: finite inputs give a finite sum)."""
    k = composite_terms(sigma, t, d, fp32)
    w = k["alpha"] * k["T"]
    acc = w.sum(1)
    comp = (w[..., None] * rgb.double()).sum(1)
    if white:
        comp = comp + (1.0 - acc)[:, None]
    return dict(comp=comp, acc=acc, w=w, depth=(w * t.double()).sum(1))


def composite_bwd(rgb: Tensor, sigma: Tensor, t: Tensor, d: Tensor, white: bool, g_comp=None, g_acc=None, g_w=None, g_depth=None,
                  fp32: bool = True) -> Dict[str, Tensor]:
    """d_rgb (n,N,3), d_sigma (n,N), their magnitudes and the per-sample a, dist, e; None upstream gradients are zero.  Keys as
    `train_stage_model.composite_bwd` (g_lam_abs is zero: mode 2 has no bg_lambda)."""
    k = composite_terms(sigma, t, d, fp32)
    n, N = t.shape
    z = lambda *s: torch.zeros(*s, dtype=torch.float64, device=t.device)
    gc = g_comp.double() if g_comp is not None else z(n, 3)
    ga = g_acc.double().reshape(n) if g_acc is not None else z(n)
    gw = g_w.double() if g_w is not None else z(n, N)
    gd = g_depth.double().reshape(n) if g_depth is not None else z(n)
    c, t64 = rgb.double(), t.double()
    w = k["alpha"] * k["T"]
    gd = torch.where(torch.isfinite((w * t64).sum(1)), gd, torch.zeros_like(gd))
    wh = 1.0 if white else 0.0
    G = (c * gc[:, None, :]).sum(-1) + gw + (ga - wh * gc.sum(-1))[:, None] + gd[:, None] * t64
    Gm = (c * gc[:, None, :]).abs().sum(-1) + gw.abs() + (ga.abs() + wh * gc.abs().sum(-1))[:, None] + (gd[:, None] * t64).abs()
    r = k["dalpha"] / (U * k["a"])
    Tm = k["T"] * (1.0 + torch.cumsum(r, 1) - r)
    wm = (k["alpha"] + k["dalpha"] / U) * Tm
    S = _rev_excl_cumsum(G * w)
    Sm = _rev_excl_cumsum(Gm * wm)
    dalpha = G * k["T"] - S / k["a"]
    dalpha_m = Gm * Tm + Sm / k["a"]
    de = k["dist"] * k["e"]
    return dict(d_sigma=dalpha * de, d_sigma_mag=dalpha_m * de, d_rgb=w[..., None] * gc[:, None, :],
                d_rgb_mag=wm[..., None] * gc.abs()[:, None, :], G_mag=Gm, g_lam_abs=z(n), a=k["a"], dist=k["dist"], e=k["e"])
