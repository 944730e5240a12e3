"""TEST INFRASTRUCTURE ONLY -- float64 model of what the NEO_PREC_TC field kernel (`neo360_b200/csrc/field_tc.cu`) computes.

`neo360_oracle.field` is the reference's formulation in fp32; the tensor-core kernel computes a re-associated formulation with
fp16 operands.  Comparing the two needs a bound loose enough for the fp16 rounding (~1e-2), and that bound hides layout bugs that move
the result by a few 1e-3.  This module restates the kernel's own formulation point by point in float64, with every fp16 rounding the
kernel applies made explicit, so that the kernel can be held to the size of its fp32 accumulation and geometry rounding instead:

* projected maps  P = fp16(fp16(F) . fp16(Wsel)^T) per map and view, Wsel = the latent columns of layers 0 and 3 ([P0 | P3]);
* lookups: bilinear blend of the fp16 texels with the kernel's `tap_quad` semantics (align_corners=True, zeros padding; a
  coordinate outside [-1, W) x [-1, H), NaN or huge, contributes nothing);
* positional encoding rounded to fp16; trunk weights fp16; b0 / b3 fp16 (they ride on the constant-one encoding column);
  b1, b2 and the head biases fp32 (they seed accumulators);
* layers 0..3 with ReLU and an fp16 round between layers; the blends are added into the layer-0 / layer-3 accumulators;
* folded head: fp16((Wv0[:, :128] Wb) / nv) and fp16(w_sigma / nv) summed over the views, the direction term
  fp16(mean_v dir_enc) . fp16(Wv0[:, 128:]), then bq = bv0 + Wv0[:, :128] bb, ReLU, fp16 -> Wv1 -> ReLU, fp16 -> Wrgb ->
  sigmoid * 1.002 - 0.001;  sigma = softplus(sigma_raw + b_sigma - 1);
* quirks Q1 (direction of ray (b*N+s) mod B of the ray's chunk) and Q2 (bg lookups at far(1-s) + 3s), as in the kernel.

`fp16=False` turns every rounding into the identity: the model is then an exact re-association of `neo360_oracle.field` /
`mlp_forward` (pinned to it on the CPU by tests/test_tc_model.py).  `mutation` applies one deliberate value-level bug (MUTATIONS), used
to show that the GPU bounds below would catch it.  Nothing under `neo360_b200/` imports this file.
"""
from __future__ import annotations

from typing import Dict, Optional

import torch
import torch.nn.functional as F

from . import neo360_oracle as orc

Tensor = torch.Tensor

# Bounds of the TC field kernel against this model (fp16=True), set from the errors measured over the cases of
# tests/test_gpu_tc_kernels.py on an H100 80GB HBM3 at a 700 W power limit (DESIGN.md section 2 lists them).  Per point:
# |rgb - model| <= RGB_TOL, |sigma - model| <= SIGMA_TOL * (1 + sigma); per case, the mean of those errors <= *_MEAN_TOL.
# The per-point maximum is not the size of one fp32 rounding: the kernel's fp32 geometry (fast-math for the background) moves the
# level-9 encodings sin(2^9 x) by up to ~1 fp16 ulp, and once one fp16 rounding of a point differs, the later roundings of that point
# decorrelate, so its result differs from the model by fp16 rounding noise.  The mean over many points stays small.
RGB_TOL = 1e-2
SIGMA_TOL = 4e-3
RGB_MEAN_TOL = 1e-3
SIGMA_MEAN_TOL = 4e-4

MUTATIONS = ("pmap_swap", "sigma_no_inv", "b0_off", "b3_off", "tap_edge", "no_q1", "no_w3enc", "dir_colmap")
FAR_UNC = 3.0


def _round(on: bool):
    return (lambda x: x.half().double()) if on else (lambda x: x)


def q1_source(n: int, N: int, chunk: int, device=None) -> Tensor:
    """(n, N) index of the ray whose view direction conditions point (ray, sample): ray (j mod B) of the ray's chunk, j = flat
    (ray, sample) index inside the chunk, B = the chunk's ray count (quirk Q1; chunk <= 0 = one chunk of n rays)."""
    ch = chunk if chunk > 0 else n
    rid = torch.arange(n, device=device)[:, None]
    c0 = (rid // ch) * ch
    bc = torch.clamp(n - c0, max=ch)
    j = (rid - c0) * N + torch.arange(N, device=device)[None, :]
    return c0 + j % bc


def latent_coords(p_cam: Tensor, sc: orc.Scene):
    """Grid coordinates of the pixel-aligned latent lookup, with the oracle's arithmetic (`neo360_oracle.local_lookup`: fp32
    camera constants and latent scaling, the rest in the dtype of p_cam)."""
    dev = p_cam.device
    uv = -p_cam[..., :2] / (p_cam[..., 2:] + 1e-9)
    uv = uv * torch.tensor([sc.focal, -sc.focal], device=dev) + torch.tensor([sc.cx, sc.cy], device=dev)
    Hl, Wl = sc.latent.shape[-2:]
    ls = torch.tensor([float(Wl), float(Hl)], device=dev)
    ls = ls / (ls - 1) * 2.0
    scale = ls / torch.tensor([float(sc.img_w), float(sc.img_h)], device=dev)
    uv = uv * scale - 1.0
    return uv[..., 0], uv[..., 1]


def blend(fmap: Tensor, gx: Tensor, gy: Tensor, edge_bug: bool = False) -> Tensor:
    """`tap_quad` + the per-thread blend of `blend_maps`: fmap (NV, C, H, W), gx / gy (NV, M) -> (NV, M, C).
    `edge_bug`: the right / bottom taps past the last texel read the last texel instead of contributing zero."""
    NV, C, H, W = fmap.shape
    ix = ((gx + 1) / 2) * (W - 1)
    iy = ((gy + 1) / 2) * (H - 1)
    inr = (ix >= -1) & (ix < W) & (iy >= -1) & (iy < H)          # False for NaN
    ix = torch.where(inr, ix, torch.full_like(ix, -1.0))
    iy = torch.where(inr, iy, torch.full_like(iy, -1.0))
    x0, y0 = torch.floor(ix), torch.floor(iy)
    fx, fy = ix - x0, iy - y0
    gx1, gy1 = (x0 + 1) - ix, (y0 + 1) - iy
    flat = fmap.reshape(NV, C, H * W).permute(0, 2, 1)
    out = torch.zeros(NV, gx.shape[1], C, dtype=fmap.dtype, device=fmap.device)
    for dx, dy, w in ((0, 0, gx1 * gy1), (1, 0, fx * gy1), (0, 1, gx1 * fy), (1, 1, fx * fy)):
        xx, yy = x0 + dx, y0 + dy
        vx = (xx >= 0) & ((xx <= W) if (edge_bug and dx) else (xx < W))
        vy = (yy >= 0) & ((yy <= H) if (edge_bug and dy) else (yy < H))
        ok = inr & vx & vy
        idx = (yy.clamp(0, H - 1) * W + xx.clamp(0, W - 1)).long()
        val = torch.gather(flat, 1, idx[..., None].expand(-1, -1, C))
        out = out + val * torch.where(ok, w, torch.zeros_like(w))[..., None]
    return out


def tc_field(rays: Dict[str, Tensor], far: Tensor, t_vals: Tensor, mlp_index: int, sc: orc.Scene, P: Dict[str, Tensor],
             chunk: int = 0, ray_order: Optional[Tensor] = None, fp16: bool = True, mutation: Optional[str] = None):
    """The TC field of one branch, point by point: same inputs as `NeRF_TP.field_eval` -> rgb (n, N, 3), sigma (n, N, 1), float64.

    Runs on the device of `t_vals`.  `ray_order` only schedules the kernel; it is checked to be a permutation and does not change the
    result (each point is computed on its own)."""
    if mutation is not None and mutation not in MUTATIONS:
        raise ValueError(f"unknown mutation {mutation!r}")
    h = _round(fp16)
    dev = t_vals.device
    f64 = lambda x: x.detach().to(device=dev, dtype=torch.float64)
    o, d, vd = (f64(rays[k]) for k in ("rays_o", "rays_d", "viewdirs"))
    t = f64(t_vals)
    far = f64(far).reshape(-1)
    n, N = t.shape
    if ray_order is not None and not torch.equal(torch.sort(ray_order.reshape(-1).long().cpu()).values, torch.arange(n)):
        raise ValueError("ray_order must be a permutation of the rays")
    pre = orc.MLP_NAMES[mlp_index]
    bg = bool(mlp_index & 1)
    Wt = lambda name: f64(P[pre + name + ".weight"])
    Bs = lambda name: f64(P[pre + name + ".bias"])
    poses = f64(sc.src_poses)
    nv = poses.shape[0]
    ich = 4 if bg else 3
    enc_dim = 21 * ich

    # geometry: encoded point xe and lookup point xl (fg: the sample point; bg: unit-sphere point / far(1-s) + 3s, quirk Q2)
    if bg:
        xe = orc.depth2pts_outside(o, d, t)[..., :3]
        tl = far[:, None] * (1.0 - t) + FAR_UNC * t
        xl = o[:, None, :] + tl[..., None] * d[:, None, :]
    else:
        xe = o[:, None, :] + t[..., None] * d[:, None, :]
        xl = xe
    M = n * N
    ce = orc.world2camera(xe.reshape(M, 3), poses)                                  # (NV, M, 3)
    cl = orc.world2camera(xl.reshape(M, 3), poses) if bg else ce
    x_in = torch.cat([ce, t.reshape(1, M, 1).expand(nv, M, 1)], -1) if bg else ce
    enc = h(orc.pos_enc(x_in, 0, 10))                                               # (NV, M, enc_dim)

    # projected maps [P0 | P3] of the latent and the three planes, and their blends at the lookup points
    W0, W3 = Wt("pts_linears.0"), Wt("pts_linears.3")
    maps = [(sc.latent, 0)] + [(m, 512) for m in (sc.planes_xz, sc.planes_xy, sc.planes_yz)]
    lgx, lgy = latent_coords(cl, sc)
    coords = [(lgx, lgy), (cl[..., 0], cl[..., 2]), (cl[..., 0], cl[..., 1]), (cl[..., 1], cl[..., 2])]
    acc = torch.zeros(nv, M, 256, dtype=torch.float64, device=dev)
    for (fm, off), (gx, gy) in zip(maps, coords):
        fm = f64(fm)
        C = fm.shape[1]
        col = enc_dim + off
        wsel = h(torch.cat([W0[:, col:col + C], W3[:, 128 + col:128 + col + C]], 0))   # (256, C): logical channel order
        if mutation == "pmap_swap":
            wsel = wsel[torch.tensor([1, 0] + list(range(2, 256)), device=dev)]
        pm = h(torch.einsum("vchw,pc->vphw", h(fm), wsel))
        acc = acc + blend(pm, gx, gy, edge_bug=(mutation == "tap_edge"))
    bl0, bl3 = acc[..., :128], acc[..., 128:]

    # trunk, per view
    relu_h = lambda x: h(torch.relu(x))
    b0 = torch.zeros(128, dtype=torch.float64, device=dev) if mutation == "b0_off" else h(Bs("pts_linears.0"))
    b3 = torch.zeros(128, dtype=torch.float64, device=dev) if mutation == "b3_off" else h(Bs("pts_linears.3"))
    x = relu_h(bl0 + enc @ h(W0[:, :enc_dim]).T + b0)
    x = relu_h(x @ h(Wt("pts_linears.1")).T + Bs("pts_linears.1"))
    x = relu_h(x @ h(Wt("pts_linears.2")).T + Bs("pts_linears.2"))
    a3 = bl3 + x @ h(W3[:, :128]).T + b3
    if mutation != "no_w3enc":
        a3 = a3 + enc @ h(W3[:, 128:128 + enc_dim]).T
    h3 = relu_h(a3)                                                                 # (NV, M, 128)

    # folded head, summed over the views
    Wv0 = Wt("views_linear.0")
    w_q = h((Wv0[:, :128] @ Wt("bottleneck_layer")) / nv)
    w_s = h(Wt("density_layer") if mutation == "sigma_no_inv" else Wt("density_layer") / nv)
    hq = (h3 @ w_q.T).sum(0)                                                        # (M, 64)
    hs = (h3 @ w_s.T).sum(0)                                                        # (M, 1)
    src = torch.arange(n, device=dev)[:, None].expand(n, N) if mutation == "no_q1" else q1_source(n, N, chunk, dev)
    dc = orc.world2camera_dirs(vd[src.reshape(-1)], poses)                          # (NV, M, 3)
    dmean = h(orc.pos_enc(dc, 0, 4).mean(0))                                        # (M, 27)
    if mutation == "dir_colmap":
        dmean = dmean[:, torch.tensor([0, 1, 2, 4, 3] + list(range(5, 27)), device=dev)]
    hq = hq + dmean @ h(Wv0[:, 128:]).T
    bq = Bs("views_linear.0") + Wv0[:, :128] @ Bs("bottleneck_layer")
    q = relu_h(hq + bq)
    v1 = relu_h(q @ h(Wt("views_linear.1")).T + Bs("views_linear.1"))
    raw = v1 @ h(Wt("rgb_layer")).T + Bs("rgb_layer")
    rgb = torch.sigmoid(raw) * 1.002 - 0.001
    sigma = F.softplus(hs + Bs("density_layer") - 1.0)
    return rgb.reshape(n, N, 3), sigma.reshape(n, N, 1)
