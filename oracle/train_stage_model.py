"""TEST INFRASTRUCTURE ONLY -- float64 restatements of the hand-written CUDA of the NeO-360 training step.

* composite_fwd / composite_bwd: `composite_kernel` and `composite_bwd_kernel` (csrc/sampling.cu), in_sphere 1 (fg: last interval
  far - t_N, distances times |d|) and 0 (bg: descending s, last interval 1e10), written out with the kernels' own formulas:
      T_i = prod_{j<i} a_j,  a_j = 1 - alpha_j + 1e-10,  w_i = alpha_i T_i,
      G_i = g_comp . c_i + g_w_i + g_acc - white sum(g_comp) + g_depth t_i,
      S_i = sum_{j>i} G_j w_j + g_lam T_N,   dalpha_i = G_i T_i - S_i / a_i,   dsigma_i = dalpha_i delta_i e_i,   dc_i = w_i g_comp.
  `composite_bwd` also returns a MAGNITUDE per output element: the same expression with every term in absolute value
  (|G_i| T_i + (sum_{j>i} |G_j| w_j + |g_lam| T_N) / a_i, ...), the unit the GPU bounds are stated in, so that cancellation in dalpha
  is allowed for and nothing more.  alpha = 1 - e is formed after the kernel's expf has rounded e, so alpha is known only to an absolute
  ~2^-23 e below 0.5, and from 0.5 up the kernel may round 1 - e to the neighbouring fp32 value when 1 - e lies that close to a rounding
  boundary (then a = 1 - alpha, and every T behind it, moves by 2^-24 / a relative).  The magnitudes count both (composite_terms).
  With `fp32=True` (default) the values the kernels round before any decision are rounded the same way: delta and sigma * delta in fp32
  (so e = exp(-sigma delta) is evaluated at the kernel's own argument), alpha = float32(1 - e) and the 1e-10 as its fp32 value.  After a
  sample with e < 2^-25 the kernel has a = 1e-10 where exact arithmetic gives e + 1e-10, so downstream weights are defined only to an
  absolute ~6e-8 T; taking alpha from the fp32 rounding puts the model on the kernel's side of that.  Forward outputs are held in
  absolute units (they are <= 1, depth <= far); backward outputs in the magnitude unit.  With `fp32=False` everything is float64 of
  the inputs, and the backward equals torch.autograd through `neo360_oracle.composite` (tests/test_train_stage_model.py).
* lookup_taps / lookup_fwd / lookup_bwd: the tri-plane lookup (`index_grid`) and the pixel-aligned lookup (`get_local_feats`) of
  `index_kernel` / `index_bwd_kernel` (csrc/field_fp32.cu): the four bilinear taps (grid_sample, align_corners, zero padding) of every
  row (view, point) in float64 from the same fp32 points and cameras.  The forward is a gather, the backward an `index_add_` into
  channel-last gradient maps.  The backward also returns, per map element, sum |w g| and the count n_t of non-zero contributions; the
  taps carry a first-order float64 estimate of each row's fp32 tap-coordinate error |dix| + |diy|.  Bilinear weights with zero padding
  are continuous in the coordinate, so a coordinate error moves every weight by at most that much.
Everything follows the dtype and device of its inputs.  Nothing under `neo360_b200/` imports this file.
"""
from __future__ import annotations

from typing import Dict, Optional

import torch

from . import neo360_oracle as orc

Tensor = torch.Tensor
U = 2.0 ** -24                      # fp32 unit roundoff
EPS32 = float(torch.tensor(1e-10, dtype=torch.float32))


# ---------------------------------------------------------------- compositing

def _f32(x: Tensor, on: bool) -> Tensor:
    return x.float().double() if on else x


def composite_terms(sigma: Tensor, t: Tensor, d: Optional[Tensor], far: Optional[Tensor], in_sphere: bool, fp32: bool = True):
    """Per sample: distances delta, e = exp(-sigma delta), alpha, a = 1 - alpha + 1e-10, exclusive T, T_N (float64)."""
    t64, s64 = t.double(), sigma.double()
    if in_sphere:
        nxt = torch.cat([t64[:, 1:], far.double().reshape(-1, 1)], 1)
        d64 = d.double()
        if fp32:    # __fsqrt_rn(dot3_(d, d)) and the fp32 product (nxt - t) * |d|
            d32 = d.float()
            dn = torch.sqrt((d32[:, 0] * d32[:, 0] + d32[:, 1] * d32[:, 1]) + d32[:, 2] * d32[:, 2]).double()
            dist = ((nxt.float() - t.float()).double() * dn[:, None]).float().double()
        else:
            dist = (nxt - t64) * torch.linalg.norm(d64, dim=-1, keepdim=True)
    else:
        last = torch.full_like(t64[:, :1], 1e10)
        dist = torch.cat([_f32(t64[:, :-1] - t64[:, 1:], fp32), last.float().double() if fp32 else last], 1)
    sd = _f32(s64 * dist, fp32)
    e = torch.exp(-sd)
    alpha = _f32(1.0 - e, fp32)
    a = 1.0 - alpha + (EPS32 if fp32 else 1e-10)
    incl = torch.cumprod(a, 1)
    T = torch.cat([torch.ones_like(incl[:, :1]), incl[:, :-1]], 1)
    # how far the kernel's alpha can be from this one: its expf is within 2 ulp of e.  Below 0.5, 1 - e is exact in fp32, so alpha moves
    # with e (4U e, plus the model's own rounding U alpha).  From 0.5 up the fp32 rounding of 1 - e absorbs that, unless 1 - e lies within
    # 4U e of a rounding boundary: then the kernel may hold the neighbouring fp32 value.
    dalpha = torch.zeros_like(alpha)
    if fp32:
        a32 = alpha.float()
        up = (torch.nextafter(a32, torch.full_like(a32, 2.0)) - a32).double()
        down = (a32 - torch.nextafter(a32, torch.zeros_like(a32))).double()
        margin = torch.minimum(up, down) / 2 - (1.0 - e - alpha).abs()
        flip = margin <= 4 * U * e
        dalpha = torch.where(alpha < 0.5, 4 * U * e + U * alpha, torch.where(flip, torch.maximum(up, down), torch.zeros_like(alpha)))
    return dict(dist=dist, e=e, alpha=alpha, a=a, T=T, TN=incl[:, -1], dalpha=dalpha)


def composite_fwd(rgb: Tensor, sigma: Tensor, t: Tensor, d, far, white: bool, in_sphere: bool, fp32: bool = True) -> Dict[str, Tensor]:
    """comp (n,3), acc (n), w (n,N), lam (n, fg only), depth (n) in float64."""
    k = composite_terms(sigma, t, d, far, in_sphere, fp32)
    w = k["alpha"] * k["T"]
    acc = w.sum(1)
    comp = (w[..., None] * rgb.double()).sum(1)
    if white:
        comp = comp + (1.0 - acc)[:, None]
    return dict(comp=comp, acc=acc, w=w, lam=k["TN"] if in_sphere else None, depth=(w * t.double()).sum(1))


def _rev_excl_cumsum(x: Tensor) -> Tensor:
    """sum_{j>i} x_j, summed from the far end (no cancellation against the terms before i)."""
    inc = torch.flip(torch.cumsum(torch.flip(x, [1]), 1), [1])
    return torch.cat([inc[:, 1:], torch.zeros_like(inc[:, :1])], 1)


def composite_bwd(rgb: Tensor, sigma: Tensor, t: Tensor, d, far, white: bool, in_sphere: bool, g_comp=None, g_acc=None, g_w=None,
                  g_lam=None, g_depth=None, fp32: bool = True) -> Dict[str, Tensor]:
    """d_rgb (n,N,3), d_sigma (n,N) and their magnitudes; None upstream gradients are zero.  Also the per-sample a, dist, e (for the
    denormal floor of the GPU bound)."""
    k = composite_terms(sigma, t, d, far, in_sphere, fp32)
    n, N = t.shape
    z = lambda *s: torch.zeros(*s, dtype=torch.float64, device=t.device)
    gc = g_comp.double() if g_comp is not None else z(n, 3)
    ga = g_acc.double().reshape(n) if g_acc is not None else z(n)
    gw = g_w.double() if g_w is not None else z(n, N)
    gl = g_lam.double().reshape(n) if g_lam is not None else z(n)
    gd = g_depth.double().reshape(n) if g_depth is not None else z(n)
    c, t64 = rgb.double(), t.double()
    w = k["alpha"] * k["T"]
    wh = 1.0 if white else 0.0
    G = (c * gc[:, None, :]).sum(-1) + gw + (ga - wh * gc.sum(-1))[:, None] + gd[:, None] * t64
    Gm = (c * gc[:, None, :]).abs().sum(-1) + gw.abs() + (ga.abs() + wh * gc.abs().sum(-1))[:, None] + (gd[:, None] * t64).abs()
    # the kernel's alpha_j may differ by dalpha_j (composite_terms): in units of 2^-24, alpha counts as alpha + dalpha / U and T_k as
    # T_k (1 + sum_{j<k} dalpha_j / (U a_j))
    r = k["dalpha"] / (U * k["a"])
    Tm = k["T"] * (1.0 + torch.cumsum(r, 1) - r)
    TNm = k["TN"] * (1.0 + r.sum(1))
    wm = (k["alpha"] + k["dalpha"] / U) * Tm
    S = _rev_excl_cumsum(G * w) + (gl * k["TN"])[:, None]
    Sm = _rev_excl_cumsum(Gm * wm) + (gl.abs() * TNm)[:, None]
    dalpha = G * k["T"] - S / k["a"]
    dalpha_m = Gm * Tm + Sm / k["a"]
    de = k["dist"] * k["e"]
    return dict(d_sigma=dalpha * de, d_sigma_mag=dalpha_m * de, d_rgb=w[..., None] * gc[:, None, :],
                d_rgb_mag=wm[..., None] * gc.abs()[:, None, :], G_mag=Gm, g_lam_abs=gl.abs(), a=k["a"], dist=k["dist"], e=k["e"])


# ---------------------------------------------------------------- lookups

def _taps(gx: Tensor, gy: Tensor, dgx: Tensor, dgy: Tensor, W: int, H: int):
    """bilinear_taps (csrc/common.cuh) in float64: flat indices (R,4) of nw, ne, sw, se (clamped), weights (R,4) (0 out of range),
    the coordinate error |dix| + |diy| (R,) from the grid-coordinate errors dgx, dgy, and x0, y0, ix, iy."""
    ix = (gx + 1) / 2 * (W - 1)
    iy = (gy + 1) / 2 * (H - 1)
    dix = dgx * (W - 1) / 2 + 2 * U * (ix.abs() + (W - 1) / 2)        # the fp32 (gx + 1), * (W - 1)
    diy = dgy * (H - 1) / 2 + 2 * U * (iy.abs() + (H - 1) / 2)
    finite = torch.isfinite(ix) & torch.isfinite(iy) & (ix.abs() < 1e9) & (iy.abs() < 1e9)
    x0 = torch.where(finite, torch.floor(ix), torch.full_like(ix, -2.0))
    y0 = torch.where(finite, torch.floor(iy), torch.full_like(iy, -2.0))
    fx, fy = torch.where(finite, ix - x0, 0.0), torch.where(finite, iy - y0, 0.0)
    idx, wts = [], []
    for xx, yy, ww in ((x0, y0, (1 - fx) * (1 - fy)), (x0 + 1, y0, fx * (1 - fy)), (x0, y0 + 1, (1 - fx) * fy), (x0 + 1, y0 + 1, fx * fy)):
        ok = (xx >= 0) & (xx <= W - 1) & (yy >= 0) & (yy <= H - 1)
        idx.append((yy.clamp(0, H - 1) * W + xx.clamp(0, W - 1)).long())
        wts.append(ww * ok)
    return dict(idx=torch.stack(idx, -1), w=torch.stack(wts, -1), derr=torch.where(finite, dix + diy, torch.zeros_like(dix)),
                x0=x0, y0=y0, ix=ix, iy=iy, finite=finite, W=W, H=H)


def _camera(pts: Tensor, poses: Tensor):
    """Camera-frame points (NV*M, 3) in float64 (rows ordered (view, point)) and a first-order bound of the fp32 error of
    `to_camera` / `view_xform_kernel` (three fma roundings plus the rounding of -(R^T t))."""
    p64, c2w = pts.double().reshape(-1, 3), poses.double()
    cam = orc.world2camera(p64, c2w)
    rt = c2w[:, :3, :3].transpose(1, 2)
    tr_abs = (rt.abs() @ c2w[:, :3, 3:].abs())[..., 0]                       # (NV,3)
    mag = torch.matmul(rt.abs()[:, None], p64.abs()[None, :, :, None])[..., 0]  # (NV,M,3)
    err = U * (3 * mag + 4 * tr_abs[:, None, :] + cam.abs())
    return cam.reshape(-1, 3), err.reshape(-1, 3)


def lookup_taps(pts: Tensor, poses: Tensor, plane_hw, lat_hw, focal: float, cx: float, cy: float, img_wh, local: bool):
    """Taps of every row (view, point) of points pts (M,3): local=True -> one tap set of the latent grid, plus z_cam per row;
    local=False -> three tap sets (xz, xy, yz) of the planes."""
    c, dc = _camera(pts, poses)
    if not local:
        Hp, Wp = plane_hw
        pairs = ((0, 2), (0, 1), (1, 2))
        return [_taps(c[:, i], c[:, j], dc[:, i], dc[:, j], Wp, Hp) for i, j in pairs]
    Hl, Wl = lat_hw
    img_w, img_h = img_wh
    z = c[:, 2] + 1e-9
    dz = dc[:, 2] + U * z.abs()
    qx, qy = -c[:, 0] / z, -c[:, 1] / z
    dqx = (dc[:, 0] + qx.abs() * dz) / z.abs() + U * qx.abs()
    dqy = (dc[:, 1] + qy.abs() * dz) / z.abs() + U * qy.abs()
    f32 = lambda x: float(torch.tensor(x, dtype=torch.float32))
    focal, cx, cy = f32(focal), f32(cx), f32(cy)
    u, v = qx * focal + cx, qy * (-focal) + cy
    du = abs(focal) * dqx + U * (2 * (qx * focal).abs() + u.abs())
    dv = abs(focal) * dqy + U * (2 * (qy * focal).abs() + v.abs())
    # latent scaling in fp32, as the scene builder and `neo360_oracle.local_lookup` compute it
    ls = torch.tensor([float(Wl), float(Hl)], dtype=torch.float32)
    sx, sy = (ls / (ls - 1) * 2.0 / torch.tensor([float(img_w), float(img_h)], dtype=torch.float32)).tolist()
    gx, gy = u * sx - 1.0, v * sy - 1.0
    dgx = sx * du + U * (2 * (u * sx).abs() + gx.abs())
    dgy = sy * dv + U * (2 * (v * sy).abs() + gy.abs())
    tp = _taps(gx, gy, dgx, dgy, Wl, Hl)
    tp["z"] = c[:, 2]
    return [tp]


def lookup_fwd(taps, maps, nv: int, chunk_elems: int = 1 << 26):
    """Gather: maps = one channel-last (NV,H,W,C) tensor per tap set; rows (NV*M, C) = sum over the tap sets of sum_tap w F[v, idx].
    Also sum |w F| and the coordinate-error term sum over the tap sets of 4 (|dix| + |diy|) max_texels |F[v, :, :, c]|."""
    R, C = taps[0]["idx"].shape[0], maps[0].shape[-1]
    M = R // nv
    dev = maps[0].device
    view = torch.arange(nv, device=dev).repeat_interleave(M)
    val = torch.zeros(R, C, dtype=torch.float64, device=dev)
    mag, derr = torch.zeros_like(val), torch.zeros_like(val)
    cs = max(1, min(C, chunk_elems // max(4 * R, 1)))
    for tp, F in zip(taps, maps):
        gi = view[:, None] * (tp["H"] * tp["W"]) + tp["idx"]
        flat = F.reshape(nv * tp["H"] * tp["W"], C)
        fmax = F.double().abs().reshape(nv, -1, C).amax(1)                   # (NV, C)
        derr += 4 * tp["derr"][:, None] * fmax[view]
        for c0 in range(0, C, cs):
            term = flat[:, c0:c0 + cs].double()[gi] * tp["w"][..., None]
            val[:, c0:c0 + cs] += term.sum(1)
            mag[:, c0:c0 + cs] += term.abs().sum(1)
    return dict(val=val, mag=mag, derr=derr)


def lookup_bwd(tp, g: Tensor, nv: int, chunk_elems: int = 1 << 26):
    """index_add_ of one tap set: rows g (NV*M, C) -> channel-last (NV,H,W,C) float64: the scatter sum_rows w g, sum |w g|,
    the count n_t of non-zero contributions per texel, and sum |g| (|dix| + |diy|) over the rows whose taps reach the texel
    (the coordinate-error term; rows within their coordinate error of a texel edge spread it over the 4 x 4 texels around them)."""
    R, C = g.shape
    M = R // nv
    H, W = tp["H"], tp["W"]
    dev = g.device
    view = torch.arange(nv, device=dev).repeat_interleave(M)
    gi = (view[:, None] * (H * W) + tp["idx"]).reshape(-1)
    wf = tp["w"].reshape(-1)
    nz = wf != 0
    cnt = torch.zeros(nv * H * W, dtype=torch.float64, device=dev).index_add_(0, gi[nz], torch.ones_like(wf[nz]))
    # rows near a texel edge: their fp32 taps may be the neighbouring texels
    fx, fy = tp["ix"] - tp["x0"], tp["iy"] - tp["y0"]
    d = tp["derr"]
    edge = ((fx < d) | (fx > 1 - d) | (fy < d) | (fy > 1 - d)) & tp["finite"]
    er = torch.nonzero(edge)[:, 0]
    nb_idx, nb_ok = [], []
    for oy in (-1, 0, 1, 2):
        for ox in (-1, 0, 1, 2):
            xx, yy = tp["x0"][er] + ox, tp["y0"][er] + oy
            nb_ok.append((xx >= 0) & (xx <= W - 1) & (yy >= 0) & (yy <= H - 1))
            nb_idx.append(view[er] * (H * W) + (yy.clamp(0, H - 1) * W + xx.clamp(0, W - 1)).long())
    nb_idx, nb_ok = torch.stack(nb_idx, 1), torch.stack(nb_ok, 1)
    inner = ~edge[:, None] & (tp["w"] != 0)
    val = torch.zeros(nv * H * W, C, dtype=torch.float64, device=dev)
    mag, derr = torch.zeros_like(val), torch.zeros_like(val)
    cs = max(1, min(C, chunk_elems // max(4 * R, 1)))
    ii = torch.nonzero(inner.reshape(-1))[:, 0]
    for c0 in range(0, C, cs):
        gc = g[:, c0:c0 + cs].double()
        src = (tp["w"][..., None] * gc[:, None, :]).reshape(-1, gc.shape[1])
        val[:, c0:c0 + cs].index_add_(0, gi, src)
        mag[:, c0:c0 + cs].index_add_(0, gi, src.abs())
        del src
        gd = gc.abs() * d[:, None]
        derr[:, c0:c0 + cs].index_add_(0, gi[ii], gd.repeat_interleave(4, 0)[ii])
        if er.numel():
            ok = nb_ok.reshape(-1)
            derr[:, c0:c0 + cs].index_add_(0, nb_idx.reshape(-1)[ok], gd[er].repeat_interleave(16, 0)[ok])
    shp = (nv, H, W, C)
    return dict(val=val.reshape(shp), mag=mag.reshape(shp), derr=derr.reshape(shp), n=cnt.reshape(nv, H, W),
                reach=(cnt.reshape(nv, H, W) > 0) | (derr.reshape(shp).amax(-1) > 0))
