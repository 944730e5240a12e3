"""TEST INFRASTRUCTURE ONLY -- float64 models of the ray and pose backward kernels of vanilla NeRF's pose refinement.

* `vanilla_encode_bwd`: neo_vanilla_encode_bwd (csrc/vanilla.cu).  The encoding of a point x is [x, sin(2^k x), sin(2^k x + pi/2)]
  (models/vanilla_nerf/helper.py:445-449), so dL/dx_j = g_j + sum_k 2^k (g_sin cos(2^k x_j) - g_cos sin(2^k x_j)); the points are
  x = o + t viewdirs (cast_rays along viewdirs, quirk Q15), so g_o = sum_samples dL/dx and g_viewdirs = sum_samples t dL/dx + the same
  form for the direction encoding (4 octaves).  Also returns, per ray, the sum of |terms| that bounds the fp32 kernel's error.
* `sample_rays_bwd`: neo_sample_rays_bwd (csrc/sampling.cu).  d = R c for the camera-frame direction c, viewdirs = rays_d = d / |d|
  (quirk Q3), rays_o = t: g_d = (g_v - v (v . g_v)) / |d|, g_R += g_d c^T, g_t += g_rays_o, summed per view.
* `rays_from_pose`: datasets/ray_utils.py get_rays(..., output_view_dirs=True) restated out of place.  The reference normalises rays_d in
  place through its viewdirs alias, which autograd refuses ("modified by an inplace operation"), so the pose gradients of the golden
  vectors are taken through this restatement of the same arithmetic.
* `mip_dir_enc_bwd`: neo_mip_encode_bwd (csrc/mip.cu), the direction encoding's derivative; Mip-NeRF 360's IPE features give the rays
  no gradient, as the reference's detached `contract`.
* `mlp_input_grad`: the input-row gradient of the tensor-core dense chain (training._MLPTrainTC) at the bf16 rounding points of
  oracle/dense_train_model.py.
Pinned to torch.autograd through the reference's own helpers (and, for mlp_input_grad with rounding off, through autograd of
dense_train_model.forward) by tests/test_camera_grad_model.py."""
from __future__ import annotations

import torch

Tensor = torch.Tensor


def _enc_grad(x: Tensor, g: Tensor, deg: int):
    """dL/dx (..., 3) of the positional encoding of x (..., 3) with upstream g (..., 3 + 6 deg), and the sum of |terms|."""
    s, a = g[..., :3].clone(), g[..., :3].abs()
    for k in range(deg):
        sc = 2.0 ** k
        gs, gc = g[..., 3 + 3 * k:6 + 3 * k], g[..., 3 + 3 * deg + 3 * k:6 + 3 * deg + 3 * k]
        cs, sn = torch.cos(sc * x), torch.sin(sc * x)
        s = s + sc * (gs * cs - gc * sn)
        a = a + sc * ((gs * cs).abs() + (gc * sn).abs())
    return s, a


def vanilla_encode_bwd(o: Tensor, vd: Tensor, t: Tensor, g_enc: Tensor, g_denc: Tensor, x: Tensor = None):
    """o, vd (n,3), t (n,N), g_enc (n*N, 63), g_denc (n, 27), float64 -> g_o, g_vd (n,3) and the per-ray sums of |terms| mag_o, mag_vd
    (n,3).  x (n,N,3): the points at which the encoding was taken (default o + t vd; a test of the fp32 kernel passes its fp32 points)."""
    n, N = t.shape
    if x is None:
        x = o[:, None, :] + t[..., None] * vd[:, None, :]
    gx, ax = _enc_grad(x, g_enc.reshape(n, N, 63), 10)
    gd, ad = _enc_grad(vd, g_denc, 4)
    g_o, g_vd = gx.sum(1), (t[..., None] * gx).sum(1) + gd
    return g_o, g_vd, ax.sum(1), (t.abs()[..., None] * ax).sum(1) + ad


def camera_dirs(H: int, W: int, focal: float, dtype=torch.float64) -> Tensor:
    """get_ray_directions (ray_utils.py:84-104): (H*W, 3) = ((i - W/2)/f, -(j - H/2)/f, -1) in row-major pixel order, computed in
    float32 as the reference (and neo_sample_rays) do, returned in `dtype`."""
    j, i = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing="ij")
    return torch.stack([(i - W / 2) / focal, -(j - H / 2) / focal, -torch.ones_like(i)], -1).reshape(-1, 3).to(dtype)


def orthonormal(c2w: Tensor) -> Tensor:
    """c2w (..., 3, 4) with its rotation replaced by the nearest orthonormal matrix (U V^T of its SVD), in float64."""
    c = c2w.double()
    U, _, Vh = torch.linalg.svd(c[..., :3])
    return torch.cat([U @ Vh, c[..., 3:]], -1)


def rays_from_pose(dirs: Tensor, c2w: Tensor):
    """get_rays(dirs, c2w (3,4), output_view_dirs=True) out of place: rays_o, viewdirs, rays_d (== viewdirs), all (n,3)."""
    d = dirs.reshape(-1, 3) @ c2w[:, :3].T
    v = d / torch.norm(d, dim=-1, keepdim=True)
    return c2w[:, 3].expand(v.shape), v, v


def sample_rays_bwd(pix: Tensor, T: int, H: int, W: int, focal: float, c2w: Tensor, g_o=None, g_vd=None, g_rd=None):
    """pix (n) int64 into the (T,H,W) stack, c2w (T,3,4) float64, upstream gradients (n,3) or None -> g_c2w (T,3,4) and the per-view sum
    of |terms| (T,3,4)."""
    pix = pix.long()
    dt = c2w.dtype
    t, r = pix // (H * W), pix % (H * W)
    c = camera_dirs(H, W, focal, dt)[r]
    R = c2w[t, :, :3]
    d = (R @ c[..., None])[..., 0]
    nrm = torch.norm(d, dim=-1, keepdim=True)
    v = d / nrm
    z = torch.zeros_like(d)
    gv = (z if g_vd is None else g_vd.to(dt)) + (z if g_rd is None else g_rd.to(dt))
    gd = (gv - v * (v * gv).sum(-1, keepdim=True)) / nrm
    terms = torch.cat([gd[:, :, None] * c[:, None, :], (z if g_o is None else g_o.to(dt))[:, :, None]], -1)     # (n,3,4)
    g = torch.zeros(T, 3, 4, dtype=dt).index_add_(0, t, terms)
    mag = torch.zeros(T, 3, 4, dtype=dt).index_add_(0, t, terms.abs())
    return g, mag


def mlp_input_grad(g_sig, g_yb, S, P, F_in: int, rnd=True, skip_scale: float = 1.0):
    """The input-row gradient that `training._MLPTrainTC` returns when its features require grad, at the rounding points of
    oracle/dense_train_model.py (S, P from its `forward` / `params_of`; the same adjoint as its `backward`):
        g_feats = dz_0 bf(w_0)[:, :F] + dz_5 bf(w_5)[:, W:W+F]   (the second term only with the skip, depth > 5),
    each product accumulated in fp32 by a bf16 GEMM and the two added in fp32.  `skip_scale` scales the skip term (a test's mutation)."""
    from oracle import dense_train_model as dtm
    r = lambda x: dtm.bf(x, rnd)
    depth, W = len(P["w"]), P["w"][0].shape[0]
    xd = S["xd"]
    dh = g_sig @ P["wsig"]
    if "wb" in P:
        dbeta = r(r(g_yb) @ r(P["wvb"]))
        dh = dh + dbeta @ r(P["wb"])
    dz = r(dh * (xd > 0))
    out = 0
    for i in range(depth - 1, -1, -1):
        if i == 0:
            out = out + dz @ r(P["w"][0])[:, :F_in]
        if i == 5 and depth > 5:
            out = out + skip_scale * (dz @ r(P["w"][5])[:, W:W + F_in])
        if i > 0:
            X = S["X"][i]
            dz = r((dz @ r(P["w"][i]))[:, :W] * (X[:, :W] > 0))
    return out


def mip_dir_enc_bwd(vd: Tensor, g_denc: Tensor):
    """neo_mip_encode_bwd: g_viewdirs (n,3) of the direction encoding pos_enc(viewdirs, 0, 4) (models/mipnerf360/model.py:152) and the
    per-ray sums of |terms|.  The IPE features give no gradient: the reference's contract detaches them (helper.py:63-66)."""
    return _enc_grad(vd, g_denc, 4)
