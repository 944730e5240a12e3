"""CPU: the float64 models of the vanilla NeRF, Mip-NeRF 360 and GridEncoder tensor-core paths (oracle/tc_paths_model.py), which the
GPU tests in test_gpu_tc_paths.py hold the kernels to.  Pinned here without a GPU:

* with fp16=False each model equals its oracle to <= 1e-9 in float64 (`vanilla_oracle.mlp_forward`, `mip_oracle.mlp` on
  `ipe_features`, `GridEncoder.dense_torch` at the same pillars);
* every value-level bug of each model's mutation catalogue moves its output by more than 3x a GPU bound, so the GPU test, which compares
  the kernel with the unmutated model at those bounds, would fail for the same bug in the kernel.  Each catalogue also reports whether
  the older end-to-end test's bound, on that test's own inputs, would have caught the bug.
"""
import os

import numpy as np
import pytest
import torch

from neo360_b200 import synth
from oracle import mip_oracle as mo
from oracle import neo360_oracle as orc
from oracle import tc_paths_model as tpm
from oracle import vanilla_oracle as vo

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
T = lambda a: torch.from_numpy(np.asarray(a))


def md(a, b):
    return float((a.double() - b.double()).abs().max())


def frame_rays(W, H, view, sel):
    """Rays (float64) and radii of pixels `sel` of a W x H frame of target camera `view`."""
    ro, vd, rd, radii = orc.rays_from_pose(orc.ray_directions(H, W, 0.8 * W), synth.target_pose(view, 100)[:3, :4])
    f = lambda x: x[sel].double().contiguous()
    return {"rays_o": f(ro), "rays_d": f(rd), "viewdirs": f(vd)}, f(radii)


def random_t(n, N, near, far, seed):
    g = torch.Generator().manual_seed(seed)
    return near + (far - near) * torch.sort(torch.rand(n, N, generator=g, dtype=torch.float64), -1).values


def mip_tdist(n, N, near, far, seed):
    """Sorted s in [0, 1] with both ends, mapped to t as the renderer's s_to_t does."""
    g = torch.Generator().manual_seed(seed)
    s = torch.sort(torch.rand(n, N + 1, generator=g, dtype=torch.float64), -1).values
    s[:, 0], s[:, -1] = 0.0, 1.0
    return 1.0 / (s / far + (1 - s) / near)


# ---------------- fp16 off: each model is its oracle ----------------

@pytest.mark.parametrize("pre", ["coarse_mlp.", "fine_mlp."])
def test_vanilla_model_without_rounding_is_the_oracle(pre):
    P = {k: v.double() for k, v in synth.make_vanilla_params(5).items()}
    rays, _ = frame_rays(37, 23, 4, slice(100, 131))
    t = random_t(31, 13, 0.2, 3.0, 1)
    with torch.no_grad():
        rgb, sig = tpm.vanilla_tc_field(P, pre, rays, t, fp16=False)
        pts = rays["rays_o"][:, None, :] + t[..., None] * rays["viewdirs"][:, None, :]
        raw_rgb, raw_sig = vo.mlp_forward(P, pre, orc.pos_enc(pts, 0, 10), orc.pos_enc(rays["viewdirs"], 0, 4))
    assert md(rgb, torch.sigmoid(raw_rgb) * 1.002 - 0.001) <= 1e-9
    assert md(sig, torch.nn.functional.softplus(raw_sig - 1.0)) <= 1e-9


@pytest.mark.parametrize("lvl", [0, 2])
@pytest.mark.parametrize("far", [6.0, 100.0])
def test_mip_model_without_rounding_is_the_oracle(lvl, far):
    P = {k: v.double() for k, v in synth.make_mip_params(4, width=256).items()}
    pre, depth, no_rgb = f"mlps.{lvl}.", (4 if lvl < 2 else 8), lvl < 2
    rays, radii = frame_rays(40, 30, 7, slice(0, 1200, 41))
    td = mip_tdist(rays["rays_o"].shape[0], 11, 0.2, far, lvl)
    with torch.no_grad():
        dens, rgb = tpm.mip_tc_field(P, pre, depth, no_rgb, rays, radii, td, fp16=False)
        mean, cov = mo.cast_cone(td, rays["rays_o"], rays["rays_d"], radii[:, None])
        z, zc = mo.contract(mean, cov)
        rd, rr = mo.mlp(P, pre, mo.ipe_features(z, zc, P[pre + "pos_basis_t"]), rays["viewdirs"], depth, no_rgb)
    assert dens.shape == rd.shape and rgb.shape == rr.shape
    assert md(dens, rd) <= 1e-9 * (1 + float(rd.abs().max())) and md(rgb, rr) <= 1e-9


def small_grid_encoder(G):
    from neo360_b200.encoder import GridEncoder
    torch.manual_seed(3)
    enc = GridEncoder().eval().double()
    enc.GRID = G
    return enc


def encoder_poses(nv):
    """Synthetic source cameras plus an identity camera (grid cells on z_cam = 0 and behind the camera) and one at (0, 0, 0.5)."""
    poses = synth.make_scene((36, 22), nv, (4, 4), 0)["src_poses"].double()
    poses[0] = torch.eye(4, dtype=torch.float64)
    if nv > 1:
        poses[1] = torch.eye(4, dtype=torch.float64)
        poses[1, 2, 3] = 0.5
    return poses


@pytest.mark.parametrize("nv,lat_hw", [(1, (11, 18)), (3, (19, 12))])
def test_encoder_model_without_rounding_is_dense_torch(nv, lat_hw):
    """On an 8^3 grid (the model takes G from the module): every pillar of every view and axis.  dense_torch builds its grid in the
    default dtype, so both run with float64 as the default."""
    G = 8
    enc = small_grid_encoder(G)
    lh, lw = lat_hw
    W, H = 2 * lw, 2 * lh
    g = torch.Generator().manual_seed(nv)
    latent = torch.rand(nv, 512, lh, lw, generator=g, dtype=torch.float64) ** 2 * 2
    poses = encoder_poses(nv)
    focal, c = torch.full((nv,), 0.8 * W, dtype=torch.float64), torch.tensor([[W / 2.0, H / 2.0]] * nv, dtype=torch.float64)
    pil = torch.tensor([(v, a, p, q) for v in range(nv) for a in range(3) for p in range(G) for q in range(G)])
    dtype = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        with torch.no_grad():
            xz, xy, yz = enc.dense_torch(latent, poses, focal, c, W, H)
            got = tpm.encoder_tc_dense(enc, latent, poses, focal, c, W, H, pil, fp16=False)
    finally:
        torch.set_default_dtype(dtype)
    planes = {0: yz, 1: xz, 2: xy}
    ref = torch.stack([planes[a][v, :, p, q] for v, a, p, q in pil.tolist()])
    assert float(ref.abs().max()) > 0.1
    assert md(got, ref) <= 1e-9 * float(ref.abs().max())
    # the scene exercises what the kernel must get right: cells behind the camera, on z_cam = 0, and lookups outside the latent
    _, cam, _, uv = tpm.encoder_geometry(pil, G, poses, float(focal[0]), c[0], W, H, (lh, lw))
    assert bool((cam[..., 2] >= 1e-3).any()) and bool((cam[..., 2] < 1e-3).any()) and bool((cam[..., 2] == 0).any())
    assert bool((uv.abs() > 1).any()) and bool((uv.abs() < 1).all(-1).any())


# ---------------- mutation catalogues ----------------

def van_render(P, rays, nc, nf, white, mutation=None):
    """vanilla_oracle.render with the TC model as the field (float64)."""
    o, d, vd = rays["rays_o"], rays["rays_d"], rays["viewdirs"]
    out, w = [], None
    for lvl, pre in enumerate(("coarse_mlp.", "fine_mlp.")):
        t = vo.sample_along_rays(o, vd, nc, 0.2, 3.0)[0] if lvl == 0 else vo.sample_pdf(o, vd, t, w, nf)[0]
        rgb, sig = tpm.vanilla_tc_field(P, pre, rays, t, mutation=mutation)
        comp, acc, w, _ = vo.composite(rgb, sig, t, d, white)
        out.append((comp, acc))
    return out


def test_vanilla_mutation_catalogue_exceeds_gpu_bounds():
    """Each bug of tc_paths_model.VANILLA_MUTATIONS moves rgb or sigma by more than 3x a GPU bound on these inputs (both MLPs, 31 frame
    rays x 21 samples, and a nearly empty variant of the weights whose sigma is seen through the transmittance).  Also reported: the
    bug's rendering against the reference vectors of test_gpu_parity.py::test_vanilla_nerf_tc_vs_reference_vectors[v_tiny] at that
    test's bound (L-inf 3e-2 on rgb / acc, PSNR 40 dB, both levels)."""
    g = np.load(os.path.join(GOLDEN, "vanilla_reference_vectors.npz"))
    _, _, _, nc, nf, seed = [int(x) for x in g["v_tiny_cfg"]]
    P0 = synth.make_vanilla_params(seed)
    old_rays = {k: T(g[f"v_tiny_{k}"]).double() for k in ("rays_o", "rays_d", "viewdirs")}
    cases = []
    for shift in (1.0, -25.0):
        P = synth.make_vanilla_params(9, density_bias_shift=shift)
        rays, _ = frame_rays(64, 48, 12, slice(1000, 3000, 64))
        t = random_t(rays["rays_o"].shape[0], 21, 0.2, 3.0, 4)
        for pre in ("coarse_mlp.", "fine_mlp."):
            with torch.no_grad():
                cases.append((P, pre, rays, t, tpm.vanilla_tc_field(P, pre, rays, t)))
    report = []
    for mut in tpm.VANILLA_MUTATIONS:
        seen = 0.0
        with torch.no_grad():
            for P, pre, rays, t, (rgb0, sig0) in cases:
                rgb, sig = tpm.vanilla_tc_field(P, pre, rays, t, mutation=mut)
                dr, ds = (rgb - rgb0).abs().amax(-1), tpm.sigma_error(sig, sig0)
                seen = max(seen, float(dr.max()) / tpm.VAN_RGB_TOL, float(ds.max()) / tpm.VAN_SIGMA_TOL,
                           float(dr.mean()) / tpm.VAN_RGB_MEAN_TOL, float(ds.mean()) / tpm.VAN_SIGMA_MEAN_TOL)
            ren = van_render(P0, old_rays, nc, nf, True, mut)
        old = []
        for lvl in range(2):
            ref_rgb, ref_acc = T(g[f"v_tiny_eval{lvl}_rgb"]).double(), T(g[f"v_tiny_eval{lvl}_acc"]).double()
            old.append((md(ren[lvl][0], ref_rgb), md(ren[lvl][1], ref_acc), orc.psnr(ren[lvl][0], ref_rgb)))
        caught = [e_rgb >= 3e-2 or e_acc >= 3e-2 or ps <= 40.0 for e_rgb, e_acc, ps in old]
        report.append(f"{mut:15s} {seen:8.1f} x GPU bound | old test (v_tiny): " +
                      ", ".join(f"level {l} rgb {o[0]:.1e} acc {o[1]:.1e} {o[2]:.1f} dB ({'caught' if c else 'MISSED'})"
                                for l, (o, c) in enumerate(zip(old, caught))))
        assert seen > 3.0, report[-1]
    print("\n" + "\n".join(report))


def mip_render(P, batch, npp, nn_, near, far, mutation=None):
    """mip_oracle.render (train_frac 1, deterministic) with the TC model as the field (float64)."""
    o = batch["rays_o"]
    B = o.shape[0]
    s_to_t = lambda s: 1 / (s * (1 / far) + (1 - s) * (1 / near))
    sdist = torch.cat([torch.zeros(B, 1), torch.ones(B, 1)], -1).double()
    weights = torch.ones(B, 1, dtype=torch.float64)
    prod, out = 1, []
    for lvl in range(3):
        n = npp if lvl < 2 else nn_
        dil = 0.0025 + 0.5 / prod
        prod *= n
        if lvl > 0:
            sdist, weights = mo.max_dilate_weights(sdist, weights, dil)
            sdist, weights = sdist[..., 1:-1], weights[..., 1:-1]
        logits = torch.where(sdist[..., 1:] > sdist[..., :-1], torch.log(weights), torch.full_like(weights, -torch.inf))
        sdist = mo.sample_intervals(sdist, logits, n)
        td = s_to_t(sdist)
        dens, rgb = tpm.mip_tc_field(P, f"mlps.{lvl}.", 4 if lvl < 2 else 8, lvl < 2, batch, batch["radii"], td, mutation=mutation)
        weights = mo.alpha_weights(dens, td, batch["rays_d"])
        out.append((weights[..., None] * rgb).sum(-2) + torch.clip(1 - weights.sum(-1)[..., None], min=0))
    return out


def test_mip_mutation_catalogue_exceeds_gpu_bounds():
    """Each bug of tc_paths_model.MIP_MUTATIONS moves density or rgb by more than 3x a GPU bound (all three MLPs at width 256, 30 frame
    rays x 16 intervals, far 6 and 100).  Also reported: the bug's renderings against the reference vectors of
    test_gpu_parity.py::test_mip360_tc_vs_reference_vectors[m_tiny] at that test's bound (L-inf 3e-2, PSNR 35 dB per level)."""
    P = synth.make_mip_params(6, width=256)
    cases = []
    for far in (6.0, 100.0):
        rays, radii = frame_rays(40, 30, 21, slice(0, 1200, 40))
        td = mip_tdist(rays["rays_o"].shape[0], 16, 0.2, far, int(far))
        for lvl in range(3):
            with torch.no_grad():
                base = tpm.mip_tc_field(P, f"mlps.{lvl}.", 4 if lvl < 2 else 8, lvl < 2, rays, radii, td)
            cases.append((lvl, rays, radii, td, base))
    g = np.load(os.path.join(GOLDEN, "mip360_reference_vectors.npz"))
    _, _, _, npp, nn_, seed = [int(x) for x in g["m_tiny_cfg"]]
    near, far = [float(x) for x in g["m_tiny_near_far"]]
    P0 = synth.make_mip_params(seed)
    batch = {k: T(g[f"m_tiny_{k}"]).double() for k in ("rays_o", "rays_d", "viewdirs", "radii")}
    batch["radii"] = batch["radii"].reshape(-1, 1)
    report = []
    for mut in tpm.MIP_MUTATIONS:
        seen = 0.0
        with torch.no_grad():
            for lvl, rays, radii, td, (d0, c0) in cases:
                dens, rgb = tpm.mip_tc_field(P, f"mlps.{lvl}.", 4 if lvl < 2 else 8, lvl < 2, rays, radii, td, mutation=mut)
                dr, ds = (rgb - c0).abs().amax(-1), tpm.sigma_error(dens, d0)
                seen = max(seen, float(dr.max()) / tpm.MIP_RGB_TOL, float(ds.max()) / tpm.MIP_SIGMA_TOL,
                           float(dr.mean()) / tpm.MIP_RGB_MEAN_TOL, float(ds.mean()) / tpm.MIP_SIGMA_MEAN_TOL)
            ren = mip_render(P0, batch, npp, nn_, near, far, mut)
        old = [(md(ren[i], T(g[f"m_tiny_eval{i}_rgb"])), orc.psnr(ren[i], T(g[f"m_tiny_eval{i}_rgb"]).double())) for i in range(3)]
        report.append(f"{mut:13s} {seen:8.1f} x GPU bound | old test (m_tiny): " +
                      ", ".join(f"level {i} {e:.1e} {ps:.1f} dB ({'caught' if e >= 3e-2 or ps <= 35.0 else 'MISSED'})"
                                for i, (e, ps) in enumerate(old)))
        assert seen > 3.0, report[-1]
    print("\n" + "\n".join(report))


def seeded_pillars(nv, G, per, seed):
    """`per` pillars per view and axis: the four corners, two more border pillars, the rest seeded."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for v in range(nv):
        for a in range(3):
            fixed = [(0, 0), (0, G - 1), (G - 1, 0), (G - 1, G - 1), (0, int(torch.randint(G, (1,), generator=g))),
                     (int(torch.randint(G, (1,), generator=g)), G - 1)]
            pq = fixed + [tuple(torch.randint(G, (2,), generator=g).tolist()) for _ in range(per - len(fixed))]
            out += [(v, a, p, q) for p, q in pq]
    return torch.tensor(out)


def test_encoder_mutation_catalogue_exceeds_gpu_bounds():
    """Each bug of tc_paths_model.ENCODER_MUTATIONS moves the pillar sums by more than 3x a GPU bound (relative to the case's largest
    |pillar sum|) on the GPU test's inputs at a subset of its pillars (NV = 3, latent 11 x 18, cameras including the identity pose).
    Also reported: the same bug at 8 pillars per view and axis of test_encoder.py::test_grid_encoder_cuda_dense_part's inputs (ResNet
    latent of the reference images), against that test's bound of 2e-2 of the scale (measured here against the unmutated model)."""
    from neo360_b200.encoder import GridEncoder
    torch.manual_seed(3)
    enc = GridEncoder().eval()
    nv, lh, lw = 3, 11, 18
    W, H = 2 * lw, 2 * lh
    latent = torch.rand(nv, 512, lh, lw, generator=torch.Generator().manual_seed(1)) ** 2 * 2
    poses = encoder_poses(nv).float()
    focal, c = torch.full((nv,), 0.8 * W), torch.tensor([[W / 2.0, H / 2.0]] * nv)
    pil = seeded_pillars(nv, 64, 8, 0)
    ge = np.load(os.path.join(GOLDEN, "encoder_reference_vectors.npz"))
    seed, W0, H0, NV0 = [int(x) for x in ge["cfg"]]
    torch.manual_seed(seed)
    enc0 = GridEncoder().eval()
    sc0 = synth.make_scene((W0, H0), NV0, (12, 16), seed)
    with torch.no_grad():
        base = tpm.encoder_tc_dense(enc, latent, poses, focal, c, W, H, pil)
        lat0 = enc0.spatial_encoder(T(ge["imgs"]))
        pil0 = seeded_pillars(NV0, 64, 8, 1)
        base0 = tpm.encoder_tc_dense(enc0, lat0, sc0["src_poses"], sc0["src_focal"], sc0["src_c"], W0, H0, pil0)
    scale, scale0 = float(base.abs().max()), float(base0.abs().max())
    report = []
    for mut in tpm.ENCODER_MUTATIONS:
        with torch.no_grad():
            d = (tpm.encoder_tc_dense(enc, latent, poses, focal, c, W, H, pil, mutation=mut) - base).abs() / scale
            d0 = float((tpm.encoder_tc_dense(enc0, lat0, sc0["src_poses"], sc0["src_focal"], sc0["src_c"], W0, H0, pil0,
                                              mutation=mut) - base0).abs().max()) / scale0
        seen = max(float(d.max()) / tpm.ENC_TOL, float(d.mean()) / tpm.ENC_MEAN_TOL)
        report.append(f"{mut:14s} {seen:8.1f} x GPU bound | old test's inputs: {d0:.1e} of scale "
                      f"({'caught' if d0 >= 2e-2 else 'MISSED'} by 2e-2)")
        assert seen > 3.0, report[-1]
    print("\n" + "\n".join(report))
