"""CPU: the float64 models of the ray and pose backward (oracle/camera_grad_model.py) against torch.autograd through the reference's own
helpers (vanilla pos_enc / cast_rays, ray_utils.get_ray_directions / get_rays), `cameras.PoseCorrection` at omega = 0, and host-side
argument checks of the new entry points."""
import pytest
import torch

from oracle import camera_grad_model as cgm
from oracle import ref_shim

needs_ref = pytest.mark.skipif(not ref_shim.available(), reason="reference sources not present")


@pytest.fixture(scope="module")
def ns():
    return ref_shim.load()


@needs_ref
@pytest.mark.parametrize("n,N", [(1, 1), (5, 17), (7, 65)])
def test_vanilla_encode_bwd_matches_autograd_through_reference(ns, n, N):
    g = torch.Generator().manual_seed(10 * n + N)
    o = (torch.rand(n, 3, generator=g, dtype=torch.float64) * 4 - 2).requires_grad_(True)
    vd = torch.nn.functional.normalize(torch.randn(n, 3, generator=g, dtype=torch.float64), dim=-1).requires_grad_(True)
    t = torch.sort(torch.rand(n, N, generator=g, dtype=torch.float64) * 3 + 0.2, -1).values
    pts = ns.van_helper.cast_rays(t, o, vd)                                         # o + t viewdirs (helper.py:20)
    enc = ns.van_helper.pos_enc(pts, 0, 10).reshape(n * N, 63)
    denc = ns.van_helper.pos_enc(vd, 0, 4)
    g_enc, g_denc = torch.randn(n * N, 63, generator=g, dtype=torch.float64), torch.randn(n, 27, generator=g, dtype=torch.float64)
    ((enc * g_enc).sum() + (denc * g_denc).sum()).backward()
    g_o, g_vd, mag_o, mag_vd = cgm.vanilla_encode_bwd(o.detach(), vd.detach(), t, g_enc, g_denc)
    assert torch.allclose(g_o, o.grad, rtol=0, atol=1e-12 * float(mag_o.max()))
    assert torch.allclose(g_vd, vd.grad, rtol=0, atol=1e-12 * float(mag_vd.max()))
    assert bool((mag_o >= g_o.abs()).all()) and bool((mag_vd >= g_vd.abs()).all())


@needs_ref
def test_rays_from_pose_is_the_reference_get_rays(ns):
    from neo360_b200 import synth
    H, W, f = 12, 16, 13.0
    pose = synth.target_pose(3, 100)[:3, :4].double()
    dirs = ns.ray_utils.get_ray_directions(H, W, f).double()
    assert torch.equal(dirs.reshape(-1, 3), cgm.camera_dirs(H, W, f))
    ro, vd, rd = ns.ray_utils.get_rays(dirs, pose, output_view_dirs=True)
    o2, v2, r2 = cgm.rays_from_pose(dirs, pose)
    assert torch.allclose(ro, o2, atol=0, rtol=0) and torch.allclose(vd, v2, atol=1e-15) and torch.allclose(rd, r2, atol=1e-15)


@pytest.mark.parametrize("T,n", [(1, 1), (3, 200)])
def test_sample_rays_bwd_matches_autograd(T, n):
    from neo360_b200 import synth
    H, W, f = 9, 11, 7.5
    g = torch.Generator().manual_seed(T + n)
    c2w = torch.stack([synth.target_pose(7 * k, 100)[:3, :4].double() for k in range(T)]).requires_grad_(True)
    pix = torch.randint(0, T * H * W, (n,), generator=g)
    dirs = cgm.camera_dirs(H, W, f)
    ro, vd, rd = zip(*[cgm.rays_from_pose(dirs, c2w[k]) for k in range(T)])
    flat = lambda x: torch.cat(x, 0)[pix]
    go, gv, gr = (torch.randn(n, 3, generator=g, dtype=torch.float64) for _ in range(3))
    ((flat(ro) * go).sum() + (flat(vd) * gv).sum() + (flat(rd) * gr).sum()).backward()
    got, mag = cgm.sample_rays_bwd(pix, T, H, W, f, c2w.detach(), go, gv, gr)
    assert torch.allclose(got, c2w.grad, rtol=0, atol=1e-12 * float(mag.max()))
    only_o, _ = cgm.sample_rays_bwd(pix, T, H, W, f, c2w.detach(), go, None, None)
    assert bool((only_o[..., :3] == 0).all())


@needs_ref
def test_radii_do_not_change_under_a_pose_correction(ns):
    """radii (ray_utils.py:153-160) are norms of differences of rotated directions: a rotation R exp([w]x) or a translation leaves them
    unchanged, so their gradient contributes nothing to a pose correction and neo_sample_rays_bwd gives them none."""
    from neo360_b200 import synth
    from neo360_b200.cameras import so3_exp
    H, W, f = 10, 12, 9.0
    pose = cgm.orthonormal(synth.target_pose(11, 100)[:3, :4])
    dirs = ns.ray_utils.get_ray_directions(H, W, f).double()
    moved = torch.cat([pose[:, :3] @ so3_exp(torch.tensor([0.3, -0.2, 0.5], dtype=torch.float64)), pose[:, 3:] + 0.7], 1)
    r0 = ns.ray_utils.get_rays(dirs, pose, output_view_dirs=True, output_radii=True)[3]
    r1 = ns.ray_utils.get_rays(dirs, moved, output_view_dirs=True, output_radii=True)[3]
    assert torch.allclose(r0, r1, rtol=1e-13, atol=0)


def test_pose_correction_at_zero_has_the_analytic_gradient():
    from neo360_b200 import synth
    from neo360_b200.cameras import PoseCorrection, skew
    T = 3
    c2w = torch.stack([cgm.orthonormal(synth.target_pose(5 * k, 100)[:3, :4]) for k in range(T)])
    pc = PoseCorrection(T).double()
    out = pc(c2w)
    assert torch.equal(out, c2w)
    G = torch.randn(T, 3, 4, generator=torch.Generator().manual_seed(4), dtype=torch.float64)
    (out * G).sum().backward()
    assert bool(torch.isfinite(pc.omega.grad).all())
    e = torch.eye(3, dtype=torch.float64)
    want = torch.stack([torch.stack([(G[v, :, :3] * (c2w[v, :, :3] @ skew(e[a]))).sum() for a in range(3)]) for v in range(T)])
    assert torch.allclose(pc.omega.grad, want, rtol=1e-13, atol=1e-13)
    assert torch.equal(pc.tau.grad, G[:, :, 3])
    # 4x4 poses keep their last row; a small rotation is a rotation
    c44 = torch.cat([c2w, torch.tensor([0, 0, 0, 1.0], dtype=torch.float64).expand(T, 1, 4)], 1)
    with torch.no_grad():
        pc.omega.copy_(torch.tensor([[1e-5, 0, 0], [0.2, -0.1, 0.3], [0, 0, 2.0]]))
    o44 = pc(c44)
    assert torch.equal(o44[:, 3], c44[:, 3])
    R = o44[:, :3, :3]
    assert torch.allclose(R.transpose(1, 2) @ R, torch.eye(3, dtype=torch.float64).expand(T, 3, 3), atol=1e-14)
    with pytest.raises(ValueError):
        pc(c2w[:2])


def test_series_branch_continues_the_closed_form():
    from neo360_b200.cameras import so3_exp
    w = torch.tensor([1.0, -2.0, 0.5], dtype=torch.float64)
    w = w / w.norm()
    for s in (0.999e-3, 1.001e-3):          # either side of the branch point th^2 = 1e-6
        th = torch.tensor(s, dtype=torch.float64)
        K = torch.zeros(3, 3, dtype=torch.float64)
        K[0, 1], K[0, 2], K[1, 2] = -w[2] * th, w[1] * th, -w[0] * th
        K = K - K.T
        assert torch.allclose(so3_exp(w * th), torch.linalg.matrix_exp(K), rtol=0, atol=1e-15)


def test_new_entry_points_reject_bad_arguments_without_gpu():
    from neo360_b200 import build, _lib as L
    build.build()
    lib = L.load()
    p = 1 << 20
    assert lib.neo_vanilla_encode_bwd(p, p, p, 4, 8, p, p, p, None, None) == -1
    assert lib.neo_vanilla_encode_bwd(p, p, p, 0, 8, p, p, p, p, None) == -1
    assert b"neo_vanilla_encode_bwd" in lib.neo_last_error()
    assert lib.neo_sample_rays_bwd_workspace_bytes(100, 3) >= 100 * 13 * 4 + 3 * 12 * 4
    assert lib.neo_sample_rays_bwd(8, p, 0, 4, 4, 1.0, p, None, None, None, p, p, 1 << 20, None) == -1          # no views
    assert lib.neo_sample_rays_bwd(8, p, 1, 4, 4, 1.0, p, None, None, None, None, p, 1 << 20, None) == -1       # no g_c2w
    assert lib.neo_sample_rays_bwd(8, p, 1, 4, 4, 1.0, p, None, None, None, p, p, 16, None) not in (0, -1)      # workspace too small
    assert b"workspace" in lib.neo_last_error()


@needs_ref
def test_mip_dir_enc_bwd_matches_autograd_through_reference(ns):
    g = torch.Generator().manual_seed(8)
    vd = torch.randn(9, 3, generator=g, dtype=torch.float64).requires_grad_(True)
    gd = torch.randn(9, 27, generator=g, dtype=torch.float64)
    (ns.mip_helper.pos_enc(vd, 0, 4, True) * gd).sum().backward()
    got, mag = cgm.mip_dir_enc_bwd(vd.detach(), gd)
    assert torch.allclose(got, vd.grad, rtol=0, atol=1e-12 * float(mag.max()))


@pytest.mark.parametrize("kind", ["vanilla", "prop", "mip"])
def test_mlp_input_grad_without_rounding_is_autograd(kind):
    """With every bf() the identity, the input-row model is autograd of dense_train_model.forward w.r.t. its features (both the layer-0
    and the skip layer's columns); dropping half of the skip term moves it."""
    from neo360_b200 import mip, vanilla
    from oracle import dense_train_model as dtm
    torch.manual_seed(1)
    m, F = (vanilla.NeRFMLP(), 63) if kind == "vanilla" else ((mip.PropMLP(), 504) if kind == "prop" else (mip.NeRFMLP(netwidth=256), 504))
    P = dtm.params_of(m)
    g = torch.Generator().manual_seed(2)
    feats = torch.randn(40, F, generator=g, dtype=torch.float64).clamp(-1, 1).requires_grad_(True)
    sig, yb, S = dtm.forward(feats, P, rnd=False)
    gs = torch.randn(40, 1, generator=g, dtype=torch.float64)
    gy = torch.randn(40, 128, generator=g, dtype=torch.float64) if yb is not None else None
    ((sig * gs).sum() + ((yb * gy).sum() if yb is not None else 0)).backward()
    got = cgm.mlp_input_grad(gs, gy, S, P, F, rnd=False)
    assert torch.allclose(got, feats.grad, rtol=1e-12, atol=1e-12)
    if len(P["w"]) > 5:
        half = cgm.mlp_input_grad(gs, gy, S, P, F, rnd=False, skip_scale=0.5)
        assert dtm.rel_err(half, feats.grad) > 1e-2
