"""GPU: meshes of vanilla NeRF, Mip-NeRF 360 and PixelNeRF (neo360_b200/mesh.py, neo_vanilla_field_eval, neo_mip_field_eval,
PixelNeRF.field).  Each model's density grid against its float64 oracle or fp16 model, the render's field against the new entry bit for
bit, direction independence of sigma, vertex colours against a direct field evaluation, and whole meshes to PLY."""
import numpy as np
import pytest
import torch

from neo360_b200 import synth
from oracle import mesh_model as mm
from oracle import mip_oracle as mo
from oracle import mip_point_model as mpm
from oracle import neo360_oracle as orc
from oracle import pixelnerf_oracle as por
from oracle import tc_paths_model as tpm
from oracle import vanilla_oracle as vo

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
UNIT = ((-1.0, -1.0, -1.0), (1.0, 1.0, 1.0))
BOX2 = ((-2.0, -2.0, -2.0), (2.0, 2.0, 2.0))      # Mip-NeRF 360: half the lattice lies outside the unit sphere, where it contracts
# Mip-NeRF 360 fp32 grid against the float64 point-Gaussian oracle, in sigma's pre-activation units (tpm.sigma_error): measured
# 8.8e-7 max over the three levels on an H100 80GB HBM3 at a 700 W power limit; the bound is about 3x that.
MIP_FP32_SIGMA_TOL = 3e-6


@pytest.fixture(scope="module", autouse=True)
def built():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from neo360_b200 import build
    build.build()


def lattice(shape, bbox):
    """float32 lattice points of make_grid(shape, bbox), (nz*ny*nx, 3), as the kernels round them."""
    from neo360_b200 import mesh
    g = mesh.make_grid(shape, bbox)
    ax = [mm.lattice(list(g.origin), list(g.step), n, a, True) for a, n in enumerate((g.nx, g.ny, g.nz))]
    Z, Y, X = np.meshgrid(ax[2], ax[1], ax[0], indexing="ij")
    return torch.from_numpy(np.stack([X, Y, Z], -1).reshape(-1, 3)), g


def vanilla_net(precision="fp32", seed=4):
    from neo360_b200.vanilla import NeRF
    P = synth.make_vanilla_params(seed)
    net = NeRF(num_coarse_samples=16, num_fine_samples=8).eval()
    net.precision = precision
    net.load_state_dict(P)
    return net.to(DEV), P


def mip_net(precision="fp32", seed=2):
    from neo360_b200.mip import MipNeRF360
    P = synth.make_mip_params(seed)
    net = MipNeRF360(num_prop_samples=16, num_nerf_samples=8, precision=precision).eval()
    net.load_state_dict(P)
    return net.to(DEV), P


def pixel_net(nv, precision="fp32", seed=11):
    from neo360_b200 import PixelNeRF
    W, H = 64, 48
    sc = synth.make_scene((W, H), nv, (8, 8), seed)
    net = PixelNeRF(num_coarse_samples=16, num_fine_samples=8, num_src_views=nv)
    net.load_state_dict({**net.state_dict(), **synth.make_pixelnerf_params(seed)})
    net = net.to(DEV).eval()
    net.precision = precision
    latent = sc["latent"].to(DEV)
    net.encoder.forward = lambda x: latent            # the synthetic encoder output, as tests/test_gpu_pixelnerf.py does
    batch = {"src_imgs": torch.zeros(nv, 3, H, W, device=DEV), "src_poses": sc["src_poses"].to(DEV),
             "src_focal": sc["src_focal"].to(DEV), "src_c": sc["src_c"].to(DEV)}
    osc = por.scene(sc["latent"], sc["src_poses"], sc["src_focal"], sc["src_c"], (W, H))
    return net, batch, osc, synth.make_pixelnerf_params(seed)


def grid_rays(g):
    """The rays density_grid evaluates: every x-row of the lattice, from neo_grid_rays."""
    import ctypes as C
    from neo360_b200 import _lib as L
    rows = g.ny * g.nz
    o, d, t = torch.empty(rows, 3, device=DEV), torch.empty(rows, 3, device=DEV), torch.empty(rows, g.nx, device=DEV)
    L.check(L.load().neo_grid_rays(C.byref(g), 0, rows, L.ptr(o), L.ptr(d), L.ptr(t), torch.cuda.current_stream().cuda_stream))
    return {"rays_o": o, "rays_d": d, "viewdirs": d}, t


# ---------------- vanilla NeRF ----------------

@pytest.mark.parametrize("precision", ["fp32", "tc"])
def test_vanilla_field_eval_is_the_render_field(precision):
    """neo_vanilla_field_eval at the render's own rays and t of each level gives forward(debug=True)'s sigma and rgb_s bit for bit."""
    net, _ = vanilla_net(precision)
    W, H = 64, 48
    ro, vd, rd, _ = orc.rays_from_pose(orc.ray_directions(H, W, 0.8 * W), synth.target_pose(3, 100)[:3, :4])
    rays = {"rays_o": ro.to(DEV), "rays_d": rd.to(DEV), "viewdirs": vd.to(DEV)}
    for randomized in (False, True):
        with torch.no_grad():
            net(rays, randomized, False, 0.2, 3.0, debug=True)
        dbg = net.last_debug
        for lvl in range(2):
            rgb, sig = net.field(rays, dbg["t"][lvl], lvl)
            assert torch.equal(sig, dbg["sigma"][lvl][..., 0]) and torch.equal(rgb, dbg["rgb_s"][lvl]), (randomized, lvl)


@pytest.mark.parametrize("level", [0, 1])
def test_vanilla_density_grid_fp32_vs_oracle(level):
    net, P = vanilla_net("fp32")
    shape = (13, 14, 15)
    sig = net.density_grid(shape, UNIT, level=level, precision="fp32").reshape(-1).cpu()
    pts, _ = lattice(shape, UNIT)
    with torch.no_grad():
        _, raw = vo.mlp_forward(P, ("coarse_mlp.", "fine_mlp.")[level], orc.pos_enc(pts, 0, 10)[None], torch.zeros(1, 27))
    ref = torch.nn.functional.softplus(raw.reshape(-1) - 1.0)
    err = float((sig - ref).abs().max())
    print(f"vanilla fp32 grid level {level}: max |sigma - oracle| = {err:.2e}, sigma up to {float(ref.max()):.3g}")
    assert err < 2e-4 and float(ref.max()) > 0.1


def test_vanilla_density_grid_tc_vs_model():
    """The tc grid against tc_paths_model.vanilla_tc_field on the lattice rays, within test_gpu_tc_paths.py's VAN_SIGMA bounds."""
    net, P = vanilla_net("tc")
    shape = (17, 16, 18)
    sig = net.density_grid(shape, UNIT, precision="tc")
    _, g = lattice(shape, UNIT)
    rays, t = grid_rays(g)
    with torch.no_grad():
        _, ms = tpm.vanilla_tc_field(P, "fine_mlp.", rays, t)
    e = tpm.sigma_error(sig.reshape(-1), ms.reshape(-1))
    print(f"vanilla tc grid: sigma error (pre-activation units) max {float(e.max()):.2e} mean {float(e.mean()):.2e}")
    assert float(e.max()) <= tpm.VAN_SIGMA_TOL and float(e.mean()) <= tpm.VAN_SIGMA_MEAN_TOL


# ---------------- Mip-NeRF 360 ----------------

def mip_oracle_density(P, lvl, pts, var):
    depth = 4 if lvl < 2 else 8
    pre = f"mlps.{lvl}."
    P64 = {k: v.double().to(DEV) for k, v in P.items() if k.startswith(pre)}
    feats = mpm.point_features(pts.double().to(DEV)[None], var, P64[pre + "pos_basis_t"])
    dens, _ = mo.mlp(P64, pre, feats, torch.tensor([[1.0, 0.0, 0.0]], dtype=torch.float64, device=DEV), depth, lvl < 2)
    return dens.reshape(-1)


@pytest.mark.parametrize("level", [0, 1, 2])
def test_mip_density_grid_fp32_vs_oracle(level):
    from neo360_b200 import mesh
    net, P = mip_net("fp32")
    shape = (15, 16, 17)
    pts, g = lattice(shape, BOX2)
    sig = net.density_grid(shape, BOX2, level=level, precision="fp32").reshape(-1)
    assert bool((pts.norm(dim=-1) > 1).any())
    ref = mip_oracle_density(P, level, pts, mesh.grid_var(g))
    e = tpm.sigma_error(sig, ref)
    print(f"mip fp32 grid level {level}: sigma error (pre-activation units) max {float(e.max()):.2e}; sigma up to {float(ref.max()):.3g}")
    assert float(e.max()) < MIP_FP32_SIGMA_TOL


@pytest.mark.parametrize("level", [0, 1, 2])
def test_mip_density_grid_tc_vs_model(level):
    """The tc grid against mip_point_model.mip_tc_gaussian_field at the lattice points, within test_gpu_tc_paths.py's MIP_SIGMA bounds."""
    from neo360_b200 import mesh
    net, P = mip_net("tc")
    shape = (15, 16, 17)
    pts, g = lattice(shape, BOX2)
    sig = net.density_grid(shape, BOX2, level=level, precision="tc").reshape(-1)
    rays, t = grid_rays(g)
    gauss = mpm.point_gaussian(pts.double().to(DEV).reshape(t.shape[0], t.shape[1], 3), mesh.grid_var(g))
    with torch.no_grad():
        md, _ = mpm.mip_tc_gaussian_field(P, f"mlps.{level}.", 4 if level < 2 else 8, level < 2, rays["viewdirs"], *gauss)
    e = tpm.sigma_error(sig, md.reshape(-1))
    print(f"mip tc grid level {level}: sigma error (pre-activation units) max {float(e.max()):.2e} mean {float(e.mean()):.2e}")
    assert float(e.max()) <= tpm.MIP_SIGMA_TOL and float(e.mean()) <= tpm.MIP_SIGMA_MEAN_TOL


# ---------------- PixelNeRF ----------------

@pytest.mark.parametrize("nv", [1, 3])
def test_pixelnerf_density_grid_fp32(nv):
    """The grid is PixelNeRF.field on the lattice rays bit for bit, and within 2e-4 of pixelnerf_oracle."""
    net, batch, osc, P = pixel_net(nv)
    shape = (13, 14, 15)
    sig = net.density_grid(shape, UNIT, precision="fp32", batch=batch)
    pts, g = lattice(shape, UNIT)
    rays, t = grid_rays(g)
    _, direct = net.field({**batch, **rays}, t, 1, precision="fp32")
    assert torch.equal(sig.reshape(direct.shape), direct)
    with torch.no_grad():
        st = por.stages(pts.reshape(-1, 1, 3), torch.tensor([[1.0, 0.0, 0.0]]).expand(pts.shape[0], 3), osc, 1)
        _, raw = por.mlp_forward(P, "fine_mlp.", st["enc"], st["dir_tile"], st["latent"], nv)
    ref = torch.relu(raw.reshape(-1))
    err = float((sig.reshape(-1).cpu() - ref).abs().max())
    print(f"pixelnerf fp32 grid nv {nv}: max |sigma - oracle| = {err:.2e}, sigma up to {float(ref.max()):.3g}")
    assert err < 2e-4 and float(ref.max()) > 0.05


def test_pixelnerf_density_grid_tc_is_the_field():
    net, batch, _, _ = pixel_net(3)
    shape = (13, 14, 15)
    sig = net.density_grid(shape, UNIT, precision="tc", batch=batch)
    _, g = lattice(shape, UNIT)
    rays, t = grid_rays(g)
    _, direct = net.field({**batch, **rays}, t, 1, precision="tc")
    assert torch.equal(sig.reshape(direct.shape), direct)
    assert net.precision == "fp32"                    # a precision argument does not change the module's own


# ---------------- every model ----------------

def models():
    return [("vanilla", lambda p: (vanilla_net(p)[0], None)), ("mip360", lambda p: (mip_net(p)[0], None)),
            ("pixelnerf", lambda p: pixel_net(3, p)[:2])]


def direct_field(kind, net, batch, rays, t, level, precision, var):
    if kind == "vanilla":
        return net.field(rays, t, level, precision=precision)
    if kind == "mip360":
        return net.field(rays, t, level, var, precision=precision)
    return net.field({**batch, **rays}, t, level, chunk=t.shape[0], precision=precision)


@pytest.mark.parametrize("precision", ["fp32", "tc"])
@pytest.mark.parametrize("kind", ["vanilla", "mip360", "pixelnerf"])
def test_sigma_does_not_depend_on_the_view_direction(kind, precision):
    net, batch = dict(models())[kind](precision)
    g = torch.Generator().manual_seed(5)
    o = ((torch.rand(257, 3, generator=g) - 0.5) * 1.6).to(DEV)
    t = torch.zeros(257, 1, device=DEV)
    var = (1e-4, 2e-4, 3e-4)
    sig = []
    for k in range(3):
        d = torch.nn.functional.normalize(torch.randn(257, 3, generator=g), dim=-1).to(DEV)
        sig.append(direct_field(kind, net, batch, {"rays_o": o, "rays_d": d, "viewdirs": d}, t, 1 if kind != "mip360" else 2, precision, var)[1])
    assert torch.equal(sig[0], sig[1]) and torch.equal(sig[0], sig[2])


@pytest.mark.parametrize("precision", ["fp32", "tc"])
@pytest.mark.parametrize("kind", ["vanilla", "mip360", "pixelnerf"])
def test_colors_equal_a_direct_field_eval(kind, precision):
    from neo360_b200 import mesh
    net, batch = dict(models())[kind](precision)
    bbox = BOX2 if kind == "mip360" else UNIT
    R = 24
    sig = mesh.density_grid(net, R, bbox, batch=batch)
    iso = float(sig[sig > 0].median())                 # PixelNeRF's sigma = relu(...) is 0 over much of the box
    m = mesh.extract_mesh(net, batch, R, iso=iso, bbox=bbox)
    V = m["verts"].shape[0]
    assert V > 0 and m["colors"].shape == (V, 3)
    var = mesh.grid_var(mesh.make_grid(R, bbox))
    vd = (-m["normals"]).contiguous()
    t0 = torch.zeros(V, 1, device=DEV)
    level = 2 if kind == "mip360" else 1
    rgb, _ = direct_field(kind, net, batch, {"rays_o": m["verts"], "rays_d": vd, "viewdirs": vd}, t0, level, precision, var)
    assert torch.equal(rgb.reshape(V, 3), m["colors"])
    if kind == "pixelnerf":
        # quirk Q1 with N = 1 and chunk = V: each vertex is conditioned on its own direction, so permuting the vertices together with
        # their directions permutes the colours, while reversing the directions changes them
        perm = torch.randperm(V, generator=torch.Generator().manual_seed(0)).to(DEV)
        rp, _ = direct_field(kind, net, batch, {"rays_o": m["verts"][perm].contiguous(), "rays_d": vd[perm].contiguous(),
                                                "viewdirs": vd[perm].contiguous()}, t0, level, precision, var)
        assert torch.equal(rp.reshape(V, 3), m["colors"][perm])
        rev, _ = direct_field(kind, net, batch, {"rays_o": m["verts"], "rays_d": -vd, "viewdirs": -vd}, t0, level, precision, var)
        assert not torch.equal(rev.reshape(V, 3), m["colors"])


@pytest.mark.parametrize("kind", ["mip360", "pixelnerf"])
def test_colors_in_budgeted_calls(kind, monkeypatch):
    """With a budget that splits the vertices into many calls, the colours still equal one direct field evaluation of every vertex:
    each call is its own chunk, and with N = 1 PixelNeRF's quirk-Q1 ray is still the vertex itself."""
    from neo360_b200 import mesh
    net, batch = dict(models())[kind]("tc")
    bbox = BOX2 if kind == "mip360" else UNIT
    g = torch.Generator().manual_seed(3)
    V = 1000
    verts = ((torch.rand(V, 3, generator=g) - 0.5) * 1.5).to(DEV)
    normals = torch.nn.functional.normalize(torch.randn(V, 3, generator=g), dim=-1).to(DEV)
    var = mesh.grid_var(mesh.make_grid(32, bbox))
    monkeypatch.setattr(mesh, "SLAB_BUDGET", mesh.workspace_bytes(net, 97, "tc") + 97 * 40)
    assert mesh.slab_rows(net, 1, V, "tc") < V // 5
    got = mesh.vertex_colors(net, verts, normals, batch=batch, var=var)
    vd = (-normals).contiguous()
    want, _ = direct_field(kind, net, batch, {"rays_o": verts, "rays_d": vd, "viewdirs": vd}, torch.zeros(V, 1, device=DEV),
                           2 if kind == "mip360" else 1, "tc", var)
    assert torch.equal(got, want.reshape(V, 3))


@pytest.mark.parametrize("kind", ["vanilla", "mip360", "pixelnerf"])
def test_mesh_to_ply_end_to_end(kind, tmp_path):
    """R = 64: extract_mesh, write_ply and back; the faces equal oracle/mesh_model.py on the same grid."""
    from neo360_b200 import mesh, output
    net, batch = dict(models())[kind]("tc")
    bbox = BOX2 if kind == "mip360" else UNIT
    sig = mesh.density_grid(net, 64, bbox, batch=batch)
    iso = float(torch.quantile(sig[sig > 0], 0.6))
    m = mesh.extract_mesh(net, batch, 64, iso=iso, bbox=bbox)
    assert m["faces"].shape[0] > 100 and bool(torch.isfinite(m["colors"]).all())
    g = mesh.make_grid(64, bbox)
    _, f_ref = mm.marching_tetrahedra(sig.cpu().numpy(), list(g.origin), list(g.step), iso, fp32=True)
    assert np.array_equal(m["faces"].cpu().numpy(), f_ref)
    vert, faces = mm.read_ply(output.write_ply(str(tmp_path / f"{kind}.ply"), m))
    assert np.array_equal(np.stack([vert["x"], vert["y"], vert["z"]], -1), m["verts"].cpu().numpy())
    assert np.array_equal(faces, m["faces"].cpu().numpy())
    c = np.rint(np.clip(m["colors"].cpu().numpy(), 0, 1) * 255).astype(np.uint8)
    assert np.array_equal(np.stack([vert["red"], vert["green"], vert["blue"]], -1), c)


def test_errors():
    from neo360_b200 import mesh
    net, _ = mip_net("fp32")
    sig = mesh.density_grid(net, 9, BOX2, level=0)                # proposal levels give density grids
    assert sig.shape == (9, 9, 9)
    with pytest.raises(ValueError, match="colour"):
        mesh.extract_mesh(net, None, 9, iso=float(sig.median()), bbox=BOX2, level=0)
    with pytest.raises(ValueError, match="colour"):
        mesh.vertex_colors(net, torch.zeros(3, 3, device=DEV), torch.ones(3, 3, device=DEV), level=1, var=(0.0, 0.0, 0.0))
    pnet, batch, _, _ = pixel_net(1)
    with pytest.raises(ValueError, match="source views"):
        mesh.density_grid(pnet, 9)
    with pytest.raises(ValueError, match="source views"):
        mesh.extract_mesh(pnet, {"src_imgs": batch["src_imgs"]}, 9, iso=0.0)
