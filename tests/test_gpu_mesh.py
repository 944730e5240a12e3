"""GPU: the geometry export (csrc/mesh.cu, neo360_b200/mesh.py).  Marching tetrahedra against the NumPy model (oracle/mesh_model.py)
face for face and bit for bit; the density grid against the oracle's NeRFPPMLP; normals and vertex colours; a whole scene to PLY."""
import numpy as np
import pytest
import torch

from neo360_b200 import synth
from oracle import mesh_model as mm
from oracle import neo360_oracle as orc

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cuda():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from neo360_b200 import build
    build.build()
    return torch.device("cuda:0")


def lattice_xyz(shape, bbox):
    """float32 lattice coordinates of make_grid(shape, bbox), (nz, ny, nx, 3), with the kernels' rounding."""
    from neo360_b200 import mesh
    g = mesh.make_grid(shape, bbox)
    ax = [mm.lattice(list(g.origin), list(g.step), n, a, True) for a, n in enumerate((g.nx, g.ny, g.nz))]
    Z, Y, X = np.meshgrid(ax[2], ax[1], ax[0], indexing="ij")
    return np.stack([X, Y, Z], -1), list(g.origin), list(g.step)


def analytic(name, shape, bbox=((-1, -1, -1), (1, 1, 1))):
    P, _, _ = lattice_xyz(shape, bbox)
    X, Y, Z = (P[..., a].astype(np.float64) for a in range(3))
    if name == "sphere":
        s = 0.6 - np.sqrt(X ** 2 + Y ** 2 + Z ** 2)
    elif name == "two_spheres":
        s = np.maximum(0.35 - np.sqrt((X + 0.45) ** 2 + Y ** 2 + (Z - 0.1) ** 2), 0.3 - np.sqrt((X - 0.45) ** 2 + (Y - 0.1) ** 2 + Z ** 2))
    elif name == "torus":
        s = 0.25 - np.sqrt((np.sqrt(X ** 2 + Y ** 2) - 0.55) ** 2 + Z ** 2)
    else:                                       # smooth random field: a few random Fourier modes
        g = np.random.default_rng(7)
        s = np.zeros_like(X)
        for _ in range(12):
            k = g.normal(size=3) * 3.0
            s += np.cos(k[0] * X + k[1] * Y + k[2] * Z + g.uniform(0, 2 * np.pi)) * g.uniform(0.2, 1.0)
    return s.astype(np.float32)


def run_mt(cuda, sig, iso, bbox=((-1, -1, -1), (1, 1, 1))):
    from neo360_b200 import mesh
    v, f = mesh.marching_tetrahedra(torch.from_numpy(sig).to(cuda), iso, bbox)
    return v.cpu().numpy(), f.cpu().numpy()


FIELDS = [("sphere", (40, 40, 40)), ("two_spheres", (41, 40, 39)), ("torus", (37, 45, 43)), ("random", (33, 29, 47))]


@pytest.mark.parametrize("name,shape", FIELDS)
def test_kernel_equals_model(cuda, name, shape):
    """Identical V, F and face arrays; vertices bit-identical to the model's fp32 operation order and within 4e-6 of float64."""
    sig = analytic(name, shape)
    _, origin, step = lattice_xyz(shape, ((-1, -1, -1), (1, 1, 1)))
    v, f = run_mt(cuda, sig, 0.0)
    v32, f_ref = mm.marching_tetrahedra(sig, origin, step, 0.0, fp32=True)
    v64, _ = mm.marching_tetrahedra(sig, origin, step, 0.0)
    assert v.shape == v32.shape and f.shape == f_ref.shape and f.shape[0] > 0
    assert np.array_equal(f, f_ref)
    assert np.array_equal(v.view(np.uint32), v32.view(np.uint32))
    assert np.abs(v - v64).max() < 4e-6
    if name != "random":
        cu, cd = mm.edge_face_counts(f)
        assert (cu == 2).all() and (cd == 1).all()
        assert mm.euler_characteristic(f) == {"sphere": 2, "two_spheres": 4, "torus": 0}[name]
        assert mm.signed_volume(v, f) > 0


@pytest.mark.parametrize("case", ["ties", "all_inside", "all_outside", "R2", "ragged"])
def test_corner_cases(cuda, case):
    g = np.random.default_rng(3)
    iso = 0.5
    if case == "ties":            # many values exactly at iso: they count as inside
        sig = (g.integers(0, 3, size=(9, 10, 11)) * 0.25 + 0.25).astype(np.float32)
    elif case == "all_inside":
        sig = np.full((6, 7, 8), iso, dtype=np.float32)
    elif case == "all_outside":
        sig = np.full((6, 7, 8), np.nextafter(np.float32(iso), np.float32(0)), dtype=np.float32)
    elif case == "R2":
        sig = g.random((2, 2, 2)).astype(np.float32)
        sig[0, 0, 0], sig[1, 1, 1] = 1.0, 0.0
    else:                          # 7 * 13 * 37 points: no block size divides it
        sig = g.random((7, 13, 37)).astype(np.float32)
    bbox = ((-0.3, 0.1, -2.0), (0.9, 0.7, 1.0))
    _, origin, step = lattice_xyz(sig.shape, bbox)
    v, f = run_mt(cuda, sig, iso, bbox)
    v32, f_ref = mm.marching_tetrahedra(sig, origin, step, iso, fp32=True)
    assert np.array_equal(f, f_ref) and np.array_equal(v.view(np.uint32), v32.view(np.uint32))
    if case.startswith("all"):
        assert v.shape == (0, 3) and f.shape == (0, 3)
    else:
        assert f.shape[0] > 0


def test_two_calls_are_bit_identical(cuda):
    from neo360_b200 import mesh
    sig = torch.from_numpy(analytic("random", (64, 64, 64))).to(cuda)
    a = mesh.marching_tetrahedra(sig, 0.1)
    b = mesh.marching_tetrahedra(sig, 0.1)
    assert torch.equal(a[0].view(torch.int32), b[0].view(torch.int32)) and torch.equal(a[1], b[1])


def test_normals_match_the_model(cuda):
    from neo360_b200 import mesh
    bbox = ((-1, -1, -1), (1, 1, 1))
    for name, shape in FIELDS:
        sig = analytic(name, shape)
        _, origin, step = lattice_xyz(shape, bbox)
        st = torch.from_numpy(sig).to(cuda)
        v, _ = mesh.marching_tetrahedra(st, 0.0, bbox)
        n = mesh.grid_normals(st, v, bbox).cpu().numpy().astype(np.float64)
        ref = mm.grid_normals(sig, origin, step, v.cpu().numpy())
        assert np.abs(n - ref).max() < 1e-4, name


# ---------------- density grid and colours of a scene ----------------

def make_net(cuda, nv, precisions=("fp32",), precision="fp32", img_wh=(64, 48), plane_hw=(24, 32), seed=0):
    from neo360_b200 import NeRF_TP
    sc = synth.make_scene(img_wh, nv, plane_hw, seed)
    P = synth.make_mlp_params(seed)
    net = NeRF_TP(num_coarse_samples=8, num_fine_samples=4, num_src_views=nv, precision=precision).eval()
    net.load_state_dict(P)
    net = net.to(cuda)
    net.set_scene(*[sc[k].to(cuda) for k in ("planes_xz", "planes_xy", "planes_yz", "latent", "src_poses", "src_focal", "src_c")],
                  sc["img_wh"], precisions=list(precisions))
    W, H = img_wh
    osc = orc.Scene(sc["planes_xz"], sc["planes_xy"], sc["planes_yz"], sc["latent"], sc["src_poses"],
                    float(sc["src_focal"][0]), float(sc["src_c"][0, 0]), float(sc["src_c"][0, 1]), W, H)
    return net, osc, P, sc


def oracle_sigma(osc, P, pts, nv, pre):
    """The oracle's NeRFPPMLP density at world points (M, 3); the direction input does not reach the density head."""
    cam = orc.world2camera(pts, osc.src_poses)
    world = orc.triplane_lookup(cam, osc).reshape(-1, 128)
    local = orc.local_lookup(cam, osc).reshape(-1, 512)
    enc = orc.pos_enc(cam, 0, 10)
    _, raw = orc.mlp_forward(P, pre, enc, torch.zeros(nv * pts.shape[0], 27), world, local, nv)
    return torch.nn.functional.softplus(raw[:, 0] - 1.0)


BOX = ((-1.2, -1.1, -1.0), (1.0, 1.2, 1.1))


@pytest.mark.parametrize("nv", [1, 3])
@pytest.mark.parametrize("level", [0, 1])
def test_density_grid_fp32_vs_oracle(cuda, nv, level):
    net, osc, P, _ = make_net(cuda, nv)
    shape = (17, 16, 18)
    sig = net.density_grid(shape, BOX, level=level, precision="fp32", slab_rays=100).cpu()
    pts, _, _ = lattice_xyz(shape, BOX)
    pts = torch.from_numpy(pts.reshape(-1, 3))
    with torch.no_grad():
        ref = oracle_sigma(osc, P, pts, nv, ("fg_coarse_mlp." if level == 0 else "fg_fine_mlp."))
    outside = (pts * pts).sum(-1) > 1
    ref[outside] = 0
    assert bool(outside.any()) and bool((sig.reshape(-1)[outside] == 0).all())
    assert float((sig.reshape(-1) - ref).abs().max()) < 2e-4
    assert float(ref.abs().max()) > 0.1


def test_density_grid_tc_vs_oracle(cuda):
    """Bounds of the TC field in tests/test_gpu_parity.py: |sigma| 2e-2 + 2%."""
    net, osc, P, _ = make_net(cuda, 3, precisions=("fp32", "tc"))
    shape = (17, 17, 17)
    sig = net.density_grid(shape, BOX, precision="tc").cpu().reshape(-1)
    pts, _, _ = lattice_xyz(shape, BOX)
    pts = torch.from_numpy(pts.reshape(-1, 3))
    with torch.no_grad():
        ref = oracle_sigma(osc, P, pts, 3, "fg_fine_mlp.")
    ref[(pts * pts).sum(-1) > 1] = 0
    ds = (sig - ref).abs()
    assert float((ds - 0.02 * ref.abs()).max()) < 2e-2, float(ds.max())


def test_density_does_not_depend_on_the_view_direction(cuda):
    """The density head reads only the view mean of the trunk: field_eval with two different viewdirs gives the same sigma bits."""
    from neo360_b200 import mesh
    net, _, _, _ = make_net(cuda, 3)
    g = torch.Generator().manual_seed(1)
    o = ((torch.rand(300, 3, generator=g) - 0.5) * 1.2).to(cuda)
    d = torch.nn.functional.normalize(torch.randn(300, 3, generator=g), dim=-1).to(cuda)
    t = (torch.rand(300, 9, generator=g) * 0.3).to(cuda)
    far = torch.ones(300, device=cuda)
    _, s1 = net.field_eval({"rays_o": o, "rays_d": d, "viewdirs": d}, far, t, 2, precision="fp32")
    _, s2 = net.field_eval({"rays_o": o, "rays_d": d, "viewdirs": -d.flip(0)}, far, t, 2, precision="fp32")
    assert torch.equal(s1, s2)
    # and the density grid is the same through any slab split
    a = mesh.density_grid(net, (9, 10, 11), BOX, precision="fp32", slab_rays=7)
    b = mesh.density_grid(net, (9, 10, 11), BOX, precision="fp32")
    assert torch.equal(a, b)


@pytest.mark.parametrize("precision", ["fp32", "tc"])
def test_colors_equal_a_direct_field_eval(cuda, precision):
    from neo360_b200 import mesh
    net, _, _, _ = make_net(cuda, 3, precisions=("fp32", "tc"), precision=precision)
    sig = net.density_grid(24)
    iso = float(sig[sig > 0].median())
    m = mesh.extract_mesh(net, None, 24, iso=iso)
    V = m["verts"].shape[0]
    assert V > 0 and m["colors"].shape == (V, 3) and m["faces"].dtype == torch.int32
    vd = (-m["normals"]).contiguous()
    rgb, _ = net.field_eval({"rays_o": m["verts"], "rays_d": vd, "viewdirs": vd}, torch.zeros(V, device=cuda),
                            torch.zeros(V, 1, device=cuda), 2, chunk=V, precision=precision)
    assert torch.equal(rgb.reshape(V, 3), m["colors"])
    # each vertex is coloured along its own direction: reversing the directions changes the colours
    rev, _ = net.field_eval({"rays_o": m["verts"], "rays_d": -vd, "viewdirs": -vd}, torch.zeros(V, device=cuda),
                            torch.zeros(V, 1, device=cuda), 2, chunk=V, precision=precision)
    assert not torch.equal(rev.reshape(V, 3), m["colors"])
    n = torch.linalg.norm(m["normals"], dim=-1)
    assert float((n - 1).abs().max()) < 1e-5


def test_bench_scene_mesh_to_ply(cuda, tmp_path):
    """The bench scene (640x480, 3 views, 120x160 planes) at R = 128 through a batch with explicit planes, then PLY and back."""
    from neo360_b200 import mesh, output
    net, _, _, sc = make_net(cuda, 3, precisions=(), precision="tc", img_wh=(640, 480), plane_hw=(120, 160))
    batch = {k: sc[k].to(cuda) for k in ("planes_xz", "planes_xy", "planes_yz", "latent", "src_poses", "src_focal", "src_c")}
    batch["src_imgs"] = torch.zeros(3, 3, 480, 640, device=cuda)
    sig = mesh.density_grid(net, 128, batch=batch)
    iso = float(sig[sig > 0].median())
    m = mesh.extract_mesh(net, batch, 128, iso=iso)
    assert m["verts"].shape[0] > 1000 and m["faces"].shape[0] > 1000
    assert int(m["faces"].min()) >= 0 and int(m["faces"].max()) < m["verts"].shape[0]
    assert bool(torch.isfinite(m["colors"]).all()) and bool(torch.isfinite(m["normals"]).all())
    vert, faces = mm.read_ply(output.write_ply(str(tmp_path / "scene.ply"), m))
    assert np.array_equal(np.stack([vert["x"], vert["y"], vert["z"]], -1), m["verts"].cpu().numpy())
    assert np.array_equal(np.stack([vert["nx"], vert["ny"], vert["nz"]], -1), m["normals"].cpu().numpy())
    assert np.array_equal(faces, m["faces"].cpu().numpy())
    c = np.rint(np.clip(m["colors"].cpu().numpy(), 0, 1) * 255).astype(np.uint8)
    assert np.array_equal(np.stack([vert["red"], vert["green"], vert["blue"]], -1), c)
    # the mesh of a level set closed by the unit sphere: every edge in two faces, consistently wound
    cu, cd = mm.edge_face_counts(m["faces"].cpu().numpy())
    assert (cu == 2).all() and (cd == 1).all()
