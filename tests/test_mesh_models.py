"""CPU: meshing vanilla NeRF, Mip-NeRF 360 and PixelNeRF.  The point-Gaussian encoding of the oracle against the reference's own
contract / lift_and_diagonalize / integrated_pos_enc; the frustum features of the refactored tc model; argument validation of
neo_vanilla_field_eval and neo_mip_field_eval without a GPU; the slab-size rule."""
import ctypes as C
import os
import re

import pytest
import torch

from oracle import mip_oracle as mo
from oracle import mip_point_model as mpm
from oracle import ref_shim
from oracle import tc_paths_model as tpm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from neo360_b200 import build, _lib
    build.build()
    return _lib.load()


def points(seed=0):
    """(2, 40, 3) float64 points inside and outside the unit sphere (|x| up to about 3)."""
    g = torch.Generator().manual_seed(seed)
    p = torch.randn(2, 40, 3, generator=g, dtype=torch.float64)
    return p * torch.linspace(0.05, 3.0, 40, dtype=torch.float64)[None, :, None] / p.norm(dim=-1, keepdim=True)


@pytest.mark.skipif(not ref_shim.available(), reason="needs the reference sources")
@pytest.mark.parametrize("var", [(0.0, 0.0, 0.0), (1e-4, 4e-4, 9e-4), (0.01, 0.01, 0.01)])
def test_point_gaussian_encoding_equals_the_reference(var):
    ns = ref_shim.load()
    h = ns.mip_helper
    from neo360_b200.mip_basis import POS_BASIS_T
    basis = POS_BASIS_T.double()
    pts = points()
    assert bool((pts.norm(dim=-1) < 1).any()) and bool((pts.norm(dim=-1) > 1).any())
    mean, cov = mpm.point_gaussian(pts, var)
    z, zc = h.contract(mean, cov, is_train=False)
    fm, fv = h.lift_and_diagonalize(z, zc, basis)
    ref = h.integrated_pos_enc(fm, fv, 0, 12)
    got = mpm.point_features(pts, var, basis)
    assert got.shape == ref.shape == (2, 40, 504)
    assert float((got - ref).abs().max()) < 1e-6


def frustum_case(seed=1, n=6, N=9):
    g = torch.Generator().manual_seed(seed)
    o = torch.randn(n, 3, generator=g, dtype=torch.float64)
    d = torch.randn(n, 3, generator=g, dtype=torch.float64)
    rad = torch.rand(n, 1, generator=g, dtype=torch.float64) * 0.01
    td = torch.sort(torch.rand(n, N + 1, generator=g, dtype=torch.float64) * 4 + 0.5, -1).values
    return o, d, rad, td


def test_frustum_features_unchanged():
    """With the render's frustums as its source, the Gaussian-input model gives tc_paths_model's frustum features and its whole tc
    field bit for bit, with and without fp16 rounding: only the Gaussian's source differs between the two."""
    from neo360_b200 import mip
    from neo360_b200.mip_basis import POS_BASIS_T
    o, d, rad, td = frustum_case()
    basis = POS_BASIS_T.double()
    assert torch.equal(mpm.gaussian_features(*mo.cast_cone(td, o, d, rad), basis), tpm.mip_features(o, d, rad, td, basis))
    torch.manual_seed(0)
    P = {k: v.double() for k, v in mip.MipNeRF360().state_dict().items()}
    vd = torch.nn.functional.normalize(d, dim=-1)
    rays = {"rays_o": o, "rays_d": d, "viewdirs": vd}
    for lvl, depth in ((0, 4), (2, 8)):
        for fp16 in (True, False):
            want = tpm.mip_tc_field(P, f"mlps.{lvl}.", depth, lvl < 2, rays, rad, td, fp16=fp16)
            got = mpm.mip_tc_gaussian_field(P, f"mlps.{lvl}.", depth, lvl < 2, vd, *mo.cast_cone(td, o, d, rad), fp16=fp16)
            assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1]), (lvl, fp16)


def test_point_tc_field_without_rounding_is_the_oracle():
    """The tc model at point Gaussians with fp16 rounding off equals mip_oracle.mlp on point_features."""
    from neo360_b200 import mip
    torch.manual_seed(0)
    net = mip.MipNeRF360()
    P = {k: v.double() for k, v in net.state_dict().items()}
    pts = points(2)[:, :8]
    vd = torch.nn.functional.normalize(torch.randn(2, 3, dtype=torch.float64), dim=-1)
    var = (1e-4, 2e-4, 3e-4)
    for lvl, depth in ((0, 4), (2, 8)):
        pre = f"mlps.{lvl}."
        dens, rgb = mpm.mip_tc_gaussian_field(P, pre, depth, lvl < 2, vd, *mpm.point_gaussian(pts, var), fp16=False)
        rd, rr = mo.mlp(P, pre, mpm.point_features(pts, var, P[pre + "pos_basis_t"]), vd, depth, lvl < 2)
        assert float((dens - rd).abs().max()) < 1e-9 and float((rgb - rr).abs().max()) < 1e-9


NEW = ("neo_vanilla_field_workspace_bytes", "neo_vanilla_field_eval", "neo_mip_field_workspace_bytes", "neo_mip_field_eval")


def test_new_argtypes_match_the_header():
    from neo360_b200 import _lib as L
    hdr = open(os.path.join(ROOT, "include", "neo360_b200.h")).read()
    for name in NEW:
        m = re.search(r"(\w+)\s+" + name + r"\(([^)]*)\);", hdr)
        assert m, name
        params = [p.strip() for p in m.group(2).split(",")]
        res, args = L.SYMBOLS[name]
        assert {"int": C.c_int, "size_t": C.c_size_t}[m.group(1)] == res, name
        assert len(params) == len(args), name
        for p, a in zip(params, args):
            if "*" in p or "[" in p:
                assert a is C.c_void_p or issubclass(a, C._Pointer), (name, p)
            elif p.startswith("long long"):
                assert a is C.c_longlong, (name, p)
            elif p.startswith("size_t"):
                assert a is C.c_size_t, (name, p)
            else:
                assert p.startswith("int") and a is C.c_int, (name, p)


def rays(n=4):
    from neo360_b200 import _lib as L
    r = L.NeoRays()
    r.n_rays, r.chunk = n, 0
    r.rays_o = r.rays_d = r.viewdirs = 1 << 20
    return r


def test_vanilla_field_eval_rejects_bad_arguments_without_gpu(lib):
    """The pointers are never dereferenced: every call fails validation before a launch (the handle is a dummy)."""
    p = 1 << 20
    h = C.create_string_buffer(4096)
    r = rays()
    N = 5
    ws = lib.neo_vanilla_field_workspace_bytes(4 * N, 1)
    assert ws > 0 and lib.neo_vanilla_field_workspace_bytes(4 * N, 0) == 0 and lib.neo_vanilla_field_workspace_bytes(0, 1) == 0
    ev = lambda *a: lib.neo_vanilla_field_eval(*a)
    assert ev(None, C.byref(r), p, N, 1, 1, p, p, p, ws, None) == -1                   # handle
    assert ev(h, None, p, N, 1, 1, p, p, p, ws, None) == -1                            # rays
    assert ev(h, C.byref(r), None, N, 1, 1, p, p, p, ws, None) == -1                   # t
    assert ev(h, C.byref(r), p, N, 1, 1, None, p, p, ws, None) == -1                   # rgb
    assert ev(h, C.byref(r), p, N, 1, 1, p, None, p, ws, None) == -1                   # sigma
    assert ev(h, C.byref(r), p, 0, 1, 1, p, p, p, ws, None) == -1                      # N
    assert ev(h, C.byref(rays(0)), p, N, 1, 1, p, p, p, ws, None) == -1                # no rays
    assert ev(h, C.byref(r), p, N, 2, 1, p, p, p, ws, None) == -1                      # level
    assert b"level" in lib.neo_last_error()
    assert ev(h, C.byref(r), p, N, 1, 7, p, p, p, ws, None) == -1                      # precision
    assert ev(h, C.byref(r), p, N, 1, 1, p, p, p, ws - 1, None) == -3                  # workspace size
    assert ev(h, C.byref(r), p, N, 1, 1, p, p, None, ws, None) == -3                   # no workspace


def mip_mlps(rgb_head=True):
    from neo360_b200 import _lib as L
    p = 1 << 20
    arr = (L.NeoMipMLPParams * 3)()
    for lvl in range(3):
        m = arr[lvl]
        m.depth, m.width, m.basis = (8, 1024, p) if lvl == 2 else (4, 256, p)
        for i in range(m.depth):
            m.w[i] = m.b[i] = p
        m.wsig = m.bsig = p
        if lvl == 2 and rgb_head:
            m.wb = m.bb = m.wv0 = m.bv0 = m.wrgb = m.brgb = p
    return arr


def test_mip_field_eval_rejects_bad_arguments_without_gpu(lib):
    p = 1 << 20
    arr = mip_mlps()
    r = rays()
    N = 3
    var = (C.c_float * 3)(1e-4, 1e-4, 1e-4)
    ws = lib.neo_mip_field_workspace_bytes(4 * N, 1024, 0)
    assert ws > lib.neo_mip_field_workspace_bytes(4 * N, 256, 0) > 0
    assert lib.neo_mip_field_workspace_bytes(4 * N, 1024, 5) == 0 and lib.neo_mip_field_workspace_bytes(-1, 1024, 1) == 0
    ev = lambda *a: lib.neo_mip_field_eval(*a)
    for prec in (0, 1):
        w = lib.neo_mip_field_workspace_bytes(4 * N, 1024, prec)
        assert ev(None, 2, C.byref(r), p, N, var, prec, p, p, p, w, None) == -1            # mlps
        assert ev(arr, 2, None, p, N, var, prec, p, p, p, w, None) == -1                   # rays
        assert ev(arr, 2, C.byref(r), None, N, var, prec, p, p, p, w, None) == -1          # t
        assert ev(arr, 2, C.byref(r), p, N, None, prec, p, p, p, w, None) == -1            # var
        assert ev(arr, 2, C.byref(r), p, N, var, prec, p, None, p, w, None) == -1          # density
        assert ev(arr, 3, C.byref(r), p, N, var, prec, p, p, p, w, None) == -1             # level
        assert ev(arr, -1, C.byref(r), p, N, var, prec, p, p, p, w, None) == -1
        for lvl in (0, 1):                                                                 # rgb at a proposal level
            assert ev(arr, lvl, C.byref(r), p, N, var, prec, p, p, p, w, None) == -1
            assert b"colour" in lib.neo_last_error()
        assert ev(arr, 2, C.byref(r), p, N, (C.c_float * 3)(1e-4, -1.0, 0.0), prec, p, p, p, w, None) == -1   # var < 0
        assert ev(arr, 2, C.byref(r), p, N, (C.c_float * 3)(float("nan"), 0, 0), prec, p, p, p, w, None) == -1
        assert ev(mip_mlps(rgb_head=False), 2, C.byref(r), p, N, var, prec, None, p, p, w, None) == -1   # level 2 without its colour head
        assert ev(arr, 2, C.byref(r), p, 0, var, prec, p, p, p, w, None) == -1             # N
        assert ev(arr, 2, C.byref(r), p, N, var, prec, p, p, p, w - 1, None) == -3         # workspace size
        assert ev(arr, 2, C.byref(r), p, N, var, prec, p, p, None, w, None) == -3
    assert ev(arr, 2, C.byref(r), p, N, var, 4, p, p, p, ws, None) == -1                   # precision


@pytest.mark.parametrize("precision", ["fp32", "tc"])
def test_mip_slab_rule_keeps_the_workspace_under_the_budget(lib, precision):
    """R = 512: the rows the rule picks, and no more, fit SLAB_BUDGET by the workspace query (plus rays, t and rgb)."""
    from neo360_b200 import mesh, mip
    net = mip.MipNeRF360()
    R = 512
    rows = mesh.slab_rows(net, R, R * R, precision)
    ws = lib.neo_mip_field_workspace_bytes(rows * R, 1024, {"fp32": 0, "tc": 1}[precision])
    cost = lambda r: lib.neo_mip_field_workspace_bytes(r * R, 1024, {"fp32": 0, "tc": 1}[precision]) + r * 24 + r * R * 16
    assert 1 <= rows < R * R
    assert cost(rows) <= mesh.SLAB_BUDGET < cost(rows + 1)
    assert ws / (rows * R) > 5000                      # kB of workspace per point: far more than a fixed 16384-row slab could take
    assert 16384 * R * ws / (rows * R) > 50e9


def test_default_levels_and_model_rules():
    from neo360_b200 import mesh
    assert {k: mesh._level(k, None) for k in mesh.LEVELS} == {"neo360": 1, "vanilla": 1, "pixelnerf": 1, "mip360": 2}
    with pytest.raises(ValueError):
        mesh._level("vanilla", 2)
    with pytest.raises(ValueError):
        mesh._src_batch("pixelnerf", None)
    with pytest.raises(ValueError):
        mesh._src_batch("pixelnerf", {"src_imgs": None})
    with pytest.raises(TypeError):
        mesh._kind(torch.nn.Linear(2, 2))
    g = mesh.make_grid(5, ((-2, -2, -2), (2, 2, 2)))
    assert mesh.grid_var(g) == pytest.approx((1.0 / 12,) * 3)
