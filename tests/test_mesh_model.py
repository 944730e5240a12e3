"""CPU: the NumPy marching-tetrahedra model (oracle/mesh_model.py) on analytic fields.  Closed level sets give closed, consistently
and outwardly wound meshes with the Euler characteristic of their topology, and vertices near the analytic surface."""
import math

import numpy as np
import pytest

from oracle import mesh_model as mm


def grid(R, lo=-1.0, hi=1.0):
    h = (hi - lo) / (R - 1)
    origin, step = (lo, lo, lo), (h, h, h)
    x = mm.lattice(origin, step, R, 0, False)
    Z, Y, X = np.meshgrid(x, x, x, indexing="ij")
    return origin, step, X, Y, Z


def sphere(X, Y, Z, c=(0.0, 0.0, 0.0), r=0.6):
    return r - np.sqrt((X - c[0]) ** 2 + (Y - c[1]) ** 2 + (Z - c[2]) ** 2)


def torus(X, Y, Z, R0=0.55, r=0.25):
    return r - np.sqrt((np.sqrt(X ** 2 + Y ** 2) - R0) ** 2 + Z ** 2)


def check_closed_oriented(faces):
    cu, cd = mm.edge_face_counts(faces)
    assert (cu == 2).all(), "every edge must be in exactly two faces"
    assert (cd == 1).all(), "every directed edge once: consistent winding"


def test_kuhn_tetrahedra_tile_the_cube_positively():
    vols = []
    for tet in mm.TETS:
        p = np.array([mm.corner(c) for c in tet], dtype=np.float64)
        vols.append(np.linalg.det(p[1:] - p[0]) / 6.0)
    assert np.allclose(vols, 1.0 / 6.0)
    # every tetrahedron is a chain of corners, so each of its edges is an owned edge of its lower corner
    for tet in range(6):
        for a in range(4):
            for b in range(a + 1, 4):
                lo, ty = mm._edge_ref(tet, (a, b))
                assert ty in range(7) and lo in mm.TETS[tet]


@pytest.mark.parametrize("m", range(16))
def test_case_triangles_face_the_outside(m):
    """In the standard tetrahedron every case's triangles (midpoint vertices) have normals pointing to the outside corners."""
    P = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]], dtype=np.float64)
    ins = [c for c in range(4) if (m >> c) & 1]
    out = [c for c in range(4) if not (m >> c) & 1]
    tris = mm.tet_triangles(m)
    assert len(tris) == {0: 0, 1: 1, 2: 2, 3: 1, 4: 0}[len(ins)]
    for tri in tris:
        v = np.array([(P[a] + P[b]) / 2 for a, b in tri])
        n = np.cross(v[1] - v[0], v[2] - v[0])
        c = v.mean(0)
        assert all(np.dot(n, P[o] - c) > 0 for o in out) and all(np.dot(n, P[i] - c) < 0 for i in ins)


@pytest.mark.parametrize("R", [24, 33])
def test_sphere_is_closed_genus_zero_and_outward(R):
    origin, step, X, Y, Z = grid(R)
    r = 0.6
    v, f = mm.marching_tetrahedra(sphere(X, Y, Z, r=r), origin, step, 0.0)
    check_closed_oriented(f)
    assert mm.euler_characteristic(f) == 2 and mm.components(f) == 1
    h = step[0]
    vol = mm.signed_volume(v, f)
    assert abs(vol - 4.0 / 3.0 * math.pi * r ** 3) < 4 * math.pi * r ** 2 * h, vol
    assert vol > 0
    assert np.abs(np.linalg.norm(v, axis=1) - r).max() < h


def test_two_spheres():
    origin, step, X, Y, Z = grid(40)
    s = np.maximum(sphere(X, Y, Z, (-0.45, 0.0, 0.1), 0.35), sphere(X, Y, Z, (0.45, 0.1, 0.0), 0.3))
    v, f = mm.marching_tetrahedra(s, origin, step, 0.0)
    check_closed_oriented(f)
    assert mm.components(f) == 2 and mm.euler_characteristic(f) == 4
    exact = 4.0 / 3.0 * math.pi * (0.35 ** 3 + 0.3 ** 3)
    assert abs(mm.signed_volume(v, f) - exact) < 4 * math.pi * (0.35 ** 2 + 0.3 ** 2) * step[0]


def test_torus_has_euler_characteristic_zero():
    origin, step, X, Y, Z = grid(41)
    v, f = mm.marching_tetrahedra(torus(X, Y, Z), origin, step, 0.0)
    check_closed_oriented(f)
    assert mm.euler_characteristic(f) == 0 and mm.components(f) == 1
    d = np.abs(0.25 - np.sqrt((np.sqrt(v[:, 0] ** 2 + v[:, 1] ** 2) - 0.55) ** 2 + v[:, 2] ** 2))
    assert d.max() < step[0]
    assert mm.signed_volume(v, f) > 0


def test_ties_count_as_inside():
    """sigma == iso is inside: a grid equal to iso except one lower point gives the small closed surface around that point."""
    s = np.full((5, 5, 5), 2.0, dtype=np.float32)
    s[2, 2, 2] = 1.0
    v, f = mm.marching_tetrahedra(s, (0, 0, 0), (1, 1, 1), 2.0)
    check_closed_oriented(f)
    assert mm.euler_characteristic(f) == 2
    # w = (iso - s_a) / (s_b - s_a) is 0 or 1 on every edge: the vertices sit on the neighbouring lattice points
    assert np.all(np.abs(np.linalg.norm(v - 2.0, axis=1, ord=np.inf) - 1.0) < 1e-12)
    # the winding faces lower sigma, i.e. inward here: the inside region surrounds the surface
    assert mm.signed_volume(v, f) < 0


def test_fp32_order_matches_float64_closely():
    origin, step, X, Y, Z = grid(20)
    s = sphere(X, Y, Z, r=0.55).astype(np.float32)
    v64, f64 = mm.marching_tetrahedra(s, origin, step, 0.0)
    v32, f32 = mm.marching_tetrahedra(s, origin, step, 0.0, fp32=True)
    assert v32.dtype == np.float32 and np.array_equal(f64, f32)
    assert np.abs(v32 - v64).max() < 1e-6


def test_normals_point_outward_on_a_sphere():
    origin, step, X, Y, Z = grid(32)
    s = sphere(X, Y, Z, r=0.6)
    v, f = mm.marching_tetrahedra(s, origin, step, 0.0)
    n = mm.grid_normals(s, origin, step, v)
    radial = v / np.linalg.norm(v, axis=1, keepdims=True)
    assert np.abs(np.linalg.norm(n, axis=1) - 1).max() < 1e-12
    assert (np.einsum("ij,ij->i", n, radial) > 0.98).all()
