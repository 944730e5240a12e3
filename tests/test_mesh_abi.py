"""CPU: the geometry-export entry points (csrc/mesh.cu) reject bad arguments before any launch, the host grid and PLY logic."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from neo360_b200 import build, _lib
    build.build()
    return _lib.load()


def grid(nx=4, ny=5, nz=6, step=0.5):
    from neo360_b200 import _lib as L
    g = L.NeoGrid()
    g.nx, g.ny, g.nz = nx, ny, nz
    for a in range(3):
        g.origin[a] = -1.0
        g.step[a] = step
    return g


def test_grid_struct_layout_matches_header():
    from neo360_b200 import _lib as L
    src = ('#include <stdio.h>\n#include <stddef.h>\n#include "neo360_b200.h"\n'
           'int main(){printf("%zu %zu %zu\\n", sizeof(NeoGrid), offsetof(NeoGrid, origin), offsetof(NeoGrid, step));return 0;}\n')
    with tempfile.TemporaryDirectory() as td:
        open(os.path.join(td, "s.c"), "w").write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), os.path.join(td, "s.c"), "-o", os.path.join(td, "s")])
        got = [int(x) for x in subprocess.check_output([os.path.join(td, "s")]).split()]
    assert got == [C.sizeof(L.NeoGrid), L.NeoGrid.origin.offset, L.NeoGrid.step.offset]


def test_workspace_bytes_validates_the_grid(lib):
    g = grid()
    assert lib.neo_mt_workspace_bytes(C.byref(g)) >= 4 * 5 * 6 * 5
    for bad in (grid(nx=1), grid(nz=0), grid(step=0.0), grid(step=-0.1), grid(step=float("inf")), grid(1024, 1024, 512)):
        assert lib.neo_mt_workspace_bytes(C.byref(bad)) == 0
    assert lib.neo_mt_workspace_bytes(None) == 0
    g.origin[1] = float("nan")
    assert lib.neo_mt_workspace_bytes(C.byref(g)) == 0 and b"origin" in lib.neo_last_error()


def test_entry_points_reject_bad_arguments_without_gpu(lib):
    """The pointers are never dereferenced: every call fails validation before a launch."""
    p = 1 << 20
    g = grid()
    ws = lib.neo_mt_workspace_bytes(C.byref(g))
    nv, nf = C.c_int(), C.c_int()
    assert lib.neo_mt_count(None, C.byref(g), 0.0, p, ws, C.byref(nv), C.byref(nf), None) == -1              # sigma
    assert lib.neo_mt_count(p, C.byref(g), 0.0, None, ws, C.byref(nv), C.byref(nf), None) == -1              # workspace
    assert lib.neo_mt_count(p, C.byref(g), 0.0, p + 16, ws, C.byref(nv), C.byref(nf), None) == -1            # alignment
    assert lib.neo_mt_count(p, C.byref(g), float("nan"), p, ws, C.byref(nv), C.byref(nf), None) == -1        # iso
    assert lib.neo_mt_count(p, C.byref(g), 0.0, p, ws, None, C.byref(nf), None) == -1                        # n_verts
    assert lib.neo_mt_count(p, C.byref(g), 0.0, p, ws - 1, C.byref(nv), C.byref(nf), None) == -3             # workspace size
    assert lib.neo_mt_count(p, C.byref(grid(nx=1)), 0.0, p, ws, C.byref(nv), C.byref(nf), None) == -1
    assert lib.neo_mt_emit(p, C.byref(g), 0.0, p, ws, None, 3, p, 1, None) == -1                             # NULL verts, V > 0
    assert lib.neo_mt_emit(p, C.byref(g), 0.0, p, ws, p, 3, None, 1, None) == -1                             # NULL faces, F > 0
    assert lib.neo_mt_emit(p, C.byref(g), 0.0, p, ws, p, -1, p, 1, None) == -1
    assert lib.neo_grid_normals(p, C.byref(g), None, 4, p, None) == -1
    assert lib.neo_grid_normals(p, C.byref(g), p, -1, p, None) == -1
    assert lib.neo_grid_normals(None, C.byref(g), None, 0, None, None) == 0                                  # nothing to do
    assert lib.neo_grid_rays(C.byref(g), 0, 31, p, p, p, None) == -1                                        # 5 * 6 = 30 rows
    assert lib.neo_grid_rays(C.byref(g), -1, 2, p, p, p, None) == -1
    assert lib.neo_grid_rays(C.byref(g), 0, 4, p, None, p, None) == -1
    assert lib.neo_grid_mask_sphere(C.byref(g), 29, 2, p, None) == -1
    assert lib.neo_grid_mask_sphere(C.byref(g), 0, 0, p, None) == -1
    assert b"neo_grid_mask_sphere" in lib.neo_last_error()


def test_make_grid_spans_the_box():
    from neo360_b200 import mesh
    g = mesh.make_grid((5, 9, 17), ((-1.0, -0.5, 0.0), (1.0, 0.5, 2.0)))
    assert (g.nx, g.ny, g.nz) == (17, 9, 5)
    assert list(g.origin) == [-1.0, -0.5, 0.0]
    assert list(g.step) == [np.float32(2.0 / 16), np.float32(1.0 / 8), np.float32(2.0 / 4)]
    assert mesh.make_grid(3).nx == 3
    with pytest.raises(ValueError):
        mesh.make_grid(1)
    with pytest.raises(ValueError):
        mesh.make_grid(8, ((0, 0, 0), (1, 0, 1)))


@pytest.mark.parametrize("with_attrs", [True, False])
def test_write_ply_round_trip(tmp_path, with_attrs):
    from neo360_b200 import output
    from oracle import mesh_model as mm
    g = torch.Generator().manual_seed(0)
    m = {"verts": torch.randn(50, 3, generator=g), "faces": torch.randint(0, 50, (70, 3), generator=g, dtype=torch.int32)}
    if with_attrs:
        m["normals"] = torch.randn(50, 3, generator=g)
        m["colors"] = torch.rand(50, 3, generator=g) * 1.2 - 0.1
    vert, faces = mm.read_ply(output.write_ply(str(tmp_path / "m.ply"), m))
    assert np.array_equal(np.stack([vert["x"], vert["y"], vert["z"]], -1), m["verts"].numpy())
    assert np.array_equal(faces, m["faces"].numpy())
    if with_attrs:
        assert np.array_equal(np.stack([vert["nx"], vert["ny"], vert["nz"]], -1), m["normals"].numpy())
        c = np.stack([vert["red"], vert["green"], vert["blue"]], -1)
        assert np.array_equal(c, np.rint(np.clip(m["colors"].numpy(), 0, 1) * 255).astype(np.uint8))
    else:
        assert vert.dtype.names == ("x", "y", "z")
