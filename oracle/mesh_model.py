"""NumPy model of the geometry export in csrc/mesh.cu: marching tetrahedra on the Kuhn subdivision and the grid normals.

The same subdivision, edge ownership, tie rule (inside means sigma >= iso) and output order as the CUDA kernels, written as whole-array
NumPy.  `marching_tetrahedra(..., fp32=False)` places the vertices in float64; `fp32=True` repeats the kernels' fp32 operation order
(lattice x = origin + i * step, w = (iso - s_a) / (s_b - s_a), x = p_a + w * (p_b - p_a), each operation rounded to nearest), so its
vertices equal the kernels' bit for bit.  Grids are (nz, ny, nx) arrays with x fastest; origin and step are (x, y, z).
"""
from __future__ import annotations

import numpy as np

# owned edge types of a lattice point, as corner codes dx | dy << 1 | dz << 2
EDGE_CODES = (1, 2, 4, 3, 5, 6, 7)
TYPE_OF_CODE = {c: t for t, c in enumerate(EDGE_CODES)}
# the 6 Kuhn tetrahedra of a cell, each in positive orientation
TETS = ((0, 1, 3, 7), (1, 0, 5, 7), (2, 0, 3, 7), (0, 2, 6, 7), (0, 4, 5, 7), (4, 0, 6, 7))


def corner(c: int):
    """(dx, dy, dz) of corner code c."""
    return c & 1, (c >> 1) & 1, (c >> 2) & 1


def _odd(q) -> bool:
    return sum(q[a] > q[b] for a in range(4) for b in range(a + 1, 4)) % 2 == 1


def tet_triangles(m: int):
    """Triangles of a tetrahedron whose local corners with bit l of m set are inside: a list of triangles, each three (a, b) pairs of
    local corners whose edge carries the vertex.  Wound counter-clockwise seen from the outside corners."""
    n = bin(m).count("1")
    if n in (0, 4):
        return []
    if n == 2:
        ins = [c for c in range(4) if (m >> c) & 1]
        out = [c for c in range(4) if not (m >> c) & 1]
        q = ins + out
        if _odd(q):
            q[2], q[3] = q[3], q[2]
        i0, i1, o0, o1 = q
        return [((i0, o0), (i0, o1), (i1, o1)), ((i0, o0), (i1, o1), (i1, o0))]
    lone = [c for c in range(4) if ((m >> c) & 1) == (n == 1)][0]
    q = [lone] + [c for c in range(4) if c != lone]
    if _odd(q):
        q[2], q[3] = q[3], q[2]
    a, j, k, l = q
    return [((a, j), (a, k), (a, l))] if n == 1 else [((a, j), (a, l), (a, k))]


def _edge_ref(tet, pair):
    """(lower corner code, owned edge type) of the edge between two local corners of a tetrahedron."""
    c0, c1 = TETS[tet][pair[0]], TETS[tet][pair[1]]
    lo = c0 if (c0 & c1) == c0 else c1
    assert (c0 & c1) in (c0, c1)
    return lo, TYPE_OF_CODE[c0 ^ c1]


def lattice(origin, step, n: int, axis: int, fp32: bool) -> np.ndarray:
    if fp32:
        return np.float32(origin[axis]) + np.arange(n, dtype=np.float32) * np.float32(step[axis])
    return float(np.float32(origin[axis])) + np.arange(n, dtype=np.float64) * float(np.float32(step[axis]))


def marching_tetrahedra(sigma: np.ndarray, origin, step, iso: float, fp32: bool = False):
    """sigma (nz, ny, nx) -> verts (V, 3) float64 (float32 with fp32=True), faces (F, 3) int64."""
    sig = np.asarray(sigma, dtype=np.float32)
    nz, ny, nx = sig.shape
    iso32 = np.float32(iso)
    inside = sig >= iso32
    P = sig.size
    # ---- vertices: owned edges whose end points straddle iso, in (point, type) order ----
    mask = np.zeros((nz, ny, nx, 7), dtype=bool)
    for t, c in enumerate(EDGE_CODES):
        dx, dy, dz = corner(c)
        a = inside[:nz - dz, :ny - dy, :nx - dx]
        b = inside[dz:, dy:, dx:]
        mask[:nz - dz, :ny - dy, :nx - dx, t] = a != b
    mask = mask.reshape(P, 7)
    vid = np.full((P, 7), -1, dtype=np.int64)
    vid[mask] = np.arange(int(mask.sum()))
    p, t = np.nonzero(mask)
    codes = np.asarray(EDGE_CODES)[t]
    i, j, k = p % nx, (p // nx) % ny, p // (nx * ny)
    di, dj, dk = codes & 1, (codes >> 1) & 1, (codes >> 2) & 1
    flat = sig.reshape(-1)
    sa = flat[p]
    sb = flat[p + dk * nx * ny + dj * nx + di]
    X = [lattice(origin, step, n, ax, fp32) for ax, n in enumerate((nx, ny, nz))]
    pa = [X[0][i], X[1][j], X[2][k]]
    pb = [X[0][i + di], X[1][j + dj], X[2][k + dk]]
    if fp32:
        w = (iso32 - sa) / (sb - sa)
    else:
        w = (float(iso32) - sa.astype(np.float64)) / (sb.astype(np.float64) - sa.astype(np.float64))
    verts = np.stack([pa[a] + w * (pb[a] - pa[a]) for a in range(3)], -1)
    # ---- faces: cells in point order, then tetrahedron, then triangle ----
    bits = np.zeros((nz - 1, ny - 1, nx - 1), dtype=np.int64)
    for c in range(8):
        dx, dy, dz = corner(c)
        bits |= inside[dz:nz - 1 + dz, dy:ny - 1 + dy, dx:nx - 1 + dx].astype(np.int64) << c
    kk, jj, ii = np.meshgrid(np.arange(nz - 1), np.arange(ny - 1), np.arange(nx - 1), indexing="ij")
    pcell = ((kk * ny + jj) * nx + ii).reshape(-1)
    bits = bits.reshape(-1)
    out = np.full((pcell.size, 6, 2, 3), -1, dtype=np.int64)
    for tet in range(6):
        m = np.zeros_like(bits)
        for l, c in enumerate(TETS[tet]):
            m |= ((bits >> c) & 1) << l
        for mm in range(16):
            sel = np.nonzero(m == mm)[0]
            if sel.size == 0:
                continue
            for s, tri in enumerate(tet_triangles(mm)):
                for b, pair in enumerate(tri):
                    lo, ty = _edge_ref(tet, pair)
                    dx, dy, dz = corner(lo)
                    out[sel, tet, s, b] = vid[pcell[sel] + dz * nx * ny + dy * nx + dx, ty]
    out = out.reshape(-1, 3)
    faces = out[out[:, 0] >= 0]
    assert (faces >= 0).all()
    return verts, faces


def grid_normals(sigma: np.ndarray, origin, step, verts: np.ndarray) -> np.ndarray:
    """-grad sigma / |grad sigma| at each vertex, float64: central differences at the lattice points (one-sided on the faces),
    trilinearly interpolated in the (clamped) cell that holds the vertex."""
    sig = np.asarray(sigma, dtype=np.float64)
    nz, ny, nx = sig.shape
    o = np.asarray([float(np.float32(x)) for x in origin])
    h = np.asarray([float(np.float32(x)) for x in step])
    gz, gy, gx = np.gradient(sig, h[2], h[1], h[0])
    G = np.stack([gx, gy, gz], -1)
    v = np.asarray(verts, dtype=np.float64)
    u = (v - o) / h
    n = np.asarray([nx, ny, nz])
    c0 = np.clip(np.floor(u).astype(np.int64), 0, n - 2)
    f = np.clip(u - c0, 0.0, 1.0)
    g = np.zeros_like(v)
    for c in range(8):
        dx, dy, dz = corner(c)
        w = (f[:, 0] if dx else 1 - f[:, 0]) * (f[:, 1] if dy else 1 - f[:, 1]) * (f[:, 2] if dz else 1 - f[:, 2])
        g += w[:, None] * G[c0[:, 2] + dz, c0[:, 1] + dy, c0[:, 0] + dx]
    ln = np.linalg.norm(g, axis=-1, keepdims=True)
    return np.where(ln > 0, -g / np.where(ln > 0, ln, 1.0), 0.0)


# ---- mesh properties the tests check ----

def edge_face_counts(faces: np.ndarray):
    """(undirected edge -> number of faces, directed edge -> number of faces)."""
    f = np.asarray(faces, dtype=np.int64)
    d = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    und = np.sort(d, axis=1)
    _, cu = np.unique(und, axis=0, return_counts=True)
    _, cd = np.unique(d, axis=0, return_counts=True)
    return cu, cd


def euler_characteristic(faces: np.ndarray) -> int:
    f = np.asarray(faces, dtype=np.int64)
    cu, _ = edge_face_counts(f)
    return int(np.unique(f).size) - int(cu.size) + int(f.shape[0])


def components(faces: np.ndarray) -> int:
    """Connected components of the faces (shared vertex ids)."""
    f = np.asarray(faces, dtype=np.int64)
    parent = np.arange(int(f.max()) + 1 if f.size else 0)

    def find(x):
        while parent[x] != x:
            parent[x] = parent[parent[x]]
            x = parent[x]
        return x

    for a, b in np.concatenate([f[:, [0, 1]], f[:, [1, 2]]]):
        ra, rb = find(a), find(b)
        if ra != rb:
            parent[ra] = rb
    return len({find(x) for x in np.unique(f)})


def signed_volume(verts: np.ndarray, faces: np.ndarray) -> float:
    v = np.asarray(verts, dtype=np.float64)[np.asarray(faces)]
    return float(np.einsum("ij,ij->i", v[:, 0], np.cross(v[:, 1], v[:, 2])).sum() / 6.0)


def read_ply(path: str):
    """Reads what neo360_b200.output.write_ply writes: (vertex record array, faces (F, 3) int32)."""
    with open(path, "rb") as fh:
        lines = []
        while not lines or lines[-1] != "end_header":
            lines.append(fh.readline().decode("ascii").rstrip("\n"))
        body = fh.read()
    assert lines[0] == "ply" and lines[1] == "format binary_little_endian 1.0"
    types = {"float": "<f4", "uchar": "u1"}
    n_v = n_f = 0
    fields = []
    for ln in lines[2:]:
        w = ln.split()
        if w[:2] == ["element", "vertex"]:
            n_v = int(w[2])
        elif w[:2] == ["element", "face"]:
            n_f = int(w[2])
        elif w[0] == "property" and w[1] != "list":
            fields.append((w[2], types[w[1]]))
    vdt = np.dtype(fields)
    vert = np.frombuffer(body, dtype=vdt, count=n_v)
    face = np.frombuffer(body, dtype=[("n", "u1"), ("i", "<i4", (3,))], count=n_f, offset=n_v * vdt.itemsize)
    assert (face["n"] == 3).all() and len(body) == n_v * vdt.itemsize + n_f * 13
    return vert, face["i"].copy()
