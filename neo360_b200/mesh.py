"""Coloured meshes of a NeO-360 scene's foreground: density grid, marching tetrahedra, normals and vertex colours, all on the GPU.

    density_grid(net, R, ...)       sigma of a foreground MLP on an (R_z, R_y, R_x) lattice: each x-row is one ray through
                                    neo_field_eval (`fp32` or `tc`), built on the device by neo_grid_rays; sigma = 0 outside the unit sphere
    marching_tetrahedra(sigma, iso) neo_mt_count + neo_mt_emit: a closed, outward-wound mesh of {sigma >= iso} (csrc/mesh.cu)
    grid_normals(sigma, verts)      neo_grid_normals: -grad sigma / |grad sigma| at the vertices
    vertex_colors(net, verts, n)    the foreground rgb of each vertex seen from outside, along -normal (neo_field_eval, one sample per ray)
    extract_mesh(net, batch, ...)   all four: dict(verts, faces, normals, colors) on the device; output.write_ply writes it

The foreground branch is an object-centric field inside the unit sphere: the reference samples it only there (helper.py:24-75, t in
[0, far] of intersect_sphere), so the grid defines sigma = 0 at lattice points with |x| > 1 and the level set closes at the sphere.
The density head reads only the trunk's view mean (models/neo360/model.py:110-158), so sigma does not depend on the view direction.
Meshing the background branch and PixelNeRF is not supported (DESIGN.md section 8).
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional

import torch

from . import _lib as L
from .renderer import PRECISIONS

UNIT_BOX = ((-1.0, -1.0, -1.0), (1.0, 1.0, 1.0))


def make_grid(resolution, bbox=UNIT_BOX) -> L.NeoGrid:
    """NeoGrid of `resolution` (R, or (R_z, R_y, R_x)) points spanning bbox = ((x0, y0, z0), (x1, y1, z1)), both corners included:
    step = (hi - lo) / (R - 1) per axis, rounded to fp32 like the origin."""
    rz, ry, rx = (resolution,) * 3 if isinstance(resolution, int) else tuple(int(r) for r in resolution)
    lo, hi = bbox
    g = L.NeoGrid()
    g.nx, g.ny, g.nz = rx, ry, rz
    for a, n in enumerate((rx, ry, rz)):
        if n < 2:
            raise ValueError(f"resolution needs at least 2 points per axis, got {resolution}")
        if not float(hi[a]) > float(lo[a]):
            raise ValueError(f"bbox must have lo < hi on every axis, got {bbox}")
        g.origin[a] = float(lo[a])
        g.step[a] = (float(hi[a]) - float(lo[a])) / (n - 1)
    return g


def _grid_of(sigma: torch.Tensor, bbox) -> L.NeoGrid:
    if sigma.dim() != 3 or sigma.dtype != torch.float32 or not sigma.is_cuda:
        raise ValueError("sigma must be an (R_z, R_y, R_x) fp32 CUDA tensor")
    return make_grid(tuple(sigma.shape), bbox)


def _precision(net, precision):
    p = precision or net.precision
    if p not in PRECISIONS:
        raise ValueError(f"precision must be one of {sorted(PRECISIONS)}, got {p!r}")
    return p


def _mlp_index(level: int) -> int:
    if level not in (0, 1):
        raise ValueError(f"level must be 0 (coarse) or 1 (fine), got {level}")
    return 2 * level            # fg_coarse, fg_fine in the scene's MLP order


def density_grid(net, resolution, bbox=UNIT_BOX, level: int = 1, precision: Optional[str] = None, slab_rays: int = 16384,
                 batch: Optional[Dict[str, torch.Tensor]] = None) -> torch.Tensor:
    """sigma (R_z, R_y, R_x) of the foreground MLP of `level` (0 coarse, 1 fine) at the lattice points of make_grid(resolution, bbox),
    0 where x*x + y*y + z*z > 1.  `precision` "fp32" or "tc" (default: the module's).  The scene comes from `batch` exactly as `forward`
    gets it (src_* with an encoder, explicit planes_* / latent) or from the last set_scene.  Each x-row is a ray o = (x0, y_j, z_k),
    d = viewdirs = (1, 0, 0), t_i = i * step_x; `slab_rays` rows go through one neo_field_eval call, which bounds the scratch."""
    prec = _precision(net, precision)
    mi = _mlp_index(level)
    if slab_rays < 1:
        raise ValueError("slab_rays must be positive")
    sc = net._ensure_scene(batch if batch is not None else {}, prec)
    g = make_grid(resolution, bbox)
    dev = next(net.fg_fine_mlp.parameters()).device
    rows, nx = g.ny * g.nz, g.nx
    slab = min(slab_rays, rows)
    sigma = torch.empty(g.nz, g.ny, nx, device=dev)
    flat = sigma.view(rows, nx)
    o = torch.empty(slab, 3, device=dev)
    d = torch.empty(slab, 3, device=dev)
    t = torch.empty(slab, nx, device=dev)
    far = torch.zeros(slab, device=dev)           # only the background branch reads far
    rgb = torch.empty(slab, nx, 3, device=dev)    # the field kernels always write colour; not part of the result
    lib = L.load()
    with torch.cuda.device(dev):
        s = torch.cuda.current_stream().cuda_stream
        for r0 in range(0, rows, slab):
            n = min(slab, rows - r0)
            L.check(lib.neo_grid_rays(C.byref(g), r0, n, L.ptr(o), L.ptr(d), L.ptr(t), s))
            r = L.NeoRays()
            r.n_rays, r.chunk = n, 0
            r.rays_o, r.rays_d, r.viewdirs = L.ptr(o), L.ptr(d), L.ptr(d)
            out = flat[r0:r0 + n]
            L.check(lib.neo_field_eval(sc.handle, C.byref(r), L.ptr(far), L.ptr(t), nx, mi, PRECISIONS[prec], L.ptr(rgb), L.ptr(out), s))
            L.check(lib.neo_grid_mask_sphere(C.byref(g), r0, n, L.ptr(out), s))
    return sigma


def marching_tetrahedra(sigma: torch.Tensor, iso: float, bbox=UNIT_BOX):
    """Mesh of {sigma >= iso} over the lattice of `sigma`'s shape on `bbox`: verts (V, 3) fp32 and faces (F, 3) int32 on the device,
    wound counter-clockwise seen from lower sigma.  Ordering and arithmetic: include/neo360_b200.h (neo_mt_count)."""
    g = _grid_of(sigma, bbox)
    sig = sigma.contiguous()
    lib = L.load()
    need = lib.neo_mt_workspace_bytes(C.byref(g))
    if need == 0:
        raise RuntimeError("neo360_b200: " + lib.neo_last_error().decode())
    dev = sig.device
    ws = torch.empty(need, dtype=torch.uint8, device=dev)
    nv, nf = C.c_int(), C.c_int()
    with torch.cuda.device(dev):
        s = torch.cuda.current_stream().cuda_stream
        L.check(lib.neo_mt_count(L.ptr(sig), C.byref(g), float(iso), L.ptr(ws), need, C.byref(nv), C.byref(nf), s))
        verts = torch.empty(nv.value, 3, device=dev)
        faces = torch.empty(nf.value, 3, dtype=torch.int32, device=dev)
        L.check(lib.neo_mt_emit(L.ptr(sig), C.byref(g), float(iso), L.ptr(ws), need, L.ptr(verts) if nv.value else None, nv.value,
                                L.ptr(faces) if nf.value else None, nf.value, s))
    return verts, faces


def grid_normals(sigma: torch.Tensor, verts: torch.Tensor, bbox=UNIT_BOX) -> torch.Tensor:
    """(V, 3) unit -grad sigma at the vertices (central differences on the grid, trilinearly interpolated); 0 where the gradient is 0."""
    g = _grid_of(sigma, bbox)
    v = verts.contiguous().float()
    out = torch.empty_like(v)
    if v.shape[0]:
        with torch.cuda.device(v.device):
            L.check(L.load().neo_grid_normals(L.ptr(sigma.contiguous()), C.byref(g), L.ptr(v), v.shape[0], L.ptr(out),
                                              torch.cuda.current_stream().cuda_stream))
    return out


def vertex_colors(net, verts: torch.Tensor, normals: torch.Tensor, level: int = 1, precision: Optional[str] = None,
                  batch: Optional[Dict[str, torch.Tensor]] = None) -> torch.Tensor:
    """(V, 3) foreground rgb of `level` at each vertex, seen from outside: one ray per vertex with rays_o = the vertex,
    viewdirs = rays_d = -normal, one sample at t = 0.  With N = 1 sample and chunk = V, the quirk-Q1 conditioning ray (b*N + s) mod B
    of field_fp32_kernel and field_tc_kernel (whose direction record dir_frag_kernel builds from viewdirs[src]) is the vertex itself,
    so every vertex is coloured along its own direction."""
    prec = _precision(net, precision)
    mi = _mlp_index(level)
    V = verts.shape[0]
    if V == 0:
        return torch.empty(0, 3, device=verts.device)
    net._ensure_scene(batch if batch is not None else {}, prec)
    vd = (-normals).contiguous().float()
    rays = {"rays_o": verts.contiguous().float(), "rays_d": vd, "viewdirs": vd}
    far = torch.zeros(V, device=verts.device)
    t = torch.zeros(V, 1, device=verts.device)
    rgb, _ = net.field_eval(rays, far, t, mi, chunk=V, precision=prec)
    return rgb.reshape(V, 3)


@torch.no_grad()
def extract_mesh(net, batch: Optional[Dict[str, torch.Tensor]], resolution=256, *, iso: float, bbox=UNIT_BOX, level: int = 1,
                 precision: Optional[str] = None, colors: bool = True) -> Dict[str, torch.Tensor]:
    """Coloured mesh of the foreground's {sigma >= iso}: dict(verts (V,3) f32, faces (F,3) int32, normals (V,3) f32, colors (V,3) f32)
    on the device (colors only with colors=True).  `iso` has no default: it depends on the trained field.  Sigma, normals and colours
    all come from the foreground MLP of `level`."""
    sigma = density_grid(net, resolution, bbox, level, precision, batch=batch)
    verts, faces = marching_tetrahedra(sigma, iso, bbox)
    out = {"verts": verts, "faces": faces, "normals": grid_normals(sigma, verts, bbox)}
    if colors:
        out["colors"] = vertex_colors(net, verts, out["normals"], level, precision, batch)
    return out
