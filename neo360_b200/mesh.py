"""Coloured meshes of a trained field on the GPU: density grid, marching tetrahedra, normals and vertex colours.

    density_grid(net, R, ...)       sigma of one MLP of the model on an (R_z, R_y, R_x) lattice: each x-row is one ray of the model's
                                    field at caller-given points (`fp32` or `tc`), built on the device by neo_grid_rays
    marching_tetrahedra(sigma, iso) neo_mt_count + neo_mt_emit: a closed, outward-wound mesh of {sigma >= iso} (csrc/mesh.cu)
    grid_normals(sigma, verts)      neo_grid_normals: -grad sigma / |grad sigma| at the vertices
    vertex_colors(net, verts, n)    the rgb of each vertex seen from outside, along -normal (one sample per ray)
    extract_mesh(net, batch, ...)   all four: dict(verts, faces, normals, colors) on the device; output.write_ply writes it

Models and their field at (rays, t), the one step that differs between them:
    NeRF_TP       (NeO-360)      neo_field_eval of the foreground MLP: level 0 coarse, 1 fine (default); the scene from `batch` or set_scene
    vanilla.NeRF                 neo_vanilla_field_eval: level 0 coarse, 1 fine (default); no batch
    mip.MipNeRF360               neo_mip_field_eval: levels 0 and 1 are the proposal MLPs (density only: colours raise), 2 the NeRF MLP
                                 (default); no batch
    PixelNeRF                    PixelNeRF.field: level 0 coarse, 1 fine (default); `batch` is required (its src_* entries, as `forward`
                                 takes them)

Per-model rules:
  * NeO-360's foreground branch is an object-centric field inside the unit sphere: the reference samples it only there (helper.py:24-75,
    t in [0, far] of intersect_sphere), so its grid defines sigma = 0 at lattice points with |x| > 1 and the level set closes at the
    sphere.  The other models have no such sphere: their sigma is meshed as evaluated over the caller's `bbox` (default the unit cube).
  * Mip-NeRF 360's MLP reads a Gaussian, not a point.  At a lattice point the Gaussian has its mean at the point and covariance
    diag(var), by default var = h_a^2 / 12 per axis (h the lattice step): the second moment of the uniform distribution over one cell,
    so a coarser grid samples a prefiltered field, as the model itself does at a coarser footprint.  The vertex colours use the grid's var.
  * Every model's density head ignores the view direction (NeO-360 and PixelNeRF read the trunk's view mean; vanilla NeRF and Mip-NeRF 360
    branch the direction in after it), so the grid's direction (1, 0, 0) does not change sigma.
  * Slabs: NeO-360 evaluates 16384 rows per call by default.  For the other models `slab_rays=None` takes the most rows whose scratch
    (the field's workspace query plus the slab's rays, t and rgb) fits in SLAB_BUDGET bytes: Mip-NeRF 360's NeRF MLP needs about 7 kB
    (tc) to 12 kB (fp32) of workspace per point.
Meshing the NeO-360 background branch is not supported (DESIGN.md section 8).
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


SLAB_BUDGET = 2 << 30         # bytes of slab scratch for the models without a fixed slab size
NEO360_SLAB_RAYS = 16384


def _kind(net) -> str:
    from .mip import MipNeRF360
    from .pixelnerf import PixelNeRF
    from .renderer import NeRF_TP
    from .vanilla import NeRF
    for cls, kind in ((NeRF_TP, "neo360"), (NeRF, "vanilla"), (MipNeRF360, "mip360"), (PixelNeRF, "pixelnerf")):
        if isinstance(net, cls):
            return kind
    raise TypeError(f"meshing supports NeRF_TP, vanilla.NeRF, mip.MipNeRF360 and PixelNeRF, got {type(net).__name__}")


LEVELS = {"neo360": (0, 1), "vanilla": (0, 1), "pixelnerf": (0, 1), "mip360": (0, 1, 2)}


def _level(kind: str, level: Optional[int]) -> int:
    """The model's level; None = its last (NeO-360's fine foreground, vanilla / PixelNeRF fine, Mip-NeRF 360's NeRF MLP)."""
    if level is None:
        return LEVELS[kind][-1]
    if level not in LEVELS[kind]:
        raise ValueError(f"level must be one of {LEVELS[kind]} for this model, got {level}")
    return level


def _precision(net, precision):
    p = precision or getattr(net, "precision", "fp32")
    if p not in PRECISIONS:
        raise ValueError(f"precision must be one of {sorted(PRECISIONS)}, got {p!r}")
    return p


def _src_batch(kind: str, batch):
    if kind != "pixelnerf":
        return batch
    need = ("src_imgs", "src_poses", "src_focal", "src_c")
    if batch is None or any(k not in batch for k in need):
        raise ValueError(f"PixelNeRF needs `batch` with its source views: {need}")
    return {k: batch[k] for k in need}


def grid_var(g: L.NeoGrid):
    """Mip-NeRF 360's default per-axis variance of a lattice point's Gaussian: h_a^2 / 12, the second moment of one cell."""
    return tuple(float(g.step[a]) ** 2 / 12.0 for a in range(3))


def workspace_bytes(net, M: int, precision: str) -> int:
    """Bytes of workspace the field of a model other than NeO-360 takes for M points (its workspace query)."""
    kind, lib, P = _kind(net), L.load(), PRECISIONS[precision]
    if kind == "vanilla":
        return int(lib.neo_vanilla_field_workspace_bytes(M, P))
    if kind == "mip360":
        return int(lib.neo_mip_field_workspace_bytes(M, max(m.netwidth for m in net.mlps), P))
    if kind == "pixelnerf":
        return int(lib.neo_pixelnerf_tc_workspace_bytes(net.num_src_views, M)) if precision == "tc" else 0
    raise ValueError("NeO-360 slabs have a fixed size")


def slab_rows(net, nx: int, rows: int, precision: str, budget: Optional[int] = None) -> int:
    """The most grid rows (of nx points) per field call whose scratch fits in `budget` (default SLAB_BUDGET): the workspace query of
    rows * nx points plus the slab's rays (24 B per row), t and rgb (16 B per point).  At least one row; rows * nx stays below 2^31."""
    budget = SLAB_BUDGET if budget is None else budget
    cost = lambda r: workspace_bytes(net, r * nx, precision) + r * 24 + r * nx * 16
    lo, hi = 1, min(rows, ((1 << 31) - 1) // nx)
    while lo < hi:
        mid = (lo + hi + 1) // 2
        if cost(mid) <= budget:
            lo = mid
        else:
            hi = mid - 1
    return lo


def _field(net, kind: str, level: int, prec: str, batch, var):
    """f(rays, t) -> (rgb or None, sigma (n, N)): the model's field of `level` at the points of `rays` and t (n, N), in `prec`."""
    if kind == "neo360":
        def f(rays, t, chunk=0, want_rgb=True):
            far = torch.zeros(t.shape[0], device=t.device)          # only the background branch reads far
            rgb, sig = net.field_eval(rays, far, t, 2 * level, chunk=chunk, precision=prec)   # fg_coarse, fg_fine in the scene's MLP order
            return rgb, sig.reshape(t.shape)
    elif kind == "vanilla":
        def f(rays, t, chunk=0, want_rgb=True):
            return net.field(rays, t, level, precision=prec)
    elif kind == "mip360":
        def f(rays, t, chunk=0, want_rgb=True):
            if want_rgb and level < 2:
                raise ValueError(f"Mip-NeRF 360's proposal level {level} has no colour head")
            return net.field(rays, t, level, var, precision=prec, rgb=want_rgb)
    else:
        def f(rays, t, chunk=0, want_rgb=True):
            return net.field({**batch, **rays}, t, level, chunk=chunk or None, precision=prec)
    return f


def density_grid(net, resolution, bbox=UNIT_BOX, level: Optional[int] = None, precision: Optional[str] = None, slab_rays: Optional[int] = None,
                 batch: Optional[Dict[str, torch.Tensor]] = None, var=None) -> torch.Tensor:
    """sigma (R_z, R_y, R_x) of one MLP of `net` (NeRF_TP, vanilla.NeRF, mip.MipNeRF360 or PixelNeRF; `level` as in the module
    docstring, default the model's last) at the lattice points of make_grid(resolution, bbox).  `precision` "fp32" or "tc" (default: the
    module's).  Each x-row is a ray o = (x0, y_j, z_k), d = viewdirs = (1, 0, 0), t_i = i * step_x; `slab_rays` rows go through one field
    call, which bounds the scratch (default: 16384 for NeRF_TP, the SLAB_BUDGET rule for the others).
    NeRF_TP: sigma = 0 where x*x + y*y + z*z > 1; the scene comes from `batch` exactly as `forward` gets it (src_* with an encoder,
    explicit planes_* / latent) or from the last set_scene.  PixelNeRF: `batch` holds the source views (required).  Mip-NeRF 360: the
    Gaussians' per-axis variance `var` (default grid_var of the lattice)."""
    kind = _kind(net)
    prec = _precision(net, precision)
    level = _level(kind, level)
    batch = _src_batch(kind, batch)
    if slab_rays is not None and slab_rays < 1:
        raise ValueError("slab_rays must be positive")
    g = make_grid(resolution, bbox)
    if kind == "mip360" and var is None:
        var = grid_var(g)
    if kind == "neo360":
        net._ensure_scene(batch if batch is not None else {}, prec)
    dev = next(net.parameters()).device
    rows, nx = g.ny * g.nz, g.nx
    slab = min(slab_rays or (NEO360_SLAB_RAYS if kind == "neo360" else slab_rows(net, nx, rows, prec)), rows)
    field = _field(net, kind, level, prec, batch, var)
    sigma = torch.empty(g.nz, g.ny, nx, device=dev)
    flat = sigma.view(rows, nx)
    o = torch.empty(slab, 3, device=dev)
    d = torch.empty(slab, 3, device=dev)
    t = torch.empty(slab, nx, device=dev)
    lib = L.load()
    with L.on(dev) as s:
        for r0 in range(0, rows, slab):
            n = min(slab, rows - r0)
            L.check(lib.neo_grid_rays(C.byref(g), r0, n, L.ptr(o), L.ptr(d), L.ptr(t), s))
            out = flat[r0:r0 + n]
            _, sig = field({"rays_o": o[:n], "rays_d": d[:n], "viewdirs": d[:n]}, t[:n], want_rgb=False)
            out.copy_(sig)
            if kind == "neo360":
                L.check(lib.neo_grid_mask_sphere(C.byref(g), r0, n, L.ptr(out), s))
    return sigma


def marching_tetrahedra(sigma: torch.Tensor, iso: float, bbox=UNIT_BOX):
    """Mesh of {sigma >= iso} over the lattice of `sigma`'s shape on `bbox`: verts (V, 3) fp32 and faces (F, 3) int32 on the device,
    wound counter-clockwise seen from lower sigma.  Ordering and arithmetic: include/neo360_b200.h (neo_mt_count)."""
    g = _grid_of(sigma, bbox)
    sig = sigma.contiguous()
    lib = L.load()
    dev = sig.device
    ws = L.workspace(lib.neo_mt_workspace_bytes(C.byref(g)), dev)
    nv, nf = C.c_int(), C.c_int()
    with L.on(dev) as s:
        L.check(lib.neo_mt_count(L.ptr(sig), C.byref(g), float(iso), L.ptr(ws), ws.numel(), C.byref(nv), C.byref(nf), s))
        verts = torch.empty(nv.value, 3, device=dev)
        faces = torch.empty(nf.value, 3, dtype=torch.int32, device=dev)
        L.check(lib.neo_mt_emit(L.ptr(sig), C.byref(g), float(iso), L.ptr(ws), ws.numel(), L.ptr(verts) if nv.value else None, nv.value,
                                L.ptr(faces) if nf.value else None, nf.value, s))
    return verts, faces


def grid_normals(sigma: torch.Tensor, verts: torch.Tensor, bbox=UNIT_BOX) -> torch.Tensor:
    """(V, 3) unit -grad sigma at the vertices (central differences on the grid, trilinearly interpolated); 0 where the gradient is 0."""
    g = _grid_of(sigma, bbox)
    v = verts.contiguous().float()
    out = torch.empty_like(v)
    if v.shape[0]:
        with L.on(v) as s:
            L.check(L.load().neo_grid_normals(L.ptr(sigma.contiguous()), C.byref(g), L.ptr(v), v.shape[0], L.ptr(out), s))
    return out


def vertex_colors(net, verts: torch.Tensor, normals: torch.Tensor, level: Optional[int] = None, precision: Optional[str] = None,
                  batch: Optional[Dict[str, torch.Tensor]] = None, var=None) -> torch.Tensor:
    """(V, 3) rgb of `level` at each vertex, seen from outside: one ray per vertex with rays_o = the vertex, viewdirs = rays_d = -normal,
    one sample at t = 0.  NeO-360 takes all V rays in one call; the other models take them in calls of at most slab_rows(net, 1, V)
    rays, which bounds Mip-NeRF 360's workspace.  Each call's chunk is its own ray count B.  NeO-360 and PixelNeRF condition sample
    b*N + s of a chunk of B rays on ray (b*N + s) mod B (quirk Q1: field_fp32_kernel, field_tc_kernel, neo_pixelnerf_field(_tc)); with
    N = 1 that ray is the vertex itself, so every vertex is coloured along its own direction.  Vanilla NeRF and Mip-NeRF 360 condition
    on each ray's own direction anyway.  Mip-NeRF 360 needs `var` (extract_mesh passes the grid's); its proposal levels raise."""
    kind = _kind(net)
    prec = _precision(net, precision)
    level = _level(kind, level)
    batch = _src_batch(kind, batch)
    if kind == "mip360":
        if level < 2:
            raise ValueError(f"Mip-NeRF 360's proposal level {level} has no colour head")
        if var is None:
            raise ValueError("Mip-NeRF 360 vertex colours need the Gaussians' `var` (mesh.grid_var of the lattice)")
    V = verts.shape[0]
    if V == 0:
        return torch.empty(0, 3, device=verts.device)
    if kind == "neo360":
        net._ensure_scene(batch if batch is not None else {}, prec)
    vd = (-normals).contiguous().float()
    rays = {"rays_o": verts.contiguous().float(), "rays_d": vd, "viewdirs": vd}
    t = torch.zeros(V, 1, device=verts.device)
    field = _field(net, kind, level, prec, batch, var)
    step = V if kind == "neo360" else slab_rows(net, 1, V, prec)
    out = torch.empty(V, 3, device=verts.device)
    for i in range(0, V, step):
        n = min(step, V - i)
        rgb, _ = field({k: v[i:i + n] for k, v in rays.items()}, t[i:i + n], chunk=n)
        out[i:i + n] = rgb.reshape(n, 3)
    return out


@torch.no_grad()
def extract_mesh(net, batch: Optional[Dict[str, torch.Tensor]], resolution=256, *, iso: float, bbox=UNIT_BOX, level: Optional[int] = None,
                 precision: Optional[str] = None, colors: bool = True, var=None) -> Dict[str, torch.Tensor]:
    """Coloured mesh of {sigma >= iso} of one MLP of `net`: dict(verts (V,3) f32, faces (F,3) int32, normals (V,3) f32, colors (V,3)
    f32) on the device (colors only with colors=True).  `iso` has no default: it depends on the trained field.  Sigma, normals and
    colours all come from the MLP of `level` (default the model's last; see the module docstring for `batch` and `var`)."""
    if _kind(net) == "mip360" and var is None:
        var = grid_var(make_grid(resolution, bbox))
    sigma = density_grid(net, resolution, bbox, level, precision, batch=batch, var=var)
    verts, faces = marching_tetrahedra(sigma, iso, bbox)
    out = {"verts": verts, "faces": faces, "normals": grid_normals(sigma, verts, bbox)}
    if colors:
        out["colors"] = vertex_colors(net, verts, out["normals"], level, precision, batch, var)
    return out
