"""Stage-level operators with the reference's names and argument meaning, each a thin call into the C ABI
(include/neo360_b200.h).  They exist so the parity tests read like tests of the reference's helpers:

    intersect_sphere        models/neo360/helper.py:253-273
    sample_along_rays       models/neo360/helper.py:24-75
    sample_pdf              models/neo360/helper.py:218-249
    volumetric_rendering    models/neo360/helper.py:128-171
    get_rays                datasets/ray_utils.py:84-104,133-176 (differentiable w.r.t. c2w when it requires grad)
    sample_rays             datasets/nerds360_ae.py:730-748 (pixel sampling of a training batch; differentiable w.r.t. c2w likewise)
    index_grid / get_local_feats / field_eval   need a Scene (see renderer.py)

CUDA only; there is no CPU fallback."""
import torch

from . import _lib as L


def _stream():
    return torch.cuda.current_stream().cuda_stream


class _on:
    """Device guard: kernels and the stream handed to the library belong to the device of the call's tensors, not to whatever device
    happens to be current in the process (ADVICE round 1)."""

    def __init__(self, t):
        self.g = torch.cuda.device(t.device)

    def __enter__(self):
        self.g.__enter__()

    def __exit__(self, *e):
        return self.g.__exit__(*e)


def _f32(t):
    if not t.is_cuda:
        raise RuntimeError("neo360_b200 ops run on CUDA tensors only (no CPU fallback)")
    return t.contiguous().float()


class _RaysFromPoses(torch.autograd.Function):
    """neo_sample_rays under autograd w.r.t. c2w (T,3,4): the same kernel and the same bits forward, `neo_sample_rays_bwd` backward (a
    fixed-order reduction per view).  radii and target carry no gradient: radii does not change under a rotation of the pose or a
    translation, so a pose correction loses nothing by it."""

    @staticmethod
    def forward(ctx, c2w, pix, H, W, focal, img, check):
        lib = L.load()
        m = c2w.detach().contiguous().float()
        n, T = pix.numel(), m.shape[0]
        o = torch.empty(n, 3, device=m.device); vd = torch.empty_like(o); rd = torch.empty_like(o)
        rad = torch.empty(n, 1, device=m.device)
        tgt = torch.empty(n, 3, device=m.device) if img is not None else None
        err = torch.zeros(1, dtype=torch.int32, device=m.device)
        with _on(m):
            L.check(lib.neo_sample_rays(n, pix.data_ptr(), T, H, W, float(focal), L.ptr(m), L.ptr(img), L.ptr(o), L.ptr(vd), L.ptr(rd),
                                        L.ptr(rad), L.ptr(tgt), L.ptr(err), _stream()))
        if check and int(err.item()):   # the reference's fancy indexing raises IndexError synchronously
            raise IndexError("sample_rays: pix_inds out of range")
        ctx.save_for_backward(m, pix)
        ctx.dims = (H, W, float(focal))
        ctx.mark_non_differentiable(rad)
        if tgt is None:
            return o, vd, rd, rad
        ctx.mark_non_differentiable(tgt)
        return o, vd, rd, rad, tgt

    @staticmethod
    def backward(ctx, g_o, g_vd, g_rd, *_):
        lib = L.load()
        m, pix = ctx.saved_tensors
        H, W, focal = ctx.dims
        n, T = pix.numel(), m.shape[0]
        f = lambda g: None if g is None else g.contiguous().float()
        need = lib.neo_sample_rays_bwd_workspace_bytes(n, T)
        ws = torch.empty(max(need, 1), dtype=torch.uint8, device=m.device)
        g_c2w = torch.empty(T, 3, 4, device=m.device)
        with _on(m):
            L.check(lib.neo_sample_rays_bwd(n, pix.data_ptr(), T, H, W, focal, L.ptr(m), L.ptr(f(g_o)), L.ptr(f(g_vd)), L.ptr(f(g_rd)),
                                            L.ptr(g_c2w), L.ptr(ws), need, _stream()))
        return g_c2w, None, None, None, None, None, None


def _pose_grad(c2w) -> bool:
    return torch.is_grad_enabled() and c2w.requires_grad


def get_rays(H, W, focal, c2w, output_radii=True):
    """c2w (3,4) or (4,4) CUDA -> rays_o, viewdirs, rays_d, radii  (quirk Q3: rays_d == viewdirs, unit norm).  When c2w requires grad
    the rays are differentiable w.r.t. it (neo_sample_rays_bwd over the frame's pixels; the same bits forward); radii is not."""
    if _pose_grad(c2w):
        m = _f32(c2w[:3, :4])
        pix = torch.arange(H * W, dtype=torch.int64, device=m.device)
        o, vd, rd, rad = _RaysFromPoses.apply(m[None], pix, H, W, focal, None, False)
        return (o, vd, rd, rad.reshape(-1)) if output_radii else (o, vd, rd)
    lib = L.load()
    m = _f32(c2w[:3, :4])
    n = H * W
    o = torch.empty(n, 3, device=m.device); vd = torch.empty_like(o); rd = torch.empty_like(o)
    rad = torch.empty(n, device=m.device) if output_radii else None
    with _on(m):
        L.check(lib.neo_get_rays(H, W, float(focal), L.ptr(m), L.ptr(o), L.ptr(vd), L.ptr(rd), L.ptr(rad), _stream()))
    return (o, vd, rd, rad) if output_radii else (o, vd, rd)


def sample_rays(pix_inds, H, W, focal, c2w, images=None, check=True):
    """The `pix_inds`-selected rays of the (T, H, W) stack of target views (nerds360_ae.py:730-748) without building the stack.
    pix_inds (n) int64 CUDA, c2w (T,3,4) CUDA, images (T,H,W,3) fp32 CUDA or None -> rays_o, viewdirs, rays_d, radii (n,1), target.
    When c2w requires grad, rays_o, viewdirs and rays_d are differentiable w.r.t. it (neo_sample_rays_bwd; the same bits forward)."""
    lib = L.load()
    m = _f32(c2w[:, :3, :4])
    if not pix_inds.is_cuda or pix_inds.dtype != torch.int64:
        raise RuntimeError("sample_rays: pix_inds must be an int64 CUDA tensor")
    pix = pix_inds.contiguous()
    n, T = pix.numel(), m.shape[0]
    img = None
    if images is not None:
        img = _f32(images)
        if tuple(img.shape) != (T, H, W, 3):
            raise ValueError(f"sample_rays: images must be ({T}, {H}, {W}, 3), got {tuple(img.shape)}")
    if _pose_grad(c2w):
        out = _RaysFromPoses.apply(m, pix, H, W, focal, img, check)
        return out if img is not None else (*out, None)
    o = torch.empty(n, 3, device=m.device); vd = torch.empty_like(o); rd = torch.empty_like(o)
    rad = torch.empty(n, 1, device=m.device)
    tgt = torch.empty(n, 3, device=m.device) if img is not None else None
    err = torch.zeros(1, dtype=torch.int32, device=m.device)
    with _on(m):
        L.check(lib.neo_sample_rays(n, pix.data_ptr(), T, H, W, float(focal), L.ptr(m), L.ptr(img), L.ptr(o), L.ptr(vd), L.ptr(rd), L.ptr(rad),
                                    L.ptr(tgt), L.ptr(err), _stream()))
    if check and int(err.item()):   # the reference's fancy indexing raises IndexError synchronously
        raise IndexError("sample_rays: pix_inds out of range")
    return o, vd, rd, rad, tgt


def intersect_sphere(rays_o, rays_d):
    lib = L.load()
    o, d = _f32(rays_o), _f32(rays_d)
    n = o.shape[0]
    far = torch.empty(n, 1, device=o.device)
    err = torch.zeros(1, dtype=torch.int32, device=o.device)
    with _on(o):
        L.check(lib.neo_intersect_sphere(L.ptr(o), L.ptr(d), n, L.ptr(far), L.ptr(err), _stream()))
    if int(err.item()):   # the reference asserts synchronously here (helper.py:271)
        raise AssertionError("1.0 - p_norm_sq should be greater than 0")
    return far


def sample_along_rays(rays_o, rays_d, num_samples, near, far, randomized, lindisp, in_sphere, far_uncontracted=4.0,
                      u_rand=None):
    """`near` must be the reference's 1e-4 (model.py:277), lindisp False.  randomized draws torch.rand like helper.py:50
    unless u_rand (n, num_samples+1) is given."""
    assert not lindisp, "lindisp is not on the NeO-360 path (model.py:175 default False)"
    lib = L.load()
    o, d, fr = _f32(rays_o), _f32(rays_d), _f32(far).reshape(-1)
    n, N = o.shape[0], num_samples + 1
    if randomized and u_rand is None:
        u_rand = torch.rand((n, N), device=o.device)
    u = _f32(u_rand) if u_rand is not None else None
    t = torch.empty(n, N, device=o.device)
    if in_sphere:
        pts = torch.empty(n, N, 3, device=o.device)
        with _on(o):
            L.check(lib.neo_sample_along_rays(L.ptr(o), L.ptr(d), L.ptr(fr), n, num_samples, 1, float(far_uncontracted),
                                              L.ptr(u), L.ptr(t), L.ptr(pts), None, _stream()))
        return t, pts
    pts = torch.empty(n, N, 4, device=o.device)
    lin = torch.empty(n, N, 3, device=o.device)
    with _on(o):
        L.check(lib.neo_sample_along_rays(L.ptr(o), L.ptr(d), L.ptr(fr), n, num_samples, 0, float(far_uncontracted),
                                          L.ptr(u), L.ptr(t), L.ptr(pts), L.ptr(lin), _stream()))
    return t, pts, lin


def sample_pdf(t_vals, weights, origins, directions, num_samples, randomized, in_sphere, far, far_uncontracted=3.0,
               u_rand=None):
    """Takes the FULL previous t_vals (n,N) and weights (n,N): bins = mids(t_vals), weights[..., 1:-1] are formed
    inside, as NeRF_TP.forward does at model.py:308-331."""
    lib = L.load()
    o, d, fr = _f32(origins), _f32(directions), _f32(far).reshape(-1)
    t_old, w = _f32(t_vals), _f32(weights)
    n, n_old = t_old.shape
    N1 = n_old + num_samples
    if randomized and u_rand is None:
        u_rand = torch.rand((n, num_samples), device=o.device)
    u = _f32(u_rand) if u_rand is not None else None
    t = torch.empty(n, N1, device=o.device)
    if in_sphere:
        pts = torch.empty(n, N1, 3, device=o.device)
        with _on(o):
            L.check(lib.neo_sample_pdf(L.ptr(o), L.ptr(d), L.ptr(fr), L.ptr(t_old), L.ptr(w), n, n_old, num_samples, 1,
                                       float(far_uncontracted), L.ptr(u), L.ptr(t), L.ptr(pts), None, _stream()))
        return t, pts
    pts = torch.empty(n, N1, 4, device=o.device)
    lin = torch.empty(n, N1, 3, device=o.device)
    with _on(o):
        L.check(lib.neo_sample_pdf(L.ptr(o), L.ptr(d), L.ptr(fr), L.ptr(t_old), L.ptr(w), n, n_old, num_samples, 0,
                                   float(far_uncontracted), L.ptr(u), L.ptr(t), L.ptr(pts), L.ptr(lin), _stream()))
    return t, pts, lin


def volumetric_rendering(rgb, density, t_vals, dirs, white_bkgd, in_sphere, t_far=None, out_depth=None):
    lib = L.load()
    rgb, sig, t, d = _f32(rgb), _f32(density).reshape(density.shape[0], -1), _f32(t_vals), _f32(dirs)
    n, N = t.shape
    far = _f32(t_far).reshape(-1) if t_far is not None else None
    comp = torch.empty(n, 3, device=t.device); acc = torch.empty(n, device=t.device)
    w = torch.empty(n, N, device=t.device); depth = torch.empty(n, device=t.device)
    lam = torch.empty(n, 1, device=t.device) if in_sphere else None
    with _on(t):
        L.check(lib.neo_volumetric_rendering(L.ptr(rgb), L.ptr(sig), L.ptr(t), L.ptr(d), L.ptr(far), n, N, int(bool(white_bkgd)),
                                             int(bool(in_sphere)), L.ptr(comp), L.ptr(acc), L.ptr(w), L.ptr(lam), L.ptr(depth),
                                             _stream()))
    if out_depth is not None:
        return comp, acc, w, lam, depth
    return comp, acc, w, lam
