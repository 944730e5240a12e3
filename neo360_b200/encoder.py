"""Tri-plane builder of NeO-360 (`GridEncoder`, SURVEY.md section 8(f1)) behind the reference's own module surface.

    reference                                                     here
    ---------------------------------------------------------     ----------------------------------------------------------------
    models/neo360/encoder_pn.py:13-210   SpatialEncoder            SpatialEncoder: same sub-module names (torchvision ResNet-34 trunk, host
                                                                   framework convolutions), `.latent` / `.latent_scaling` as the renderer reads them
    encoder_tp_fusion_conv.py:262-470    GridEncoder.__init__      GridEncoder.__init__: same sub-modules in the same construction order
                                                                   (state dicts and seeded initialisations are interchangeable)
    encoder_tp_fusion_conv.py:472-597    GridEncoder.forward       forward(): ResNet features and the three floor-plan conv stacks stay in the
                                                                   host framework; everything between them -- 64^3 x NV grid lookup,
                                                                   DepthPillarEncoder, three pillar aggregators, softmax-weighted pillar sums
                                                                   (2.7 TFLOP per scene) -- runs in hand-written CUDA on the tensor cores
                                                                   (`neo_grid_encoder_dense`, csrc/encoder.cu + csrc/gemm_tc.cu) when no
                                                                   gradient is required.  Under autograd on CUDA tensors (`dense_train`) the
                                                                   grid lookup and the softmax pillar sums run forward and backward in
                                                                   hand-written fp32 CUDA (`neo_grid_encoder_features(_bwd)`,
                                                                   `neo_grid_encoder_pool(_bwd)`) and the dense layers as framework fp32
                                                                   GEMMs; with `train_precision="tc"` the whole dense part trains on the
                                                                   tensor cores instead (`dense_train_tc`: bf16 operands, fp32
                                                                   accumulation, `_DenseTC`); under autograd on the CPU the same algebra
                                                                   runs as framework ops (`dense_torch`).
"""
from __future__ import annotations

import ctypes as C
import functools
import math

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _lib as L
from . import bf16
from .training import check_train_precision


def _init_linear_kaiming(m):
    """encoder_tp_fusion_conv.py:258-263"""
    if type(m) == nn.Linear:
        nn.init.kaiming_normal_(m.weight)
        nn.init.uniform_(m.bias, -1e-3, 1e-3)


class _ResNet34Trunk(nn.Module):
    """encoder_pn.py:13-30: the first three stages of torchvision's ResNet-34 (the full net is built first so that a seeded
    construction consumes the generator exactly like the reference)."""

    def __init__(self):
        super().__init__()
        import torchvision
        norm = functools.partial(nn.BatchNorm2d, affine=True, track_running_stats=True)
        net = torchvision.models.resnet34(weights=None, norm_layer=norm)
        self.conv1, self.bn1, self.relu, self.maxpool = net.conv1, net.bn1, net.relu, net.maxpool
        self.layer1, self.layer2, self.layer3 = net.layer1, net.layer2, net.layer3


class _UpsampleBilinear(torch.autograd.Function):
    """F.interpolate(x, size, mode="bilinear", align_corners=True) with the gather adjoint neo_upsample_bilinear_bwd as its backward (every
    input element written once, no atomics).  The forward is F.interpolate itself, so values are bit-identical."""

    @staticmethod
    def forward(ctx, x, size):
        ctx.in_shape = x.shape
        return F.interpolate(x, size, mode="bilinear", align_corners=True)

    @staticmethod
    def backward(ctx, g):
        lib = L.load()
        n, c, hi, wi = ctx.in_shape
        gc = g.contiguous().float()
        g_in = torch.empty(ctx.in_shape, device=gc.device)
        with L.on(gc) as s:
            L.check(lib.neo_upsample_bilinear_bwd(L.ptr(gc), n * c, hi, wi, gc.shape[-2], gc.shape[-1], L.ptr(g_in), s))
        return g_in, None


def upsample_bilinear(x, size):
    """F.interpolate(x, size, mode="bilinear", align_corners=True).  Under torch.use_deterministic_algorithms, where the framework's backward
    of this op raises, a CUDA input that needs a gradient goes through `_UpsampleBilinear`."""
    if torch.are_deterministic_algorithms_enabled() and x.is_cuda and torch.is_grad_enabled() and x.requires_grad:
        return _UpsampleBilinear.apply(x, tuple(int(v) for v in size))
    return F.interpolate(x, size, mode="bilinear", align_corners=True)


class _Upsample(nn.Upsample):
    """nn.Upsample(mode="bilinear", align_corners=True) that differentiates through `upsample_bilinear` (no parameters or buffers, so the
    state dict is nn.Upsample's)."""

    def forward(self, x):
        if torch.are_deterministic_algorithms_enabled() and x.is_cuda and torch.is_grad_enabled() and x.requires_grad:
            if self.size is not None:
                size = self.size
            else:
                size = [int(math.floor(d * self.scale_factor)) for d in x.shape[-2:]]
            return upsample_bilinear(x, size)
        return super().forward(x)


class SpatialEncoder(nn.Module):
    """encoder_pn.py:32-210 with the reference's defaults as GridEncoder passes them (resnet34, 4 layers, bilinear, zeros padding)."""

    def __init__(self):
        super().__init__()
        self.model = _ResNet34Trunk()
        self.latent_size = 512
        self.register_buffer("latent", torch.empty(1, 1, 1, 1), persistent=False)
        self.register_buffer("latent_scaling", torch.empty(2, dtype=torch.float32), persistent=False)

    def forward(self, x):
        x = self.model.relu(self.model.bn1(self.model.conv1(x)))
        feats = [x]
        x = self.model.layer1(self.model.maxpool(x))
        feats.append(x)
        x = self.model.layer2(x)
        feats.append(x)
        x = self.model.layer3(x)
        feats.append(x)
        size = feats[0].shape[-2:]
        self.latent = torch.cat([upsample_bilinear(f, size) for f in feats], 1)
        ls = torch.tensor([self.latent.shape[-1], self.latent.shape[-2]], dtype=torch.float32, device=self.latent.device)
        self.latent_scaling = ls / (ls - 1) * 2.0
        return self.latent


class DepthPillarEncoder(nn.Module):
    """encoder_tp_fusion_conv.py:234-250"""

    def __init__(self, inp_ch, LS):
        super().__init__()
        self.common_branch = nn.Sequential(nn.Linear(inp_ch, LS), nn.ReLU(inplace=True), nn.Linear(LS, LS), nn.ReLU(inplace=True))
        self.depth_encoder = nn.Linear(LS, LS)
        self.common_branch.apply(_init_linear_kaiming)
        self.depth_encoder.apply(_init_linear_kaiming)

    def forward(self, x):
        return self.depth_encoder(self.common_branch(x))


def _floorplan_convnet():
    """encoder_tp_fusion_conv.py:372-398 (identical for xy / yz / xz): 512 -> 256 (s2) -> 128 (s2) -> 128 -> up x2 -> 128 -> up (120,160) -> 128."""
    return nn.Sequential(
        nn.Conv2d(512, 256, 3, stride=2, padding=1), nn.BatchNorm2d(256), nn.ReLU(inplace=True),
        nn.Conv2d(256, 128, 3, stride=2, padding=1), nn.BatchNorm2d(128), nn.ReLU(inplace=True),
        nn.Conv2d(128, 128, 3, stride=1, padding=1), nn.BatchNorm2d(128), nn.ReLU(inplace=True),
        _Upsample(scale_factor=2, mode="bilinear", align_corners=True),
        nn.Conv2d(128, 128, 3, padding=1), nn.BatchNorm2d(128), nn.ReLU(inplace=True),
        _Upsample(size=(120, 160), mode="bilinear", align_corners=True),
        nn.Conv2d(128, 128, 3, padding=1))


class _Features(torch.autograd.Function):
    """Grid lookup rows: latent_cl (NV,Hl,Wl,512) channel-last -> X (NV*G^3, 518) = [latent lookup | cam xyz | masked unit direction], the
    input of depth_fc.  Returned as a view of a 520-wide buffer (16-byte rows); the gradient flows to the latent only (poses do not train)."""

    @staticmethod
    def forward(ctx, latent_cl, poses, focal, cx, cy, W, H):
        lib = L.load()
        lat = latent_cl.detach().contiguous().float()
        nv, lh, lw, _ = lat.shape
        pose_c = poses.detach().contiguous().float()
        X = torch.empty(nv * GridEncoder.GRID ** 3, 520, device=lat.device)
        geo = (nv, lh, lw, int(W), int(H))
        with L.on(lat) as s:
            L.check(lib.neo_grid_encoder_features(L.ptr(lat), *geo, L.ptr(pose_c), focal, cx, cy, L.ptr(X), X.shape[1], s))
        ctx.save_for_backward(pose_c)
        ctx.geo, ctx.cam = geo, (focal, cx, cy)
        ctx.det = torch.are_deterministic_algorithms_enabled()
        return X[:, :518]

    @staticmethod
    def backward(ctx, g_X):
        (pose_c,) = ctx.saved_tensors
        return _lookup_bwd(ctx, pose_c, g_X.contiguous().float()), None, None, None, None, None, None


class _Pool(torch.autograd.Function):
    """Softmax pillar sums: lat (NV*G^3, 512), logits (3, NV*G^3) by axis (yz, xz, xy) -> floor plans xz, xy, yz (NV,512,G,G)."""

    @staticmethod
    def forward(ctx, lat, logits):
        lib = L.load()
        lat_c, lg = lat.detach().contiguous().float(), logits.detach().contiguous().float()
        G = GridEncoder.GRID
        nv = lat_c.shape[0] // G ** 3
        out = [torch.empty(nv, 512, G, G, device=lat_c.device) for _ in range(3)]
        with L.on(lat_c) as s:
            L.check(lib.neo_grid_encoder_pool(L.ptr(lat_c), L.ptr(lg), nv, *[L.ptr(t) for t in out], s))
        ctx.save_for_backward(lat_c, lg)
        return tuple(out)

    @staticmethod
    def backward(ctx, g_xz, g_xy, g_yz):
        lib = L.load()
        lat_c, lg = ctx.saved_tensors
        nv = lat_c.shape[0] // GridEncoder.GRID ** 3
        d_lat, d_logits = torch.empty_like(lat_c), torch.empty_like(lg)
        gs = [None if g is None else g.contiguous().float() for g in (g_xz, g_xy, g_yz)]
        with L.on(lat_c) as s:
            L.check(lib.neo_grid_encoder_pool_bwd(L.ptr(lat_c), L.ptr(lg), nv, *[L.ptr(g) for g in gs], L.ptr(d_lat), L.ptr(d_logits), s))
        return d_lat, d_logits


class _DenseTC(torch.autograd.Function):
    """The dense part of `GridEncoder.dense_train` on the tensor cores (csrc/encoder.cu, gemm_tc.cu, dense_train.cu: bf16 operands, fp32
    accumulation, no floating-point atomics); oracle/encoder_train_tc_model.py states the formulation and its rounding points.
    latent_cl (NV,Hl,Wl,512) channel-last, params = depth_fc's three (w, b), then per aggregator in axis order (yz, xz, xy) its
    Linear(513, 512) w, b and Linear(512, 1) w, b -> floor plans xz, xy, yz (NV,512,G,G) fp32.  Activations live in bf16: the lookup rows
    X (R, 576), h0, h1 (R, 512), L = [lat | x y z | 0] (R, 576) and the three aggregators' hidden layers side by side in A (R, 1536), the
    output of one GEMM over L with their first layers stacked (row block a = aggregator a's 512 latent columns, its coordinate column at
    column 512 + a, zeros elsewhere)."""

    @staticmethod
    def forward(ctx, latent_cl, poses, focal, cx, cy, W, H, *params):
        lib = L.load()
        lat = latent_cl.detach().contiguous().float()
        nv, lh, lw, _ = lat.shape
        dev = lat.device
        pose_c = poses.detach().contiguous().float()
        R = nv * GridEncoder.GRID ** 3
        P = [t.detach().contiguous().float() for t in params]
        w, b = P[0:6:2], P[1:6:2]
        u, c, q, e = P[6::4], P[7::4], P[8::4], P[9::4]
        bf = lambda *shape: torch.empty(*shape, dtype=torch.bfloat16, device=dev)
        U = torch.zeros(1536, 576, device=dev)                  # the stacked first layers (fp32 master values)
        for a in range(3):
            U[512 * a:512 * (a + 1), :512] = u[a][:, :512]
            U[512 * a:512 * (a + 1), 512 + a] = u[a][:, 512]
        cs = torch.cat(c)
        X, H0, H1, Lb, A = bf(R, 576), bf(R, 512), bf(R, 512), bf(R, 576), bf(R, 1536)
        Wp = [bf(512, 576), bf(512, 512), bf(512, 512)]
        Up = bf(1536, 576)
        WT = [bf(512, 512) for _ in range(3)]                   # W_i^T (W_0: its 512 lookup columns), the data gradients' operands
        UT = bf(512, 1536)                                      # U[:, :512]^T
        logits = torch.empty(3, R, device=dev)
        out = [torch.empty(nv, 512, GridEncoder.GRID, GridEncoder.GRID, device=dev) for _ in range(3)]
        geo, cam = (nv, lh, lw, int(W), int(H)), (focal, cx, cy)
        lb, ldl = bf16.rows(Lb)
        with L.on(dev) as s:
            for i, wi in enumerate(w):
                bf16.pack(wi, Wp[i], False, s)
                bf16.pack(wi, WT[i], True, s)
            bf16.pack(U, Up, False, s)
            bf16.pack(U, UT, True, s)
            L.check(lib.neo_grid_encoder_features_bf16(L.ptr(lat), *geo, L.ptr(pose_c), *cam, *bf16.rows(X), s))
            bf16.gemm(X, Wp[0], b[0], H0, 0, s)
            bf16.gemm(H0, Wp[1], b[1], H1, 0, s)
            bf16.gemm(H1, Wp[2], b[2], Lb[:, :512], 1, s)
            L.check(lib.neo_grid_encoder_coords_bf16(lb, nv, ldl, s))
            bf16.gemm(Lb, Up, cs, A, 0, s)
            for a in range(3):
                bf16.rowdot(A[:, 512 * a:512 * (a + 1)], q[a], e[a], logits[a], s)
            L.check(lib.neo_grid_encoder_pool_bf16(lb, ldl, L.ptr(logits), nv, *[L.ptr(t) for t in out], s))
        ctx.save_for_backward(X, H0, H1, Lb, A, logits, *WT, UT, pose_c, *q)
        ctx.geo, ctx.cam = geo, cam
        ctx.det = torch.are_deterministic_algorithms_enabled()
        return tuple(out)

    @staticmethod
    def backward(ctx, g_xz, g_xy, g_yz):
        lib = L.load()
        X, H0, H1, Lb, A, logits, *rest = ctx.saved_tensors
        WT, UT, pose_c, q = rest[0:3], rest[3], rest[4], rest[5:8]
        nv = ctx.geo[0]
        R, dev = X.shape[0], X.device
        bf = lambda *shape: torch.empty(*shape, dtype=torch.bfloat16, device=dev)
        gs = [None if g is None else g.contiguous().float() for g in (g_xz, g_xy, g_yz)]
        ws = L.workspace(max(lib.neo_tc_wgrad_bf16_workspace_bytes(R, *c) for c in ((64, 512), (1536, 576), (512, 512), (512, 576))), dev)
        d_pool, d_lg = torch.empty(R, 512, device=dev), torch.empty(3, R, device=dev)
        dA, g1 = bf(R, 1536), bf(R, 64)
        agg = []
        with L.on(dev) as s:
            L.check(lib.neo_grid_encoder_pool_bwd_bf16(*bf16.rows(Lb), L.ptr(logits), nv, *[L.ptr(g) for g in gs], L.ptr(d_pool), L.ptr(d_lg),
                                                       s))
            for a in range(3):
                cols = slice(512 * a, 512 * (a + 1))
                bf16.relu_rank1(d_lg[a], q[a], A[:, cols], dA[:, cols], s)
                bf16.pack(d_lg[a][:, None], g1, False, s)
                gq = torch.empty(64, 512, device=dev)
                bf16.wgrad(g1, A[:, cols], gq, None, ws, s)
                agg.append((gq[:1].clone(), d_lg[a].sum().reshape(1)))
            gU, gc = torch.empty(1536, 515, device=dev), torch.empty(1536, device=dev)
            bf16.wgrad(dA, Lb, gU, gc, ws, s)
            d_agg = torch.empty(R, 512, device=dev)
            bf16.gemm(dA, UT, None, d_agg, 2, s)
            del dA
            G = [bf(R, 512), bf(R, 512)]
            L.check(lib.neo_grid_encoder_lat_grad_bf16(L.ptr(d_pool), L.ptr(d_agg), nv, L.ptr(G[0]), s))
            del d_pool, d_agg
            grads = [None] * 6
            for i, x in ((2, H1), (1, H0), (0, X)):
                gw, gb = torch.empty(512, 518 if i == 0 else 512, device=dev), torch.empty(512, device=dev)
                bf16.wgrad(G[0], x, gw, gb, ws, s)
                grads[2 * i], grads[2 * i + 1] = gw, gb
                if i > 0:
                    bf16.dgrad(G[0], WT[i], x, None, None, G[1], s)
                    G.reverse()
            g_lat = None
            if ctx.needs_input_grad[0]:
                g_X = torch.empty(R, 512, device=dev)
                bf16.gemm(G[0], WT[0], None, g_X, 2, s)
                g_lat = _lookup_bwd(ctx, pose_c, g_X)
        for a in range(3):
            rows = slice(512 * a, 512 * (a + 1))
            grads += [torch.cat([gU[rows, :512], gU[rows, 512 + a:513 + a]], 1), gc[rows].clone(), *agg[a]]
        return (g_lat, None, None, None, None, None, None, *grads)


def _lookup_bwd(ctx, pose_c, g):
    """Latent gradient (NV,Hl,Wl,512) of the lookup rows' 512 lookup columns g (R, ld) fp32: the order-fixed scatter under
    torch.use_deterministic_algorithms (ctx.det, recorded in the forward), the atomic one otherwise."""
    lib = L.load()
    nv, lh, lw, _, _ = ctx.geo
    g_lat = torch.zeros(nv, lh, lw, 512, device=g.device)
    with L.on(g) as s:
        if ctx.det:                 # order-fixed scatter: bit-reproducible
            ws = L.workspace(lib.neo_grid_encoder_features_bwd_det_workspace_bytes(nv, lh, lw), g.device)
            L.check(lib.neo_grid_encoder_features_bwd_det(*ctx.geo, L.ptr(pose_c), *ctx.cam, L.ptr(g), g.stride(0), L.ptr(g_lat), L.ptr(ws),
                                                          ws.numel(), s))
        else:
            L.check(lib.neo_grid_encoder_features_bwd(*ctx.geo, L.ptr(pose_c), *ctx.cam, L.ptr(g), g.stride(0), L.ptr(g_lat), s))
    return g_lat


class GridEncoder(nn.Module):
    GRID = 64

    def __init__(self, encoder_type="resnet", train_precision="fp32", **unused):
        super().__init__()
        # "fp32": the dense part trains through framework fp32 GEMMs (dense_train); "tc": on the tensor cores (dense_train_tc)
        self.train_precision = train_precision
        if encoder_type != "resnet":
            raise NotImplementedError("reference default only (encoder_type='resnet')")
        self.grid_size = [self.GRID] * 3
        self.spatial_encoder = SpatialEncoder()
        LS = self.latent_size = self.spatial_encoder.latent_size
        self.depth_fc = DepthPillarEncoder(inp_ch=LS + 3 + 3, LS=LS)
        mk = lambda: nn.Sequential(nn.Linear(LS + 1, LS), nn.ReLU(inplace=True), nn.Linear(LS, 1))
        self.pillar_aggregator_xz, self.pillar_aggregator_yz, self.pillar_aggregator_xy = mk(), mk(), mk()
        self.floorplan_convnet_xy, self.floorplan_convnet_yz, self.floorplan_convnet_xz = _floorplan_convnet(), _floorplan_convnet(), _floorplan_convnet()
        for m in (self.floorplan_convnet_xy, self.floorplan_convnet_yz, self.floorplan_convnet_xz,
                  self.pillar_aggregator_xz, self.pillar_aggregator_yz, self.pillar_aggregator_xy):
            m.apply(_init_linear_kaiming)
        self._ws = None
        self._latent_key = None         # (images, their version, the ResNet's tensor versions, latent, latent_scaling) of the cached latent

    @property
    def train_precision(self) -> str:
        return self._train_precision

    @train_precision.setter
    def train_precision(self, p: str):
        self._train_precision = check_train_precision(p)

    # ---- the dense part, framework ops (autograd; also the fp32 reference of the CUDA path in the tests) ----
    def dense_torch(self, latent, poses, focal, c, W, H):
        """encoder_tp_fusion_conv.py:483-570"""
        G, NV, dev = self.GRID, latent.shape[0], latent.device
        ax = [torch.linspace(-1, 1, G, device=dev), torch.linspace(-1, 1, G, device=dev), torch.linspace(0, 1, G, device=dev)]
        world = torch.stack(torch.meshgrid(*ax, indexing="ij"), -1).reshape(1, -1, 3).expand(NV, -1, -1)     # (NV, G^3, 3)
        rot = poses[:, :3, :3].transpose(1, 2)
        trans = -torch.bmm(rot, poses[:, :3, 3:])
        cam = torch.matmul(rot[:, None], world.unsqueeze(-1))[..., 0] + trans[:, None, :, 0]
        mask = cam[:, :, 2] < 1e-3
        d = world - poses[:, None, :3, -1]
        d = d / torch.norm(d + 1e-9, dim=-1)[:, :, None] * mask[:, :, None]
        f2 = torch.stack([focal[0], -focal[0]]).reshape(1, 1, 2)
        uv = -cam[..., :2] / (cam[..., 2:] + 1e-9) * f2 + c[0].reshape(1, 1, 2)
        ls = torch.tensor([latent.shape[-1], latent.shape[-2]], dtype=torch.float32, device=dev)
        uv = uv * ((ls / (ls - 1) * 2.0) / torch.tensor([W, H], dtype=torch.float32, device=dev)) - 1.0
        feat = F.grid_sample(latent, uv.unsqueeze(2), align_corners=True, mode="bilinear", padding_mode="zeros")[..., 0]     # (NV, 512, G^3)
        x = torch.cat([feat, cam.permute(0, 2, 1), d.permute(0, 2, 1)], 1).permute(0, 2, 1)
        lat = self.depth_fc(x).reshape(NV, G, G, G, -1)
        wg = world.reshape(NV, G, G, G, 3)
        w_yz = torch.softmax(self.pillar_aggregator_yz(torch.cat([lat, wg[..., 0:1]], -1)), dim=1)
        w_xz = torch.softmax(self.pillar_aggregator_xz(torch.cat([lat, wg[..., 1:2]], -1)), dim=2)
        w_xy = torch.softmax(self.pillar_aggregator_xy(torch.cat([lat, wg[..., 2:3]], -1)), dim=3)
        fp = lambda t: t.permute(0, 3, 1, 2)
        return fp((lat * w_xz).sum(2)), fp((lat * w_xy).sum(3)), fp((lat * w_yz).sum(1))      # xz, xy, yz: (NV, 512, 64, 64)

    # ---- the dense part for training on CUDA: hand-written lookup and pillar sums (forward and backward), framework fp32 GEMMs ----
    def dense_train(self, latent, poses, focal, c, W, H):
        """The algebra of `dense_torch`, differentiable with respect to `latent` and every parameter of depth_fc and the three aggregators.
        The dense layers are fp32 `F.linear` on the modules' own parameters (TF32 when torch.backends.cuda.matmul.allow_tf32 is set); each
        aggregator's coordinate input (column 512) is applied as a rank-1 term over the grid axis it depends on."""
        if not latent.is_cuda:
            raise RuntimeError("neo360_b200 needs CUDA tensors (no CPU fallback)")
        G, NV = self.GRID, latent.shape[0]
        lin = lambda m, x: F.linear(x, m.weight, m.bias)
        X = _Features.apply(latent.permute(0, 2, 3, 1), poses, float(focal[0]), float(c[0, 0]), float(c[0, 1]), W, H)
        fc = self.depth_fc
        h = torch.relu_(lin(fc.common_branch[0], X))
        h = torch.relu_(lin(fc.common_branch[2], h))
        lat = lin(fc.depth_encoder, h)                                                    # (NV*G^3, 512)
        ax = [torch.linspace(-1, 1, G, device=latent.device), torch.linspace(-1, 1, G, device=latent.device),
              torch.linspace(0, 1, G, device=latent.device)]
        logits = []
        for axis, name in enumerate(("yz", "xz", "xy")):
            agg = getattr(self, f"pillar_aggregator_{name}")
            w0 = agg[0].weight
            shape = [1, 1, 1, 1]
            shape[1 + axis] = G
            a = F.linear(lat, w0[:, :512], agg[0].bias)
            a.view(NV, G, G, G, -1).add_(ax[axis].reshape(*shape, 1) * w0[:, 512])           # + coordinate (x, y or z) times column 512
            logits.append(lin(agg[2], torch.relu_(a)).reshape(-1))
        return _Pool.apply(lat, torch.stack(logits))

    # ---- the dense part for training on the tensor cores: bf16 products, hand-written lookup and pillar sums (forward and backward) ----
    def dense_train_tc(self, latent, poses, focal, c, W, H):
        """`dense_train` with every dense layer on the tensor cores (`_DenseTC`), differentiable with respect to `latent` and every
        parameter of depth_fc and the three aggregators."""
        if not latent.is_cuda:
            raise RuntimeError("neo360_b200 needs CUDA tensors (no CPU fallback)")
        fc = self.depth_fc
        params = [t for m in (fc.common_branch[0], fc.common_branch[2], fc.depth_encoder) for t in (m.weight, m.bias)]
        for name in ("yz", "xz", "xy"):
            agg = getattr(self, f"pillar_aggregator_{name}")
            params += [agg[0].weight, agg[0].bias, agg[2].weight, agg[2].bias]
        return _DenseTC.apply(latent.permute(0, 2, 3, 1), poses, float(focal[0]), float(c[0, 0]), float(c[0, 1]), int(W), int(H), *params)

    # ---- the dense part, hand-written CUDA (wgmma) ----
    def dense_cuda(self, latent, poses, focal, c, W, H):
        if not latent.is_cuda:
            raise RuntimeError("neo360_b200 needs CUDA tensors (no CPU fallback)")
        lib = L.load()
        dev = latent.device
        lat = latent.detach().contiguous().float()
        NV, _, lh, lw = lat.shape
        keep = []
        f = lambda t: (keep.append(t.detach().contiguous().float()) or L.ptr(keep[-1]))
        p = L.NeoGridEncoderParams()
        fc = [self.depth_fc.common_branch[0], self.depth_fc.common_branch[2], self.depth_fc.depth_encoder]
        for i, m in enumerate(fc):
            p.fc_w[i], p.fc_b[i] = f(m.weight), f(m.bias)
        for pl in ("xz", "yz", "xy"):
            agg = getattr(self, f"pillar_aggregator_{pl}")
            setattr(p, f"agg_{pl}_w0", f(agg[0].weight)); setattr(p, f"agg_{pl}_b0", f(agg[0].bias))
            setattr(p, f"agg_{pl}_w1", f(agg[2].weight)); setattr(p, f"agg_{pl}_b1", f(agg[2].bias))
        self._ws = L.grow(self._ws, lib.neo_grid_encoder_workspace_bytes(NV, lh, lw), dev)
        out = [torch.empty(NV, 512, self.GRID, self.GRID, device=dev) for _ in range(3)]
        pose_c = poses.detach().contiguous().float()
        with L.on(dev) as s:
            L.check(lib.neo_grid_encoder_dense(C.byref(p), L.ptr(lat), NV, lh, lw, int(W), int(H), L.ptr(pose_c), float(focal[0]),
                                               float(c[0, 0]), float(c[0, 1]), L.ptr(out[0]), L.ptr(out[1]), L.ptr(out[2]),
                                               L.ptr(self._ws), self._ws.numel(), s))
        return out[0], out[1], out[2]

    def _spatial_latent(self, images):
        """spatial_encoder(images).  A frozen spatial encoder in eval mode (test-time optimisation, `training.test_time_optimizer`) is a
        fixed function of its input, so it runs once per set of `images`: compared by identity and in-place version, as
        NeRF_TP._same_source compares its sources, and by the version of every ResNet parameter and buffer (load_state_dict).  The
        cached latent is put back in `spatial_encoder.latent`, where the renderer reads it."""
        se = self.spatial_encoder
        frozen = not se.training and not images.requires_grad and not any(p.requires_grad for p in se.parameters())
        if not frozen:
            self._latent_key = None
            return se(images)
        key = (images, images._version, tuple((t.data_ptr(), t._version) for t in list(se.parameters()) + list(se.buffers())
                                              if t is not se.latent and t is not se.latent_scaling))
        old = self._latent_key
        if old is not None and old[0] is images and old[1:3] == key[1:3]:
            se.latent, se.latent_scaling = old[3], old[4]
            return old[3]
        with torch.no_grad():
            latent = se(images)
        self._latent_key = key + (latent, se.latent_scaling)
        return latent

    def forward(self, images, poses, focal, c):
        """images (NV,3,H,W), poses (NV,4,4) camera-to-world, focal (NV,), c (NV,2) -> scene_grid_xz, scene_grid_xy, scene_grid_yz (NV,128,120,160)."""
        NV, _, H, W = images.shape
        latent = self._spatial_latent(images)
        trained = [self.depth_fc, self.pillar_aggregator_xz, self.pillar_aggregator_yz, self.pillar_aggregator_xy]
        needs_grad = torch.is_grad_enabled() and (latent.requires_grad or any(q.requires_grad for m in trained for q in m.parameters()))
        if needs_grad:
            if not latent.is_cuda:
                dense = self.dense_torch
            else:
                dense = self.dense_train_tc if self.train_precision == "tc" else self.dense_train
            fxz, fxy, fyz = dense(latent, poses.float(), focal.float(), c.float(), W, H)
        else:
            fxz, fxy, fyz = self.dense_cuda(latent, poses, focal, c, W, H)
        return self.floorplan_convnet_xz(fxz), self.floorplan_convnet_xy(fxy), self.floorplan_convnet_yz(fyz)
