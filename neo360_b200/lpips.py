"""LPIPS (VGG) for evaluation and fine-tuning: LitModel.lpips_each with piqa's LPIPS(network="vgg") (models/interface.py:113-122) and
NeRF_TP.lpips_loss with lpips.LPIPS(net="vgg") (models/neo360/model.py:1283-1309).

What runs where
  * the VGG-16 trunk (torchvision's vgg16().features[:30]): framework convolutions, parameters frozen, as the ResNet trunk of the encoder;
  * hand-written CUDA (csrc/lpips.cu, definition in its header): input clipping, the NHWC -> NCHW copy and either scaling form
    (`neo_lpips_prepare`), channel normalisation, the weighted squared distance and the spatial means (`neo_lpips_head`), and their
    adjoints (`neo_lpips_prepare_bwd`, `neo_lpips_head_bwd`).  Deterministic, no floating-point atomics.
Weights are the user's files (`LPIPS.from_files`): torchvision's `vgg16-*.pth` and the LPIPS v0.1 `vgg.pth` that lpips and piqa download.
The 1x1 layers have no dropout: the term is always evaluated as in eval mode (DESIGN.md section 8).
There is no CPU fallback; `head_torch` is the framework form of the head, the baseline of tools/bench_lpips.py and of the tests.
"""
from __future__ import annotations

import ctypes as C
from typing import List, Sequence

import torch
import torch.nn as nn

from . import _lib as L

Tensor = torch.Tensor

VGG16_CFG = (64, 64, "M", 128, 128, "M", 256, 256, 256, "M", 512, 512, 512, "M", 512, 512, 512)   # features[:30]: no last pool
TAPS = (3, 8, 15, 22, 29)                   # relu1_2, relu2_2, relu3_3, relu4_3, relu5_3
CHANNELS = (64, 128, 256, 512, 512)
EPS = 1e-10                                 # lpips' normalize_tensor
FORM_PIQA, FORM_LPIPS = 0, 1                # scaling of evaluation (piqa) and of the fine-tuning loss (lpips)
MIN_SIZE = 16                               # relu5_3 is (H >> 4, W >> 4)


def _vgg16_features() -> nn.Sequential:
    layers, c_in = [], 3
    for v in VGG16_CFG:
        if v == "M":
            layers.append(nn.MaxPool2d(kernel_size=2, stride=2))
        else:
            layers += [nn.Conv2d(c_in, v, kernel_size=3, padding=1), nn.ReLU()]
            c_in = v
    return nn.Sequential(*layers)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _ptrs(ts: Sequence[Tensor]):
    return (C.c_void_p * len(ts))(*[t.data_ptr() for t in ts])


def _check_features(fx: Sequence[Tensor], fy: Sequence[Tensor], w: Sequence[Tensor]):
    """(n, H, W) of the frames the five feature pairs come from; raises on a shape, dtype or device the kernels do not take."""
    if not (len(fx) == len(fy) == len(w) == 5):
        raise ValueError("LPIPS head: five feature maps of each image and five weight vectors")
    n, _, H, W = fx[0].shape
    for k, (a, b, wk) in enumerate(zip(fx, fy, w)):
        want = (n, CHANNELS[k], H >> k, W >> k)
        if tuple(a.shape) != want or tuple(b.shape) != want or wk.numel() != CHANNELS[k]:
            raise ValueError(f"LPIPS head layer {k}: features {tuple(a.shape)} / {tuple(b.shape)}, weights {wk.numel()}; expected {want}")
        for t in (a, b, wk):
            if not (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous() and t.device == fx[0].device):
                raise RuntimeError("neo360_b200 needs contiguous fp32 CUDA tensors on one device (no CPU fallback)")
    return n, H, W


def head(fx: Sequence[Tensor], fy: Sequence[Tensor], w: Sequence[Tensor], per_layer: bool = False):
    """neo_lpips_head: per-frame LPIPS (n,) float64 from the five NCHW feature maps of each image and the 1x1 weights; with `per_layer`
    also the (n, 5) layer values."""
    n, H, W = _check_features(fx, fy, w)
    lib = L.load()
    nbytes = lib.neo_lpips_workspace_bytes(n, H, W)
    if nbytes == 0:
        raise ValueError(f"LPIPS needs n >= 1 frames of at least {MIN_SIZE}x{MIN_SIZE} pixels, got n {n}, {H}x{W}")
    dev = fx[0].device
    ws = torch.empty(nbytes // 8, dtype=torch.float64, device=dev)
    out = torch.empty(n, dtype=torch.float64, device=dev)
    lay = torch.empty(n, 5, dtype=torch.float64, device=dev) if per_layer else None
    with torch.cuda.device(dev):
        L.check(lib.neo_lpips_head(_ptrs(fx), _ptrs(fy), _ptrs(w), n, H, W, out.data_ptr(), None if lay is None else lay.data_ptr(),
                                   ws.data_ptr(), nbytes, _stream()))
    return (out, lay) if per_layer else out


def head_bwd(fx: Sequence[Tensor], fy: Sequence[Tensor], w: Sequence[Tensor], g: Tensor, with_y: bool = False):
    """neo_lpips_head_bwd: the gradients of sum_f g_f LPIPS_f with respect to the five fx maps (and, with `with_y`, the fy maps)."""
    n, H, W = _check_features(fx, fy, w)
    if g.shape != (n,):
        raise ValueError(f"LPIPS head backward: upstream gradient {tuple(g.shape)}, expected ({n},)")
    gc = g.detach().to(device=fx[0].device, dtype=torch.float32).contiguous()
    gx = [torch.empty_like(t) for t in fx]
    gy = [torch.empty_like(t) for t in fy] if with_y else None
    with torch.cuda.device(gc.device):
        L.check(L.load().neo_lpips_head_bwd(_ptrs(fx), _ptrs(fy), _ptrs(w), n, H, W, gc.data_ptr(), _ptrs(gx), None if gy is None else _ptrs(gy),
                                            _stream()))
    return gx, gy


class _Head(torch.autograd.Function):
    """head() under autograd: (5 weights, 5 fx, 5 fy) -> (n,) float64; gradients flow to the feature maps, not to the weights."""

    @staticmethod
    def forward(ctx, *t):
        ts = [x.detach().contiguous() for x in t]
        ctx.save_for_backward(*ts)
        return head(ts[5:10], ts[10:], ts[:5])

    @staticmethod
    def backward(ctx, g):
        ts = ctx.saved_tensors
        with_y = any(ctx.needs_input_grad[10:])
        gx, gy = head_bwd(ts[5:10], ts[10:], ts[:5], g, with_y)
        return (None,) * 5 + tuple(gx) + (tuple(gy) if with_y else (None,) * 5)


class _Prepare(torch.autograd.Function):
    """neo_lpips_prepare: (n, H, W, 3) frames -> clipped, scaled (n, 3, H, W) trunk input; backward neo_lpips_prepare_bwd."""

    @staticmethod
    def forward(ctx, img, form):
        x = img.detach().contiguous().float()
        if not x.is_cuda:
            raise RuntimeError("neo360_b200 needs CUDA tensors (no CPU fallback)")
        if x.dim() != 4 or x.shape[-1] != 3:
            raise ValueError(f"LPIPS takes (n, H, W, 3) frames, got {tuple(img.shape)}")
        n, H, W, _ = x.shape
        out = torch.empty(n, 3, H, W, device=x.device)
        with torch.cuda.device(x.device):
            L.check(L.load().neo_lpips_prepare(x.data_ptr(), n, H, W, int(form), out.data_ptr(), _stream()))
        ctx.save_for_backward(x)
        ctx.form = int(form)
        return out

    @staticmethod
    def backward(ctx, g):
        (x,) = ctx.saved_tensors
        n, H, W, _ = x.shape
        gi = torch.empty_like(x)
        with torch.cuda.device(x.device):
            L.check(L.load().neo_lpips_prepare_bwd(x.data_ptr(), g.contiguous().float().data_ptr(), n, H, W, ctx.form, gi.data_ptr(), _stream()))
        return gi, None


def prepare(img: Tensor, form: int = FORM_PIQA) -> Tensor:
    """Clip (n, H, W, 3) frames to [0, 1] and scale them into the (n, 3, H, W) trunk input (form 0: piqa, 1: lpips)."""
    return _Prepare.apply(img, form)


def head_torch(fx: Sequence[Tensor], fy: Sequence[Tensor], w: Sequence[Tensor]) -> Tensor:
    """The head as lpips computes it, in framework ops on any device: normalize_tensor, squared difference, the 1x1 layer, then the
    spatial mean, summed over the layers.  Per-frame values (n,) in the features' dtype."""
    total = 0
    for a, b, wk in zip(fx, fy, w):
        u = a / (torch.sqrt(torch.sum(a ** 2, dim=1, keepdim=True)) + EPS)
        v = b / (torch.sqrt(torch.sum(b ** 2, dim=1, keepdim=True)) + EPS)
        d = torch.nn.functional.conv2d((u - v) ** 2, wk.reshape(1, -1, 1, 1).to(a.dtype))
        total = total + d.mean(dim=(2, 3)).reshape(-1)
    return total


class LPIPS(nn.Module):
    """The VGG-16 trunk (frozen) and the five 1x1 weights.  `forward(x, y, form)` takes (n, H, W, 3) frames and returns per-frame LPIPS
    as float64 (n,); gradients flow to the frames (the training loss differentiates with respect to the rendered colours)."""

    def __init__(self):
        super().__init__()
        self.features = _vgg16_features()
        self.lin = nn.ParameterList([nn.Parameter(torch.zeros(c)) for c in CHANNELS])
        self.requires_grad_(False)

    @classmethod
    def from_files(cls, vgg16_path: str, lin_path: str) -> "LPIPS":
        """torchvision's vgg16 state dict (`features.N.weight|bias`; `classifier.*` is ignored) and the LPIPS v0.1 vgg weights, in lpips'
        layout (`lin{k}.model.1.weight`) or piqa's (`{k}.1.weight`), each (1, C_k, 1, 1).  A missing, unknown or mis-shaped key raises."""
        m = cls()
        m.load_vgg16(torch.load(vgg16_path, map_location="cpu", weights_only=True))
        m.load_lin(torch.load(lin_path, map_location="cpu", weights_only=True))
        return m

    def load_vgg16(self, sd: dict) -> None:
        own = self.features.state_dict()
        got = {k[len("features."):]: v for k, v in sd.items() if k.startswith("features.")}
        extra = [k for k in sd if not k.startswith("classifier.") and not (k.startswith("features.") and k[len("features."):] in own)]
        if extra:
            raise KeyError(f"vgg16 weights: unexpected key {extra[0]!r}")
        for k, t in own.items():
            if k not in got:
                raise KeyError(f"vgg16 weights: missing key 'features.{k}'")
            if tuple(got[k].shape) != tuple(t.shape):
                raise ValueError(f"vgg16 weights: 'features.{k}' is {tuple(got[k].shape)}, expected {tuple(t.shape)}")
        self.features.load_state_dict(got)

    def load_lin(self, sd: dict) -> None:
        layout = "lin{}.model.1.weight" if "lin0.model.1.weight" in sd else "{}.1.weight"
        for k, c in enumerate(CHANNELS):
            key = layout.format(k)
            if key not in sd:
                raise KeyError(f"LPIPS lin weights: missing key {key!r}")
            if tuple(sd[key].shape) != (1, c, 1, 1):
                raise ValueError(f"LPIPS lin weights: {key!r} is {tuple(sd[key].shape)}, expected (1, {c}, 1, 1)")
            self.lin[k].data.copy_(sd[key].reshape(c))

    def trunk(self, x: Tensor) -> List[Tensor]:
        """relu1_2 .. relu5_3 of the (n, 3, H, W) trunk input, contiguous NCHW."""
        feats = []
        for i, layer in enumerate(self.features):
            x = layer(x)
            if i in TAPS:
                feats.append(x.contiguous())
        return feats

    def forward(self, x: Tensor, y: Tensor, form: int = FORM_PIQA) -> Tensor:
        if x.shape != y.shape:
            raise ValueError(f"LPIPS: shape mismatch {tuple(x.shape)} vs {tuple(y.shape)}")
        fx = self.trunk(prepare(x, form))           # separate calls of the same shape, as the reference runs them
        fy = self.trunk(prepare(y, form))
        return _Head.apply(*[w.contiguous() for w in self.lin], *fx, *fy)
