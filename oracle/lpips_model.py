"""TEST INFRASTRUCTURE ONLY.  Float64 models of LPIPS (VGG) as csrc/lpips.cu pins it, the head's adjoint, a-priori fp32 error bounds for
neo_lpips_head and neo_lpips_head_bwd, an fp32 emulation of neo_lpips_prepare, and seeded weights in the layouts users' files have.

Neither piqa nor lpips is installed here, so both definitions are written out from their sources:
* `lpips_piqa_f64`: piqa's LPIPS(network="vgg") -- (x - mean) / std with ImageNet mean / std; per layer the spatial mean of (u - v)^2
  and then the 1x1 layer;
* `lpips_lpips_f64`: lpips.LPIPS(net="vgg") on 2x - 1 -- ((2x - 1) - shift) / scale; per layer the 1x1 layer and then the spatial mean.
Both clip to [0, 1] first and normalise with eps = 1e-10.  In exact arithmetic they are equal.

Bounds, with u = 2^-24 and the fp32 features taken as exact inputs (every intermediate a normal fp32 number):
* head, per pixel of a layer with C channels: the kernel's norm (an fma chain of C squares, a square root, + eps) is within (C/2 + 2) u
  relative, each of u, v within (C/2 + 3) u, e = u - v within (C/2 + 4) u (|u| + |v|), e^2 within (C + 9) u |e| (|u| + |v|), and the
  fma chain over the channels adds C u of each term.  So |d~ - d| <= (2C + 12) u m_p with m_p = sum_c |w_c| |e_c| (|u_c| + |v_c|).  A
  layer's value is within the mean of that plus the double sums' (P / 128 + 20) 2^-53 of the mean of d; a frame's within the sum.
* backward, per element j: with D = ||f|| + eps, T = sum_c |w_c| |f_c| (|u_c| + |v_c|) and a = 2 g / P, the two terms carry
  (C + 10) u |a| |w_j| (|u_j| + |v_j|) / D and (3C + 17) u |a| |f_j| T / (||f|| D^2); the bound is (3C + 24) u times their magnitudes'
  sum.  A zero-norm pixel's gradient is exactly 0.
"""
import numpy as np
import torch
import torch.nn.functional as F

CHANNELS = (64, 128, 256, 512, 512)
TAPS = (3, 8, 15, 22, 29)
CONVS = (0, 2, 5, 7, 10, 12, 14, 17, 19, 21, 24, 26, 28)
EPS = 1e-10
U = 2.0 ** -24
MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
SHIFT, SCALE = (-0.030, -0.088, -0.188), (0.458, 0.448, 0.450)


# ---- weights ---------------------------------------------------------------------------------------------------------------------
def vgg16_state(seed: int = 0, classifier: bool = True) -> dict:
    """Seeded torchvision-layout vgg16 state dict (`features.N.weight|bias`, and `classifier.*` as the real file has), He-scaled so the
    features keep their magnitude through the 13 layers."""
    g = torch.Generator().manual_seed(seed)
    sd, c_in = {}, 3
    cfg = [c for c in (64, 64, 128, 128, 256, 256, 256, 512, 512, 512, 512, 512, 512)]
    for i, c in zip(CONVS, cfg):
        sd[f"features.{i}.weight"] = torch.randn(c, c_in, 3, 3, generator=g) * (2.0 / (9 * c_in)) ** 0.5
        sd[f"features.{i}.bias"] = 0.05 * torch.randn(c, generator=g)
        c_in = c
    if classifier:
        sd["classifier.0.weight"] = torch.randn(8, 4, generator=g)
        sd["classifier.0.bias"] = torch.randn(8, generator=g)
    return sd


def lin_weights(seed: int = 0):
    """Five seeded non-negative 1x1 weight vectors (LPIPS v0.1 weights are non-negative), of a different scale per layer so that using
    one layer's weights for another's is visible."""
    g = torch.Generator().manual_seed(seed)
    return [torch.rand(c, generator=g) * ((k + 1) / c) for k, c in enumerate(CHANNELS)]


def lin_state(ws, layout: str) -> dict:
    """The lin weights in lpips' (`lin{k}.model.1.weight`) or piqa's (`{k}.1.weight`) layout, each (1, C, 1, 1)."""
    key = {"lpips": "lin{}.model.1.weight", "piqa": "{}.1.weight"}[layout]
    return {key.format(k): w.reshape(1, -1, 1, 1).clone() for k, w in enumerate(ws)}


# ---- float64 models --------------------------------------------------------------------------------------------------------------
def trunk_f64(vgg_sd: dict, x: torch.Tensor):
    """relu1_2 .. relu5_3 of torchvision's vgg16().features[:30] in float64 on (n, 3, H, W)."""
    feats, conv = [], iter(CONVS)
    h = x.double()
    i = 0
    while i < 30:
        if i in (4, 9, 16, 23):
            h = F.max_pool2d(h, 2, 2)
            i += 1
            continue
        j = next(conv)
        h = torch.relu(F.conv2d(h, vgg_sd[f"features.{j}.weight"].to(h), vgg_sd[f"features.{j}.bias"].to(h), padding=1))
        i += 2
        if i - 1 in TAPS:
            feats.append(h)
    return feats


def _unit(f):
    return f / (torch.sqrt((f * f).sum(1, keepdim=True)) + EPS)


def head_f64(fx, fy, ws, order: str = "lpips", eps: float = EPS):
    """(per-frame (n,), per-layer (n, 5)) in float64.  order "lpips": 1x1 layer then spatial mean; "piqa": spatial mean then 1x1."""
    vals = []
    for a, b, w in zip(fx, fy, ws):
        a, b, w = a.double(), b.double(), w.double().to(a.device).reshape(1, -1, 1, 1)
        u = a / (torch.sqrt((a * a).sum(1, keepdim=True)) + eps)
        v = b / (torch.sqrt((b * b).sum(1, keepdim=True)) + eps)
        e2 = (u - v) ** 2
        vals.append((w * e2).sum(1).mean((1, 2)) if order == "lpips" else (w * e2.mean((2, 3), keepdim=True)).sum((1, 2, 3)))
    per = torch.stack(vals, 1)
    return per.sum(1), per


def scale_f64(img: torch.Tensor, form: int) -> torch.Tensor:
    """(n, H, W, 3) -> clipped and scaled (n, 3, H, W) in float64; form 0 piqa, 1 lpips."""
    x = img.double().clamp(0, 1).permute(0, 3, 1, 2)
    if form == 0:
        m, s = torch.tensor(MEAN, dtype=torch.float64), torch.tensor(STD, dtype=torch.float64)
        return (x - m.view(1, 3, 1, 1).to(x.device)) / s.view(1, 3, 1, 1).to(x.device)
    sh, sc = torch.tensor(SHIFT, dtype=torch.float64), torch.tensor(SCALE, dtype=torch.float64)
    return ((2 * x - 1) - sh.view(1, 3, 1, 1).to(x.device)) / sc.view(1, 3, 1, 1).to(x.device)


def lpips_piqa_f64(x, y, vgg_sd, ws):
    return head_f64(trunk_f64(vgg_sd, scale_f64(x, 0)), trunk_f64(vgg_sd, scale_f64(y, 0)), ws, "piqa")[0]


def lpips_lpips_f64(x, y, vgg_sd, ws):
    return head_f64(trunk_f64(vgg_sd, scale_f64(x, 1)), trunk_f64(vgg_sd, scale_f64(y, 1)), ws, "lpips")[0]


def adjoint_f64(fx, fy, ws, g, projection: bool = True):
    """Gradients of sum_f g_f LPIPS_f with respect to fx and fy (float64 lists), 0 at zero-norm pixels.  `projection=False` drops the
    term through the norm (a mutant)."""
    gx, gy = [], []
    g = g.double()
    for a, b, w in zip(fx, fy, ws):
        a, b, w = a.double(), b.double(), w.double().to(a.device).reshape(1, -1, 1, 1)
        P = a.shape[2] * a.shape[3]
        coef = (2 * g / P).view(-1, 1, 1, 1).to(a.device)
        out = []
        for f, o in ((a, b), (b, a)):        # d/dv of w (u - v)^2 is d/du with the roles exchanged
            n = torch.sqrt((f * f).sum(1, keepdim=True))
            D = n + EPS
            r = w * (f / D - o / (torch.sqrt((o * o).sum(1, keepdim=True)) + EPS))
            t = (r * f).sum(1, keepdim=True)
            grad = coef * (r / D - (f * t / (n * D * D) if projection else 0))
            out.append(torch.where(n > 0, grad, torch.zeros_like(grad)))
        gx.append(out[0])
        gy.append(out[1])
    return gx, gy


# ---- bounds ----------------------------------------------------------------------------------------------------------------------
def head_bound(fx, fy, ws):
    """(per-frame (n,), per-layer (n, 5)) a-priori bounds of neo_lpips_head's values (module docstring)."""
    lay = []
    for a, b, w in zip(fx, fy, ws):
        a, b, w = a.double(), b.double(), w.double().to(a.device).reshape(1, -1, 1, 1)
        C, P = a.shape[1], a.shape[2] * a.shape[3]
        u, v = _unit(a), _unit(b)
        m = (w.abs() * (u - v).abs() * (u.abs() + v.abs())).sum(1).mean((1, 2))
        d = (w * (u - v) ** 2).sum(1).mean((1, 2))
        lay.append((2 * C + 12) * U * m + (P / 128 + 20) * 2.0 ** -53 * d)
    per = torch.stack(lay, 1)
    vals = head_f64(fx, fy, ws)[0]
    return per.sum(1) + 5 * 2.0 ** -53 * vals.abs(), per


def bwd_bound(fx, fy, ws, g):
    """Per-element bounds of neo_lpips_head_bwd's g_fx and g_fy (float64 lists shaped as the features)."""
    bx, by = [], []
    g = g.double()
    for a, b, w in zip(fx, fy, ws):
        a, b, w = a.double(), b.double(), w.double().to(a.device).reshape(1, -1, 1, 1)
        C, P = a.shape[1], a.shape[2] * a.shape[3]
        coef = (2 * g / P).abs().view(-1, 1, 1, 1).to(a.device)
        u, v = _unit(a), _unit(b)
        mag = w.abs() * (u.abs() + v.abs())
        out = []
        for f in (a, b):
            n = torch.sqrt((f * f).sum(1, keepdim=True))
            D = n + EPS
            T = (mag * f.abs()).sum(1, keepdim=True)
            e = coef * (mag / D + f.abs() * T / (n * D * D))
            out.append(torch.where(n > 0, (3 * C + 24) * U * e, torch.zeros_like(e)))
        bx.append(out[0])
        by.append(out[1])
    return bx, by


# ---- fp32 emulation of neo_lpips_prepare -----------------------------------------------------------------------------------------
def prepare_f32(img: np.ndarray, form: int) -> np.ndarray:
    """neo_lpips_prepare step by step in numpy float32 (IEEE, round to nearest): (n, H, W, 3) -> (n, 3, H, W)."""
    x = np.clip(img.astype(np.float32), np.float32(0), np.float32(1))
    if form == 0:
        out = (x - np.asarray(MEAN, np.float32)) / np.asarray(STD, np.float32)
    else:
        out = ((np.float32(2) * x - np.float32(1)) - np.asarray(SHIFT, np.float32)) / np.asarray(SCALE, np.float32)
    return np.ascontiguousarray(out.transpose(0, 3, 1, 2))


def prepare_bwd_f32(img: np.ndarray, g_out: np.ndarray, form: int) -> np.ndarray:
    """neo_lpips_prepare_bwd in numpy float32: g / std (form 0) or (g / scale) * 2 (form 1), zero outside [0, 1] (bounds inclusive)."""
    g = g_out.astype(np.float32).transpose(0, 2, 3, 1)
    d = g / np.asarray(STD, np.float32) if form == 0 else (g / np.asarray(SCALE, np.float32)) * np.float32(2)
    x = img.astype(np.float32)
    return np.ascontiguousarray(np.where((x >= 0) & (x <= 1), d, np.float32(0)).astype(np.float32))


# ---- test content ----------------------------------------------------------------------------------------------------------------
def plant(feats, seed: int, zero_frac: float = 0.05, tiny_frac: float = 0.05):
    """Copies of (n, C, H, W) feature maps with a seeded share of pixels set to all-zero channels and another share scaled to a norm
    near eps (1e-11 .. 1e-9, where eps matters)."""
    out = []
    for k, f in enumerate(feats):
        g = torch.Generator().manual_seed(seed * 10 + k)
        n, C, H, W = f.shape
        r = torch.rand(n, 1, H, W, generator=g).to(f.device)
        tiny = 10.0 ** (-11 + 2 * torch.rand(n, 1, H, W, generator=g)).to(f.device)
        nrm = torch.sqrt((f.double() ** 2).sum(1, keepdim=True)).clamp_min(1e-30)
        t = torch.where(r < zero_frac, torch.zeros_like(f), f)
        t = torch.where((r >= zero_frac) & (r < zero_frac + tiny_frac), (f.double() / nrm * tiny).to(f.dtype), t)
        out.append(t.contiguous())
    return out
