"""Float64 model of the PixelNeRF form of the tensor-core training trunk (csrc/field_train.cu with PIX, training._PixelTrunkTC) with
every bf16 rounding the kernels apply made explicit, its hand-written adjoint, the projection and per-point head around it, and the
mutations only this form can have.  The NeO-360 form, the shared helpers and the bounds live in oracle/field_train_model.py.

Forward (rows r = v M + j, point j seen from source view v; pixelnerf.NeRFMLP at skip_layer = netdepth = 4, so no layer-3 skip):
    p0 = rows . W0[:, 63:575]^T   (`project`: the latent columns of pts_linears.0 on looked-up latent rows, or on the latent map --
                                   the lookup is linear; fp32 rows, never rounded)
    enc = bf(_pos_enc(cam, 0, 10));  h0 = relu(enc bf(W0e)^T + b0 + p0);  h1 = relu(bf(h0) bf(W1)^T + b1);
    h2 = relu(bf(h1) bf(W2)^T + b2);  h3 = relu(bf(h2) bf(W3)^T + b3);  hbar = mean_v h3 (h3 unrounded)
Backward, g = d hbar:
    dz3 = (g / NV)[h3 > 0];  dz2 = (bf(dz3) bf(W3))[h2 > 0];  dz1 = (bf(dz2) bf(W2))[h1 > 0];  dz0 = (bf(dz1) bf(W1))[h0 > 0]
    d_p0 = dz0;  dW0e = bf(dz0)^T enc;  dW1 = bf(dz1)^T bf(h0);  dW2 = bf(dz2)^T bf(h1);  dW3 = bf(dz3)^T bf(h2);  db_l = sum_rows bf(dz_l)
With `rnd=False` every bf() is the identity and projection, trunk and `head` are pixelnerf._mlp_train re-associated exactly (head on
the view mean), which tests/test_pixelnerf_train_tc_model.py checks in float64.  The kernels are held to the bounds of
field_train_model (FWD_BOUND, BWD_BOUND, STEP_BOUND): the same products, roundings and accumulation lengths.
"""
import torch

from oracle.field_train_model import BWD_BOUND, FWD_BOUND, STEP_BOUND, bf, pos_enc, rel_err  # noqa: F401

# bugs only the PixelNeRF form can have: `forward` (skip3, p0_at_layer3), `project` (wrong_w0_cols), `head` (dbar_over_rays)
MUTATIONS = ("skip3", "p0_at_layer3", "wrong_w0_cols", "dbar_over_rays")


def project(rows, w0, mut=None):
    """p0 = rows . W0[:, 63:575]^T: the latent columns of pts_linears.0 (128, 575) applied to latent rows (NV*M, 512)."""
    lo = 62 if mut == "wrong_w0_cols" else 63
    return rows @ w0[:, lo:lo + 512].T


def forward(cam, p0, W, rnd=True, mut=None):
    """cam (NV, M, 3), p0 (NV*M, 128), W = dict(w0e, b0, w1, b1, w2, b2, w3, b3) float64 -> hbar (M, 128), saved."""
    nv, M, _ = cam.shape
    r = lambda x: bf(x, rnd)
    enc = r(pos_enc(cam).reshape(nv * M, 63))
    h0 = torch.relu(enc @ r(W["w0e"]).T + W["b0"] + p0)
    h1 = torch.relu(r(h0) @ r(W["w1"]).T + W["b1"])
    h2 = torch.relu(r(h1) @ r(W["w2"]).T + W["b2"])
    z3 = r(h2) @ r(W["w3"]).T + W["b3"]
    if mut == "skip3":                      # an encoding skip at layer 3 (the NeO-360 form's W3e product, fed the layer-0 weights)
        z3 = z3 + enc @ r(W["w0e"]).T
    if mut == "p0_at_layer3":               # the projected row seeded into layer 3 as well (the NeO-360 form's P3 slot)
        z3 = z3 + p0
    h3 = torch.relu(z3)
    return h3.reshape(nv, M, 128).mean(0), dict(enc=enc, h0=h0, h1=h1, h2=h2, h3=h3, nv=nv)


def backward(g_hbar, S, W, rnd=True, mut=None):
    """Adjoint of `forward`: g_hbar (M, 128) -> d_p0 (NV*M, 128) and dict of weight / bias gradients (nn.Linear layout)."""
    r = lambda x: bf(x, rnd)
    nv = S["nv"]
    dz3 = g_hbar.repeat(nv, 1) / nv * (S["h3"] > 0)
    dz2 = (r(dz3) @ r(W["w3"])) * (S["h2"] > 0)
    dz1 = (r(dz2) @ r(W["w2"])) * (S["h1"] > 0)
    dz0 = (r(dz1) @ r(W["w1"])) * (S["h0"] > 0)
    G = {"w0e": r(dz0).T @ S["enc"], "w1": r(dz1).T @ r(S["h0"]), "w2": r(dz2).T @ r(S["h1"]), "w3": r(dz3).T @ r(S["h2"])}
    for k, dz in (("b0", dz0), ("b1", dz1), ("b2", dz2), ("b3", dz3)):
        G[k] = r(dz).sum(0)
    return dz0, G


def head(mlp, hbar, dir_tile, nv, mut=None):
    """training.view_mean_head: raw rgb and raw sigma once per point from hbar and the view mean of the direction encodings."""
    lin = lambda m, x: torch.nn.functional.linear(x, m.weight, m.bias)
    M = hbar.shape[0]
    raw_sigma = lin(mlp.density_layer, hbar)
    if mut == "dbar_over_rays":             # rows grouped point-major: each mean runs over consecutive rows of one view
        dbar = dir_tile.reshape(M, nv, -1).mean(1)
    else:
        dbar = dir_tile.reshape(nv, M, -1).mean(0)
    q = lin(mlp.views_linear[0], torch.cat([lin(mlp.bottleneck_layer, hbar), dbar], -1))
    q = torch.relu(lin(mlp.views_linear[1], torch.relu(q)))
    return lin(mlp.rgb_layer, q), raw_sigma


def weights_of(mlp):
    """The trunk inputs of `_PixelTrunkTC` from a PixelNeRF NeRFMLP (float64 copies)."""
    p = mlp.pts_linears
    d = lambda t: t.detach().double().clone()
    return dict(w0e=d(p[0].weight[:, :63]), b0=d(p[0].bias), w1=d(p[1].weight), b1=d(p[1].bias), w2=d(p[2].weight), b2=d(p[2].bias),
                w3=d(p[3].weight), b3=d(p[3].bias))
