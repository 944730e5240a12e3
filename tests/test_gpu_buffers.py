"""The buffer contract of every C-ABI entry point: each call writes all of its outputs, nothing outside them, reads only workspace it
wrote during the same call, stays within the bytes its `*_workspace_bytes` reports, and leaves its inputs unchanged.

The harness calls the C ABI directly, so the test owns every buffer.  Each output and workspace is the interior of one larger uint8 CUDA
tensor: a guard band of at least GUARD bytes on either side, filled with a fixed byte pattern, and the interior aligned to ALIGN bytes and
exactly as large as the entry point needs (a workspace exactly `*_workspace_bytes`).  Every pointer argument of a case has one role:

  in       snapshot before the call, byte-identical after it
  out      must be fully written
  inout    an accumulator the contract adds into (seeded with the same values in both runs)
  ws       scratch written before it is read within the call
  ws-seq   state the contract carries from one call of the case to the next (neo_mt_count -> neo_mt_emit, a training forward -> its
           backward, the sort buffers of the *_bwd_det entry points, whose layout the header documents); never poisoned between those calls

Each case runs twice with the same inputs: run A fills `out` (and poisonable `ws` / `ws-seq`) interiors with 0x00, run B with 0xFF,
which is NaN in fp32, fp16 and bf16.  A workspace is poisoned only if its carve holds nothing but floating-point data; one that holds
indices, counts or keys is zero-filled in both runs, so that a missing write can never turn into an out-of-range load.  Run B also runs on
a fresh torch.cuda.Stream with its fills enqueued there and no device synchronisation before the call, so a launch on another stream shows
up as a mismatch.  Checks: every `out` bit-identical between the runs (holes, reads of unwritten workspace), every guard band intact
(writes before or past a buffer, an under-reported workspace), every `in` unchanged, and run A's outputs bit-identical to the production
wrapper's at the same inputs where a wrapper exists.

The coverage test (no GPU) holds the table to include/neo360_b200.h: every name of `_lib.SYMBOLS` has a case or an exclusion with a reason.
Run with `-m gpu -s` to see each case's shapes, roles and poisoned workspaces.
"""
import ctypes as C
import functools
import itertools
import zlib

import pytest
import torch

from neo360_b200 import _lib as L

GUARD = 4096          # bytes of guard band on either side of every interior (at least)
ALIGN = 1024          # interior alignment: every alignment the kernels check (16 B, TMA) holds
F32, F16, BF16, I32, I64, F64, U8 = torch.float32, torch.float16, torch.bfloat16, torch.int32, torch.int64, torch.float64, torch.uint8

# symbols without a case, each with its reason
EXCLUDED = {
    "neo_scene_create": "owns its allocations (the scene), no caller buffer to guard; every scene entry point below runs on one",
    "neo_scene_free": "frees the scene's own allocations",
    "neo_scene_bytes": "host query of the scene's own allocations",
    "neo_release_cached": "returns the library's kept scene blocks to the driver; no caller buffer",
    "neo_check_async": "reads the scene's own error flag; no caller buffer",
    "neo_vanilla_create": "owns its allocations (the packed weights), no caller buffer to guard",
    "neo_vanilla_free": "frees the model's own allocations",
    "neo_profile": "profiling counters, no device buffer",
    "neo_profile_read": "profiling counters, host outputs only",
    "neo_tc_enc_column": "pure host code",
    "neo_tc_trap_info": "host string",
    "neo_last_error": "host string",
    "neo_version": "host string",
    "neo_tc_gemm_f16": "checked against sentinels by tests/test_gpu_tc_kernels.py::test_gemm_f16_vs_float64 and ::test_gemm_f16_call_patterns",
    "neo_tc_rowdot_f16": "checked against sentinels by tests/test_gpu_tc_paths.py::test_rowdot_f16_vs_float64",
}


# ------------------------------------------------------------------------------------------------ buffers and cases

class Buf:
    def __init__(self, role, nbytes, data=None, poison=False, why="", exact=True, shape=None, out_cols=None):
        self.role, self.nbytes, self.data, self.poison, self.why, self.exact, self.shape = role, int(nbytes), data, poison, why, exact, shape
        self.out_cols = out_cols        # (row bytes, first written byte of a row): an `inout` whose columns from there on are `out`


def _bytes(t):
    return t.detach().contiguous().reshape(-1).view(U8)


def In(t):
    return Buf("in", t.numel() * t.element_size(), data=t.contiguous(), shape=tuple(t.shape))


def InOut(t, why, exact=True, out_from_col=None):
    """exact=False: the contract adds with atomics in no fixed order, so the two runs agree to rounding only.
    out_from_col=c (2-D t): the call writes columns c.. of every row and must leave columns ..c-1 alone.  Those columns get the `out`
    treatment (0x00 in run A, 0xFF in run B, bit-identical after the call); the others keep the seed and must still hold it."""
    cols = None if out_from_col is None else (t.shape[1] * t.element_size(), out_from_col * t.element_size())
    return Buf("inout", t.numel() * t.element_size(), data=t.contiguous(), why=why, exact=exact, shape=tuple(t.shape), out_cols=cols)


def Out(*shape, dtype=F32):
    n = 1
    for s in shape:
        n *= s
    return Buf("out", n * torch.empty((), dtype=dtype).element_size(), poison=True, shape=shape)


def Ws(nbytes, poison, why):
    return Buf("ws", nbytes, poison=poison, why=why)


def WsSeq(nbytes, poison, why):
    return Buf("ws-seq", nbytes, poison=poison, why=why)


class Spec:
    """ref: the production wrapper's outputs at the same inputs, {buffer name: tensor}; noref: why a case has none."""
    def __init__(self, bufs, call, ref=None, info="", noref=""):
        self.bufs, self.call, self.ref, self.info, self.noref = bufs, call, ref, info, noref


CASES = {}


def case(symbols, **grid):
    """Register fn(dev, **params) -> Spec once per combination of `grid`, covering the entry points `symbols`."""
    def reg(fn):
        keys = list(grid)
        for vals in itertools.product(*[grid[k] for k in keys]) if keys else [()]:
            kw = dict(zip(keys, vals))
            cid = fn.__name__ + ("[" + ",".join(f"{k}={v}" for k, v in kw.items()) + "]" if kw else "")
            CASES[cid] = (tuple(symbols), fn, kw)
        return fn
    return reg


def chk(rc):
    L.check(rc)


def gen(seed_text):
    return torch.Generator().manual_seed(zlib.crc32(seed_text.encode()))


def rnd(g, dev, *shape, lo=-1.0, hi=1.0, dtype=F32):
    return (torch.rand(shape, generator=g) * (hi - lo) + lo).to(dtype).to(dev)


def rays_in_sphere(g, dev, n):
    """Rays from inside the unit sphere, unit directions, and their far."""
    from oracle import neo360_oracle as orc
    o = (torch.rand(n, 3, generator=g) - 0.5) * 1.0
    d = torch.randn(n, 3, generator=g)
    d = d / d.norm(dim=-1, keepdim=True)
    far = orc.intersect_sphere(o, d).float().reshape(n)
    return o.to(dev), d.to(dev), far.to(dev)


def neo_rays(P, n, chunk=0, order=None):
    r = L.NeoRays()
    r.n_rays, r.chunk = n, chunk
    r.rays_o, r.rays_d, r.viewdirs = P["rays_o"], P["rays_d"], P["viewdirs"]
    r.ray_order = P.get(order) if order else None
    return r


def set_struct(S, P, prefix, keys):
    for k in keys:
        name, _, i = k.partition(".")
        if i:
            getattr(S, name)[int(i)] = P[f"{prefix}:{k}"]
        else:
            setattr(S, name, P[f"{prefix}:{k}"])
    return S


def struct_ins(prefix, tensors):
    """Guarded `in` buffers for the weights a parameter struct points at: {prefix:key: In(t)}."""
    return {f"{prefix}:{k}": In(t) for k, t in tensors.items()}


def ptrs5(P, names):
    return (C.c_void_p * 5)(*[P[n] for n in names])


AUTOGRAD = "its wrapper is an autograd function of a training step, which allocates around it"


# ------------------------------------------------------------------------------------------------ the harness

@functools.lru_cache(maxsize=None)
def _pattern(dev):
    return ((torch.arange(GUARD + ALIGN, dtype=torch.int64) * 151 + 89) % 251).to(U8).to(dev)


def _run(spec, fill, dev, stream):
    """One run: allocate and fill every guarded buffer on `stream`, make the call there, return {name: (raw, offset)}."""
    pat = _pattern(dev)
    raws = {}
    with torch.cuda.stream(stream):
        P = {}
        for name, b in spec.bufs.items():
            if b.nbytes == 0:
                P[name] = None
                continue
            raw = torch.empty(b.nbytes + 2 * GUARD + ALIGN, dtype=U8, device=dev)
            off = GUARD + (-(raw.data_ptr() + GUARD)) % ALIGN
            raw[:off].copy_(pat[:off])
            raw[off + b.nbytes:].copy_(pat[:raw.numel() - off - b.nbytes])
            it = raw[off:off + b.nbytes]
            if b.role in ("in", "inout"):
                it.copy_(_bytes(b.data))
                if b.out_cols:
                    it.view(-1, b.out_cols[0])[:, b.out_cols[1]:].fill_(fill)
            else:
                it.fill_(fill if b.poison else 0)
            raws[name] = (raw, off)
            P[name] = it.data_ptr()
        spec.call(P, stream.cuda_stream)
    stream.synchronize()
    return raws


def _first_bad(a, b):
    bad = (a != b).nonzero()
    return int(bad[0]) if bad.numel() else -1


def _check_guards(spec, raws, run):
    pat = _pattern(next(iter(raws.values()))[0].device) if raws else None
    for name, (raw, off) in raws.items():
        n = spec.bufs[name].nbytes
        front, back = raw[:off], raw[off + n:]
        i = _first_bad(front, pat[:off])
        assert i < 0, f"run {run}: {name} ({spec.bufs[name].role}): front guard band written at byte {i - off} of the interior"
        i = _first_bad(back, pat[:back.numel()])
        assert i < 0, f"run {run}: {name} ({spec.bufs[name].role}, {n} bytes): back guard band written at byte {n + i} (offset {i} past the end)"


def _interior(raws, spec, name):
    raw, off = raws[name]
    return raw[off:off + spec.bufs[name].nbytes]


def _describe(b, name, a, bb):
    """First differing fp32 element of an output (as fp32 when it is 4-byte sized)."""
    d = (a != bb).nonzero()
    i = int(d[0])
    return f"{name} ({b.role}, {b.nbytes} bytes, shape {b.shape}): {int(d.numel())} bytes differ between runs, first at byte {i} " \
           f"(element {i // 4} if fp32)"


def run_case(cid, dev):
    symbols, fn, kw = CASES[cid]
    spec = fn(dev, **kw)
    assert spec.ref is not None or spec.noref, f"{cid}: compare with the production wrapper, or say why there is none"
    roles = ", ".join(f"{k}:{b.role}" + ("+out columns" if b.out_cols else "") for k, b in spec.bufs.items() if ":" not in k)
    n_w = sum(1 for k in spec.bufs if ":" in k)
    poisoned = [k for k, b in spec.bufs.items() if b.role in ("ws", "ws-seq") and b.poison]
    zeroed = [k for k, b in spec.bufs.items() if b.role in ("ws", "ws-seq") and not b.poison]
    print(f"\n{cid}: {spec.info}\n  roles {roles}" + (f" (+{n_w} weight buffers: in)" if n_w else "") +
          f"\n  poisoned ws: {poisoned or '-'}; zero-filled ws: {zeroed or '-'}" +
          ("\n  wrapper: compared" if spec.ref is not None else f"\n  wrapper: none compared ({spec.noref})"))
    torch.cuda.synchronize()
    ra = _run(spec, 0x00, dev, torch.cuda.current_stream())
    rb = _run(spec, 0xFF, dev, torch.cuda.Stream(dev))
    _check_guards(spec, ra, "A")
    _check_guards(spec, rb, "B")
    for name, b in spec.bufs.items():
        if b.nbytes == 0:
            continue
        a, bb = _interior(ra, spec, name), _interior(rb, spec, name)
        if b.role == "in":
            for run, x in (("A", a), ("B", bb)):
                i = _first_bad(x, _bytes(b.data))
                assert i < 0, f"run {run}: input {name} written at byte {i}"
        elif b.out_cols:
            rb_, c0 = b.out_cols
            a2, b2, seed = a.view(-1, rb_), bb.view(-1, rb_), _bytes(b.data).view(-1, rb_)
            assert torch.equal(a2[:, c0:], b2[:, c0:]), _describe(b, name, a2[:, c0:].reshape(-1), b2[:, c0:].reshape(-1)) + " (written columns)"
            for run, x in (("A", a2), ("B", b2)):
                assert torch.equal(x[:, :c0], seed[:, :c0]), f"run {run}: {name}: columns before byte {c0} of a row were written"
        elif b.role == "out" or (b.role == "inout" and b.exact):
            assert torch.equal(a, bb), _describe(b, name, a, bb)
        elif b.role == "inout":
            x, y = a.view(b.data.dtype).double(), bb.view(b.data.dtype).double()
            assert not (y.isnan() & ~x.isnan()).any(), f"{name}: NaN in run B only"
            tol = 1e-5 * float(x.abs().max())           # sums of many terms in no fixed order: rounding of the largest magnitude
            assert float((x - y).abs().max()) <= tol, f"{name}: runs differ by {float((x - y).abs().max())} (> {tol})"
    if spec.ref is not None:
        with torch.no_grad():
            ref = spec.ref()
        torch.cuda.synchronize()
        for name, t in ref.items():
            got = _interior(ra, spec, name)
            want = _bytes(t)
            assert got.numel() == want.numel(), f"{name}: wrapper output has {want.numel()} bytes, the case {got.numel()}"
            assert torch.equal(got, want), f"{name}: run A differs from the production wrapper at byte {_first_bad(got, want)}"
    return spec


# ------------------------------------------------------------------------------------------------ NeO-360 scenes

@functools.lru_cache(maxsize=None)
def neo_net(nv):
    """NeRF_TP (8 + 4 samples) with a scene prepared for both precisions: image 37 x 23, planes 13 x 17, latent 18 x 11."""
    from neo360_b200 import NeRF_TP, synth
    dev = torch.device("cuda:0")
    sc = synth.make_scene((37, 23), nv, (13, 17), 40 + nv)
    net = NeRF_TP(num_coarse_samples=8, num_fine_samples=4, num_src_views=nv, precision="tc").eval()
    net.load_state_dict(synth.make_mlp_params(40 + nv))
    net = net.to(dev)
    net.set_scene(*[sc[k].to(dev) for k in ("planes_xz", "planes_xy", "planes_yz", "latent", "src_poses", "src_focal", "src_c")],
                  sc["img_wh"], precisions=["fp32", "tc"])
    return net


def _scene_geom(net):
    a = net._scene_inputs
    return a[0].shape[2], a[0].shape[3], a[3].shape[2], a[3].shape[3]     # plane_h, plane_w, lat_h, lat_w


def _ray_bufs(g, dev, n, with_order=False):
    o, d, far = rays_in_sphere(g, dev, n)
    bufs = {"rays_o": In(o), "rays_d": In(d), "viewdirs": In(d)}
    if with_order:
        bufs["ray_order"] = In(torch.randperm(n, generator=g).to(I32).to(dev))
    return bufs, {"rays_o": o, "rays_d": d, "viewdirs": d}, far


# n = 1 and ragged against the 32-ray x 2-sample TC tiles and the 8- and 4-point fp32 tiles (NV <= 6 / >= 7)
@case(["neo_field_eval"], nv=[1, 8], prec=["fp32", "tc"], mlp=[0, 1], n=[1, 33])
def field_eval(dev, nv, prec, mlp, n):
    net = neo_net(nv)
    g = gen(f"field{nv}{prec}{mlp}{n}")
    N = 7
    bufs, rays, far = _ray_bufs(g, dev, n, with_order=(prec == "tc"))
    u = torch.sort(torch.rand(n, N, generator=g), -1).values.to(dev)
    t = torch.flip(u, [-1]) if mlp & 1 else u * far[:, None] * 1.2
    bufs.update({"far": In(far), "t": In(t), "rgb": Out(n, N, 3), "sigma": Out(n, N)})
    pr = L.NEO_PREC_TC if prec == "tc" else L.NEO_PREC_FP32

    def call(P, s):
        r = neo_rays(P, n, order="ray_order" if prec == "tc" else None)
        chk(L.load().neo_field_eval(net._scene.handle, C.byref(r), P["far"], P["t"], N, mlp, pr, P["rgb"], P["sigma"], s))

    def ref():
        rgb, sig = net.field_eval(rays, far, t, mlp, precision=prec, ray_order=bufs["ray_order"].data if prec == "tc" else None)
        return {"rgb": rgb, "sigma": sig}
    return Spec(bufs, call, ref, f"nv {nv} {prec} mlp {mlp}: {n} rays x {N} samples")


@case(["neo_tc_dir_fragments"], nv=[1, 8], n=[1, 33])
def dir_fragments(dev, nv, n):
    net = neo_net(nv)
    bufs, _, _ = _ray_bufs(gen(f"dir{nv}{n}"), dev, n)
    bufs["out"] = Out(n * 64, dtype=U8)
    return Spec(bufs, lambda P, s: chk(L.load().neo_tc_dir_fragments(net._scene.handle, C.byref(neo_rays(P, n)), P["out"], s)),
                info=f"nv {nv}: {n} rays x 64 bytes", noref="no wrapper: neo_render_fwd and neo_field_eval build the fragments themselves")


@case(["neo_render_workspace_bytes", "neo_render_fwd"], prec=["fp32", "tc"], outs=["all", "min"], rand=[0, 1], n=[1, 33])
def render(dev, prec, outs, rand, n):
    net = neo_net(3 if n > 1 else 1)
    g = gen(f"render{prec}{outs}{rand}{n}")
    nc, nf = net.num_coarse_samples, net.num_fine_samples
    N = (nc + 1, nc + 1 + nf)
    bufs, rays, _ = _ray_bufs(g, dev, n)
    u = [torch.rand(n, k, generator=g).to(dev) for k in (nc + 1, nc + 1, nf, nf)] if rand else None
    if rand:
        bufs.update({f"u{i}": In(x) for i, x in enumerate(u)})
    cfg = L.NeoCfg()
    cfg.n_coarse, cfg.n_fine, cfg.white_bkgd, cfg.out_depth = nc, nf, 0, 1
    cfg.precision = L.NEO_PREC_TC if prec == "tc" else L.NEO_PREC_FP32
    need = L.load().neo_render_workspace_bytes(n, C.byref(cfg))
    bufs["ws"] = Ws(need, True, "floats and fp16 direction fragments")
    shapes = {"comp_rgb": (3,), "fg_rgb": (3,), "bg_rgb": (3,), "fg_acc": (), "bg_lambda": (1,), "depth": (), "bg_acc": (),
              "fg_w": "N", "bg_w": "N", "fg_sdist": "N", "bg_sdist": "N", "fg_t": "N", "bg_s": "N", "fg_sigma": "N", "bg_sigma": "N",
              "fg_rgb_s": "N3", "bg_rgb_s": "N3"}
    names = L.OUT_FIELDS if outs == "all" else ("comp_rgb", "depth")
    for k in names:
        for lvl in range(2):
            sh = shapes[k]
            sh = (N[lvl],) if sh == "N" else ((N[lvl], 3) if sh == "N3" else sh)
            bufs[f"{k}{lvl}"] = Out(n, *sh)

    def call(P, s):
        if rand:
            cfg.u_fg0, cfg.u_bg0, cfg.u_fg1, cfg.u_bg1 = P["u0"], P["u1"], P["u2"], P["u3"]
        out = L.NeoOut()
        for k in names:
            for lvl in range(2):
                getattr(out, k)[lvl] = P[f"{k}{lvl}"]
        chk(L.load().neo_render_fwd(net._scene.handle, C.byref(neo_rays(P, n)), C.byref(cfg), C.byref(out), P["ws"], need, s))

    def ref():
        net.precision = prec
        r = dict(rays)
        if rand:
            r["_uniforms"] = u
        res = net(r, bool(rand), False, None, None, out_depth=True, debug=True)
        got = {}
        for lvl in range(2):
            got.update({f"comp_rgb{lvl}": res[lvl][0], f"depth{lvl}": res[lvl][5]})
            if outs == "all":
                got.update({f"{k}{lvl}": v[lvl] for k, v in net.last_debug.items()})
        return got
    return Spec(bufs, call, ref, f"{prec}, outputs {outs}, randomized {rand}: {n} rays, N {N}")


# ------------------------------------------------------------------------------------------------ NeO-360 lookups

def _pts(g, dev, M):
    return ((torch.rand(M, 3, generator=g) - 0.5) * 2.2).to(dev)


@case(["neo_index_maps"], nv=[1, 8], C=[4, 128])
def index_maps(dev, nv, C):
    net = neo_net(nv)
    ph, pw, lh, lw = _scene_geom(net)
    g = gen(f"im{nv}{C}")
    M = 37
    bufs = {"pts": In(_pts(g, dev, M)), "latent": In(rnd(g, dev, nv, lh, lw, C)),
            **{p: In(rnd(g, dev, nv, ph, pw, C)) for p in ("xz", "xy", "yz")},
            "out_local": Out(nv * M, C), "out_world": Out(nv * M, C)}
    return Spec(bufs, lambda P, s: chk(L.load().neo_index_maps(net._scene.handle, P["pts"], M, C, P["latent"], P["xz"], P["xy"], P["yz"],
                                                               P["out_local"], P["out_world"], s)), info=f"nv {nv}, C {C}, M {M}",
                noref="its wrappers are the autograd lookups of training.py and pixelnerf.py, which take whole batches")


@case(["neo_index_maps_bwd", "neo_index_maps_bwd_det_workspace_bytes", "neo_index_maps_bwd_det"], nv=[1, 8], C=[4, 128], det=[0, 1])
def index_maps_bwd(dev, nv, C, det):
    net = neo_net(nv)
    ph, pw, lh, lw = _scene_geom(net)
    g = gen(f"imb{nv}{C}{det}")
    M = 37
    why = "gradient maps: the contract accumulates into them"
    bufs = {"pts": In(_pts(g, dev, M)), "g_local": In(rnd(g, dev, nv * M, C)), "g_world": In(rnd(g, dev, nv * M, C)),
            "g_latent": InOut(rnd(g, dev, nv, lh, lw, C), why, exact=bool(det)),
            **{p: InOut(rnd(g, dev, nv, ph, pw, C), why, exact=bool(det)) for p in ("g_xz", "g_xy", "g_yz")}}
    lib = L.load()
    if det:
        need = lib.neo_index_maps_bwd_det_workspace_bytes(net._scene.handle, M, C)
        bufs["ws"] = WsSeq(need, False, "keys, entry ids, segment starts and sort scratch: integers, a documented layout")

    def call(P, s):
        a = (net._scene.handle, P["pts"], M, C, P["g_local"], P["g_world"], P["g_latent"], P["g_xz"], P["g_xy"], P["g_yz"])
        chk(lib.neo_index_maps_bwd_det(*a, P["ws"], need, s) if det else lib.neo_index_maps_bwd(*a, s))
    return Spec(bufs, call, info=f"nv {nv}, C {C}, M {M}, {'deterministic' if det else 'atomic'}",
                noref="the backward of the autograd lookups of training.py and pixelnerf.py")


@case(["neo_index_grid", "neo_index_local"], nv=[1, 8])
def index_scene(dev, nv):
    net = neo_net(nv)
    g = gen(f"is{nv}")
    M = 37
    pts = _pts(g, dev, M)
    bufs = {"pts": In(pts), "grid": Out(nv * M, 128), "local": Out(nv * M, 512)}

    def call(P, s):
        chk(L.load().neo_index_grid(net._scene.handle, P["pts"], M, P["grid"], s))
        chk(L.load().neo_index_local(net._scene.handle, P["pts"], M, P["local"], s))
    return Spec(bufs, call, lambda: {"grid": net.index_grid(pts), "local": net.get_local_feats(pts)}, f"nv {nv}, M {M}")


@case(["neo_index_grid_bwd", "neo_index_local_bwd"], nv=[1, 8])
def index_scene_bwd(dev, nv):
    net = neo_net(nv)
    ph, pw, lh, lw = _scene_geom(net)
    g = gen(f"isb{nv}")
    M = 37
    why = "gradient maps: the contract accumulates into them (vector atomics)"
    bufs = {"pts": In(_pts(g, dev, M)), "g_grid": In(rnd(g, dev, nv * M, 128)), "g_local": In(rnd(g, dev, nv * M, 512)),
            **{p: InOut(rnd(g, dev, nv, ph, pw, 128), why, exact=False) for p in ("g_xz", "g_xy", "g_yz")},
            "g_latent": InOut(rnd(g, dev, nv, lh, lw, 512), why, exact=False)}

    def call(P, s):
        chk(L.load().neo_index_grid_bwd(net._scene.handle, P["pts"], M, P["g_grid"], P["g_xz"], P["g_xy"], P["g_yz"], s))
        chk(L.load().neo_index_local_bwd(net._scene.handle, P["pts"], M, P["g_local"], P["g_latent"], s))
    return Spec(bufs, call, info=f"nv {nv}, M {M}", noref="the backward of the reference-formulation lookups of training.py")


# ------------------------------------------------------------------------------------------------ NeO-360 stages

@case(["neo_get_rays"], hw=[(2, 1), (23, 37)])
def get_rays(dev, hw):
    from neo360_b200 import ops, synth
    H, W = hw
    c2w = synth.target_pose(5)[:3, :4].contiguous().to(dev)
    n = H * W
    bufs = {"c2w": In(c2w), "o": Out(n, 3), "vd": Out(n, 3), "rd": Out(n, 3), "radii": Out(n)}

    def ref():
        o, vd, rd, rad = ops.get_rays(H, W, 0.8 * W, c2w)
        return {"o": o, "vd": vd, "rd": rd, "radii": rad}
    return Spec(bufs, lambda P, s: chk(L.load().neo_get_rays(H, W, 0.8 * W, P["c2w"], P["o"], P["vd"], P["rd"], P["radii"], s)), ref,
                f"{H} x {W}")


def _pix(g, dev, n, T, H, W):
    return torch.randint(0, T * H * W, (n,), generator=g).to(I64).to(dev)


@case(["neo_sample_rays"], n=[1, 257])
def sample_rays(dev, n):
    from neo360_b200 import ops, synth
    g = gen(f"sr{n}")
    T, H, W = 3, 11, 13
    c2w = torch.stack([synth.target_pose(v)[:3, :4] for v in range(T)]).contiguous().to(dev)
    pix, img = _pix(g, dev, n, T, H, W), rnd(g, dev, T, H, W, 3, lo=0.0)
    bufs = {"pix": In(pix), "c2w": In(c2w), "img": In(img), "o": Out(n, 3), "vd": Out(n, 3), "rd": Out(n, 3), "radii": Out(n, 1),
            "target": Out(n, 3), "err": InOut(torch.zeros(1, dtype=I32, device=dev), "error flag: raised only on a bad index")}

    def call(P, s):
        chk(L.load().neo_sample_rays(n, P["pix"], T, H, W, 9.0, P["c2w"], P["img"], P["o"], P["vd"], P["rd"], P["radii"], P["target"],
                                     P["err"], s))

    def ref():
        o, vd, rd, rad, tgt = ops.sample_rays(pix, H, W, 9.0, c2w, img)
        return {"o": o, "vd": vd, "rd": rd, "radii": rad, "target": tgt}
    return Spec(bufs, call, ref, f"{n} rays of {T} views {H} x {W}")


@case(["neo_sample_rays_bwd_workspace_bytes", "neo_sample_rays_bwd"], n=[1, 257, 4099], T=[1, 3])
def sample_rays_bwd(dev, n, T):
    from neo360_b200 import synth
    g = gen(f"srb{n}{T}")
    H, W = 11, 13
    c2w = torch.stack([synth.target_pose(v)[:3, :4] for v in range(T)]).contiguous().to(dev)
    need = L.load().neo_sample_rays_bwd_workspace_bytes(n, T)
    bufs = {"pix": In(_pix(g, dev, n, T, H, W)), "c2w": In(c2w), "g_o": In(rnd(g, dev, n, 3)), "g_vd": In(rnd(g, dev, n, 3)),
            "g_rd": In(rnd(g, dev, n, 3)), "g_c2w": Out(T, 3, 4), "ws": Ws(need, True, "per-ray terms and per-block partials (floats) and each ray's view index (int): the index is only "
                                   "compared with a view, never used as an address, and 0xFF reads as -1, the kernel's own invalid-ray mark")}
    return Spec(bufs, lambda P, s: chk(L.load().neo_sample_rays_bwd(n, P["pix"], T, H, W, 9.0, P["c2w"], P["g_o"], P["g_vd"], P["g_rd"],
                                                                    P["g_c2w"], P["ws"], need, s)), info=f"{n} rays, {T} views",
                noref="its wrapper is the backward of ops.sample_rays under autograd")


@case(["neo_intersect_sphere"], n=[1, 257])
def intersect_sphere(dev, n):
    from neo360_b200 import ops
    o, d, _ = rays_in_sphere(gen(f"is{n}"), dev, n)
    bufs = {"o": In(o), "d": In(d), "far": Out(n), "err": InOut(torch.zeros(1, dtype=I32, device=dev), "error flag: raised on a miss")}
    return Spec(bufs, lambda P, s: chk(L.load().neo_intersect_sphere(P["o"], P["d"], n, P["far"], P["err"], s)),
                lambda: {"far": ops.intersect_sphere(o, d)}, f"{n} rays")


@case(["neo_sample_along_rays"], in_sphere=[0, 1], rand=[0, 1], n=[1, 129])
def sample_along_rays(dev, in_sphere, rand, n):
    g = gen(f"sar{in_sphere}{rand}{n}")
    o, d, far = rays_in_sphere(g, dev, n)
    S = 9
    bufs = {"o": In(o), "d": In(d), "far": In(far), "t": Out(n, S + 1), "pts": Out(n, S + 1, 3 if in_sphere else 4)}
    if not in_sphere:
        bufs["lin"] = Out(n, S + 1, 3)
    if rand:
        bufs["u"] = In(rnd(g, dev, n, S + 1, lo=0.0))
    def ref():
        from neo360_b200 import ops
        r = ops.sample_along_rays(o, d, S, 1e-4, far, bool(rand), False, bool(in_sphere), far_uncontracted=3.0,
                                  u_rand=bufs["u"].data if rand else None)
        return dict(zip(("t", "pts", "lin"), r))
    return Spec(bufs, lambda P, s: chk(L.load().neo_sample_along_rays(P["o"], P["d"], P["far"], n, S, in_sphere, 3.0, P.get("u"), P["t"],
                                                                      P["pts"], P.get("lin"), s)), ref, f"{n} rays, {S}+1 samples")


@case(["neo_sample_pdf"], in_sphere=[0, 1], rand=[0, 1], n=[1, 129])
def sample_pdf(dev, in_sphere, rand, n):
    g = gen(f"spdf{in_sphere}{rand}{n}")
    o, d, far = rays_in_sphere(g, dev, n)
    n_old, m = 9, 7
    t = torch.sort(torch.rand(n, n_old, generator=g), -1).values.to(dev)
    t = t * far[:, None] if in_sphere else torch.flip(t, [-1])
    bufs = {"o": In(o), "d": In(d), "far": In(far), "t_old": In(t), "w": In(rnd(g, dev, n, n_old, lo=0.0)),
            "t": Out(n, n_old + m), "pts": Out(n, n_old + m, 3 if in_sphere else 4)}
    if not in_sphere:
        bufs["lin"] = Out(n, n_old + m, 3)
    if rand:
        bufs["u"] = In(rnd(g, dev, n, m, lo=0.0))
    def ref():
        from neo360_b200 import ops
        r = ops.sample_pdf(bufs["t_old"].data, bufs["w"].data, o, d, m, bool(rand), bool(in_sphere), far, far_uncontracted=3.0,
                           u_rand=bufs["u"].data if rand else None)
        return dict(zip(("t", "pts", "lin"), r))
    return Spec(bufs, lambda P, s: chk(L.load().neo_sample_pdf(P["o"], P["d"], P["far"], P["t_old"], P["w"], n, n_old, m, in_sphere, 3.0,
                                                               P.get("u"), P["t"], P["pts"], P.get("lin"), s)), ref,
                f"{n} rays, {n_old} + {m} samples")


def _composite_inputs(g, dev, n, N, mode):
    o, d, far = rays_in_sphere(g, dev, n)
    t = torch.sort(torch.rand(n, N, generator=g), -1).values.to(dev)
    t = torch.flip(t, [-1]) if mode == 0 else t * far[:, None]
    return {"rgb": In(rnd(g, dev, n, N, 3, lo=0.0)), "sigma": In(rnd(g, dev, n, N, lo=0.0, hi=5.0)), "t": In(t), "d": In(d), "far": In(far)}


@case(["neo_volumetric_rendering"], mode=[0, 1, 2], n=[1, 129])
def volumetric_rendering(dev, mode, n):
    N = 13
    bufs = _composite_inputs(gen(f"vr{mode}{n}"), dev, n, N, mode)
    bufs.update({"comp": Out(n, 3), "acc": Out(n), "w": Out(n, N), "depth": Out(n)})
    if mode == 1:
        bufs["lam"] = Out(n)                       # the foreground's 1 - acc: the background composite and mode 2 take none
    def ref():
        from neo360_b200 import ops
        x = {k: bufs[k].data for k in ("rgb", "sigma", "t", "d", "far")}
        r = ops.volumetric_rendering(x["rgb"], x["sigma"], x["t"], x["d"], True, bool(mode), x["far"], out_depth=True)
        return {k: v for k, v in zip(("comp", "acc", "w", "lam", "depth"), r) if v is not None}
    return Spec(bufs, lambda P, s: chk(L.load().neo_volumetric_rendering(P["rgb"], P["sigma"], P["t"], P["d"], P["far"], n, N, 1, mode,
                                                                         P["comp"], P["acc"], P["w"], P.get("lam"), P["depth"], s)),
                ref if mode < 2 else None, f"mode {mode}: {n} rays x {N}",
                noref="ops.volumetric_rendering covers modes 0 and 1; mode 2 is called inside vanilla NeRF's and PixelNeRF's forward")


@case(["neo_volumetric_rendering_bwd"], mode=[0, 1], n=[1, 129])
def volumetric_rendering_bwd(dev, mode, n):
    N = 13
    g = gen(f"vrb{mode}{n}")
    bufs = _composite_inputs(g, dev, n, N, mode)
    bufs.update({"g_comp": In(rnd(g, dev, n, 3)), "g_acc": In(rnd(g, dev, n)), "g_w": In(rnd(g, dev, n, N)), "g_lam": In(rnd(g, dev, n)),
                 "g_depth": In(rnd(g, dev, n)), "d_rgb": Out(n, N, 3), "d_sigma": Out(n, N)})
    return Spec(bufs, lambda P, s: chk(L.load().neo_volumetric_rendering_bwd(
        P["rgb"], P["sigma"], P["t"], P["d"], P["far"], n, N, 1, mode, P["g_comp"], P["g_acc"], P["g_w"], P["g_lam"], P["g_depth"],
        P["d_rgb"], P["d_sigma"], s)), info=f"mode {mode}: {n} rays x {N}", noref=AUTOGRAD)


@case(["neo_vanilla_composite_bwd"], n=[1, 129])
def vanilla_composite_bwd(dev, n):
    N = 13
    g = gen(f"vcb{n}")
    bufs = _composite_inputs(g, dev, n, N, 2)
    del bufs["far"]
    bufs.update({"g_comp": In(rnd(g, dev, n, 3)), "g_acc": In(rnd(g, dev, n)), "g_w": In(rnd(g, dev, n, N)), "g_depth": In(rnd(g, dev, n)),
                 "d_rgb": Out(n, N, 3), "d_sigma": Out(n, N)})
    return Spec(bufs, lambda P, s: chk(L.load().neo_vanilla_composite_bwd(P["rgb"], P["sigma"], P["t"], P["d"], n, N, 1, P["g_comp"], P["g_acc"],
                                                                          P["g_w"], P["g_depth"], P["d_rgb"], P["d_sigma"], s)),
                info=f"{n} rays x {N}", noref=AUTOGRAD)


@case(["neo_clipped_sq_err", "neo_clipped_sq_err_masked"], n=[1, 4099])
def clipped_sq_err(dev, n):
    g = gen(f"cse{n}")
    why = "sum and count: the contract adds into them (double atomics)"
    bufs = {"pred": In(rnd(g, dev, n, 3, lo=-0.2, hi=1.2)), "gt": In(rnd(g, dev, n, 3, lo=0.0)),
            "mask": In((torch.rand(n, generator=g) < 0.5).to(U8).to(dev)),
            "sum": InOut(torch.rand(1, generator=g, dtype=F64).to(dev), why, exact=False),
            "msum": InOut(torch.rand(1, generator=g, dtype=F64).to(dev), why, exact=False),
            "mcount": InOut(torch.tensor([7], dtype=I64, device=dev), why)}

    def call(P, s):
        chk(L.load().neo_clipped_sq_err(P["pred"], P["gt"], 3 * n, P["sum"], s))
        chk(L.load().neo_clipped_sq_err_masked(P["pred"], P["gt"], P["mask"], n, P["msum"], P["mcount"], s))
    return Spec(bufs, call, info=f"{n} pixels", noref="output.psnr zeroes its own accumulator and returns a host float")


@case(["neo_ssim_workspace_bytes", "neo_ssim"], nhw=[(1, 11, 11), (3, 23, 37)])
def ssim(dev, nhw):
    from neo360_b200 import output
    n, H, W = nhw
    g = gen(f"ssim{nhw}")
    a, b = rnd(g, dev, n, H, W, 3, lo=-0.1, hi=1.1), rnd(g, dev, n, H, W, 3, lo=0.0)
    need = L.load().neo_ssim_workspace_bytes(n, H, W)
    bufs = {"pred": In(a), "gt": In(b), "ssim": Out(n, dtype=F64), "map": Out(n, H - 10, W - 10, 3),
            "ws": Ws(need, True, "filtered moments and partial sums: floats and doubles")}

    def ref():
        v, m = output.ssim_batch(a, b, return_map=True)
        return {"ssim": v, "map": m}
    return Spec(bufs, lambda P, s: chk(L.load().neo_ssim(P["pred"], P["gt"], n, H, W, P["ssim"], P["map"], P["ws"], need, s)), ref,
                f"{n} frames {H} x {W}")


LPIPS_C = (64, 128, 256, 512, 512)


def _lpips_bufs(g, dev, n, H, W):
    bufs = {}
    for k, c in enumerate(LPIPS_C):
        bufs[f"fx{k}"] = In(rnd(g, dev, n, c, H >> k, W >> k))
        bufs[f"fy{k}"] = In(rnd(g, dev, n, c, H >> k, W >> k))
        bufs[f"w{k}"] = In(rnd(g, dev, c, lo=0.0))
    return bufs


@case(["neo_lpips_workspace_bytes", "neo_lpips_head"], nhw=[(1, 16, 16), (2, 19, 23)])
def lpips_head(dev, nhw):
    from neo360_b200 import lpips
    n, H, W = nhw
    bufs = _lpips_bufs(gen(f"lp{nhw}"), dev, n, H, W)
    need = L.load().neo_lpips_workspace_bytes(n, H, W)
    bufs.update({"lpips": Out(n, dtype=F64), "per_layer": Out(n, 5, dtype=F64), "ws": Ws(need, True, "per-pixel distances and partial sums: floats")})
    names = lambda p: [f"{p}{k}" for k in range(5)]

    def ref():
        v, lay = lpips.head(*[[bufs[x].data for x in names(p)] for p in ("fx", "fy", "w")], per_layer=True)
        return {"lpips": v, "per_layer": lay}
    return Spec(bufs, lambda P, s: chk(L.load().neo_lpips_head(ptrs5(P, names("fx")), ptrs5(P, names("fy")), ptrs5(P, names("w")), n, H, W,
                                                               P["lpips"], P["per_layer"], P["ws"], need, s)), ref, f"{n} frames {H} x {W}")


@case(["neo_lpips_head_bwd"], nhw=[(1, 16, 16), (2, 19, 23)])
def lpips_head_bwd(dev, nhw):
    n, H, W = nhw
    g = gen(f"lpb{nhw}")
    bufs = _lpips_bufs(g, dev, n, H, W)
    bufs["g"] = In(rnd(g, dev, n))
    for k, c in enumerate(LPIPS_C):
        bufs[f"gx{k}"] = Out(n, c, H >> k, W >> k)
        bufs[f"gy{k}"] = Out(n, c, H >> k, W >> k)
    nm = lambda p: [f"{p}{k}" for k in range(5)]

    def ref():
        from neo360_b200 import lpips
        gx, gy = lpips.head_bwd(*[[bufs[x].data for x in nm(p)] for p in ("fx", "fy", "w")], bufs["g"].data, with_y=True)
        return {**{f"gx{k}": t for k, t in enumerate(gx)}, **{f"gy{k}": t for k, t in enumerate(gy)}}
    return Spec(bufs, lambda P, s: chk(L.load().neo_lpips_head_bwd(ptrs5(P, nm("fx")), ptrs5(P, nm("fy")), ptrs5(P, nm("w")), n, H, W, P["g"],
                                                                   ptrs5(P, nm("gx")), ptrs5(P, nm("gy")), s)), ref, f"{n} frames {H} x {W}")


@case(["neo_lpips_prepare", "neo_lpips_prepare_bwd"], form=[0, 1], nhw=[(1, 16, 16), (2, 19, 23)])
def lpips_prepare(dev, form, nhw):
    n, H, W = nhw
    g = gen(f"lpp{form}{nhw}")
    bufs = {"img": In(rnd(g, dev, n, H, W, 3, lo=-0.1, hi=1.1)), "g_out": In(rnd(g, dev, n, 3, H, W)), "out": Out(n, 3, H, W),
            "g_img": Out(n, H, W, 3)}

    def call(P, s):
        chk(L.load().neo_lpips_prepare(P["img"], n, H, W, form, P["out"], s))
        chk(L.load().neo_lpips_prepare_bwd(P["img"], P["g_out"], n, H, W, form, P["g_img"], s))

    def ref():
        from neo360_b200 import lpips
        with torch.enable_grad():
            img = bufs["img"].data.clone().requires_grad_(True)
            out = lpips.prepare(img, form)
            out.backward(bufs["g_out"].data)
        return {"out": out.detach(), "g_img": img.grad}
    return Spec(bufs, call, ref, f"form {form}, {n} frames {H} x {W}")


# ------------------------------------------------------------------------------------------------ mesh

MESH_BOX = ((-1.1, -1.0, -0.9), (1.0, 1.1, 0.9))


def _mesh_grid(shape):
    from neo360_b200 import mesh
    return mesh.make_grid(shape, MESH_BOX)


def _sphere_sigma(dev, shape, g):
    nz, ny, nx = shape
    z, y, x = torch.meshgrid(torch.linspace(-1, 1, nz), torch.linspace(-1, 1, ny), torch.linspace(-1, 1, nx), indexing="ij")
    return (1.0 - (x * x + y * y + z * z).sqrt() + 0.1 * torch.rand(shape, generator=g)).float().contiguous().to(dev)


@case(["neo_grid_rays", "neo_grid_mask_sphere"], rows=[1, 37])
def grid_rays(dev, rows):
    g = gen(f"gr{rows}")
    grid = _mesh_grid((9, 11, 13))
    row0 = 5
    bufs = {"o": Out(rows, 3), "dirs": Out(rows, 3), "t": Out(rows, grid.nx),
            "sigma": InOut(rnd(g, dev, rows, grid.nx), "density rows masked in place")}

    def call(P, s):
        chk(L.load().neo_grid_rays(C.byref(grid), row0, rows, P["o"], P["dirs"], P["t"], s))
        chk(L.load().neo_grid_mask_sphere(C.byref(grid), row0, rows, P["sigma"], s))
    return Spec(bufs, call, info=f"rows {row0}..{row0 + rows} of a 13 x 11 x 9 grid",
                noref="called inside mesh.density_grid's slab loop, which allocates and evaluates around it")


@case(["neo_mt_workspace_bytes", "neo_mt_count", "neo_mt_emit", "neo_grid_normals"], shape=[(3, 3, 3), (9, 11, 13), (17, 33, 65)])
def marching_tets(dev, shape):
    g = gen(f"mt{shape}")
    grid = _mesh_grid(shape)
    sigma = _sphere_sigma(dev, shape, g)
    lib = L.load()
    need = lib.neo_mt_workspace_bytes(C.byref(grid))
    ws = torch.zeros(need, dtype=U8, device=dev)
    nv_, nf_ = C.c_int(), C.c_int()
    s0 = torch.cuda.current_stream().cuda_stream
    chk(lib.neo_mt_count(L.ptr(sigma), C.byref(grid), 0.5, ws.data_ptr(), need, C.byref(nv_), C.byref(nf_), s0))
    nV, nF = nv_.value, nf_.value
    bufs = {"sigma": In(sigma), "ws": WsSeq(need, False, "block counts, offsets, vertex bases and masks: integers, neo_mt_count -> neo_mt_emit"),
            "verts": Out(nV, 3), "faces": Out(nF, 3, dtype=I32), "normals": Out(nV, 3)}

    def call(P, s):
        a, b = C.c_int(), C.c_int()
        chk(lib.neo_mt_count(P["sigma"], C.byref(grid), 0.5, P["ws"], need, C.byref(a), C.byref(b), s))
        assert (a.value, b.value) == (nV, nF)
        chk(lib.neo_mt_emit(P["sigma"], C.byref(grid), 0.5, P["ws"], need, P["verts"], nV, P["faces"], nF, s))
        chk(lib.neo_grid_normals(P["sigma"], C.byref(grid), P["verts"], nV, P["normals"], s))
    def ref():
        from neo360_b200 import mesh
        v, f = mesh.marching_tetrahedra(sigma, 0.5, MESH_BOX)
        return {"verts": v, "faces": f, "normals": mesh.grid_normals(sigma, v, MESH_BOX)}
    return Spec(bufs, call, ref, f"grid {shape}: {nV} vertices, {nF} faces")


# ------------------------------------------------------------------------------------------------ vanilla NeRF

@functools.lru_cache(maxsize=None)
def vanilla_net():
    from neo360_b200 import synth
    from neo360_b200.vanilla import NeRF
    net = NeRF(num_coarse_samples=8, num_fine_samples=4).eval()
    net.load_state_dict(synth.make_vanilla_params(7))
    return net.cuda()


def _van_rays(g, dev, n):
    o = (torch.rand(n, 3, generator=g) - 0.5).to(dev)
    d = torch.randn(n, 3, generator=g)
    vd = (d / d.norm(dim=-1, keepdim=True)).to(dev)
    return o, (d * 1.3).to(dev), vd


@case(["neo_vanilla_workspace_bytes", "neo_vanilla_render_fwd"], prec=["fp32", "tc"], rand=[0, 1], n=[1, 33])
def vanilla_render(dev, prec, rand, n):
    net = vanilla_net()
    h = net._ensure(dev)
    g = gen(f"vr{prec}{rand}{n}")
    nc, nf = net.num_coarse_samples, net.num_fine_samples
    N = (nc + 1, nc + 1 + nf)
    o, d, vd = _van_rays(g, dev, n)
    bufs = {"rays_o": In(o), "rays_d": In(d), "viewdirs": In(vd)}
    u = [rnd(g, dev, n, nc + 1, lo=0.0), rnd(g, dev, n, nf, lo=0.0)] if rand else None
    if rand:
        bufs.update({"u0": In(u[0]), "u1": In(u[1])})
    cfg = L.NeoVanillaCfg()
    cfg.n_coarse, cfg.n_fine, cfg.white_bkgd, cfg.near_plane, cfg.far_plane = nc, nf, 1, 0.2, 4.0
    cfg.precision = L.NEO_PREC_TC if prec == "tc" else L.NEO_PREC_FP32
    need = L.load().neo_vanilla_workspace_bytes(n, C.byref(cfg))
    bufs["ws"] = Ws(need, True, "t, weights, field outputs (floats) and the fp16 activation rows")
    shp = {"comp_rgb": (3,), "acc": (), "depth": (), "t": "N", "sigma": "N", "rgb_s": "N3", "weights": "N"}
    for k in L.VANILLA_OUT_FIELDS:
        for lvl in range(2):
            sh = shp[k]
            bufs[f"{k}{lvl}"] = Out(n, *((N[lvl],) if sh == "N" else ((N[lvl], 3) if sh == "N3" else sh)))

    def call(P, s):
        if rand:
            cfg.u0, cfg.u1 = P["u0"], P["u1"]
        out = L.NeoVanillaOut()
        for k in L.VANILLA_OUT_FIELDS:
            for lvl in range(2):
                getattr(out, k)[lvl] = P[f"{k}{lvl}"]
        chk(L.load().neo_vanilla_render_fwd(h, C.byref(neo_rays(P, n)), C.byref(cfg), C.byref(out), P["ws"], need, s))

    def ref():
        net.precision = prec
        r = {"rays_o": o, "rays_d": d, "viewdirs": vd}
        if rand:
            r["_uniforms"] = u
        net(r, bool(rand), True, 0.2, 4.0, debug=True)
        return {f"{k}{lvl}": v[lvl] for k, v in net.last_debug.items() for lvl in range(2)}
    return Spec(bufs, call, ref, f"{prec}, randomized {rand}: {n} rays, N {N} ({n * N[1]} points)")


# 297 points: ragged against enc16's 256 rows, the 128-row gemm tiles and the field kernel's 8-point tiles
@case(["neo_vanilla_field_workspace_bytes", "neo_vanilla_field_eval"], prec=["fp32", "tc"], level=[0, 1], nN=[(1, 5), (33, 9)])
def vanilla_field(dev, prec, level, nN):
    net = vanilla_net()
    h = net._ensure(dev)
    n, N = nN
    g = gen(f"vf{prec}{level}{nN}")
    o, _, vd = _van_rays(g, dev, n)
    t = torch.sort(torch.rand(n, N, generator=g), -1).values.to(dev) * 3.0
    P_ = L.NEO_PREC_TC if prec == "tc" else L.NEO_PREC_FP32
    need = L.load().neo_vanilla_field_workspace_bytes(n * N, P_)
    bufs = {"rays_o": In(o), "viewdirs": In(vd), "t": In(t), "rgb": Out(n, N, 3), "sigma": Out(n, N),
            "ws": Ws(need, True, "fp16 activation rows and fp32 head outputs (none for fp32)")}

    def call(P, s):
        r = L.NeoRays()
        r.n_rays, r.rays_o, r.rays_d, r.viewdirs = n, P["rays_o"], P["viewdirs"], P["viewdirs"]
        chk(L.load().neo_vanilla_field_eval(h, C.byref(r), P["t"], N, level, P_, P["rgb"], P["sigma"], P["ws"], need, s))

    def ref():
        rgb, sig = net.field({"rays_o": o, "viewdirs": vd}, t, level, precision=prec)
        return {"rgb": rgb, "sigma": sig}
    return Spec(bufs, call, ref, f"{prec} level {level}: {n} rays x {N} samples ({n * N} points), ws {need} bytes")


@case(["neo_vanilla_sample_along_rays", "neo_vanilla_encode", "neo_vanilla_encode_bwd"], rand=[0, 1], n=[1, 33])
def vanilla_stages(dev, rand, n):
    g = gen(f"vs{rand}{n}")
    o, _, vd = _van_rays(g, dev, n)
    nc = 8
    N = nc + 1
    t = torch.sort(torch.rand(n, N, generator=g), -1).values.to(dev) * 3.0
    bufs = {"o": In(o), "vd": In(vd), "t": In(t), "t_out": Out(n, N), "enc": Out(n * N, 63), "denc": Out(n, 27),
            "g_enc": In(rnd(g, dev, n * N, 63)), "g_denc": In(rnd(g, dev, n, 27)), "g_o": Out(n, 3), "g_vd": Out(n, 3)}
    if rand:
        bufs["u"] = In(rnd(g, dev, n, N, lo=0.0))

    def call(P, s):
        lib = L.load()
        chk(lib.neo_vanilla_sample_along_rays(P["o"], P["vd"], n, nc, 0.2, 4.0, P.get("u"), P["t_out"], s))
        chk(lib.neo_vanilla_encode(P["o"], P["vd"], P["t"], n, N, P["enc"], P["denc"], s))
        chk(lib.neo_vanilla_encode_bwd(P["o"], P["vd"], P["t"], n, N, P["g_enc"], P["g_denc"], P["g_o"], P["g_vd"], s))
    return Spec(bufs, call, info=f"{n} rays x {N}", noref=AUTOGRAD)


# ------------------------------------------------------------------------------------------------ Mip-NeRF 360

@functools.lru_cache(maxsize=None)
def mip_net():
    from neo360_b200 import synth
    from neo360_b200.mip import MipNeRF360
    net = MipNeRF360(num_prop_samples=7, num_nerf_samples=13).eval()
    net.load_state_dict(synth.make_mip_params(3), strict=False)
    return net.cuda()


def _mip_weights(m):
    t = {"basis": m.pos_basis_t}
    for i in range(m.netdepth):
        t[f"w.{i}"], t[f"b.{i}"] = m.pts_linear[i].weight, m.pts_linear[i].bias
    t["wsig"], t["bsig"] = m.density_layer.weight, m.density_layer.bias
    if not m.disable_rgb:
        t.update({"wb": m.bottleneck_layer.weight, "bb": m.bottleneck_layer.bias, "wv0": m.views_linear[0].weight,
                  "bv0": m.views_linear[0].bias, "wrgb": m.rgb_layer.weight, "brgb": m.rgb_layer.bias})
    return {k: v.detach().contiguous().float() for k, v in t.items()}


def _mip_bufs(net, levels):
    bufs, keys = {}, {}
    for l in levels:
        w = _mip_weights(net.mlps[l])
        bufs.update(struct_ins(f"mlp{l}", w))
        keys[l] = list(w)
    return bufs, keys


def _mip_params(net, P, keys):
    arr = (L.NeoMipMLPParams * 3)()
    for l, ks in keys.items():
        arr[l].depth, arr[l].width = net.mlps[l].netdepth, net.mlps[l].netwidth
        set_struct(arr[l], P, f"mlp{l}", ks)
    return arr


@case(["neo_mip_workspace_bytes", "neo_mip_render_fwd"], prec=["fp32", "tc"], rand=[0, 1], n=[1, 33])
def mip_render(dev, prec, rand, n):
    net = mip_net()
    g = gen(f"mr{prec}{rand}{n}")
    o, d, vd = _van_rays(g, dev, n)
    radii = rnd(g, dev, n, lo=0.001, hi=0.01)
    bufs, keys = _mip_bufs(net, range(3))
    bufs.update({"rays_o": In(o), "rays_d": In(d), "viewdirs": In(vd), "radii": In(radii)})
    jit = [rnd(g, dev, n, 1, lo=0.0) for _ in range(3)] if rand else None
    if rand:
        bufs.update({f"j{i}": In(j) for i, j in enumerate(jit)})
    cfg = L.NeoMipCfg()
    cfg.n_prop, cfg.n_nerf, cfg.near_plane, cfg.far_plane, cfg.train_frac = net.num_prop_samples, net.num_nerf_samples, 0.2, 6.0, 0.5
    cfg.precision = L.NEO_PREC_TC if prec == "tc" else L.NEO_PREC_FP32
    need = L.load().neo_mip_workspace_bytes(n, C.byref(cfg), net.mlps[2].netwidth)
    bufs["ws"] = Ws(need, True, "activations, features, raw heads and intervals: floats, fp16 rows and the fp16 weight images")
    ns = (cfg.n_prop, cfg.n_prop, cfg.n_nerf)
    for l in range(3):
        bufs.update({f"rgb{l}": Out(n, 3), f"density{l}": Out(n, ns[l]), f"rgb_s{l}": Out(n, ns[l], 3), f"sdist{l}": Out(n, ns[l] + 1),
                     f"weights{l}": Out(n, ns[l])})

    def call(P, s):
        if rand:
            for i in range(3):
                cfg.jitter[i] = P[f"j{i}"]
        out = L.NeoMipOut()
        for k in L.MIP_OUT_FIELDS:
            for l in range(3):
                getattr(out, k)[l] = P[f"{k}{l}"]
        chk(L.load().neo_mip_render_fwd(_mip_params(net, P, keys), P["rays_o"], P["rays_d"], P["viewdirs"], P["radii"], n, C.byref(cfg),
                                        C.byref(out), P["ws"], need, s))

    def ref():
        net.precision = prec
        b = {"rays_o": o, "rays_d": d, "viewdirs": vd, "radii": radii}
        if rand:
            b["_uniforms"] = jit
        ren, hist = net(b, 0.5, bool(rand), False, 0.2, 6.0)
        got = {}
        for l in range(3):
            got.update({f"rgb{l}": ren[l]["rgb"], f"density{l}": hist[l]["density"], f"rgb_s{l}": hist[l]["rgb"], f"sdist{l}": hist[l]["sdist"],
                        f"weights{l}": hist[l]["weights"]})
        return got
    return Spec(bufs, call, ref, f"{prec}, randomized {rand}: {n} rays, samples {ns}")


@case(["neo_mip_field_workspace_bytes", "neo_mip_field_eval"], prec=["fp32", "tc"], level=[0, 2], nN=[(1, 5), (33, 9)])
def mip_field(dev, prec, level, nN):
    net = mip_net()
    n, N = nN
    g = gen(f"mf{prec}{level}{nN}")
    o, _, vd = _van_rays(g, dev, n)
    t = torch.sort(torch.rand(n, N, generator=g), -1).values.to(dev) * 3.0
    bufs, keys = _mip_bufs(net, [level])
    P_ = L.NEO_PREC_TC if prec == "tc" else L.NEO_PREC_FP32
    need = L.load().neo_mip_field_workspace_bytes(n * N, net.mlps[level].netwidth, P_)
    var = (C.c_float * 3)(1e-4, 2e-4, 3e-4)
    bufs.update({"rays_o": In(o), "viewdirs": In(vd), "t": In(t), "density": Out(n, N),
                 "ws": Ws(need, True, "activations, features and raw heads: floats and fp16 rows")})
    if level == 2:
        bufs["rgb"] = Out(n, N, 3)

    def call(P, s):
        r = L.NeoRays()
        r.n_rays, r.rays_o, r.rays_d, r.viewdirs = n, P["rays_o"], P["viewdirs"], P["viewdirs"]
        chk(L.load().neo_mip_field_eval(_mip_params(net, P, keys), level, C.byref(r), P["t"], N, var, P_, P.get("rgb"), P["density"],
                                        P["ws"], need, s))

    def ref():
        rgb, dens = net.field({"rays_o": o, "viewdirs": vd}, t, level, list(var), precision=prec)
        return {"density": dens, **({"rgb": rgb} if level == 2 else {})}
    return Spec(bufs, call, ref, f"{prec} level {level}: {n} rays x {N} ({n * N} points), ws {need} bytes")


@case(["neo_mip_resample", "neo_mip_encode", "neo_mip_encode_bwd"], level=[0, 1], n=[1, 33])
def mip_stages(dev, level, n):
    from neo360_b200.mip_basis import POS_BASIS_T
    g = gen(f"ms{level}{n}")
    o, d, vd = _van_rays(g, dev, n)
    n_prev, n_new = 7, 13
    sp = torch.sort(torch.rand(n, n_prev + 1, generator=g), -1).values
    sp[:, 0], sp[:, -1] = 0.0, 1.0
    td = torch.sort(torch.rand(n, n_new + 1, generator=g), -1).values * 3 + 0.2
    bufs = {"sp": In(sp.to(dev)), "wp": In(rnd(g, dev, n, n_prev, lo=0.0)), "jit": In(rnd(g, dev, n, lo=0.0)), "sdist": Out(n, n_new + 1),
            "tdist": Out(n, n_new + 1), "o": In(o), "d": In(d), "vd": In(vd), "radii": In(rnd(g, dev, n, lo=0.001, hi=0.01)),
            "td": In(td.to(dev)), "basis": In(POS_BASIS_T.float().contiguous().to(dev)), "feats": Out(n * n_new, 504), "denc": Out(n, 27),
            "g_denc": In(rnd(g, dev, n, 27)), "g_vd": Out(n, 3)}

    def call(P, s):
        lib = L.load()
        chk(lib.neo_mip_resample(P["sp"] if level else None, P["wp"] if level else None, n, n_prev if level else 1, level, n_new, 0.2, 6.0,
                                 0.5, P["jit"], P["sdist"], P["tdist"], s))
        chk(lib.neo_mip_encode(P["o"], P["d"], P["vd"], P["radii"], P["td"], P["basis"], n, n_new, P["feats"], P["denc"], s))
        chk(lib.neo_mip_encode_bwd(P["vd"], n, P["g_denc"], P["g_vd"], s))
    return Spec(bufs, call, info=f"level {level}: {n} rays, {n_prev} -> {n_new}", noref=AUTOGRAD)


@case(["neo_mip_composite", "neo_mip_composite_bwd", "neo_mip_composite_bwd_rays_d"], prop=[0, 1], n=[1, 33])
def mip_composite(dev, prop, n):
    g = gen(f"mc{prop}{n}")
    N = 13
    _, d, _ = _van_rays(g, dev, n)
    td = (torch.sort(torch.rand(n, N + 1, generator=g), -1).values * 3 + 0.2).to(dev)
    bufs = {"rd": In(rnd(g, dev, n, N, lo=-2.0, hi=3.0)), "td": In(td), "d": In(d), "rgb": Out(n, 3), "w": Out(n, N), "dens": Out(n, N),
            "rgb_s": Out(n, N, 3), "g_rgb": In(rnd(g, dev, n, 3)), "g_w": In(rnd(g, dev, n, N)), "g_dens": In(rnd(g, dev, n, N)),
            "g_rgb_s": In(rnd(g, dev, n, N, 3)), "d_rd": Out(n, N), "d_rd2": Out(n, N), "g_d": Out(n, 3)}
    if not prop:
        bufs.update({"rc": In(rnd(g, dev, n, N, 3)), "d_rc": Out(n, N, 3), "d_rc2": Out(n, N, 3)})

    def call(P, s):
        lib = L.load()
        gs = (P["g_rgb"], P["g_w"], P["g_dens"], P["g_rgb_s"])
        chk(lib.neo_mip_composite(P["rd"], P.get("rc"), P["td"], P["d"], n, N, P["rgb"], P["w"], P["dens"], P["rgb_s"], s))
        chk(lib.neo_mip_composite_bwd(P["rd"], P.get("rc"), P["td"], P["d"], n, N, *gs, P["d_rd"], P.get("d_rc"), s))
        chk(lib.neo_mip_composite_bwd_rays_d(P["rd"], P.get("rc"), P["td"], P["d"], n, N, *gs, P["d_rd2"], P.get("d_rc2"), P["g_d"], s))
    return Spec(bufs, call, info=f"{'proposal' if prop else 'NeRF'} level: {n} rays x {N}", noref=AUTOGRAD)


@case(["neo_distortion_loss", "neo_distortion_loss_bwd", "neo_interlevel_loss", "neo_interlevel_loss_bwd"], n=[1, 33], iv=[0, 1])
def losses(dev, n, iv):
    g = gen(f"loss{n}{iv}")
    N, Nc, Np = 13, 13, 7
    s_c = torch.sort(torch.rand(n, Nc + 1, generator=g), -1).values
    s_p = torch.sort(torch.rand(n, Np + 1, generator=g), -1).values
    bufs = {"w": In(rnd(g, dev, n, N, lo=0.0)), "m": In(torch.sort(torch.rand(n, N, generator=g), -1).values.to(dev)),
            "g_loss": In(rnd(g, dev, n)), "loss": Out(n), "d_w": Out(n, N), "s_c": In(s_c.to(dev)), "s_p": In(s_p.to(dev)),
            "w_p": In(rnd(g, dev, n, Np, lo=0.0)), "il": Out(n), "d_wp": Out(n, Np)}
    if iv:
        bufs["interval"] = In(rnd(g, dev, n, N, lo=0.0, hi=0.1))

    def call(P, s):
        lib = L.load()
        chk(lib.neo_distortion_loss(P["w"], P["m"], P.get("interval"), 0.05, n, N, P["loss"], s))
        chk(lib.neo_distortion_loss_bwd(P["w"], P["m"], P.get("interval"), 0.05, n, N, P["g_loss"], P["d_w"], s))
        chk(lib.neo_interlevel_loss(P["s_c"], P["w"], P["s_p"], P["w_p"], n, Nc, Np, P["il"], s))
        chk(lib.neo_interlevel_loss_bwd(P["s_c"], P["w"], P["s_p"], P["w_p"], n, Nc, Np, P["g_loss"], P["d_wp"], s))
    return Spec(bufs, call, info=f"{n} rays, N {N}, interval {'per sample' if iv else 'scalar'}", noref=AUTOGRAD)


# ------------------------------------------------------------------------------------------------ PixelNeRF

@functools.lru_cache(maxsize=None)
def pixel_model(nv):
    """PixelNeRF with the synthetic latent in place of its encoder's output (as tests/test_gpu_pixelnerf.py bypasses it), and the src_*
    entries of a batch: the model builds its own cameras-only scene, hoisted latent and packed weights from them."""
    from neo360_b200 import PixelNeRF, synth
    dev = torch.device("cuda:0")
    net = PixelNeRF(num_coarse_samples=8, num_fine_samples=4, num_src_views=nv)
    net.load_state_dict({**net.state_dict(), **synth.make_pixelnerf_params(60 + nv)})
    net = net.to(dev).eval()
    sc = synth.make_scene((37, 23), nv, (4, 4), 60 + nv)
    latent = sc["latent"].to(dev)
    net.encoder.forward = lambda x: latent
    src = {"src_poses": sc["src_poses"].to(dev), "src_focal": sc["src_focal"].to(dev), "src_c": sc["src_c"].to(dev),
           "src_imgs": torch.zeros(nv, 3, 23, 37, device=dev)}
    return net, src


def pixel_scene(net, src):
    """The model's own hoisted latent (nv, lat_h, lat_w, 512) and scene, as PixelNeRF.field builds them."""
    lat = net._hoisted_latent(src["src_imgs"])
    return lat, net._ensure_scene(src, lat.shape[1:3])


def packed_weights(S, keep):
    """{field or field.i: tensor} of the weights a packed parameter struct points at, found among the tensors the model keeps."""
    by_ptr = {t.data_ptr(): t for t in keep}
    out = {}
    for name, typ in S._fields_:
        v = getattr(S, name)
        for k, x in ([(f"{name}.{i}", x) for i, x in enumerate(v)] if hasattr(typ, "_length_") else [(name, v)]):
            if isinstance(x, int) and x:
                out[k] = by_ptr[x]
    return out


# nv = 1 and 8: the fp32 kernel's tile is 8 points up to 4 views and 4 points from 5 views on; 297 points are ragged against both
@case(["neo_pixelnerf_field", "neo_pixelnerf_tc_workspace_bytes", "neo_pixelnerf_field_tc"], prec=["fp32", "tc"], nv=[1, 8], nN=[(1, 5), (33, 9)])
def pixelnerf_field(dev, prec, nv, nN):
    net, src = pixel_model(nv)
    n, N = nN
    g = gen(f"pf{prec}{nv}{nN}")
    o, d, _ = rays_in_sphere(g, dev, n)
    t = torch.sort(torch.rand(n, N, generator=g), -1).values.to(dev) * 2.0 + 0.1
    lat, sc = pixel_scene(net, src)
    S = net._ensure_weights(prec)[0]
    w = packed_weights(S, net._packed[2])
    bufs = {"rays_o": In(o), "rays_d": In(d), "viewdirs": In(d), "t": In(t), "lat": In(lat), "rgb": Out(n, N, 3), "sigma": Out(n, N),
            **struct_ins("mlp", w)}
    lib = L.load()
    need = lib.neo_pixelnerf_tc_workspace_bytes(nv, n * N) if prec == "tc" else 0
    if prec == "tc":
        bufs["ws"] = Ws(need, True, "fp16 rows [enc | latent | 0], trunk and head activations, fp32 head sums")

    def call(P, s):
        r = neo_rays(P, n, chunk=5)
        mlp = C.byref(set_struct(type(S)(), P, "mlp", w))
        if prec == "fp32":
            chk(lib.neo_pixelnerf_field(sc.handle, P["lat"], mlp, C.byref(r), P["t"], N, P["rgb"], P["sigma"], s))
        else:
            chk(lib.neo_pixelnerf_field_tc(sc.handle, P["lat"], mlp, C.byref(r), P["t"], N, P["rgb"], P["sigma"], P["ws"], need, s))

    def ref():
        rgb, sigma = net.field({"rays_o": o, "rays_d": d, "viewdirs": d, **src}, t, 0, chunk=5, precision=prec)
        return {"rgb": rgb, "sigma": sigma}
    return Spec(bufs, call, ref, f"{prec}, nv {nv}: {n} rays x {N} ({nv * n * N} rows)")


@case(["neo_pixelnerf_encode"], nv=[1, 8], n=[1, 33])
def pixelnerf_encode(dev, nv, n):
    net, src = pixel_model(nv)
    _, sc = pixel_scene(net, src)
    g = gen(f"pe{nv}{n}")
    o, d, _ = rays_in_sphere(g, dev, n)
    N = 9
    M = n * N
    bufs = {"rays_o": In(o), "rays_d": In(d), "viewdirs": In(d), "t": In(torch.rand(n, N, generator=g).to(dev) * 2.0),
            "enc": Out(nv * M, 63), "dir": Out(nv * M, 27), "pts": Out(M, 3)}
    return Spec(bufs, lambda P, s: chk(L.load().neo_pixelnerf_encode(sc.handle, C.byref(neo_rays(P, n, chunk=4)), P["t"], N, P["enc"], P["dir"],
                                                                     P["pts"], s)), info=f"nv {nv}: {n} rays x {N}",
                noref="called inside PixelNeRF's training forward, which allocates around it")


# ------------------------------------------------------------------------------------------------ training on the tensor cores

def _trunk_weights(g, dev, E, pix):
    w = {"w0": rnd(g, dev, 128, E, lo=-0.1, hi=0.1), "b0": rnd(g, dev, 128, lo=-0.1, hi=0.1)}
    for i in (1, 2):
        w[f"w{i}"], w[f"b{i}"] = rnd(g, dev, 128, 128, lo=-0.1, hi=0.1), rnd(g, dev, 128, lo=-0.1, hi=0.1)
    w["w3"], w["b3"] = rnd(g, dev, 128, 128 if pix else 128 + E, lo=-0.1, hi=0.1), rnd(g, dev, 128, lo=-0.1, hi=0.1)
    return w


@case(["neo_field_train_workspace_bytes", "neo_field_train_fwd", "neo_field_train_bwd"], nv=[1, 8], in_ch=[3, 4], M=[1, 129])
def field_train(dev, nv, in_ch, M):
    g = gen(f"ft{nv}{in_ch}{M}")
    E = 21 * in_ch
    lib = L.load()
    saved, scratch = (lib.neo_field_train_workspace_bytes(nv, M, in_ch, k) for k in (0, 1))
    w = _trunk_weights(g, dev, E, False)
    bufs = {"cam": In(rnd(g, dev, nv * M, in_ch)), "local_p": In(rnd(g, dev, nv * M, 256)), "world_p": In(rnd(g, dev, nv * M, 256)),
            **{k: In(v) for k, v in w.items()}, "hbar": Out(M, 128), "g_hbar": In(rnd(g, dev, M, 128)), "d_pm": Out(nv * M, 256),
            "saved": WsSeq(saved, True, "bf16 input rows and weight images, written by the forward, read by the backward"),
            "scratch": Ws(scratch, True, "bf16 gradient rows, weight images and fp32 partials")}
    for k in ("w0", "b0", "w1", "b1", "w2", "b2", "w3", "b3"):
        bufs["g" + k] = Out(*w[k].shape)

    def call(P, s):
        chk(lib.neo_field_train_fwd(P["cam"], P["local_p"], P["world_p"], nv, M, in_ch, *[P[k] for k in ("w0", "b0", "w1", "b1", "w2", "b2", "w3", "b3")],
                                    P["hbar"], P["saved"], saved, s))
        chk(lib.neo_field_train_bwd(P["g_hbar"], nv, M, in_ch, P["w1"], P["w2"], P["w3"], P["saved"], saved, P["d_pm"],
                                    *[P["g" + k] for k in ("w0", "b0", "w1", "b1", "w2", "b2", "w3", "b3")], P["scratch"], scratch, s))
    return Spec(bufs, call, info=f"nv {nv}, in_ch {in_ch}, M {M}: saved {saved} B, scratch {scratch} B", noref=AUTOGRAD)


@case(["neo_pixelnerf_train_workspace_bytes", "neo_pixelnerf_train_fwd", "neo_pixelnerf_train_bwd"], nv=[1, 8], M=[1, 129])
def pixelnerf_train(dev, nv, M):
    g = gen(f"pt{nv}{M}")
    lib = L.load()
    saved, scratch = (lib.neo_pixelnerf_train_workspace_bytes(nv, M, k) for k in (0, 1))
    w = _trunk_weights(g, dev, 63, True)
    bufs = {"cam": In(rnd(g, dev, nv * M, 3)), "p0": In(rnd(g, dev, nv * M, 128)), **{k: In(v) for k, v in w.items()}, "hbar": Out(M, 128),
            "g_hbar": In(rnd(g, dev, M, 128)), "d_p0": Out(nv * M, 128),
            "saved": WsSeq(saved, True, "bf16 input rows and weight images, written by the forward, read by the backward"),
            "scratch": Ws(scratch, True, "bf16 gradient rows, weight images and fp32 partials")}
    for k in ("w0", "b0", "w1", "b1", "w2", "b2", "w3", "b3"):
        bufs["g" + k] = Out(*w[k].shape)

    def call(P, s):
        chk(lib.neo_pixelnerf_train_fwd(P["cam"], P["p0"], nv, M, *[P[k] for k in ("w0", "b0", "w1", "b1", "w2", "b2", "w3", "b3")], P["hbar"],
                                        P["saved"], saved, s))
        chk(lib.neo_pixelnerf_train_bwd(P["g_hbar"], nv, M, P["w1"], P["w2"], P["w3"], P["saved"], saved, P["d_p0"],
                                        *[P["g" + k] for k in ("w0", "b0", "w1", "b1", "w2", "b2", "w3", "b3")], P["scratch"], scratch, s))
    return Spec(bufs, call, info=f"nv {nv}, M {M}: saved {saved} B, scratch {scratch} B", noref=AUTOGRAD)


# M ragged against the 128-row tiles
@case(["neo_tc_gemm_bf16"], M=[1, 129], epi=[0, 1, 2])
def gemm_bf16(dev, M, epi):
    g = gen(f"gb{M}{epi}")
    N, K = 128, 192
    bufs = {"A": In(rnd(g, dev, M, K, dtype=BF16)), "W": In(rnd(g, dev, N, K, dtype=BF16)), "bias": In(rnd(g, dev, N)),
            "C": Out(M, N, dtype=F32 if epi == 2 else BF16)}
    return Spec(bufs, lambda P, s: chk(L.load().neo_tc_gemm_bf16(P["A"], K, P["W"], K, None if epi == 2 else P["bias"], P["C"], N, M, N, K, epi, s)),
                info=f"M {M}, N {N}, K {K}, epilogue {epi}", noref=AUTOGRAD)


@case(["neo_tc_dgrad_bf16"], M=[1, 129], mask=[0, 1])
def dgrad_bf16(dev, M, mask):
    g = gen(f"dg{M}{mask}")
    N, K = 128, 192
    bufs = {"dY": In(rnd(g, dev, M, K, dtype=BF16)), "Wt": In(rnd(g, dev, N, K, dtype=BF16)), "X": In(rnd(g, dev, M, N, dtype=BF16)),
            "g_sig": In(rnd(g, dev, M)), "w_sig": In(rnd(g, dev, N)), "dX": Out(M, N, dtype=BF16)}

    def call(P, s):
        chk(L.load().neo_tc_dgrad_bf16(P["dY"], K, P["Wt"], K, P["X"] if mask else None, N, P["g_sig"] if mask else None,
                                       P["w_sig"] if mask else None, P["dX"], N, M, N, K, s))
    return Spec(bufs, call, info=f"M {M}, N {N}, K {K}, mask and rank-1 term {mask}", noref=AUTOGRAD)


@case(["neo_tc_wgrad_bf16_workspace_bytes", "neo_tc_wgrad_bf16"], M=[1, 129, 4099], kv=[192, 170])
def wgrad_bf16(dev, M, kv):
    g = gen(f"wg{M}{kv}")
    N, K = 128, 192
    need = L.load().neo_tc_wgrad_bf16_workspace_bytes(M, N, K)
    bufs = {"dY": In(rnd(g, dev, M, N, dtype=BF16)), "X": In(rnd(g, dev, M, K, dtype=BF16)), "dW": Out(N, kv), "db": Out(N),
            "ws": Ws(need, True, "fp32 split-K partials")}
    return Spec(bufs, lambda P, s: chk(L.load().neo_tc_wgrad_bf16(P["dY"], N, P["X"], K, M, N, K, P["dW"], kv, P["db"], P["ws"], need, s)),
                info=f"M {M}, N {N}, K {K}, k_valid {kv}, ws {need} B", noref=AUTOGRAD)


@case(["neo_tc_pack_bf16", "neo_tc_relu_rank1_bf16", "neo_tc_rowdot_bf16"], M=[1, 129])
def bf16_small(dev, M):
    g = gen(f"bs{M}")
    cols_in, cols_out, N, K = 70, 128, 64, 64
    bufs = {"in": In(rnd(g, dev, M, cols_in)), "packed": Out(M, cols_out, dtype=BF16), "packed_t": Out(cols_in, M, dtype=BF16),
            "g": In(rnd(g, dev, M)), "w": In(rnd(g, dev, N)), "X": In(rnd(g, dev, M, N, dtype=BF16)), "r1": Out(M, N, dtype=BF16),
            "H": In(rnd(g, dev, M, K, dtype=BF16)), "Wr": In(rnd(g, dev, 3, K)), "br": In(rnd(g, dev, 3)), "rd": Out(M, 3)}

    def call(P, s):
        lib = L.load()
        chk(lib.neo_tc_pack_bf16(P["in"], M, cols_in, cols_in, P["packed"], cols_out, cols_out, 0, s))
        chk(lib.neo_tc_pack_bf16(P["in"], M, cols_in, cols_in, P["packed_t"], cols_in, M, 1, s))
        chk(lib.neo_tc_relu_rank1_bf16(P["g"], P["w"], P["X"], N, M, N, P["r1"], N, s))
        chk(lib.neo_tc_rowdot_bf16(P["H"], K, K, P["Wr"], P["br"], 3, M, P["rd"], s))
    return Spec(bufs, call, info=f"M {M}", noref=AUTOGRAD)


# ------------------------------------------------------------------------------------------------ grid encoder (64^3 cells per view)

G3 = 64 ** 3


def _enc_geom(g, dev, nv):
    from neo360_b200 import synth
    poses = torch.stack([synth.look_at_pose(360.0 * v / nv + 10.0, 0.3, 0.8) for v in range(nv)]).contiguous().to(dev)
    return poses, 30.0, 18.5, 11.5


@functools.lru_cache(maxsize=None)
def grid_encoder():
    from neo360_b200.encoder import GridEncoder
    torch.manual_seed(3)
    return GridEncoder().eval().to(torch.device("cuda:0"))


# The encoder's rows are v * 64^3 + cell: the view count only adds whole 64^3-row blocks, which every tile divides, so nv = 2 already
# crosses a view boundary.  nv = 8 is run where both runs' buffers fit in about 20 GB; the pool case stays at nv = 1 and 2 because at
# nv = 8 its fp32 and bf16 row buffers of both runs would hold about 55 GB at once.
@case(["neo_grid_encoder_workspace_bytes", "neo_grid_encoder_dense"], nv=[1, 8])
def grid_encoder_dense(dev, nv):
    enc = grid_encoder()
    g = gen(f"ged{nv}")
    lh, lw = 6, 9
    poses, f, cx, cy = _enc_geom(g, dev, nv)
    fc = [enc.depth_fc.common_branch[0], enc.depth_fc.common_branch[2], enc.depth_fc.depth_encoder]
    w = {}
    for i, m in enumerate(fc):
        w[f"fc_w.{i}"], w[f"fc_b.{i}"] = m.weight, m.bias
    for pl in ("xz", "yz", "xy"):
        agg = getattr(enc, f"pillar_aggregator_{pl}")
        w.update({f"agg_{pl}_w0": agg[0].weight, f"agg_{pl}_b0": agg[0].bias, f"agg_{pl}_w1": agg[2].weight, f"agg_{pl}_b1": agg[2].bias})
    w = {k: v.detach().contiguous().float() for k, v in w.items()}
    latent = rnd(g, dev, nv, 512, lh, lw, lo=0.0, hi=2.0)
    need = L.load().neo_grid_encoder_workspace_bytes(nv, lh, lw)
    bufs = {"latent": In(latent), "poses": In(poses), **struct_ins("p", w),
            **{k: Out(nv, 512, 64, 64) for k in ("fxz", "fxy", "fyz")},
            "ws": Ws(need, True, "channel-last latent, fp16 rows and weights, fp32 logits")}

    def call(P, s):
        prm = set_struct(L.NeoGridEncoderParams(), P, "p", w)
        chk(L.load().neo_grid_encoder_dense(C.byref(prm), P["latent"], nv, lh, lw, 37, 23, P["poses"], f, cx, cy, P["fxz"], P["fxy"], P["fyz"],
                                            P["ws"], need, s))
    def ref():
        focal, c = torch.full((nv,), f, device=dev), torch.tensor([[cx, cy]] * nv, device=dev)
        return dict(zip(("fxz", "fxy", "fyz"), enc.dense_cuda(latent, poses, focal, c, 37, 23)))
    return Spec(bufs, call, ref, f"nv {nv}, latent {lh} x {lw}, ws {need} B")


@case(["neo_grid_encoder_features", "neo_grid_encoder_features_bf16", "neo_grid_encoder_coords_bf16"], nv=[1, 8])
def grid_encoder_features(dev, nv):
    g = gen(f"gef{nv}")
    lh, lw, ld = 6, 9, 520
    poses, f, cx, cy = _enc_geom(g, dev, nv)
    R = nv * G3
    bufs = {"lat": In(rnd(g, dev, nv, lh, lw, 512)), "poses": In(poses), "X": Out(R, ld), "X16": Out(R, ld, dtype=BF16),
            "Lc": InOut(rnd(g, dev, R, ld, dtype=BF16), "rows [lat | x y z | 0]: the call writes columns 512.. and leaves the latent",
                        out_from_col=512)}

    def call(P, s):
        lib = L.load()
        chk(lib.neo_grid_encoder_features(P["lat"], nv, lh, lw, 37, 23, P["poses"], f, cx, cy, P["X"], ld, s))
        chk(lib.neo_grid_encoder_features_bf16(P["lat"], nv, lh, lw, 37, 23, P["poses"], f, cx, cy, P["X16"], ld, s))
        chk(lib.neo_grid_encoder_coords_bf16(P["Lc"], nv, ld, s))
    return Spec(bufs, call, info=f"nv {nv}: {R} rows x {ld}", noref=AUTOGRAD)


@case(["neo_grid_encoder_features_bwd", "neo_grid_encoder_features_bwd_det_workspace_bytes", "neo_grid_encoder_features_bwd_det"], nv=[1, 8],
      det=[0, 1])
def grid_encoder_features_bwd(dev, nv, det):
    g = gen(f"gefb{nv}{det}")
    lh, lw, ldg = 6, 9, 520
    poses, f, cx, cy = _enc_geom(g, dev, nv)
    lib = L.load()
    bufs = {"poses": In(poses), "g_X": In(rnd(g, dev, nv * G3, ldg)),
            "g_lat": InOut(rnd(g, dev, nv, lh, lw, 512), "latent gradient: the contract accumulates into it", exact=bool(det))}
    need = lib.neo_grid_encoder_features_bwd_det_workspace_bytes(nv, lh, lw) if det else 0
    if det:
        bufs["ws"] = WsSeq(need, False, "keys, entry ids, segment starts and sort scratch: integers, a documented layout")

    def call(P, s):
        a = (nv, lh, lw, 37, 23, P["poses"], f, cx, cy, P["g_X"], ldg, P["g_lat"])
        chk(lib.neo_grid_encoder_features_bwd_det(*a, P["ws"], need, s) if det else lib.neo_grid_encoder_features_bwd(*a, s))
    return Spec(bufs, call, info=f"nv {nv}, {'deterministic' if det else 'atomic'}", noref=AUTOGRAD)


@case(["neo_grid_encoder_pool", "neo_grid_encoder_pool_bwd", "neo_grid_encoder_pool_bf16", "neo_grid_encoder_pool_bwd_bf16",
       "neo_grid_encoder_lat_grad_bf16"], nv=[1, 2])
def grid_encoder_pool(dev, nv):
    g = gen(f"gep{nv}")
    R, ld = nv * G3, 520
    lat = rnd(g, dev, R, 512)
    bufs = {"lat": In(lat), "lat16": In(rnd(g, dev, R, ld, dtype=BF16)), "logits": In(rnd(g, dev, 3, R, lo=-3.0, hi=3.0)),
            **{k: In(rnd(g, dev, nv, 512, 64, 64)) for k in ("g_xz", "g_xy", "g_yz")},
            **{k: Out(nv, 512, 64, 64) for k in ("fxz", "fxy", "fyz", "hxz", "hxy", "hyz")},
            "d_lat": Out(R, 512), "d_logits": Out(3, R), "d_lat2": Out(R, 512), "d_logits2": Out(3, R), "d_agg": In(rnd(g, dev, R, 512)),
            "d_lat16": Out(R, 512, dtype=BF16)}

    def call(P, s):
        lib = L.load()
        gs = (P["g_xz"], P["g_xy"], P["g_yz"])
        chk(lib.neo_grid_encoder_pool(P["lat"], P["logits"], nv, P["fxz"], P["fxy"], P["fyz"], s))
        chk(lib.neo_grid_encoder_pool_bwd(P["lat"], P["logits"], nv, *gs, P["d_lat"], P["d_logits"], s))
        chk(lib.neo_grid_encoder_pool_bf16(P["lat16"], ld, P["logits"], nv, P["hxz"], P["hxy"], P["hyz"], s))
        chk(lib.neo_grid_encoder_pool_bwd_bf16(P["lat16"], ld, P["logits"], nv, *gs, P["d_lat2"], P["d_logits2"], s))
        chk(lib.neo_grid_encoder_lat_grad_bf16(P["lat"], P["d_agg"], nv, P["d_lat16"], s))
    return Spec(bufs, call, info=f"nv {nv}: {R} rows", noref=AUTOGRAD)


@case(["neo_upsample_bilinear_bwd"], hw=[((2, 2), (3, 5)), ((6, 9), (23, 37)), ((7, 5), (7, 5))])
def upsample_bwd(dev, hw):
    (hi, wi), (ho, wo) = hw
    g = gen(f"ub{hw}")
    planes = 5
    bufs = {"g_out": In(rnd(g, dev, planes, ho, wo)), "g_in": Out(planes, hi, wi)}
    return Spec(bufs, lambda P, s: chk(L.load().neo_upsample_bilinear_bwd(P["g_out"], planes, hi, wi, ho, wo, P["g_in"], s)),
                info=f"{planes} planes {hi} x {wi} <- {ho} x {wo}", noref=AUTOGRAD)


# ------------------------------------------------------------------------------------------------ tests

def test_every_entry_point_has_a_case_or_an_exclusion():
    """Every name the library exports has a case above or an exclusion with a reason: a new entry point without a case fails here."""
    covered = {s for syms, _, _ in CASES.values() for s in syms}
    missing = sorted(set(L.SYMBOLS) - covered - set(EXCLUDED))
    assert not missing, f"entry points with neither a buffer-contract case nor an exclusion: {missing}"
    unknown = sorted((covered | set(EXCLUDED)) - set(L.SYMBOLS))
    assert not unknown, f"cases or exclusions name symbols the library does not export: {unknown}"
    both = sorted(covered & set(EXCLUDED))
    assert not both, f"symbols both covered and excluded: {both}"
    assert all(r.strip() for r in EXCLUDED.values())


@pytest.fixture(scope="module")
def cuda():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from neo360_b200 import build
    build.build()
    return torch.device("cuda:0")


@pytest.mark.gpu
@pytest.mark.parametrize("cid", list(CASES))
def test_buffer_contract(cuda, cid):
    run_case(cid, cuda)
