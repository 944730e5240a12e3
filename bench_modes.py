"""Secondary bench modes of bench.py (the headline stays `--mode frames`, BASELINE configs[1]).

  --mode strong      ONE 640x480 frame split over the ranks on chunk boundaries (neo360_b200/sharding.py) and the pixels
                     all-gathered over NCCL inside the timed region -- the reference's `alter_gather_cat` (models/interface.py:30-50).
  --mode turntable   BASELINE configs[4]: a 360-degree turntable of `--views` target views at 1280x960, 128+128 samples, views sharded
                     over the ranks first (SURVEY.md 8(e)); rays are generated on the device from the pose (datasets/ray_utils.py:84-176).
  --mode train       BASELINE configs[3]: generalisable training steps on 4096-ray batches sharded over the ranks, MSE + distortion
                     loss, flat-buffer NCCL gradient all-reduce, Adam (models/neo360/model.py:697-820, 1003-1025, 1246-1260).

Each prints one JSON line in bench.py's format (rank 0); timing = CUDA events bracketed by barrier + synchronize, max over ranks.
"""
import math
import os
import time

import torch

import bench as B


def _timed(fn, steps, warmup, dev, dist):
    def barrier():
        if dist is not None:
            dist.barrier()
        torch.cuda.synchronize()
    for s in range(warmup):
        fn(s)
    barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for s in range(steps):
        fn(warmup + s)
    e1.record()
    barrier()
    ms = torch.tensor([e0.elapsed_time(e1)], device=dev)
    if dist is not None:
        dist.all_reduce(ms, op=dist.ReduceOp.MAX)
    return float(ms.item())


def _net(dev, precision, n_coarse, n_fine, img_wh, train=False):
    from neo360_b200 import NeRF_TP, synth
    sc = synth.make_scene(img_wh, B.NV, (120, 160), seed=0)
    P = synth.make_mlp_params(0)
    net = NeRF_TP(num_coarse_samples=n_coarse, num_fine_samples=n_fine, num_src_views=B.NV, precision=precision)
    net.load_state_dict(P)
    net = net.to(dev)
    if not train:
        net.eval()
    scd = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in sc.items()}
    return net, scd, P


def run(args, rank, world, local, dev, dist, pk):
    base = {"n_gpus": world, "steps": args.steps, "warmup": args.warmup, "higher_is_better": True, "vs_baseline": None, "data": "synthetic",
            "unit": "rays/s"}
    sampler = B.ClockSampler(local) if rank == 0 else None
    if args.mode == "strong":
        from neo360_b200 import sharding
        net, sc, _ = _net(dev, args.precision, B.N_COARSE, B.N_FINE, (B.IMG_W, B.IMG_H))
        net.set_scene(*[sc[k] for k in ("planes_xz", "planes_xy", "planes_yz", "latent", "src_poses", "src_focal", "src_c")], sc["img_wh"])
        n = B.IMG_W * B.IMG_H
        a, b = sharding.shard_range(n, world, rank, B.CHUNK)
        frames = [tuple(x.to(dev) for x in B.frame_rays_cpu(v)) for v in range(4)]
        full = {}

        def step(s):
            o, d = frames[s % len(frames)]
            with torch.no_grad():
                r = net.render_rays_test({"rays_o": o[a:b], "rays_d": d[a:b], "viewdirs": d[a:b]}, chunk=B.CHUNK)
                px = torch.cat([r["rgb"], r["depth"][:, None]], 1)
                full["px"] = sharding.gather_rays(px, n, world, B.CHUNK) if dist is not None else px

        if sampler:
            sampler.start()
        ms = _timed(step, args.steps, args.warmup, dev, dist)
        if sampler:
            sampler.stop_flag = True
        # the gathered frame must be the single-rank frame, bit for bit (same 32-ray groups: shards start on chunk boundaries)
        step(0)
        o, d = frames[0]
        with torch.no_grad():
            ref = net.render_rays_test({"rays_o": o, "rays_d": d, "viewdirs": d}, chunk=B.CHUNK)
        diff = float((full["px"][:, :3] - ref["rgb"]).abs().max())
        line = dict(base, metric="rays/sec at 640x480, 192 samples/ray", value=n * args.steps / (ms * 1e-3), ms_per_step=ms / args.steps,
                    scaling="strong", dtype="f16 operands, f32 accumulate (wgmma)" if args.precision == "tc" else "f32",
                    config={"workload": "ONE neo360 640x480 frame (128+64 samples, 3 src views) split over the ranks on 1024-ray chunk boundaries, "
                                        "pixels (rgb+depth) all-gathered over NCCL inside the timed region", "rays_per_step": n,
                            "rays_per_rank": b - a, "chunk": B.CHUNK, "precision": args.precision,
                            "parallelism": f"ray ranges x{world} + all_gather (models/interface.py:30-50)"},
                    gathered_vs_single_rank_linf=diff, clocks=sampler.result() if sampler else None)
        return line

    if args.mode == "turntable":
        from neo360_b200 import ops, synth
        W, H, nc, nf = 1280, 960, 128, 128
        net, sc, _ = _net(dev, args.precision, nc, nf, (W, H))
        net.set_scene(*[sc[k] for k in ("planes_xz", "planes_xy", "planes_yz", "latent", "src_poses", "src_focal", "src_c")], sc["img_wh"])
        views = list(range(rank, args.views, world))                       # views first (SURVEY.md 8(e))
        poses = [synth.target_pose(v, args.views)[:3, :4].contiguous().pin_memory() for v in views]
        out = torch.empty(W * H, 4).pin_memory()

        def render_view(i):
            c2w = poses[i].to(dev, non_blocking=True)
            ro, vd, rd, _ = ops.get_rays(H, W, 0.8 * W, c2w)
            with torch.no_grad():
                r = net.render_rays_test({"rays_o": ro, "rays_d": rd, "viewdirs": vd}, chunk=B.CHUNK, img_wh=(W, H))
            out[:, :3].copy_(r["rgb"], non_blocking=True)
            out[:, 3].copy_(r["depth"], non_blocking=True)

        def step(s):
            for i in range(len(views)):
                render_view(i)

        if views:
            render_view(0)                                                  # warm-up: one view
        if sampler:
            sampler.start()
        ms = _timed(step, args.steps, 0, dev, dist)
        if sampler:
            sampler.stop_flag = True
        rays = args.views * W * H * args.steps
        return dict(base, metric="rays/sec, 360-degree turntable at 1280x960, 256 samples/ray", value=rays / (ms * 1e-3), ms_per_step=ms / args.steps,
                    scaling="strong", warmup=1, dtype="f16 operands, f32 accumulate (wgmma)" if args.precision == "tc" else "f32",
                    config={"workload": f"full 360-degree turntable, {args.views} novel views at 1280x960, 128+128 samples (BASELINE configs[4]), "
                                        "rays generated on the device from the pose, rgb+depth copied back to pinned host memory per view",
                            "views_per_rank": len(views), "chunk": B.CHUNK, "precision": args.precision,
                            "parallelism": f"views sharded x{world} (view v on rank v mod {world}), no collective"},
                    clocks=sampler.result() if sampler else None)

    if args.mode == "mip360":
        from neo360_b200 import ops, synth
        from neo360_b200.mip import MipNeRF360
        W, H, npp, nn_ = B.IMG_W, B.IMG_H, 64, 64
        net = MipNeRF360(num_prop_samples=npp, num_nerf_samples=nn_, precision=args.precision).eval()
        net.load_state_dict(synth.make_mip_params(0))
        net = net.to(dev)
        n = min(args.rays, W * H)
        sub = 65536                                                       # rays per library call (bounds the activation workspace: ~26 GB)
        poses = [synth.target_pose((s * world + rank) % 100, 100)[:3, :4].contiguous().pin_memory() for s in range(4)]
        out = torch.empty(n, 3).pin_memory()

        def step(s):
            c2w = poses[s % len(poses)].to(dev, non_blocking=True)
            ro, vd, rd, rad = ops.get_rays(H, W, 0.8 * W, c2w)
            with torch.no_grad():
                for i in range(0, n, sub):
                    j = min(i + sub, n)
                    ren, _ = net({"rays_o": ro[i:j], "rays_d": rd[i:j], "viewdirs": vd[i:j], "radii": rad[i:j]}, 1.0, False, False, 0.2, 100.0)
                    out[i:j].copy_(ren[2]["rgb"], non_blocking=True)

        if sampler:
            sampler.start()
        ms = _timed(step, args.steps, args.warmup, dev, dist)
        if sampler:
            sampler.stop_flag = True
        rays = n * world * args.steps
        # dense-layer MACs per ray (SURVEY.md 8(d)): two proposal MLPs 4x256 on 64 samples each, one NeRF MLP 8x1024 (+ heads) on 64
        prop = 504 * 256 + 3 * 256 * 256 + 256
        nerf = 504 * 1024 + 6 * 1024 * 1024 + (1024 + 504) * 1024 + 1024 + 1024 * 256 + (256 + 27) * 128 + 128 * 3
        flop_ray = 2.0 * (2 * npp * prop + nn_ * nerf)
        ach = rays * flop_ray / (ms * 1e-3) / 1e12
        return dict(base, metric="rays/sec at 640x480, 192 samples/ray (mipnerf360)", value=rays / (ms * 1e-3), ms_per_step=ms / args.steps,
                    scaling="weak", dtype="f16 operands, f32 accumulate (wgmma)" if args.precision == "tc" else "f32",
                    config={"workload": "mipnerf360 unbounded-contraction render, 640x480, 64+64 proposal + 64 NeRF samples (BASELINE configs[2]), "
                                        "rays generated on the device, rgb copied back to pinned host memory",
                            "rays_per_step_per_gpu": n, "rays_per_call": sub, "precision": args.precision,
                            "parallelism": f"one frame per rank x{world}, no collective", "valid_headline": n == W * H},
                    roofline={"bound": "tensor", "achieved": ach, "peak": pk["bf16_tflops"], "unit": "TFLOP/s", "frac": ach / pk["bf16_tflops"],
                              "traffic": None, "peak_source": pk["src"],
                              "flops": f"{flop_ray / 1e9:.3f} GFLOP/ray of dense layers (2*MAC, padding not counted) over the WHOLE step time "
                                       "(sampling, IPE features, packing, compositing included)"},
                    e2e={"value": rays / (ms * 1e-3), "unit": "rays/s", "h2d_bytes_per_step": 48, "d2h_bytes_per_step": n * 12},
                    clocks=sampler.result() if sampler else None)

    if args.mode == "vanilla":
        from neo360_b200 import ops, synth
        from neo360_b200.vanilla import NeRF
        W, H, nc, nf = B.IMG_W, B.IMG_H, 64, 128                          # reference defaults (models/vanilla_nerf/model.py:135-136): 65 + 193 points per ray
        net = NeRF(num_coarse_samples=nc, num_fine_samples=nf).eval()
        net.precision = args.precision
        net.load_state_dict(synth.make_vanilla_params(0))
        net = net.to(dev)
        n, sub = min(args.rays, W * H), 65536
        poses = [synth.target_pose((s * world + rank) % 100, 100)[:3, :4].contiguous().pin_memory() for s in range(4)]
        out = torch.empty(n, 3).pin_memory()

        def step(s):
            c2w = poses[s % len(poses)].to(dev, non_blocking=True)
            ro, vd, rd, _ = ops.get_rays(H, W, 0.8 * W, c2w)
            with torch.no_grad():
                for i in range(0, n, sub):
                    j = min(i + sub, n)
                    ev = net({"rays_o": ro[i:j], "rays_d": rd[i:j], "viewdirs": vd[i:j]}, False, True, 0.2, 3.0)
                    out[i:j].copy_(ev[1][0], non_blocking=True)

        if sampler:
            sampler.start()
        ms = _timed(step, args.steps, args.warmup, dev, dist)
        if sampler:
            sampler.stop_flag = True
        rays = n * world * args.steps
        flop_ray = 2.0 * 593408 * ((nc + 1) + (nc + 1 + nf))               # SURVEY.md 8(d): 593 408 MAC per point
        ach = rays * flop_ray / (ms * 1e-3) / 1e12
        return dict(base, metric="rays/sec at 640x480, vanilla NeRF 64+128 samples", value=rays / (ms * 1e-3), ms_per_step=ms / args.steps,
                    scaling="weak", dtype="f16 operands, f32 accumulate (wgmma)" if args.precision == "tc" else "f32",
                    config={"workload": "vanilla NeRF two-level render, 640x480, 64 + 128 samples (65 + 193 points per ray), rays generated on the device",
                            "rays_per_step_per_gpu": n, "rays_per_call": sub, "precision": args.precision,
                            "parallelism": f"one frame per rank x{world}, no collective", "valid_headline": n == W * H},
                    roofline={"bound": "tensor", "achieved": ach, "peak": pk["bf16_tflops"], "unit": "TFLOP/s", "frac": ach / pk["bf16_tflops"],
                              "traffic": None, "peak_source": pk["src"],
                              "flops": f"{flop_ray / 1e6:.1f} MFLOP/ray of dense layers (2*MAC) over the WHOLE step time"},
                    e2e={"value": rays / (ms * 1e-3), "unit": "rays/s", "h2d_bytes_per_step": 48, "d2h_bytes_per_step": n * 12},
                    clocks=sampler.result() if sampler else None)

    if args.mode == "encoder":
        # SURVEY.md 8(f1): GridEncoder.forward per scene (3 source views at 640x480): ResNet trunk + dense part + conv stacks; the dense part
        # (64^3 x 3 grid lookup, DepthPillarEncoder, three pillar aggregators: 2.7 TFLOP) timed as hand-written CUDA vs framework ops
        from neo360_b200.encoder import GridEncoder
        from neo360_b200 import synth
        torch.manual_seed(0)
        enc = GridEncoder().eval().to(dev)
        sc = synth.make_scene((64, 48), B.NV, (12, 16), 0)
        poses, focal, c = sc["src_poses"].to(dev), torch.full((B.NV,), 0.8 * B.IMG_W, device=dev), torch.tensor([[B.IMG_W / 2.0, B.IMG_H / 2.0]] * B.NV, device=dev)
        imgs = torch.rand(B.NV, 3, B.IMG_H, B.IMG_W, device=dev) * 2 - 1
        res = {}
        with torch.no_grad():
            lat = enc.spatial_encoder(imgs)
            for name, fn in (("dense_cuda_tc", lambda: enc.dense_cuda(lat, poses, focal, c, B.IMG_W, B.IMG_H)),
                             ("dense_framework_fp32", lambda: enc.dense_torch(lat, poses, focal, c, B.IMG_W, B.IMG_H)),
                             ("whole_forward", lambda: enc(imgs, poses, focal, c))):
                res[name] = _timed(lambda s: fn(), args.steps, args.warmup, dev, dist) / args.steps
        rows = B.NV * 64 ** 3
        flop = 2.0 * rows * (518 * 512 + 2 * 512 * 512 + 3 * (513 * 512 + 512))
        return dict(base, metric="GridEncoder scenes/sec (3 source views, 640x480)", unit="scenes/s", value=1e3 / res["whole_forward"],
                    ms_per_step=res["whole_forward"], scaling="weak", dtype="f16 operands, f32 accumulate (wgmma) for the dense part",
                    config={"workload": "GridEncoder.forward: ResNet-34 trunk (framework) + dense part (hand-written CUDA) + 3 conv stacks (framework)",
                            "rows": rows, "parallelism": "one scene per rank"},
                    dense_part_ms=res, roofline={"bound": "tensor", "achieved": flop / (res["dense_cuda_tc"] * 1e-3) / 1e12, "peak": pk["bf16_tflops"],
                                                 "unit": "TFLOP/s", "frac": flop / (res["dense_cuda_tc"] * 1e-3) / 1e12 / pk["bf16_tflops"],
                                                 "traffic": None, "peak_source": pk["src"],
                                                 "flops": f"{flop / 1e12:.2f} TFLOP of dense layers per scene over the dense part's time (gather, softmax sums included)"},
                    speedup_dense_vs_framework_fp32=res["dense_framework_fp32"] / res["dense_cuda_tc"])

    if args.mode == "train":
        from neo360_b200 import training
        return training.bench_train(args, rank, world, local, dev, dist, pk, base, sampler, _timed)
    raise ValueError(args.mode)
