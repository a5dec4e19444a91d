"""Multi-GPU parity of the frame-sharded / CFG-split step (SURVEY.md 8e): every rank runs the SAME full step on its own GPU
(unsharded native path = the reference here; it is itself pinned to the oracle by the -m gpu tests) and then its shard of
the step split over all ranks; the shard must reproduce the corresponding frames.
  python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port 29511 tools/gpu_shard_check.py
With REPORT_JSON set, rank 0 writes the full report there; exits 1 unless every case reaches 55 dB."""
import json
import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def psnr(a, b):
    a, b = a.float(), b.float()
    mse = ((a - b) ** 2).mean().item()
    rng = (b.max() - b.min()).item()
    return float("inf") if mse == 0 else 10 * math.log10(rng * rng / mse)


def main():
    import torch
    import torch.distributed as dist
    from bench import gpu_weights
    from videoswap_b200 import AnimateDiffUNet3DModel, DDIMScheduler, VideoSwapPipeline, dist_util, ops
    from videoswap_b200.pipeline import GraphedStep
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    model = AnimateDiffUNet3DModel(init="empty")
    model.load_state_dict(gpu_weights(model.cfg, dev), assign=True)
    pipe = VideoSwapPipeline(model, DDIMScheduler())
    pipe.scheduler.set_timesteps(50)
    boc = model.cfg.block_out_channels
    out = {"world": world, "cases": {}}
    ok = True
    cases = (("16f_32x32", 16, 32), ("16f_64x64_C2", 16, 64))
    if os.environ.get("SHARD_CHECK_ONLY_C2"):
        cases = cases[1:]
    for name, Fr, hw in cases:
        g = torch.Generator(device=dev).manual_seed(100)
        lat = torch.randn((1, 4, Fr, hw, hw), device=dev, generator=g).half()
        embeds = torch.randn((2, 16, 77, 768), device=dev, generator=g).half()
        res = [(0.1 * torch.randn((Fr, c, hw >> l, hw >> l), device=dev, generator=g)).half() for l, c in enumerate(boc)]
        t = 981
        # ---- reference: the whole step on this GPU (k = 1)
        dist_util.attach(model, dist_util.ShardPlan())
        ref = pipe.step(lat, t, embeds, 7.5, [torch.cat([r, r]) for r in res]).clone()
        ref_inv = model(lat, 501, embeds[1:2, 0].contiguous(), return_dict=False)[0].clone()     # no CFG, plain embeds
        torch.cuda.synchronize()
        case = {}
        # ---- CFG x frame shards
        plan = dist_util.create_comms(dist_util.make_plan(world, rank, cfg=True))
        dist_util.attach(model, plan)
        fr = plan.frame_range(Fr)
        lat_loc = plan.shard_frames(lat, 2)
        res_loc = [plan.shard_frame_major(r, Fr) for r in res]
        got = pipe.step_sharded(lat_loc, t, embeds, 7.5, plan, res_loc)
        torch.cuda.synchronize()
        case["cfg_x_frames"] = {"plan": f"cfg {plan.cfg_ranks} x frames {plan.frame_shards}", "psnr_vs_unsharded": psnr(got, ref[:, :, fr.start:fr.stop]),
                                "finite": bool(torch.isfinite(got).all().item())}
        gs = GraphedStep(pipe, lat_loc, embeds, 7.5, res_loc, plan=plan)           # NCCL exchanges captured in the graph
        g1 = gs(lat_loc, t).clone()
        g2 = gs(lat_loc, t).clone()
        torch.cuda.synchronize()
        case["cfg_x_frames"]["graph_psnr_vs_unsharded"] = psnr(g1, ref[:, :, fr.start:fr.stop])
        case["cfg_x_frames"]["graph_replay_equal"] = bool(torch.equal(g1, g2))
        del gs
        # ---- frame shards only (inversion: no CFG), all ranks one group
        plan2 = dist_util.create_comms(dist_util.make_plan(world, rank, cfg=False))
        dist_util.attach(model, plan2)
        fr2 = plan2.frame_range(Fr)
        eps = model(plan2.shard_frames(lat, 2), 501, embeds[1:2, 0].contiguous(), return_dict=False)[0]
        torch.cuda.synchronize()
        case["frames_only"] = {"plan": f"frames {plan2.frame_shards}", "psnr_vs_unsharded": psnr(eps, ref_inv[:, :, fr2.start:fr2.stop]),
                               "finite": bool(torch.isfinite(eps).all().item())}
        vals = [case["cfg_x_frames"]["psnr_vs_unsharded"], case["cfg_x_frames"]["graph_psnr_vs_unsharded"], case["frames_only"]["psnr_vs_unsharded"]]
        tmin = torch.tensor([min(vals)], device=dev)
        dist.all_reduce(tmin, op=dist.ReduceOp.MIN)
        case["min_psnr_over_ranks"] = tmin.item()
        ok = ok and tmin.item() >= 55.0
        out["cases"][name] = case
        if rank == 0:
            print(name, json.dumps(case), flush=True)
    out["ok"] = ok
    if rank == 0:
        if os.environ.get("REPORT_JSON"):            # optional: full JSON report to this path
            with open(os.environ["REPORT_JSON"], "w") as f:
                json.dump(out, f, indent=1)
        print("SHARD_CHECK", "OK" if ok else "FAILED", flush=True)
    dist.barrier()
    dist.destroy_process_group()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
