"""CPU tests of the multi-rank path (gloo, world_size 2 and 4): the rank plan, and -- with the oracle standing in for the
CUDA kernels -- that the exchanges the frame-sharded / CFG-split step performs (GroupNorm-statistics all-reduce, frames <->
pixels re-sharding around the motion modules, all-gather of the two noise predictions) reproduce the single-process
step.  The CUDA implementation of the same exchanges is checked on GPUs by tests/test_multi_gpu.py
(tools/gpu_shard_check.py under torchrun)."""
import os

import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from videoswap_b200.dist_util import make_plan, max_over_ranks, shard_jobs

TINY = dict(boc=(32, 64, 128, 128), ctx=64, groups=8)


def _tiny_problem(frames=4, hw=16):      # 16x16 latents: 2x2 pixels at the deepest level, divisible by the 2 frame shards
    from oracle import unet3d_oracle as O
    from videoswap_b200.spec import UNetConfig, unet_param_shapes
    from videoswap_b200.weights import seeded_state_dict
    cfg = UNetConfig(block_out_channels=TINY["boc"], cross_attention_dim=TINY["ctx"], norm_num_groups=TINY["groups"])
    sd = seeded_state_dict(unet_param_shapes(cfg), seed=0)
    oc = O.OracleConfig(block_out_channels=TINY["boc"], cross_attention_dim=TINY["ctx"], norm_groups=TINY["groups"])
    g = torch.Generator().manual_seed(3)
    lat = torch.randn((1, 4, frames, hw, hw), generator=g)
    ehs2 = torch.randn((2, 16, 77, TINY["ctx"]), generator=g)
    res = [0.5 * torch.randn((frames, c, max(hw >> l, 1), max(hw >> l, 1)), generator=g) for l, c in enumerate(TINY["boc"])]
    return sd, oc, lat, ehs2, res


def _init(rank, world, port):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.set_num_threads(2)
    dist.init_process_group("gloo", rank=rank, world_size=world)


def _shard_worker(rank, world, port, q, cfg_split):
    try:
        _shard_worker_body(rank, world, port, q, cfg_split)
    except Exception as e:  # noqa: BLE001  (surface the failure in the parent instead of a queue timeout)
        import traceback
        q.put((rank, None, "".join(traceback.format_exception(e))[-2000:]))


def _shard_worker_body(rank, world, port, q, cfg_split):
    _init(rank, world, port)
    from oracle import sharded
    plan = make_plan(world, rank, cfg=cfg_split)
    # every rank creates every group (torch.distributed requires it); keep the two this rank belongs to
    groups = {}
    for r in range(world):
        pr = make_plan(world, r, cfg=cfg_split)
        for key in (tuple(pr.frame_group), tuple(pr.cfg_group)):
            if key not in groups:
                groups[key] = dist.new_group(list(key))
    sd, oc, lat, ehs2, res = _tiny_problem()
    with torch.no_grad():
        out = sharded.denoise_step_sharded(sd, oc, lat, 981, 50, ehs2, 7.5 if cfg_split else 1.0, res, plan,
                                           groups[tuple(plan.frame_group)], groups[tuple(plan.cfg_group)]) if cfg_split else None
        if not cfg_split:        # inversion-like: no CFG, every rank is a frame shard
            from oracle import unet3d_oracle as O
            r = plan.frame_range(lat.shape[2])
            with sharded.frame_sharded(groups[tuple(plan.frame_group)], plan.frame_shard, plan.frame_shards):
                out = O.unet_forward(sd, oc, lat[:, :, r.start:r.stop], 501, ehs2[1:2], [m[r.start:r.stop] for m in res])
    q.put((rank, list(plan.frame_range(lat.shape[2])), out))
    max_over_ranks(1.0)
    dist.barrier()
    dist.destroy_process_group()


def _run(world, cfg_split, port_base):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = port_base + (os.getpid() % 2000)
    procs = [ctx.Process(target=_shard_worker, args=(r, world, port, q, cfg_split)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=300) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    for r in res:
        assert r[1] is not None, f"rank {r[0]} failed:\n{r[2]}"
    return res


def test_frame_shards_reproduce_the_unsharded_unet_world2():
    """2 frame shards, no CFG (the inversion loop's shape): GroupNorm all-reduce + motion-module re-sharding."""
    from oracle import unet3d_oracle as O
    sd, oc, lat, ehs2, res = _tiny_problem()
    with torch.no_grad():
        ref = O.unet_forward(sd, oc, lat, 501, ehs2[1:2], res)
    for rank, frames, out in _run(2, False, 29500):
        assert out.shape[2] == len(frames) == 2
        assert torch.allclose(out, ref[:, :, frames[0]:frames[-1] + 1], atol=2e-5), (rank, (out - ref[:, :, frames[0]:frames[-1] + 1]).abs().max())


def test_cfg_split_times_frame_shards_reproduce_the_step_world4():
    """4 ranks = CFG pair x 2 frame shards: a full denoise step (UNet halves, eps all-gather, combine, DDIM)."""
    from oracle import unet3d_oracle as O
    sd, oc, lat, ehs2, res = _tiny_problem()
    with torch.no_grad():
        ref = O.denoise_step(sd, oc, O.DDIM(), lat, 981, 50, ehs2, 7.5, res)
    got = _run(4, True, 33500)
    assert sorted(r for r, _, _ in got) == [0, 1, 2, 3]
    for rank, frames, out in got:
        assert torch.allclose(out, ref[:, :, frames[0]:frames[-1] + 1], atol=2e-5), (rank, (out - ref[:, :, frames[0]:frames[-1] + 1]).abs().max())
    # ranks 0 and 2 (the two CFG halves of frame shard 0) hold the same latents
    by = {r: o for r, _, o in got}
    assert torch.equal(by[0], by[2]) and torch.equal(by[1], by[3])


def test_cfg_split_times_four_frame_shards_reproduce_the_step_world8():
    """8 ranks = CFG pair x 4 frame shards (the layout `bench.py --gpus 8` runs): one frame per rank, so every temporal
    attention works purely on re-sharded pixels and every GroupNorm statistic is an all-reduce of four single-frame partials."""
    from oracle import unet3d_oracle as O
    sd, oc, lat, ehs2, res = _tiny_problem()
    with torch.no_grad():
        ref = O.denoise_step(sd, oc, O.DDIM(), lat, 981, 50, ehs2, 7.5, res)
    got = _run(8, True, 37500)
    assert sorted(r for r, _, _ in got) == list(range(8))
    for rank, frames, out in got:
        assert len(frames) == 1 and frames[0] == rank % 4
        assert torch.allclose(out, ref[:, :, frames[0]:frames[0] + 1], atol=2e-5), (rank, (out - ref[:, :, frames[0]:frames[0] + 1]).abs().max())


def test_plan_layout():
    p = [make_plan(8, r) for r in range(8)]
    assert [x.cfg_index for x in p] == [0, 0, 0, 0, 1, 1, 1, 1] and [x.frame_shard for x in p] == [0, 1, 2, 3] * 2
    assert p[5].frame_group == [4, 5, 6, 7] and p[5].cfg_group == [1, 5] and list(p[5].frame_range(16)) == [4, 5, 6, 7]
    q = make_plan(2, 1)
    assert (q.cfg_ranks, q.frame_shards, q.cfg_index, q.frame_group, q.cfg_group) == (2, 1, 1, [1], [0, 1])
    inv = make_plan(4, 3, cfg=False)
    assert (inv.cfg_ranks, inv.frame_shards, inv.frame_shard, inv.frame_group) == (1, 4, 3, [0, 1, 2, 3])
    one = make_plan(1, 0)
    assert one.world == 1 and one.frame_group == [0] and list(one.frame_range(16)) == list(range(16))
    x = torch.arange(2 * 4 * 16).reshape(2, 4, 16)
    assert torch.equal(p[2].shard_frames(x, 2), x[:, :, 8:12])


def test_every_communicator_gets_its_own_unique_id():
    """A ncclUniqueId serves exactly ONE communicator (the 4-GPU run of round 2 failed in ncclCommInitRank because rank 0 is
    the first rank of a frame group AND of a CFG pair and both groups took 'the id of their first rank')."""
    from videoswap_b200.dist_util import select_comm_ids
    for world, cfg in ((2, True), (4, True), (8, True), (4, False)):
        ids = [[f"frame-id-of-{r}".encode(), f"cfg-id-of-{r}".encode()] for r in range(world)]
        used = {}                                   # id -> (kind, group)
        for r in range(world):
            for name, (group, idb) in select_comm_ids(make_plan(world, r, cfg=cfg), ids).items():
                assert r in group
                key = (name, tuple(group))
                assert used.setdefault(idb, key) == key, f"id {idb} shared by {used[idb]} and {key}"
        groups = {v for v in used.values()}
        expect = {2: 1, 4: 4, 8: 6}[world] if cfg else 1        # CFG pairs + frame groups with more than one rank
        assert len(groups) == len(used) == expect, (world, cfg, groups)


def test_shard_jobs_covers_everything():
    for n in (0, 1, 7, 16):
        for w in (1, 2, 4, 8):
            got = sum((shard_jobs(n, r, w) for r in range(w)), [])
            assert got == list(range(n))
