"""Fused NVLink peer-memory exchange (needs >= 2 GPUs; skipped on the single-GPU test box):
the gather buffers every rank ends up with must equal the stacked per-rank rollouts."""
import os
import socket

import pytest
import torch

pytestmark = pytest.mark.gpu


def _worker(rank, world, port, q):
    import torch.distributed as dist
    from madrl_b200 import BatchedMAWaterWorld
    from madrl_b200.dist import PeerGather
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    try:
        # one block per SM and E > 2 SMs: the fused-exchange kernel's warps step several envs each
        sms = torch.cuda.get_device_properties(dev).multi_processor_count
        E, T, Np = 2 * sms + 7, 45, 5       # T not a multiple of the 6- and 32-step staging runs
        assert E > 2 * sms
        eng = BatchedMAWaterWorld(E, Np, 5, device=dev, seed=9, env_id_base=rank * E, n_coop=1, radius=0.04)
        eng.set_launch(blocks_per_sm=1)
        eng.reset()
        ok = True
        for mode in ("root", "all"):
            pg = PeerGather(eng, T, Np, mode=mode)
            for k in range(3):                                  # exercises both buffer sets
                act = torch.randn(T, E, Np, 2, device=dev,
                                  generator=torch.Generator(dev).manual_seed(100 * k + rank)) * 0.7
                pg.arm(k)
                obs, rew, done, info = eng.rollout(act, auto_reset=True)
                got = pg.complete()
                torch.cuda.synchronize()
                # reference exchange: plain NCCL all_gather of the local outputs
                r_rew = torch.empty((world,) + tuple(rew.shape), device=dev)
                dist.all_gather_into_tensor(r_rew.view(world * T, E, Np), rew)
                r_info = torch.empty((world,) + tuple(info.shape), dtype=torch.int32, device=dev)
                dist.all_gather_into_tensor(r_info.view(world * T, E, 2), info)
                r_done = torch.empty((world,) + tuple(done.shape), dtype=torch.uint8, device=dev)
                dist.all_gather_into_tensor(r_done.view(world * T, E), done)
                if got is not None:                         # env-major [W,E,T,..] -> time-major [W,T,E,..]
                    g_rew, g_done, g_info = got
                    ok = ok and torch.equal(g_rew.permute(0, 2, 1, 3), r_rew) and \
                        torch.equal(g_info.permute(0, 2, 1, 3), r_info) and \
                        torch.equal(g_done.permute(0, 2, 1), r_done)
                else:
                    ok = ok and mode == "root" and rank != 0
            pg.close()
        # copy-engine gather to the root, overlapped on a side stream; both completion protocols
        # (stream memory operations / round 1's NCCL all-reduce), with the full trajectory packed in
        from madrl_b200.dist import AsyncRootGather
        for completion in ("memops", "nccl"):
            ag = AsyncRootGather(T, E, Np, 2, dev, completion=completion, obs_dim=eng.obs_dim, act_shape=(Np, 2))
            ok = ok and ag.completion == completion
            seen = []
            for k in range(5):                     # > n_sets: exercises the release / reuse handshake
                act = torch.randn(T, E, Np, 2, device=dev, generator=torch.Generator(dev).manual_seed(7 * k + rank)) * 0.7
                ag.before_reuse(k)
                pk = ag.packed(k)
                pk.act.copy_(act)
                eng.rollout(pk.act, auto_reset=True, out=(pk.obs, pk.rew, pk.done, pk.info))
                ag.submit(k, consume=lambda g: seen.append(g.clone()))   # root: snapshot inside the protocol
                ag.before_reuse(k)                 # wait for this exchange before checking it
                torch.cuda.synchronize()
                ref = torch.empty(world * pk.nbytes, dtype=torch.uint8, device=dev)
                dist.all_gather_into_tensor(ref, pk.buf)
                got = ag.result(k)
                if rank == 0:
                    ok = ok and torch.equal(got.reshape(-1), ref) and torch.equal(seen[-1].reshape(-1), ref)
                    ok = ok and torch.equal(pk.view_of(got[1], 'obs'), pk.view_of(ref.view(world, -1)[1], 'obs'))
                else:
                    ok = ok and got is None and not seen
            ag.close()
        q.put((rank, bool(ok)))
    finally:
        dist.destroy_process_group()


def test_fused_exchange_equals_nccl_all_gather():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.SimpleQueue()
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    world = 2
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(300)
        assert p.exitcode == 0
    res = dict(q.get() for _ in range(world))
    assert res == {0: True, 1: True}
