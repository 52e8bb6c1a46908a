"""Sample processing and evaluation pooled over the ranks of a sharded batch (``group=``), on the GPU:

  * with a one-rank group every pooled call returns the bits of ``group=None``;
  * an evaluation over several ranks refuses an engine not built by ``dist.make_sharded``;
  * two processes, each holding half of a C2-like Waterworld batch through ``dist.make_sharded`` (ragged: 31 and 32
    envs), over gloo on one GPU -- and over NCCL on two GPUs where the box has them: every pooled output has the
    same bytes on both ranks and matches the unsharded single-process call (counts, lengths, path counts, bin
    counts and the fallback decision exactly; float32 standardiser state and simplev within one float32 ulp;
    float64 moments, explained variances and mean returns at rtol 1e-12; the rltools baseline with obsnorm within
    1e-9 of the unsharded fit; evaluate_heuristic on Waterworld and Pursuit exactly).
"""
import pytest
import torch
import torch.distributed as dist

import sharded_edges as se

pytestmark = pytest.mark.gpu

# ---- one rank -------------------------------------------------------------------------------------------------


@pytest.fixture(scope="module")
def one_rank_group():
    dist.init_process_group("gloo", store=dist.HashStore(), rank=0, world_size=1)
    try:
        yield dist.group.WORLD
    finally:
        dist.destroy_process_group()


def test_one_rank_group_gives_the_bits_of_no_group(one_rank_group):
    se.bits_equal(se.pooled_suite("cuda:0", one_rank_group), se.pooled_suite("cuda:0", None))


# ---- two ranks ------------------------------------------------------------------------------------------------


def _two_ranks(ctx, payload):
    """The pooled suite on this rank's half, and the refusal of an engine that does not know its shard."""
    from madrl_b200 import BatchedMAWaterWorld, evaluate_heuristic
    res = se.pooled_suite(ctx.dev, ctx.group, ctx.rank, ctx.world)
    unsharded = BatchedMAWaterWorld(4, 5, 5, device=ctx.dev, seed=1, max_path_length=5, n_poison=10, n_sensors=30)
    res["refused"] = se.refused(lambda: evaluate_heuristic(unsharded, 4, 0.99, "decentralized", group=ctx.group))
    return res


def _check_two(got, full):
    assert got[0]["refused"] == got[1]["refused"] == "refused"
    assert [(r["lo"], r["lo"] + r["done"].shape[1]) for r in (got[0], got[1])] == [(0, 31), (31, 63)]
    se.check_pooled(got, full)


def test_two_gloo_ranks_on_one_gpu_pool_to_the_unsharded_batch():
    _check_two(se.run_ranks(2, "gloo", _two_ranks, None), se.pooled_suite("cuda:0", None))


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_nccl_ranks_pool_to_the_unsharded_batch():
    _check_two(se.run_ranks(2, "nccl", _two_ranks, None), se.pooled_suite("cuda:0", None))
