"""CPU: the layout of the sharded optimizer (oracle/shard_oracle.py): the partition of the flat buffer over W ranks, the
segments of each shard, consolidation / re-sharding, and the constructor's refusal of mixed dtypes."""
import numpy as np
import pytest
import torch

import shard_oracle

NUMELS = [768 * 768, 5, 1000 * 33, 1, 64, 63, 65, 2048 * 130, 70001]


@pytest.mark.parametrize("world", [1, 2, 3, 8])
def test_partition_covers_every_element_once(world):
    offsets, padded, shard = shard_oracle.partition(NUMELS, world)
    assert padded % (world * shard_oracle.ALIGN) == 0 and padded == world * shard
    assert padded - sum(NUMELS) < world * shard_oracle.ALIGN
    hits = np.zeros(padded, dtype=np.int64)
    for r in range(world):
        lo, hi = r * shard, (r + 1) * shard
        covered = lo
        for i, a, b in shard_oracle.segments(NUMELS, world, r):
            assert a == covered, (r, i, a, covered)          # segments are contiguous, in parameter order
            assert offsets[i] <= a < b <= offsets[i] + NUMELS[i]
            hits[a:b] += 1
            covered = b
        assert covered <= hi
        assert covered == hi or covered == sum(NUMELS)        # only the padding is left out
    assert np.all(hits[:sum(NUMELS)] == 1) and np.all(hits[sum(NUMELS):] == 0)


@pytest.mark.parametrize("world,other", [(1, 8), (2, 3), (3, 2), (8, 1), (3, 8)])
def test_consolidate_and_reshard_round_trip(world, other):
    rng = np.random.default_rng(world * 10 + other)
    shapes = [(768, 768), (5,), (1000, 33), (1,), (8, 8), (63,), (65,), (2048, 130), (70001,)]
    tensors = [rng.standard_normal(s).astype(np.float32) for s in shapes]
    shards = shard_oracle.shard(tensors, world)
    back = shard_oracle.consolidate(shards, shapes)
    assert all(np.array_equal(a, b) for a, b in zip(tensors, back))
    again = shard_oracle.consolidate(shard_oracle.shard(back, other), shapes)
    assert all(np.array_equal(a, b) for a, b in zip(tensors, again))


def test_mixed_dtypes_are_refused():
    from atlas_b200._lib import AtlasB200Error
    from atlas_b200.sharded import OSS

    module = torch.nn.Sequential(torch.nn.Linear(4, 4).to(torch.bfloat16), torch.nn.Linear(4, 4).to(torch.float16))
    with pytest.raises(AtlasB200Error, match="mix dtypes"):
        OSS(module.parameters(), lr=1e-3)


def test_only_adamw_fp32copy_is_accepted():
    from atlas_b200._lib import AtlasB200Error
    from atlas_b200.sharded import OSS

    with pytest.raises(AtlasB200Error, match="not implemented"):
        OSS([torch.nn.Parameter(torch.zeros(4))], optim=torch.optim.SGD, lr=1e-3)
