"""wf_shard_columns: the main-trace columns each rank of a sharded proof owns. Needs no device."""
import pytest

from winterfell_b200 import dist as wd


@pytest.mark.parametrize("world", [2, 4, 8])
def test_blocks_partition_the_columns_in_whole_segments(world):
    for w in range(1, 256):
        blocks = [wd.shard_columns(w, world, r) for r in range(world)]
        nseg = (w + 7) // 8
        end = 0
        for r, (first, count) in enumerate(blocks):
            assert first == end, (w, world, r, blocks)              # contiguous, in rank order
            end = first + count
            assert first % 8 == 0 or count == 0, (w, world, r)       # blocks start on a segment
            if end < w:
                assert count % 8 == 0, (w, world, r)                 # whole segments, except the one holding the last column
        assert end == w, (w, world, blocks)                          # every column, once
        counts = [(c + 7) // 8 for _, c in blocks]
        assert sum(counts) == nseg and max(counts) - min(counts) <= 1, (w, world, blocks)
        if nseg % world == 0:                                        # the even split of the whole-segment shapes
            assert counts == [nseg // world] * world, (w, world, blocks)


def test_uneven_shapes():
    assert [wd.shard_columns(6, 4, r) for r in range(4)] == [(0, 6), (6, 0), (6, 0), (6, 0)]
    assert [wd.shard_columns(20, 2, r) for r in range(2)] == [(0, 16), (16, 4)]
    # about 70 columns fit a description: nine segments over eight ranks
    assert [wd.shard_columns(70, 8, r) for r in range(8)] == [(0, 16), (16, 8), (24, 8), (32, 8), (40, 8), (48, 8), (56, 8), (64, 6)]


@pytest.mark.parametrize("world", [0, 3, 5, 6, 7, 12])
def test_world_not_a_power_of_two_is_refused(world):
    with pytest.raises(ValueError):
        wd.shard_columns(16, world, 0)


@pytest.mark.parametrize("width,world,rank", [(0, 2, 0), (256, 2, 0), (16, 2, 2), (16, 4, 7)])
def test_bad_width_or_rank_is_refused(width, world, rank):
    with pytest.raises(ValueError):
        wd.shard_columns(width, world, rank)
