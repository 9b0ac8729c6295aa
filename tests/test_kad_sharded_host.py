"""The shard plan of the sharded KAD entries (fad_kad_shard_plan, host only): contiguous ranges of work units that
partition the units in order, each holding at most its ideal share of the tiles plus one unit's tiles, with empty
shards when there are more shards than units."""
import numpy as np
import pytest
from hypothesis import given, settings, strategies as st

from fadtk_b200 import _native


def pair_unit_tiles(T: int) -> list[int]:
    """tiles of the whole-set units over T tile rows: row u, then row T - 1 - u (once when they are the same row)"""
    return [(T - u) + (u + 1 if T - 1 - u != u else 0) for u in range((T + 1) // 2)]


def check_plan(tiles, shards):
    b = _native.Engine.kad_shard_plan(tiles, shards)
    assert b.shape == (shards + 1,) and b[0] == 0 and b[-1] == len(tiles)
    assert (np.diff(b) >= 0).all()                                  # contiguous ranges in unit order: a partition
    t = np.asarray(tiles, dtype=np.int64)
    ideal = t.sum() / shards
    for s in range(shards):
        part = t[b[s]:b[s + 1]]
        if part.size:
            assert part.sum() <= ideal + part.max(), (s, part.sum(), ideal, part.max())
    assert (np.diff(b) == 0).sum() >= shards - len(tiles)          # more shards than units: the rest are empty
    return b


@settings(max_examples=300, deadline=None)
@given(st.lists(st.integers(1, 5000), min_size=0, max_size=400), st.integers(1, 64))
def test_plan_partitions_ragged_units(tiles, shards):
    """work-list units of any size (the per-song pass)"""
    check_plan(tiles, shards)


@settings(max_examples=200, deadline=None)
@given(st.integers(1, 4000), st.integers(1, 16))
def test_plan_of_pair_units(T, shards):
    """the whole-set and bandwidth passes: ceil(T / 2) units of T + 1 tiles (T - u for the middle row of an odd T)"""
    tiles = pair_unit_tiles(T)
    assert sum(tiles) == T * (T + 1) // 2                          # every tile of the upper triangle once
    b = check_plan(tiles, shards)
    if shards <= len(tiles):                                        # near-equal units: no shard is empty
        assert (np.diff(b) > 0).all()


def test_plan_examples():
    assert list(_native.Engine.kad_shard_plan([3, 3, 3, 3], 2)) == [0, 2, 4]
    assert list(_native.Engine.kad_shard_plan([1, 1, 1], 8)) == [0, 1, 1, 2, 2, 2, 3, 3, 3]
    assert list(_native.Engine.kad_shard_plan([], 3)) == [0, 0, 0, 0]
    assert list(_native.Engine.kad_shard_plan([5], 1)) == [0, 1]


@pytest.mark.parametrize("tiles,shards,msg", [([1, 2], 0, "shards >= 1"), ([1, 0, 2], 2, "at least one tile")])
def test_plan_rejections(tiles, shards, msg):
    with pytest.raises(_native.NativeError, match=msg):
        _native.Engine.kad_shard_plan(tiles, shards)
